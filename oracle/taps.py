"""CPU oracle of the jittered regulariser taps -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/taps.c``, the restatement of shade()'s kd_grad / ks_grad / normal_grad / perturbed_nrm_grad
(render/render.py:50-97; the contract is stated in nvdiffrecmc_b200/csrc/taps.cu), whose tap is texture.c's look-up, included by the C
file.  Two builds of the same source: fp32 (``taps_oracle()``, compared bit for bit with the kernels' forward and one-writer gradients, and
per element with their scatters) and fp64 (``taps_oracle(True)``, checked by finite differences and against the reference's own shade()).
``oracle.build()`` compiles both from ``oracle.LIBS``.  The library also exports texture.c's functions, so ``TapsOracle.SIGS`` extends
``TextureOracle.SIGS``.
"""
import numpy as np

from oracle import _I, _P, TERMS, CLib
from oracle.texture import TextureOracle

BUFFERS = ["kd_grad", "ks_grad", "normal_grad", "perturbed_nrm_grad"]
OPERANDS = ["kd", "ks", "gb_normal", "perturbed_nrm", "kd_jitter", "ks_jitter"]


class TapsOracle(CLib):
    LIB = "taps"
    SIGS = dict(TextureOracle.SIGS, **{
        "taps_sizeof_real": ([], _I),
        "taps_fwd": ([_I] * 4 + [_P] * 12, None),
        "taps_bwd": ([_I] * 4 + [_P] * 18 + [_I], None),
    })

    def _ops(self, rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter):
        B, H, W = np.shape(rast)[:3]
        ckd = np.shape(kd)[3]
        shapes = [(B, H, W, 4), (B, H, W, 2), (B, H, W, ckd), (B, H, W, 3), (B, H, W, 3), (B, H, W, 3), (B, H, W, ckd), (B, H, W, 3)]
        ops = [None if x is None else self._a(x) for x in (rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter)]
        for x, s in zip(ops, shapes):
            assert x is None or x.shape == s, (x.shape, s)
        assert (kd_jitter is None) == (ks_jitter is None)
        return (B, H, W, ckd), ops

    @staticmethod
    def _p(x):
        return None if x is None else x.ctypes.data

    def forward(self, rast, jitter, kd, ks, gb_normal, perturbed_nrm=None, kd_jitter=None, ks_jitter=None):
        """-> {"kd_grad": [B,H,W,Ckd+1], "ks_grad", "normal_grad"[, "perturbed_nrm_grad"]: [B,H,W,4]}"""
        (B, H, W, ckd), ops = self._ops(rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter)
        outs = [np.zeros((B, H, W, ckd + 1), self.dt)] + [np.zeros((B, H, W, 4), self.dt) for _ in range(3)]
        self.lib.taps_fwd(B, H, W, ckd, *[self._p(x) for x in ops], *[o.ctypes.data for o in outs])
        return dict(zip(BUFFERS[:4 if perturbed_nrm is not None else 3], outs))

    def backward(self, rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter, grads, terms="sum"):
        """grads: the upstream gradient of each buffer, keyed as forward's result.  -> {operand: gradient} for kd, ks, gb_normal (and
        perturbed_nrm, kd_jitter, ks_jitter when given).  terms: the scattered gradients (kd, ks, gb_normal, perturbed_nrm) as the sum of
        their terms, the sum of their absolute values ("abs") or the number of non-zero terms ("count"); kd_jitter / ks_jitter have one
        writer and are the same in every mode."""
        (B, H, W, ckd), ops = self._ops(rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter)
        has_pn, mlp = perturbed_nrm is not None, kd_jitter is not None
        g = [self._a(grads[k], (B, H, W, ckd + 1 if k == "kd_grad" else 4)) if (k != "perturbed_nrm_grad" or has_pn) else None for k in BUFFERS]
        d = [np.zeros((B, H, W, ckd), self.dt), np.zeros((B, H, W, 3), self.dt), np.zeros((B, H, W, 3), self.dt),
             np.zeros((B, H, W, 3), self.dt) if has_pn else None, np.zeros((B, H, W, ckd), self.dt) if mlp else None,
             np.zeros((B, H, W, 3), self.dt) if mlp else None]
        self.lib.taps_bwd(B, H, W, ckd, *[self._p(x) for x in ops], *[self._p(x) for x in g], *[self._p(x) for x in d], TERMS[terms])
        return {k: v for k, v in zip(OPERANDS, d) if v is not None}


taps_oracle = TapsOracle.get
