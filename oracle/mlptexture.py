"""CPU oracle of the fused MLP texture -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/mlptexture.c`` (the contract is stated in nvdiffrecmc_b200/csrc/mlptexture.cu), which includes
``oracle/hashgrid.c`` for the encoding, so the library also exports the hash-grid oracle's functions and ``MlpTextureOracle`` is a
``HashGridOracle`` (``levels``, ``forward``, ``backward``) with the MLP texture added.  Two builds of the same source: fp32
(``mlptexture_oracle()``, compared bit for bit with the CUDA output, saved encoding, d texc and d W) and fp64 (``mlptexture_oracle(f64=True)``,
checked by finite differences).  ``oracle.build()`` compiles both from ``oracle.LIBS``.
"""
import ctypes as C
import os

import numpy as np

from oracle import _HERE, _I, _I64, _P, LIBS, TERMS
from oracle.hashgrid import HashGridOracle

SOURCES = [os.path.join(_HERE, s) for s in LIBS["mlptexture"]]      # paths of the library's source and the hashgrid.c it includes
MLPTEX_CHUNK = 1024          # MCS_MLPTEX_CHUNK: points per d W chunk partial


class MlpTextureOracle(HashGridOracle):
    LIB = "mlptexture"
    SIGS = dict(HashGridOracle.SIGS, **{
        "mlt_exp": ([_P, _I64, _P], None),
        "mlt_fwd": ([_P, _I64] + [_P] * 3 + [_I, _P, _P, _P, C.c_uint32, _I, _I] + [_P] * 3, None),
        "mlt_bwd": ([_P, _I64] + [_P] * 3 + [_I, _P, _P, _P, C.c_uint32, _I, _I] + [_P] * 5 + [_I], None),
    })

    def exp(self, x):
        """The MLP texture's exp (csrc/mlptexture.cu, fp32 build; libm exp in the fp64 build)."""
        x = self._a(x); y = np.zeros_like(x)
        self.lib.mlt_exp(x.ctypes.data, x.size, y.ctypes.data)
        return y

    def _mlp_args(self, t, aabb, min_max, params, lv, weights):
        t = self._a(t).reshape(-1, 3); aabb = self._a(aabb).reshape(2, 3); C = int(np.asarray(weights[-1]).shape[0])
        mm = self._a(min_max).reshape(2, C); p = self._a(params)
        hidden = len(weights) - 1
        assert lv["n_levels"] == 16 and all(np.asarray(w).shape == (32, 32) for w in weights[:-1]) and np.asarray(weights[-1]).shape == (C, 32)
        w = self._a(np.concatenate([np.asarray(x).reshape(-1) for x in weights]))
        keep, a = self._args(lv)
        return (t, aabb, mm, p, w, keep), [t.ctypes.data, t.shape[0], aabb.ctypes.data, mm.ctypes.data, p.ctypes.data, *a, hidden, C, w.ctypes.data]

    def mlptex_forward(self, t, aabb, min_max, params, lv, weights):
        """MLPTexture3D.sample's contract (csrc/mlptexture.cu): t [n,3] -> (out [n,C], the encoding [n,32]).  weights: the hidden + 1
        Linear weights, [32,32] ... [C,32]."""
        keep, a = self._mlp_args(t, aabb, min_max, params, lv, weights)
        n, C = keep[0].shape[0], keep[2].shape[1]
        out = np.zeros((n, C), self.dt); enc = np.zeros((n, 32), self.dt)
        self.lib.mlt_fwd(*a, out.ctypes.data, enc.ctypes.data)
        return out, enc

    def mlptex_backward(self, t, aabb, min_max, params, lv, weights, d_out, want_params=True, want_t=True, want_w=True, terms="sum"):
        """-> (d params or None, d t or None, [d W per layer] or None): the true gradients (no x128 on d params).  terms: d params in
        hg_bwd's mode ("sum", "abs" or "count")."""
        keep, a = self._mlp_args(t, aabb, min_max, params, lv, weights)
        n, C, p = keep[0].shape[0], keep[2].shape[1], keep[3]
        g = self._a(d_out).reshape(n, C)
        dp = np.zeros_like(p) if want_params else None
        dt = np.zeros((n, 3), self.dt) if want_t else None
        dw = np.zeros(keep[4].size, self.dt) if want_w else None
        self.lib.mlt_bwd(*a, g.ctypes.data, dp.ctypes.data if want_params else None, dt.ctypes.data if want_t else None,
                               dw.ctypes.data if want_w else None, TERMS[terms])
        if want_w:
            sizes = [np.asarray(x).size for x in weights]
            dw = [d.reshape(np.asarray(x).shape) for d, x in zip(np.split(dw, np.cumsum(sizes)[:-1]), weights)]
        return dp, dt, dw


mlptexture_oracle = MlpTextureOracle.get
