"""CPU oracle of the image-space regularisers -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/regularizer.c``, the restatement of the reference's ``shading_loss``, ``material_smoothness_grad``
and ``chroma_loss`` (render/regularizer.py:15-49; the contract is stated in nvdiffrecmc_b200/csrc/regularizer.cu).  Two builds of the
same source: fp32 (``RegularizerOracle.get()``, compared bit for bit with the CUDA gradients of material_smoothness_grad and chroma_loss)
and fp64 (``RegularizerOracle.get(True)``, checked by finite differences and the per-element bar).  ``oracle.build()`` compiles both
from ``oracle.LIBS``.
"""
import os

import numpy as np

from oracle import _HERE, _I, _P, LIBS, REAL, CLib

SOURCES = [os.path.join(_HERE, s) for s in LIBS["regularizer"]]      # path of the library's source


class RegularizerOracle(CLib):
    LIB = "regularizer"
    SIGS = {
        "reg_sizeof_real": ([], _I),
        "reg_shading_loss_fwd": ([_I] + [_P] * 3 + [REAL, REAL, _P, _P], None),
        "reg_shading_loss_bwd": ([_I] + [_P] * 3 + [REAL, REAL, _P, REAL, _P, _P], None),
        "reg_material_smoothness_grad_fwd": ([_I] + [_P] * 3 + [REAL] * 3 + [_P], None),
        "reg_material_smoothness_grad_bwd": ([_I] + [_P] * 3 + [REAL] * 4 + [_P] * 3, None),
        "reg_chroma_loss_fwd": ([_I, _P, _P, REAL, _P], None),
        "reg_chroma_loss_bwd": ([_I, _P, _P, REAL, REAL, _P], None),
    }

    def _px4(self, *arrs):
        """[...,4] arrays of one shape -> (leading shape, pixel count, contiguous `real` copies)."""
        lead = np.shape(arrs[0])[:-1]
        out = [self._a(a) for a in arrs]
        assert all(a.shape == lead + (4,) for a in out), "every operand must be [...,4] of one shape"
        return lead, int(np.prod(lead)), out

    def shading_loss(self, diffuse_light, specular_light, color_ref, lambda_diffuse, lambda_specular, d_loss=None):
        """Forward -> (loss, means = (mean diffuse luma, mean specular luma)); with d_loss (the upstream gradient of the loss) ->
        (d diffuse_light, d specular_light), full [...,4], from this precision's own forward means."""
        lead, n, (d, s, r) = self._px4(diffuse_light, specular_light, color_ref)
        loss, means = np.zeros(1, self.dt), np.zeros(2, self.dt)
        self.lib.reg_shading_loss_fwd(n, d.ctypes.data, s.ctypes.data, r.ctypes.data, lambda_diffuse, lambda_specular, loss.ctypes.data,
                                      means.ctypes.data)
        if d_loss is None:
            return loss[0], means
        gd, gs = np.zeros_like(d), np.zeros_like(s)
        self.lib.reg_shading_loss_bwd(n, d.ctypes.data, s.ctypes.data, r.ctypes.data, lambda_diffuse, lambda_specular, means.ctypes.data,
                                      d_loss, gd.ctypes.data, gs.ctypes.data)
        return gd, gs

    def material_smoothness_grad(self, kd_grad, ks_grad, nrm_grad, lambda_kd=0.25, lambda_ks=0.1, lambda_nrm=0.0, d_loss=None):
        """Forward -> loss; with d_loss -> (d kd_grad, d ks_grad, d nrm_grad), full [...,4]."""
        lead, n, (k, s, m) = self._px4(kd_grad, ks_grad, nrm_grad)
        if d_loss is None:
            loss = np.zeros(1, self.dt)
            self.lib.reg_material_smoothness_grad_fwd(n, k.ctypes.data, s.ctypes.data, m.ctypes.data, lambda_kd, lambda_ks, lambda_nrm,
                                                      loss.ctypes.data)
            return loss[0]
        g = [np.zeros_like(k) for _ in range(3)]
        self.lib.reg_material_smoothness_grad_bwd(n, k.ctypes.data, s.ctypes.data, m.ctypes.data, lambda_kd, lambda_ks, lambda_nrm, d_loss,
                                                  *[x.ctypes.data for x in g])
        return tuple(g)

    def chroma_loss(self, kd, color_ref, lambda_chroma, d_loss=None):
        """Forward -> loss; with d_loss -> d kd, full [...,4] (alpha 0)."""
        lead, n, (k, r) = self._px4(kd, color_ref)
        if d_loss is None:
            loss = np.zeros(1, self.dt)
            self.lib.reg_chroma_loss_fwd(n, k.ctypes.data, r.ctypes.data, lambda_chroma, loss.ctypes.data)
            return loss[0]
        g = np.zeros_like(k)
        self.lib.reg_chroma_loss_bwd(n, k.ctypes.data, r.ctypes.data, lambda_chroma, d_loss, g.ctypes.data)
        return g
