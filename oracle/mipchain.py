"""CPU oracle of Texture2D's automatic mip chain -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/mipchain.c``, the restatement of the chain forward, its backward folded over every level, and
Texture2D's clamp_ / normalize_ (render/texture.py:20-30,89-100; the contract is stated in nvdiffrecmc_b200/csrc/texture.cu).  Two builds
of the same source: fp32 (``mipchain_oracle()``, compared bit for bit with the kernels) and fp64 (``mipchain_oracle(True)``).
``oracle.build()`` compiles both from ``oracle.LIBS``.
"""
import ctypes as C
import os

import numpy as np

from oracle import _HERE, _I, _P, LIBS, CLib

SOURCES = [os.path.join(_HERE, s) for s in LIBS["mipchain"]]      # path of the library's source


def mip_shapes(H, W):
    """(H_k, W_k) of the automatic chain of an H x W texture: halve both sides until either is 1."""
    shapes = [(H, W)]
    while shapes[-1][0] > 1 and shapes[-1][1] > 1:
        shapes.append((shapes[-1][0] // 2, shapes[-1][1] // 2))
    return shapes


class MipChainOracle(CLib):
    LIB = "mipchain"
    SIGS = {
        "mip_sizeof_real": ([], _I),
        "mip_fwd": ([_I, _I, _I] + [_P] * 3, None),
        "mip_fold": ([_I, _I, _I] + [_P] * 4, None),
        "mip_clamp": ([_I, _I, _I] + [_P] * 5, None),
        "mip_normalize": ([_I, _I] + [_P] * 3, None),
    }

    @staticmethod
    def _table(levels):
        n = len(levels)
        return ((C.c_void_p * n)(*[None if t is None else t.ctypes.data for t in levels]), (C.c_int * n)(*[t.shape[1] for t in levels]),
                (C.c_int * n)(*[t.shape[2] for t in levels]))

    def forward(self, base):
        """levels 1..L of the automatic chain of base [Bt, H, W, C] (2 x 2 averages until either side is 1)"""
        base = self._a(base)
        Bt, H, W, Cn = base.shape
        lv = [base] + [np.zeros((Bt, h, w, Cn), self.dt) for h, w in mip_shapes(H, W)[1:]]
        ptrs, h, w = self._table(lv)
        self.lib.mip_fwd(len(lv), Cn, Bt, ptrs, h, w)
        return lv[1:]

    def fold(self, grads, shape):
        """d level 0 ([Bt, H, W, C] = shape) of a chain whose levels 0..L get the gradients grads[k] (None = none; at least one given)"""
        Bt, H, W, Cn = shape
        shapes = mip_shapes(H, W)
        assert len(grads) == len(shapes)
        gs = [None if g is None else self._a(g, (Bt, h, w, Cn)) for g, (h, w) in zip(grads, shapes)]
        ptrs = (C.c_void_p * len(gs))(*[None if g is None else g.ctypes.data for g in gs])
        d0 = np.zeros(shape, self.dt)
        self.lib.mip_fold(len(gs), Cn, Bt, ptrs, (C.c_int * len(gs))(*[s[0] for s in shapes]), (C.c_int * len(gs))(*[s[1] for s in shapes]),
                          d0.ctypes.data)
        return d0

    def clamp(self, levels, lo, hi):
        """copies of levels clamped per channel to [lo[c], hi[c]] as torch.clamp with tensor bounds"""
        lv = [self._a(t).copy() for t in levels]
        ptrs, h, w = self._table(lv)
        lo, hi = self._a(lo), self._a(hi)
        self.lib.mip_clamp(len(lv), lv[0].shape[3], lv[0].shape[0], ptrs, h, w, lo.ctypes.data, hi.ctypes.data)
        return lv

    def normalize(self, levels):
        """copies of 3-channel levels with every texel normalised as util.safe_normalize does"""
        lv = [self._a(t).copy() for t in levels]
        assert all(t.shape[3] == 3 for t in lv)
        ptrs, h, w = self._table(lv)
        self.lib.mip_normalize(len(lv), lv[0].shape[0], ptrs, h, w)
        return lv


mipchain_oracle = MipChainOracle.get
