"""CPU oracle of the filtered, mip-mapped texture look-up -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/texture.c`` (forward, d tex, d uv, d uv_da and the contract's deterministic log2; the contract is
stated in nvdiffrecmc_b200/csrc/texture.cu).  Two builds of the same source: fp32 (``texture_oracle()``, compared bit for bit with the
CUDA forward, d uv and d uv_da) and fp64 (``texture_oracle(f64=True)``, checked by finite differences).  Only ``tests/`` and the developer
tools import it; ``nvdiffrecmc_b200`` never does.
"""
import ctypes as C

import numpy as np

from oracle import TERMS, CLib, _I, _P

FILTERS = {"linear": 0, "linear-mipmap-linear": 1}
BOUNDARIES = {"wrap": 0, "clamp": 1}


def chain_shapes(H, W, n_levels):
    """(H_k, W_k) of levels 0 .. n_levels - 1 of a chain whose level 0 is H x W."""
    return [(max(1, H >> k), max(1, W >> k)) for k in range(n_levels)]


class TextureOracle(CLib):
    LIB = "texture"
    SIGS = {
        "tex_sizeof_real": ([], _I),
        "tex_log2f": ([C.c_float], C.c_float),
        "tex_fwd": ([_I, _I] + [_P] * 6 + [_I] * 5 + [_P], None),
        "tex_bwd": ([_I, _I] + [_P] * 6 + [_I] * 5 + [_P] * 4 + [_I], None),
    }

    def log2(self, x):
        """The contract's fp32 log2, elementwise."""
        return np.array([self.lib.tex_log2f(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32).reshape(np.shape(x))

    def _levels(self, levels):
        lv = [self._a(t) for t in levels]
        n = len(lv)
        ptrs = (C.c_void_p * n)(*[t.ctypes.data for t in lv])
        h = (C.c_int * n)(*[t.shape[1] for t in lv])
        w = (C.c_int * n)(*[t.shape[2] for t in lv])
        bs = (C.c_int64 * n)(*[0 if t.shape[0] == 1 else t.shape[1] * t.shape[2] * t.shape[3] for t in lv])
        return lv, [n, lv[0].shape[3], ptrs, h, w, bs]

    def _uv(self, uv, uv_da, filter_mode):
        uv = self._a(uv)
        mip = FILTERS[filter_mode]
        da = self._a(uv_da) if mip else None
        return uv, da, mip

    def forward(self, levels, uv, uv_da=None, filter_mode="linear", boundary_mode="wrap"):
        """levels: [tex, mip1, ...] each [Bt, H_k, W_k, C]; 'linear' reads levels[0] only.  -> [B, h, w, C]"""
        if FILTERS[filter_mode] == 0:
            levels = levels[:1]
        keep, a = self._levels(levels)
        uv, da, mip = self._uv(uv, uv_da, filter_mode)
        B, H, W = uv.shape[:3]
        out = np.zeros((B, H, W, keep[0].shape[3]), self.dt)
        self.lib.tex_fwd(*a, uv.ctypes.data, da.ctypes.data if da is not None else None, B, H, W, mip, BOUNDARIES[boundary_mode], out.ctypes.data)
        return out

    def backward(self, levels, uv, uv_da, d_out, filter_mode="linear", boundary_mode="wrap", want_tex=True, want_uv=True, want_uv_da=True,
                 terms="sum"):
        """-> (list of d level or None, d uv or None, d uv_da or None); 'linear' returns one d level and no d uv_da.  terms: d tex as the
        sum of its terms (w_lvl w_ij) g_c, the sum of their absolute values ("abs") or the number of non-zero terms ("count")."""
        if FILTERS[filter_mode] == 0:
            levels = levels[:1]
        keep, a = self._levels(levels)
        uv, da, mip = self._uv(uv, uv_da, filter_mode)
        B, H, W = uv.shape[:3]
        g = self._a(d_out)
        assert g.shape == (B, H, W, keep[0].shape[3])
        dt = [np.zeros_like(t) for t in keep] if want_tex else None
        dtp = (C.c_void_p * len(keep))(*[t.ctypes.data for t in dt]) if want_tex else None
        duv = np.zeros_like(uv) if want_uv else None
        dda = np.zeros((B, H, W, 4), self.dt) if (want_uv_da and mip) else None
        ptr = lambda x: x.ctypes.data if x is not None else None
        self.lib.tex_bwd(*a, uv.ctypes.data, ptr(da), B, H, W, mip, BOUNDARIES[boundary_mode], g.ctypes.data, dtp, ptr(duv), ptr(dda),
                         TERMS[terms])
        return dt, duv, dda


texture_oracle = TextureOracle.get
