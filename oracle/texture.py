"""CPU oracle of the filtered, mip-mapped texture look-up -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/texture.c`` (forward, d tex, d uv, d uv_da and the contract's deterministic log2; the contract is
stated in nvdiffrecmc_b200/csrc/texture.cu).  Two builds of the same source: fp32 (``TextureOracle()``, compared bit for bit with the
CUDA forward, d uv and d uv_da) and fp64 (``TextureOracle(f64=True)``, checked by finite differences).  Only ``tests/`` and the developer
tools import it; ``nvdiffrecmc_b200`` never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
_SRC = os.path.join(_HERE, "texture.c")
FILTERS = {"linear": 0, "linear-mipmap-linear": 1}
BOUNDARIES = {"wrap": 0, "clamp": 1}


def _lib_path(f64):
    return os.path.join(_BUILD, "libtexture_f64.so" if f64 else "libtexture_f32.so")


def build(force=False):
    """Compile oracle/texture.c with gcc (fp32 + fp64); -ffp-contract=off is what makes the fp32 build bit-comparable."""
    os.makedirs(_BUILD, exist_ok=True)
    for f64 in (False, True):
        out = _lib_path(f64)
        if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(_SRC):
            continue
        tmp = out + ".%d.tmp" % os.getpid()
        cmd = ["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", tmp, _SRC, "-lm"]
        if f64:
            cmd.insert(1, "-DORACLE_F64")
        subprocess.run(cmd, check=True)
        os.replace(tmp, out)


def chain_shapes(H, W, n_levels):
    """(H_k, W_k) of levels 0 .. n_levels - 1 of a chain whose level 0 is H x W."""
    return [(max(1, H >> k), max(1, W >> k)) for k in range(n_levels)]


class TextureOracle:
    def __init__(self, f64=False):
        build()
        self.f64 = f64
        self.dt = np.float64 if f64 else np.float32
        self.lib = C.CDLL(_lib_path(f64))
        assert self.lib.tex_sizeof_real() == (8 if f64 else 4)
        self.lib.tex_log2f.argtypes = [C.c_float]
        self.lib.tex_log2f.restype = C.c_float

    def log2(self, x):
        """The contract's fp32 log2, elementwise."""
        return np.array([self.lib.tex_log2f(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32).reshape(np.shape(x))

    def _a(self, x):
        return np.ascontiguousarray(np.asarray(x, dtype=self.dt))

    def _levels(self, levels):
        lv = [self._a(t) for t in levels]
        n = len(lv)
        ptrs = (C.c_void_p * n)(*[t.ctypes.data for t in lv])
        h = (C.c_int * n)(*[t.shape[1] for t in lv])
        w = (C.c_int * n)(*[t.shape[2] for t in lv])
        bs = (C.c_int64 * n)(*[0 if t.shape[0] == 1 else t.shape[1] * t.shape[2] * t.shape[3] for t in lv])
        return lv, [C.c_int(n), C.c_int(lv[0].shape[3]), ptrs, h, w, bs]

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
        self.lib.tex_fwd(*a, C.c_void_p(uv.ctypes.data), C.c_void_p(da.ctypes.data) if da is not None else None, C.c_int(B), C.c_int(H), C.c_int(W),
                         C.c_int(mip), C.c_int(BOUNDARIES[boundary_mode]), C.c_void_p(out.ctypes.data))
        return out

    def backward(self, levels, uv, uv_da, d_out, filter_mode="linear", boundary_mode="wrap", want_tex=True, want_uv=True, want_uv_da=True):
        """-> (list of d level or None, d uv or None, d uv_da or None); 'linear' returns one d level and no d uv_da."""
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
        self.lib.tex_bwd(*a, C.c_void_p(uv.ctypes.data), C.c_void_p(da.ctypes.data) if da is not None else None, C.c_int(B), C.c_int(H), C.c_int(W),
                         C.c_int(mip), C.c_int(BOUNDARIES[boundary_mode]), C.c_void_p(g.ctypes.data), dtp,
                         C.c_void_p(duv.ctypes.data) if duv is not None else None, C.c_void_p(dda.ctypes.data) if dda is not None else None)
        return dt, duv, dda


_CACHE = {}


def texture_oracle(f64=False):
    if f64 not in _CACHE:
        _CACHE[f64] = TextureOracle(f64=f64)
    return _CACHE[f64]
