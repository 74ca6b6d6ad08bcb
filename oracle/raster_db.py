"""CPU oracle of the G-buffer producer's screen-space derivatives -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Thin numpy/ctypes wrapper around ``oracle/raster_db.c`` (rast_db, interpolate's out_da, their adjoints and interpolate's forward; the
semantics are stated in nvdiffrecmc_b200/csrc/raster.cu).  Two builds of the same source: fp32 (``RasterDbOracle()``, compared with the
CUDA kernels bit for bit) and fp64 (``RasterDbOracle(f64=True)``, used to validate the derivatives and the hand-derived adjoints by
finite differences).  Only ``tests/`` and the developer tools import it; ``nvdiffrecmc_b200`` never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
_SRC = os.path.join(_HERE, "raster_db.c")


def _lib_path(f64):
    return os.path.join(_BUILD, "libraster_db_f64.so" if f64 else "libraster_db_f32.so")


def build(force=False):
    """Compile oracle/raster_db.c with gcc (fp32 + fp64).  -ffp-contract=off is mandatory: the fp32 build reproduces the kernels'
    explicitly rounded operations."""
    os.makedirs(_BUILD, exist_ok=True)
    for f64 in (False, True):
        out = _lib_path(f64)
        if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(_SRC):
            continue
        cmd = ["gcc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", out, _SRC, "-lm"]
        if f64:
            cmd.insert(1, "-DORACLE_F64")
        subprocess.run(cmd, check=True)


class RasterDbOracle:
    def __init__(self, f64=False):
        build()
        self.f64 = f64
        self.dt = np.float64 if f64 else np.float32
        self.lib = C.CDLL(_lib_path(f64))
        assert self.lib.db_sizeof_real() == (8 if f64 else 4)

    def _a(self, x):
        return np.ascontiguousarray(np.asarray(x, dtype=self.dt))

    def _geo(self, pos, rast, tris):
        pos = self._a(pos); rast = self._a(rast); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        pos_bs = pos.shape[-2] * 4 if pos.ndim == 3 else 0
        return pos, rast, tris, B, H, W, C.c_int64(pos_bs)

    def _attr(self, attr, tris, rast):
        attr = self._a(attr); rast = self._a(rast); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        Cn = attr.shape[-1]
        return attr, rast, tris, B, H, W, Cn, C.c_int64(attr.shape[-2] * Cn if attr.ndim == 3 else 0)

    def interpolate(self, attr, tris, rast):
        """out [B,H,W,C] = fma(u, A0, fma(v, A1, (1 - u - v) A2)), 0 without a hit (the kernel's operation order)."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        out = np.zeros((B, H, W, Cn), self.dt)
        self.lib.orc_interpolate_fwd(C.c_int(B), C.c_int(H), C.c_int(W), C.c_int(Cn), abs_, C.c_void_p(attr.ctypes.data), C.c_int(tris.shape[0]),
                                     C.c_void_p(tris.ctypes.data), C.c_void_p(rast.ctypes.data), C.c_void_p(out.ctypes.data))
        return out

    def rast_db(self, pos, tris, rast):
        """rast_db [B,H,W,4] = (du/dX, du/dY, dv/dX, dv/dY) of the clip-space triangle under each covered pixel (0 elsewhere)."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        db = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_rast_db(C.c_int(B), C.c_int(H), C.c_int(W), pbs, C.c_void_p(pos.ctypes.data), C.c_int(tris.shape[0]), C.c_void_p(tris.ctypes.data),
                             C.c_void_p(rast.ctypes.data), C.c_void_p(db.ctypes.data))
        return db

    def rast_db_bwd(self, pos, tris, rast, d_db):
        """d pos (shape of pos) from d rast_db."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        g = self._a(d_db); d = np.zeros_like(pos)
        self.lib.orc_rast_db_bwd(C.c_int(B), C.c_int(H), C.c_int(W), pbs, C.c_void_p(pos.ctypes.data), C.c_int(tris.shape[0]), C.c_void_p(tris.ctypes.data),
                                 C.c_void_p(rast.ctypes.data), C.c_void_p(g.ctypes.data), C.c_void_p(d.ctypes.data))
        return d

    @staticmethod
    def _sel(diff_attrs, Cn):
        if isinstance(diff_attrs, str):
            assert diff_attrs == "all"
            return Cn, None, None
        idx = np.ascontiguousarray(diff_attrs, np.int32)
        return idx.shape[0], idx, C.c_void_p(idx.ctypes.data)

    def interpolate_da(self, attr, tris, rast, db, diff_attrs="all"):
        """out_da [B,H,W,2n]: (dA/dX, dA/dY) of each selected attribute ('all' or a list of indices)."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        db = self._a(db)
        n, keep, ip = self._sel(diff_attrs, Cn)
        out = np.zeros((B, H, W, 2 * n), self.dt)
        self.lib.orc_interpolate_da(C.c_int(B), C.c_int(H), C.c_int(W), C.c_int(Cn), abs_, C.c_void_p(attr.ctypes.data), C.c_int(tris.shape[0]),
                                    C.c_void_p(tris.ctypes.data), C.c_void_p(rast.ctypes.data), C.c_void_p(db.ctypes.data), C.c_int(n), ip,
                                    C.c_void_p(out.ctypes.data))
        return out

    def interpolate_da_bwd(self, attr, tris, rast, db, d_out_da, diff_attrs="all"):
        """-> (d attr, d rast_db) of out_da."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        db = self._a(db); g = self._a(d_out_da)
        n, keep, ip = self._sel(diff_attrs, Cn)
        da = np.zeros_like(attr); ddb = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_interpolate_da_bwd(C.c_int(B), C.c_int(H), C.c_int(W), C.c_int(Cn), abs_, C.c_void_p(attr.ctypes.data), C.c_int(tris.shape[0]),
                                        C.c_void_p(tris.ctypes.data), C.c_void_p(rast.ctypes.data), C.c_void_p(db.ctypes.data), C.c_int(n), ip,
                                        C.c_void_p(g.ctypes.data), C.c_void_p(da.ctypes.data), C.c_void_p(ddb.ctypes.data))
        return da, ddb


_CACHE = {}


def raster_db_oracle(f64=False):
    if f64 not in _CACHE:
        _CACHE[f64] = RasterDbOracle(f64=f64)
    return _CACHE[f64]
