"""CPU oracle of the G-buffer producer's geometry gradients -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Thin numpy/ctypes wrapper around ``oracle/geometry.c`` (rasterize / interpolate backward, edge adjacency, analytic antialias; the
semantics are stated in nvdiffrecmc_b200/csrc/raster.cu).  Two builds of the same source: fp32 (``GeometryOracle()``, compared with
the CUDA kernels) and fp64 (``GeometryOracle(f64=True)``, used to validate the hand-derived adjoints by finite differences).  Only
``tests/`` and the developer tools import it; ``nvdiffrecmc_b200`` never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
_SRC = os.path.join(_HERE, "geometry.c")


def _lib_path(f64):
    return os.path.join(_BUILD, "libgeometry_f64.so" if f64 else "libgeometry_f32.so")


def build(force=False):
    """Compile oracle/geometry.c with gcc (fp32 + fp64).  -ffp-contract=off is mandatory: the fp32 build makes the CUDA kernel's
    discrete decisions with the same roundings."""
    os.makedirs(_BUILD, exist_ok=True)
    for f64 in (False, True):
        out = _lib_path(f64)
        if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(_SRC):
            continue
        cmd = ["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", out, _SRC, "-lm"]
        if f64:
            cmd.insert(1, "-DORACLE_F64")
        subprocess.run(cmd, check=True)


class GeometryOracle:
    def __init__(self, f64=False):
        build()
        self.f64 = f64
        self.dt = np.float64 if f64 else np.float32
        self.lib = C.CDLL(_lib_path(f64))
        assert self.lib.geo_sizeof_real() == (8 if f64 else 4)

    def _a(self, x, shape=None):
        x = np.ascontiguousarray(np.asarray(x, dtype=self.dt))
        if shape is not None:
            x = np.ascontiguousarray(np.broadcast_to(x, shape))
        return x

    def _geo(self, pos, rast, tris):
        pos = self._a(pos); rast = self._a(rast); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        pos_bs = pos.shape[-2] * 4 if pos.ndim == 3 else 0
        return pos, rast, tris, B, H, W, C.c_int64(pos_bs)

    def raster_bary(self, pos, tris, rast):
        """(u, v) [B,H,W,2] = (s0 / S, s1 / S) of the clip-space triangle under each covered pixel (0 elsewhere)."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        uv = np.zeros((B, H, W, 2), self.dt)
        self.lib.orc_raster_bary(C.c_int(B), C.c_int(H), C.c_int(W), pbs, C.c_void_p(pos.ctypes.data), C.c_int(tris.shape[0]),
                                 C.c_void_p(tris.ctypes.data), C.c_void_p(rast.ctypes.data), C.c_void_p(uv.ctypes.data))
        return uv

    def raster_bwd(self, pos, tris, rast, d_rast):
        """d pos (shape of pos) from d rast[...,0:2] through the barycentrics of pos."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        g = self._a(d_rast); d = np.zeros_like(pos)
        self.lib.orc_raster_bwd(C.c_int(B), C.c_int(H), C.c_int(W), pbs, C.c_void_p(pos.ctypes.data), C.c_int(tris.shape[0]), C.c_void_p(tris.ctypes.data),
                                C.c_void_p(rast.ctypes.data), C.c_void_p(g.ctypes.data), C.c_void_p(d.ctypes.data))
        return d

    def interpolate_bwd_rast(self, attr, tris, rast, d_out):
        """d rast [B,H,W,4] = (sum_c g (A0 - A2), sum_c g (A1 - A2), 0, 0) of interpolate."""
        attr = self._a(attr); rast = self._a(rast); g = self._a(d_out); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        Cn = attr.shape[-1]
        d = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_interpolate_bwd_rast(C.c_int(B), C.c_int(H), C.c_int(W), C.c_int(Cn), C.c_int64(attr.shape[-2] * Cn if attr.ndim == 3 else 0),
                                          C.c_void_p(attr.ctypes.data), C.c_int(tris.shape[0]), C.c_void_p(tris.ctypes.data), C.c_void_p(rast.ctypes.data),
                                          C.c_void_p(g.ctypes.data), C.c_void_p(d.ctypes.data))
        return d

    def aa_topology(self, tris):
        """int32 [T,3]: triangle across edge (tri[t,k], tri[t,(k+1)%3]), -1 boundary, -2 three or more triangles."""
        tris = np.ascontiguousarray(tris, np.int32)
        adj = np.zeros(tris.shape, np.int32)
        self.lib.orc_aa_topology(C.c_int(tris.shape[0]), C.c_void_p(tris.ctypes.data), C.c_void_p(adj.ctypes.data))
        return adj

    def _aa_args(self, color, rast, pos, tris, adj):
        color = self._a(color)
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        adj = self.aa_topology(tris) if adj is None else np.ascontiguousarray(adj, np.int32)
        keep = (color, rast, pos, tris, adj)
        args = [C.c_int(B), C.c_int(H), C.c_int(W), C.c_int(color.shape[3]), C.c_void_p(color.ctypes.data), C.c_void_p(rast.ctypes.data), pbs,
                C.c_void_p(pos.ctypes.data), C.c_int(tris.shape[0]), C.c_void_p(tris.ctypes.data), C.c_void_p(adj.ctypes.data)]
        return keep, args

    def antialias(self, color, rast, pos, tris, adj=None):
        keep, args = self._aa_args(color, rast, pos, tris, adj)
        out = np.zeros_like(keep[0])
        self.lib.orc_antialias_fwd(*args, C.c_void_p(out.ctypes.data))
        return out

    def antialias_bwd(self, color, rast, pos, tris, d_out, adj=None):
        """-> (d_color, d_pos)"""
        keep, args = self._aa_args(color, rast, pos, tris, adj)
        g = self._a(d_out, keep[0].shape)
        dc = np.zeros_like(keep[0]); dp = np.zeros_like(keep[2])
        self.lib.orc_antialias_bwd(*args, C.c_void_p(g.ctypes.data), C.c_void_p(dc.ctypes.data), C.c_void_p(dp.ctypes.data))
        return dc, dp


_CACHE = {}


def geometry_oracle(f64=False):
    if f64 not in _CACHE:
        _CACHE[f64] = GeometryOracle(f64=f64)
    return _CACHE[f64]
