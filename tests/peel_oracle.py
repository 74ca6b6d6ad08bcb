"""CPU twin of depth peeling's ray query for the peel tests: ``tests/peel_oracle.c`` (which includes ``oracle/mcoracle.c``, so the
triangle predicate is the oracle's own) compiled with the oracle's flags into a temporary directory on first use."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from common import ROOT

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "peel_oracle.c")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        import oracle
        out = os.path.join(tempfile.mkdtemp(prefix="peel_oracle_"), "libpeel_oracle.so")
        cmd = ["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-I", os.path.join(ROOT, "oracle"), "-o", out, _SRC, "-lm"]
        if oracle._cpu_has_fma():
            cmd.insert(2, "-mfma")            # as oracle.build(): only the explicit fmaf() calls of mt_eval use it
        subprocess.run(cmd, check=True)
        lib = C.CDLL(out)
        lib.orc_scene_create.restype = C.c_void_p
        lib.orc_scene_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        lib.orc_scene_destroy.argtypes = [C.c_void_p]
        lib.orc_closest_hit_after.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
        lib.orc_all_hits.argtypes = [C.c_void_p] * 4
        lib.orc_all_hits.restype = C.c_int
        assert lib.orc_sizeof_real() == 4
        _LIB = lib
    return _LIB


SEP = np.float32(1.0 + 2.0 ** -16)


def sep(t):
    """fl32(t * (1 + 2^-16)): the separation between consecutive layers along a ray."""
    return (np.asarray(t, np.float32) * SEP).astype(np.float32)


class PeelScene:
    """Brute-force fp32 scene (triangle soup, no BVH)."""

    def __init__(self, verts, tris):
        self.lib = _lib()
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
        self.tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
        self.T = self.tris.shape[0]
        self.h = self.lib.orc_scene_create(self.verts.ctypes.data, self.verts.shape[0], self.tris.ctypes.data, self.T)

    def __del__(self):
        try:
            self.lib.orc_scene_destroy(self.h)
        except Exception:
            pass

    def closest_hit(self, ro, rd, t_after=None):
        """(tri_id [n] (-1 = miss), tuv [n,3] = (t, u, v)) of the closest hit with t > sep(t_after) (t_after None: t > 0)."""
        ro = np.ascontiguousarray(ro, np.float32).reshape(-1, 3); rd = np.ascontiguousarray(rd, np.float32).reshape(-1, 3)
        ta = np.zeros(ro.shape[0], np.float32) if t_after is None else np.ascontiguousarray(t_after, np.float32).reshape(-1)
        assert ta.shape[0] == ro.shape[0]
        tid = np.zeros(ro.shape[0], np.int32); tuv = np.zeros((ro.shape[0], 3), np.float32)
        self.lib.orc_closest_hit_after(self.h, ro.shape[0], ro.ctypes.data, rd.ctypes.data, ta.ctypes.data, tid.ctypes.data, tuv.ctypes.data)
        return tid, tuv

    def peel(self, ro, rd, layers):
        """Per-layer (tri_id, tuv) lists of `layers` successive closest_hit_after calls, each starting after the previous layer's t
        (+inf once a ray has no further hit), as raster.DepthPeeler does per pixel."""
        ta = np.zeros(np.asarray(ro).reshape(-1, 3).shape[0], np.float32)
        out = []
        for _ in range(layers):
            tid, tuv = self.closest_hit(ro, rd, ta)
            out.append((tid, tuv))
            ta = np.where(tid >= 0, tuv[:, 0], np.float32(np.inf)).astype(np.float32)
        return out

    def all_hits(self, ro, rd):
        """Sorted (t [k], tri_id [k]) of every triangle the ray hits."""
        t_all = np.zeros(self.T, np.float32)
        o = np.ascontiguousarray(ro, np.float32).reshape(3); d = np.ascontiguousarray(rd, np.float32).reshape(3)
        self.lib.orc_all_hits(self.h, o.ctypes.data, d.ctypes.data, t_all.ctypes.data)
        ids = np.nonzero(t_all >= 0)[0]
        order = np.lexsort((ids, t_all[ids]))
        return t_all[ids][order], ids[order].astype(np.int32)
