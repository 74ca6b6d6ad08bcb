"""CPU oracle of DMTet's marching tetrahedra and SDF regulariser -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/dmtet.c`` (the contract is stated in nvdiffrecmc_b200/csrc/dmtet.cu).  Two builds of the same source:
fp32 (``dmtet_oracle()``, compared bit for bit with the CUDA vertices, faces, uv_idx, d pos and d sdf) and fp64 (``dmtet_oracle(f64=True)``,
checked by finite differences).  ``build()`` compiles both; ``__graft_entry__.build()`` calls it.
"""
import ctypes as C
import os

import numpy as np

from oracle import _CFLAGS, _HERE, _I, _I64, _P, REAL, CLib, _compile, _lib_path

SOURCE = os.path.join(_HERE, "dmtet.c")


def _build(f64, force=False):
    _compile(["gcc"] + _CFLAGS + (["-DORACLE_F64"] if f64 else []) + [SOURCE, "-lm"], _lib_path("dmtet", f64), [SOURCE], force)


def build(force=False):
    """Compile oracle/dmtet.c with gcc, fp32 and fp64 (-DORACLE_F64), into oracle/_build/."""
    for f64 in (False, True):
        _build(f64, force)


class DmtetOracle(CLib):
    LIB = "dmtet"
    SIGS = {
        "dmt_sizeof_real": ([], _I),
        "dmt_edges": ([_I64, _I64, _P, _P, _P], _I64),
        "dmt_adjacency": ([_I64, _I64, _P, _P, _P], None),
        "dmt_uv_side": ([_I64], _I64),
        "dmt_uvs": ([_I64, _P], None),
        "dmt_extract": ([_I64, _I64, _I64] + [_P] * 10, None),
        "dmt_backward": ([_I64, _I64] + [_P] * 7, None),
        "dmt_reg_fwd": ([_I64, _P, _P, _P], C.c_double),
        "dmt_reg_bwd": ([_I64, _I64, _P, _P, REAL, _P], None),
    }

    def __init__(self, f64=False):
        # CLib.__init__ builds from oracle.LIBS; this library has its own recipe (build() above), the loading is the same
        self.f64 = f64
        self.dt, self.real = (np.float64, C.c_double) if f64 else (np.float32, C.c_float)
        _build(f64)
        self.lib = C.CDLL(_lib_path(self.LIB, f64))
        for name, (args, res) in self.SIGS.items():
            fn = getattr(self.lib, name)          # AttributeError if the library does not export it
            fn.argtypes = [self.real if a is REAL else a for a in args]
            fn.restype = res
        assert self.lib.dmt_sizeof_real() == C.sizeof(self.real)

    def tables(self, tet, V):
        """Static tables of a grid: dict(edges [E,2], tet_edges [T,6], v2e_offsets [V+1], v2e_edges [2E]), int32."""
        tet = np.ascontiguousarray(tet, np.int64).reshape(-1, 4)
        T = tet.shape[0]
        assert T >= 1 and tet.min() >= 0 and tet.max() < V
        edges = np.zeros((6 * T, 2), np.int32); tet_edges = np.zeros((T, 6), np.int32)
        E = int(self.lib.dmt_edges(V, T, tet.ctypes.data, edges.ctypes.data, tet_edges.ctypes.data))
        edges = np.ascontiguousarray(edges[:E])
        off, adj = self.adjacency(edges, V)
        return {"edges": edges, "tet_edges": tet_edges, "v2e_offsets": off, "v2e_edges": adj}

    def adjacency(self, edges, V):
        edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
        off = np.zeros(V + 1, np.int32); adj = np.zeros(2 * edges.shape[0], np.int32)
        self.lib.dmt_adjacency(V, edges.shape[0], edges.ctypes.data, off.ctypes.data, adj.ctypes.data)
        return off, adj

    def uvs(self, T):
        N = int(self.lib.dmt_uv_side(T))
        out = np.zeros((4 * N * N, 2), np.float32)
        self.lib.dmt_uvs(T, out.ctypes.data)
        return out

    def marching_tets(self, pos, sdf, tet, tables=None):
        """-> (verts [M,3], faces [F,3] int64, uvs, uv_idx [F,3] int64, vid [E] int32)."""
        tet = np.ascontiguousarray(tet, np.int64).reshape(-1, 4)
        pos = self._a(pos).reshape(-1, 3); sdf = self._a(sdf).reshape(-1)
        V, T = pos.shape[0], tet.shape[0]
        tb = tables or self.tables(tet, V)
        E = tb["edges"].shape[0]
        counts = np.zeros(2, np.int64); vid = np.zeros(E, np.int32)
        verts = np.zeros((E, 3), self.dt); faces = np.zeros((2 * T, 3), np.int64); uv_idx = np.zeros((2 * T, 3), np.int64)
        self.lib.dmt_extract(V, E, T, pos.ctypes.data, sdf.ctypes.data, tb["edges"].ctypes.data, tet.ctypes.data, tb["tet_edges"].ctypes.data,
                             counts.ctypes.data, vid.ctypes.data, verts.ctypes.data, faces.ctypes.data, uv_idx.ctypes.data)
        M, F = int(counts[0]), int(counts[1])
        return verts[:M].copy(), faces[:F].copy(), self.uvs(T), uv_idx[:F].copy(), vid

    def backward(self, pos, sdf, tet, d_verts, tables=None):
        """-> (d pos [V,3], d sdf [V]) for the upstream gradient d_verts [M,3] of marching_tets' verts."""
        pos = self._a(pos).reshape(-1, 3); sdf = self._a(sdf).reshape(-1)
        V = pos.shape[0]
        tb = tables or self.tables(tet, V)
        vid = self.marching_tets(pos, sdf, tet, tb)[4]
        g = self._a(d_verts).reshape(-1, 3)
        assert g.shape[0] == int((vid >= 0).sum())
        dp = np.zeros((V, 3), self.dt); ds = np.zeros(V, self.dt)
        self.lib.dmt_backward(V, tb["edges"].shape[0], pos.ctypes.data, sdf.ctypes.data, tb["edges"].ctypes.data, vid.ctypes.data, g.ctypes.data,
                              dp.ctypes.data, ds.ctypes.data)
        return dp, ds

    def sdf_reg_loss(self, sdf, edges):
        """-> (loss, M): the regulariser in double and the number of sign-changing edges."""
        sdf = self._a(sdf).reshape(-1); edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
        m = C.c_int64(0)
        loss = self.lib.dmt_reg_fwd(edges.shape[0], sdf.ctypes.data, edges.ctypes.data, C.byref(m))
        return loss, int(m.value)

    def sdf_reg_loss_bwd(self, sdf, edges, d_loss=1.0):
        sdf = self._a(sdf).reshape(-1); edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
        out = np.zeros(sdf.shape[0], self.dt)
        self.lib.dmt_reg_bwd(sdf.shape[0], edges.shape[0], sdf.ctypes.data, edges.ctypes.data, float(d_loss), out.ctypes.data)
        return out


dmtet_oracle = DmtetOracle.get
