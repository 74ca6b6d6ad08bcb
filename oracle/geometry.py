"""CPU oracle of the G-buffer producer's geometry gradients -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Thin numpy/ctypes wrapper around ``oracle/geometry.c`` (rasterize / interpolate backward, edge adjacency, analytic antialias, and the
screen-space derivatives: rast_db, interpolate's out_da, their adjoints and interpolate's forward; the semantics are stated in
nvdiffrecmc_b200/csrc/raster.cu).  Two builds of the same source: fp32 (``geometry_oracle()``, compared with the CUDA kernels) and fp64
(``geometry_oracle(f64=True)``, used to validate the derivatives and the hand-derived adjoints by finite differences).  Only ``tests/``
and the developer tools import it; ``nvdiffrecmc_b200`` never does.
"""
import numpy as np

from oracle import TERMS, CLib, _I, _I64, _P


class GeometryOracle(CLib):
    LIB = "geometry"
    SIGS = {
        "geo_sizeof_real": ([], _I),
        "orc_raster_bary": ([_I] * 3 + [_I64, _P, _I] + [_P] * 3, None),
        "orc_raster_bwd": ([_I] * 3 + [_I64, _P, _I] + [_P] * 4 + [_I], None),
        "orc_interpolate_bwd_attr": ([_I] * 4 + [_I64, _I] + [_P] * 4 + [_I], None),
        "orc_interpolate_bwd_rast": ([_I] * 4 + [_I64, _P, _I] + [_P] * 4, None),
        "orc_aa_topology": ([_I, _P, _P], None),
        "orc_antialias_pair_t": ([_I] * 3 + [_P, _I64, _P, _I] + [_P] * 3, None),
        "orc_antialias_fwd": ([_I] * 4 + [_P, _P, _I64, _P, _I] + [_P] * 3, None),
        "orc_antialias_bwd_color": ([_I] * 4 + [_P, _P, _I64, _P, _I] + [_P] * 4, None),
        "orc_antialias_bwd": ([_I] * 4 + [_P, _P, _I64, _P, _I] + [_P] * 5 + [_I], None),
        "orc_interpolate_fwd": ([_I] * 4 + [_I64, _P, _I] + [_P] * 3, None),
        "orc_rast_db": ([_I] * 3 + [_I64, _P, _I] + [_P] * 3, None),
        "orc_rast_db_bwd": ([_I] * 3 + [_I64, _P, _I] + [_P] * 4 + [_I], None),
        "orc_interpolate_da": ([_I] * 4 + [_I64, _P, _I] + [_P] * 3 + [_I, _P, _P], None),
        "orc_interpolate_da_bwd": ([_I] * 4 + [_I64, _P, _I] + [_P] * 3 + [_I] + [_P] * 4 + [_I], None),
    }

    def _geo(self, pos, rast, tris):
        pos = self._a(pos); rast = self._a(rast); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        pos_bs = pos.shape[-2] * 4 if pos.ndim == 3 else 0
        return pos, rast, tris, B, H, W, pos_bs

    def _attr(self, attr, tris, rast):
        attr = self._a(attr); rast = self._a(rast); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        Cn = attr.shape[-1]
        return attr, rast, tris, B, H, W, Cn, attr.shape[-2] * Cn if attr.ndim == 3 else 0

    def raster_bary(self, pos, tris, rast):
        """(u, v) [B,H,W,2] = (s0 / S, s1 / S) of the clip-space triangle under each covered pixel (0 elsewhere)."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        uv = np.zeros((B, H, W, 2), self.dt)
        self.lib.orc_raster_bary(B, H, W, pbs, pos.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, uv.ctypes.data)
        return uv

    def raster_bwd(self, pos, tris, rast, d_rast, terms="sum"):
        """d pos (shape of pos) from d rast[...,0:2] through the barycentrics of pos.  terms: the sum of the per-pixel terms, the sum of
        their absolute values ("abs") or the number of non-zero terms ("count"), as for every scatter below."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        g = self._a(d_rast); d = np.zeros_like(pos)
        self.lib.orc_raster_bwd(B, H, W, pbs, pos.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, g.ctypes.data, d.ctypes.data,
                                TERMS[terms])
        return d

    def interpolate_bwd_attr(self, attr_shape, tris, rast, d_out, terms="sum"):
        """d attr (shape attr_shape: [V,C] or [B,V,C]) of interpolate: vertex k of the pixel's triangle gets w_k g, (w0, w1, w2) = (u, v,
        (1 - u) - v), summed in pixel, channel, vertex order."""
        rast = self._a(rast); tris = np.ascontiguousarray(tris, np.int32)
        B, H, W = rast.shape[:3]
        Cn = attr_shape[-1]
        g = self._a(d_out, (B, H, W, Cn)); d = np.zeros(attr_shape, self.dt)
        self.lib.orc_interpolate_bwd_attr(B, H, W, Cn, attr_shape[-2] * Cn if len(attr_shape) == 3 else 0, tris.shape[0], tris.ctypes.data,
                                          rast.ctypes.data, g.ctypes.data, d.ctypes.data, TERMS[terms])
        return d

    def interpolate_bwd_rast(self, attr, tris, rast, d_out):
        """d rast [B,H,W,4] = (sum_c g (A0 - A2), sum_c g (A1 - A2), 0, 0) of interpolate."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        g = self._a(d_out)
        d = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_interpolate_bwd_rast(B, H, W, Cn, abs_, attr.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, g.ctypes.data,
                                          d.ctypes.data)
        return d

    def aa_topology(self, tris):
        """int32 [T,3]: triangle across edge (tri[t,k], tri[t,(k+1)%3]), -1 boundary, -2 three or more triangles."""
        tris = np.ascontiguousarray(tris, np.int32)
        adj = np.zeros(tris.shape, np.int32)
        self.lib.orc_aa_topology(tris.shape[0], tris.ctypes.data, adj.ctypes.data)
        return adj

    def _aa_args(self, color, rast, pos, tris, adj):
        color = self._a(color)
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        adj = self.aa_topology(tris) if adj is None else np.ascontiguousarray(adj, np.int32)
        keep = (color, rast, pos, tris, adj)
        args = [B, H, W, color.shape[3], color.ctypes.data, rast.ctypes.data, pbs, pos.ctypes.data, tris.shape[0], tris.ctypes.data,
                adj.ctypes.data]
        return keep, args

    def antialias(self, color, rast, pos, tris, adj=None):
        keep, args = self._aa_args(color, rast, pos, tris, adj)
        out = np.zeros_like(keep[0])
        self.lib.orc_antialias_fwd(*args, out.ctypes.data)
        return out

    def antialias_bwd(self, color, rast, pos, tris, d_out, adj=None, scatter=False, terms="sum"):
        """-> (d_color, d_pos).  d_color is gathered per pixel in the kernel's order (the fp32 build equals k_antialias<true> bit for
        bit), or with scatter=True accumulated pair by pair; d_pos is always the pair-by-pair scatter, in the `terms` mode."""
        keep, args = self._aa_args(color, rast, pos, tris, adj)
        g = self._a(d_out, keep[0].shape)
        dc = np.zeros_like(keep[0]); dp = np.zeros_like(keep[2])
        self.lib.orc_antialias_bwd(*args, g.ctypes.data, dc.ctypes.data, dp.ctypes.data, TERMS[terms])
        if not scatter:
            self.lib.orc_antialias_bwd_color(*args, g.ctypes.data, dc.ctypes.data)
        return dc, dp

    def antialias_pair_t(self, rast, pos, tris, adj=None):
        """[B,H,W,2]: t of the crossing edge of each pixel's right (0) and down (1) pair, NaN where the pair has none (t = 1/2: no blend)."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        adj = self.aa_topology(tris) if adj is None else np.ascontiguousarray(adj, np.int32)
        t = np.zeros((B, H, W, 2), self.dt)
        self.lib.orc_antialias_pair_t(B, H, W, rast.ctypes.data, pbs, pos.ctypes.data, tris.shape[0], tris.ctypes.data, adj.ctypes.data,
                                      t.ctypes.data)
        return t

    def interpolate(self, attr, tris, rast):
        """out [B,H,W,C] = fma(u, A0, fma(v, A1, (1 - u - v) A2)), 0 without a hit (the kernel's operation order)."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        out = np.zeros((B, H, W, Cn), self.dt)
        self.lib.orc_interpolate_fwd(B, H, W, Cn, abs_, attr.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, out.ctypes.data)
        return out

    def rast_db(self, pos, tris, rast):
        """rast_db [B,H,W,4] = (du/dX, du/dY, dv/dX, dv/dY) of the clip-space triangle under each covered pixel (0 elsewhere)."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        db = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_rast_db(B, H, W, pbs, pos.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, db.ctypes.data)
        return db

    def rast_db_bwd(self, pos, tris, rast, d_db, terms="sum"):
        """d pos (shape of pos) from d rast_db, in the `terms` mode."""
        pos, rast, tris, B, H, W, pbs = self._geo(pos, rast, tris)
        g = self._a(d_db); d = np.zeros_like(pos)
        self.lib.orc_rast_db_bwd(B, H, W, pbs, pos.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, g.ctypes.data, d.ctypes.data,
                                 TERMS[terms])
        return d

    @staticmethod
    def _sel(diff_attrs, Cn):
        if isinstance(diff_attrs, str):
            assert diff_attrs == "all"
            return Cn, None, None
        idx = np.ascontiguousarray(diff_attrs, np.int32)
        return idx.shape[0], idx, idx.ctypes.data

    def interpolate_da(self, attr, tris, rast, db, diff_attrs="all"):
        """out_da [B,H,W,2n]: (dA/dX, dA/dY) of each selected attribute ('all' or a list of indices)."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        db = self._a(db)
        n, keep, ip = self._sel(diff_attrs, Cn)
        out = np.zeros((B, H, W, 2 * n), self.dt)
        self.lib.orc_interpolate_da(B, H, W, Cn, abs_, attr.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, db.ctypes.data, n, ip,
                                    out.ctypes.data)
        return out

    def interpolate_da_bwd(self, attr, tris, rast, db, d_out_da, diff_attrs="all", terms="sum"):
        """-> (d attr, d rast_db) of out_da; d attr in the `terms` mode, where the third vertex's term -(a0 + a1) counts as |a0| + |a1|
        and as one term when a0 or a1 is non-zero."""
        attr, rast, tris, B, H, W, Cn, abs_ = self._attr(attr, tris, rast)
        db = self._a(db); g = self._a(d_out_da)
        n, keep, ip = self._sel(diff_attrs, Cn)
        da = np.zeros_like(attr); ddb = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_interpolate_da_bwd(B, H, W, Cn, abs_, attr.ctypes.data, tris.shape[0], tris.ctypes.data, rast.ctypes.data, db.ctypes.data, n,
                                        ip, g.ctypes.data, da.ctypes.data, ddb.ctypes.data, TERMS[terms])
        return da, ddb


geometry_oracle = GeometryOracle.get
