"""DMTet's per-iteration geometry on the GPU: drop-ins for the reference's `marching_tets` and `sdf_reg_loss` (geometry/dmtet.py:91-153),
run by the kernels of csrc/dmtet.cu (semantics stated there).

`marching_tets(pos_nx3, sdf_n, tet_fx4) -> (verts, faces, uvs, uv_idx)` returns what the reference returns -- the same vertex order, faces,
UVs and uv_idx, bit for bit -- without sorting anything per call: the grid's edges, each tet's six edge rows, a vertex -> edge adjacency
and the UV table are built once per index tensor and cached.  One extraction makes exactly one device -> host read (the vertex and face
counts, to size the outputs).  `verts` is differentiable in `pos_nx3` and `sdf_n`; the backward is a per-vertex gather, deterministic and
free of atomics.  `uvs` depends only on the number of tets: the SAME cached tensor is returned by every call on a grid, so treat it as
read-only (the reference's callers only read it).

`sdf_reg_loss(sdf, all_edges)` returns the reference's regulariser as a 0-dim device tensor; neither it nor its backward synchronises
the host, and both can be captured in a CUDA graph.

The cache is keyed by the index tensor itself (a weak reference) and its version counter, so an in-place change of the indices, or a new
tensor at a reused address, rebuilds the tables.  Building validates the indices (ValueError if one is outside [0, V)).
"""
import weakref

import numpy as np
import torch

from . import _lib as L

__all__ = ["marching_tets", "sdf_reg_loss"]

_BASE_EDGES = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))


class _Grid:
    """Static tables of one tet grid (layout in include/mcshade.h)."""

    def __init__(self, tet, V):
        dev = tet.device
        T = tet.shape[0]
        t64 = tet.to(torch.int64)
        lo, hi = torch.stack([t64.min(), t64.max()]).tolist()
        if lo < 0 or hi >= V:
            raise ValueError("marching_tets: tet_fx4 holds vertex index %d, outside [0, %d)" % (lo if lo < 0 else hi, V))
        ends = t64[:, [i for e in _BASE_EDGES for i in e]].reshape(T * 6, 2)
        a, b = torch.minimum(ends[:, 0], ends[:, 1]), torch.maximum(ends[:, 0], ends[:, 1])
        keys, rows = torch.unique(a * V + b, sorted=True, return_inverse=True)      # lexicographic (a, b) order
        self.V, self.T, self.E = V, T, keys.shape[0]
        self.edges = torch.stack([keys // V, keys % V], 1).to(torch.int32).contiguous()
        self.tet_edges = rows.reshape(T, 6).to(torch.int32).contiguous()
        self.tets = tet.to(torch.int32, copy=True).contiguous()        # a copy: the cache must not keep its key alive
        self.v2e_offsets, self.v2e_edges = _adjacency(self.edges, V)
        self.uvs = _uv_table(T, dev)


def _adjacency(edges, V):
    """Vertex -> edge CSR: for each vertex, the rows of `edges` it is an end of, in ascending order."""
    ends = edges.reshape(-1).to(torch.int64)                    # a0, b0, a1, b1, ...: row order within each vertex
    order = torch.sort(ends, stable=True).indices
    adj = (order // 2).to(torch.int32).contiguous()
    off = torch.zeros(V + 1, dtype=torch.int64, device=edges.device)
    off[1:] = torch.cumsum(torch.bincount(ends, minlength=V), 0)
    return off.to(torch.int32).contiguous(), adj


def _uv_table(T, dev):
    """The reference's per-tet UV quads (map_uv): an N x N lattice, N = ceil(sqrt(T)), four corners per cell offset by 0.9 / N."""
    N = int(np.ceil(np.sqrt((T * 2 + 1) // 2)))
    axis = torch.linspace(0, 1 - (1 / N), N, dtype=torch.float32, device=dev)
    y, x = torch.meshgrid(axis, axis, indexing="ij")
    cell = torch.stack([x, y], -1).reshape(N * N, 1, 2)
    pad = 0.9 / N
    corner = torch.tensor([[0.0, 0.0], [pad, 0.0], [pad, pad], [0.0, pad]], dtype=torch.float32, device=dev)
    return (cell + corner).reshape(-1, 2)


class _EdgeList:
    """sdf_reg_loss's edge list in int32 and its vertex -> edge CSR."""

    def __init__(self, all_edges, V):
        if all_edges.shape[0] > 0:
            lo, hi = torch.stack([all_edges.min(), all_edges.max()]).tolist()
            if lo < 0 or hi >= V:
                raise ValueError("sdf_reg_loss: all_edges holds vertex index %d, outside [0, %d)" % (lo if lo < 0 else hi, V))
        self.V, self.E = V, all_edges.shape[0]
        self.edges = all_edges.to(torch.int32, copy=True).contiguous()
        self.v2e_offsets, self.v2e_edges = _adjacency(self.edges, V)


_GRIDS, _EDGE_LISTS = {}, {}


def _cached(cache, key, V, make):
    ent = cache.get(id(key))
    if ent is not None and ent[0]() is key and ent[1] == key._version and ent[2] == V:
        return ent[3]
    tables = make(key, V)

    def drop(ref, k=id(key)):
        e = cache.get(k)
        if e is not None and e[0] is ref:
            del cache[k]
    cache[id(key)] = (weakref.ref(key, drop), key._version, V, tables)
    return tables


def _check_index(name, t, cols):
    if not isinstance(t, torch.Tensor) or t.dtype not in (torch.int32, torch.int64):
        raise ValueError("%s must be an int32 or int64 tensor" % name)
    if t.dim() != 2 or t.shape[1] != cols:
        raise ValueError("%s must be [n,%d], got %s" % (name, cols, tuple(t.shape)))


def _check_float(name, t, shape):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise ValueError("%s must be a float32 tensor" % name)
    if t.dim() != len(shape) or any(s is not None and t.shape[i] != s for i, s in enumerate(shape)):
        raise ValueError("%s must be %s, got %s" % (name, "[" + ",".join("n" if s is None else str(s) for s in shape) + "]", tuple(t.shape)))


def _extract(pos, sdf, g):
    """Count, read the counts back (the one host read), emit.  -> (verts, faces, uv_idx, vid)."""
    dev = sdf.device
    lib = L.lib()
    vid = torch.empty(g.E, dtype=torch.int32, device=dev)
    tpre = torch.empty(g.T, 2, dtype=torch.int32, device=dev)
    counts = torch.empty(3, dtype=torch.int32, device=dev)
    ws = torch.empty(lib.mcs_dmtet_workspace_bytes(g.E, g.T) // 8, dtype=torch.int64, device=dev)
    L.check(lib.mcs_dmtet_count(sdf.data_ptr(), sdf.stride(0), g.edges.data_ptr(), g.E, g.tets.data_ptr(), g.T, vid.data_ptr(), tpre.data_ptr(),
                                counts.data_ptr(), ws.data_ptr(), L.stream_ptr()), "dmtet_count")
    M, n1, n2 = counts.tolist()
    F = n1 + 2 * n2
    verts = torch.empty(M, 3, dtype=torch.float32, device=dev)
    faces = torch.empty(F, 3, dtype=torch.int64, device=dev)
    uv_idx = torch.empty(F, 3, dtype=torch.int64, device=dev)
    if M > 0:
        L.check(lib.mcs_dmtet_emit(pos.data_ptr(), pos.stride(0), pos.stride(1), sdf.data_ptr(), sdf.stride(0), g.edges.data_ptr(), g.E,
                                   g.tets.data_ptr(), g.tet_edges.data_ptr(), g.T, vid.data_ptr(), tpre.data_ptr(), counts.data_ptr(),
                                   verts.data_ptr(), faces.data_ptr(), uv_idx.data_ptr(), L.stream_ptr()), "dmtet_emit")
    return verts, faces, uv_idx, vid


class _MarchingTets(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, sdf, g):
        verts, faces, uv_idx, vid = _extract(pos, sdf, g)
        ctx.mark_non_differentiable(faces, uv_idx)
        ctx.save_for_backward(pos, sdf)
        ctx.g, ctx.vid = g, vid
        return verts, faces, uv_idx

    @staticmethod
    def backward(ctx, d_verts, _d_faces, _d_uv_idx):
        pos, sdf = ctx.saved_tensors
        g = ctx.g
        d_pos = torch.empty(g.V, 3, dtype=torch.float32, device=pos.device)
        d_sdf = torch.empty(g.V, dtype=torch.float32, device=pos.device)
        if d_verts is None or d_verts.shape[0] == 0:
            d_pos.zero_()
            d_sdf.zero_()
        else:
            d = d_verts.to(torch.float32).contiguous()
            L.check(L.lib().mcs_dmtet_bwd(pos.data_ptr(), pos.stride(0), pos.stride(1), sdf.data_ptr(), sdf.stride(0), g.V, g.edges.data_ptr(), g.E,
                                          ctx.vid.data_ptr(), g.v2e_offsets.data_ptr(), g.v2e_edges.data_ptr(), d.data_ptr(), d_pos.data_ptr(),
                                          d_sdf.data_ptr(), L.stream_ptr()), "dmtet_bwd")
        return (d_pos if ctx.needs_input_grad[0] else None), (d_sdf if ctx.needs_input_grad[1] else None), None


def marching_tets(pos_nx3, sdf_n, tet_fx4):
    """The reference's marching_tets: pos_nx3 [V,3] and sdf_n [V] fp32 (strided views are fine), tet_fx4 [T,4] int32 or int64, all on
    one CUDA device.  -> verts [M,3] fp32, faces [F,3] int64, uvs [4 N^2, 2] fp32 (cached, shared, read-only), uv_idx [F,3] int64."""
    _check_float("marching_tets: pos_nx3", pos_nx3, (None, 3))
    _check_float("marching_tets: sdf_n", sdf_n, (pos_nx3.shape[0],))
    _check_index("marching_tets: tet_fx4", tet_fx4, 4)
    if pos_nx3.shape[0] < 1 or tet_fx4.shape[0] < 1:
        raise ValueError("marching_tets: the grid needs at least one vertex and one tet")
    L.require_cuda(pos_nx3, sdf_n, tet_fx4)
    g = _cached(_GRIDS, tet_fx4, pos_nx3.shape[0], _Grid)
    if torch.is_grad_enabled() and (pos_nx3.requires_grad or sdf_n.requires_grad):
        verts, faces, uv_idx = _MarchingTets.apply(pos_nx3, sdf_n, g)
    else:
        verts, faces, uv_idx, _ = _extract(pos_nx3.detach(), sdf_n.detach(), g)
    return verts, faces, g.uvs, uv_idx


def _reg_fwd(sdf, r):
    dev = sdf.device
    lib = L.lib()
    partials = torch.empty(3 * lib.mcs_sdf_reg_num_partials(r.E), dtype=torch.float64, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    m = torch.empty(1, dtype=torch.float32, device=dev)
    L.check(lib.mcs_sdf_reg_fwd(sdf.data_ptr(), sdf.stride(0), r.edges.data_ptr() if r.E else None, r.E, partials.data_ptr(), loss.data_ptr(),
                                m.data_ptr(), L.stream_ptr()), "sdf_reg_fwd")
    return loss, m


class _SdfRegLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sdf, r):
        loss, m = _reg_fwd(sdf, r)
        ctx.save_for_backward(sdf, m)
        ctx.r = r
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        sdf, m = ctx.saved_tensors
        r = ctx.r
        d = d_loss.to(torch.float32).contiguous()
        d_sdf = torch.empty(r.V, dtype=torch.float32, device=sdf.device)
        L.check(L.lib().mcs_sdf_reg_bwd(sdf.data_ptr(), sdf.stride(0), r.V, r.edges.data_ptr() if r.E else None, r.v2e_offsets.data_ptr(),
                                        r.v2e_edges.data_ptr() if r.E else None, m.data_ptr(), d.data_ptr(), d_sdf.data_ptr(), L.stream_ptr()),
                "sdf_reg_bwd")
        return d_sdf, None


def sdf_reg_loss(sdf, all_edges):
    """The reference's sdf_reg_loss: sdf [V] fp32 (a strided view is fine), all_edges [E,2] int32 or int64 on the same CUDA device.
    -> a 0-dim fp32 device tensor (NaN when no edge changes sign), differentiable in sdf.  The count of sign-changing edges stays on
    the device."""
    _check_float("sdf_reg_loss: sdf", sdf, (None,))
    _check_index("sdf_reg_loss: all_edges", all_edges, 2)
    if sdf.shape[0] < 1:
        raise ValueError("sdf_reg_loss: sdf is empty")
    L.require_cuda(sdf, all_edges)
    r = _cached(_EDGE_LISTS, all_edges, sdf.shape[0], _EdgeList)
    if torch.is_grad_enabled() and sdf.requires_grad:
        return _SdfRegLoss.apply(sdf, r)
    return _reg_fwd(sdf.detach(), r)[0]
