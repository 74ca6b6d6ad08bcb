"""Primary visibility, attribute interpolation and antialiasing without a rasteriser (SURVEY section 8 row f2).

Stand-ins for the nvdiffrast calls of the reference's G-buffer pass (render/render.py:208-234) and of its compositing
(`composite_buffer`, render.py:284-291): `rasterize` traces one primary ray per pixel through the LBVH that `optix_build_bvh`
already built for the shadow rays and returns nvdiffrast's `rast` tensor `(u, v, z/w, triangle_id + 1)`; given the clip-space
vertices `pos` it is differentiable with respect to them through the barycentrics.  `interpolate` evaluates vertex attributes at
those barycentrics and is differentiable with respect to the attributes and to `rast`.  `antialias` is the pixel-pair analytic
antialiasing of Laine et al. 2020, the only path from coverage (alpha) to vertex positions, so silhouette losses train the mesh;
`antialias_topology` builds the edge adjacency it needs on the device.  `DepthPeeler` returns the deeper layers of the same G-buffer
(the next surface along each primary ray), each an ordinary `rast` that `interpolate` and `antialias` take, as render_mesh's
back-to-front `composite_buffer` needs.  Screen-space derivatives come in nvdiffrast's layout: `rasterize(grad_db=True)` and
`DepthPeeler(grad_db=True)` also return `rast_db` (du/dX, du/dY, dv/dX, dv/dY in pixels, from the clip-space triangle), and
`interpolate(..., rast_db=, diff_attrs=)` returns the attribute derivatives `out_da` that render_layer turns into the denoiser's depth
guide (render.py:225-234).  `texture` is nvdiffrast's filtered look-up with its signature, in the modes the reference calls: bilinear
('linear') and trilinear on a mip chain with the level of detail taken from `uv_da` ('linear-mipmap-linear', e.g. `gb_texc_deriv`),
'wrap' or 'clamp' borders, differentiable with respect to the texture, every mip level, uv and uv_da (Texture2D.sample, texture.py:57-68,
its mip chain's backward and the regulariser taps of render.py)."""
import ctypes

import torch
from . import _lib as L


def _check_pos(pos, B, name):
    if pos.dtype != torch.float32:
        raise TypeError("%s: pos must be fp32 [V,4] or [B,V,4]" % name)
    if not (pos.dim() == 2 and pos.shape[1] == 4) and not (pos.dim() == 3 and pos.shape[2] == 4):
        raise ValueError("%s: pos must be [V,4] or [B,V,4], got %s" % (name, tuple(pos.shape)))
    if pos.dim() == 3 and pos.shape[0] != B:
        raise ValueError("%s: pos batch %d does not match %d" % (name, pos.shape[0], B))


def _check_tri(tri, name, what="tri"):
    if tri.dtype != torch.int32:
        raise TypeError("%s: %s must be int32 [T,3]" % (name, what))
    if tri.dim() != 2 or tri.shape[1] != 3 or tri.shape[0] == 0:
        raise ValueError("%s: %s must be a non-empty [T,3], got %s" % (name, what, tuple(tri.shape)))


def _rasterize_launch(optix_ctx, m, resolution, t_state=None):
    B, (H, W) = m.shape[0], resolution
    rast = torch.empty(B, H, W, 4, dtype=torch.float32, device=m.device)
    if t_state is None:
        L.check(L.lib().mcs_rasterize(optix_ctx.cpp_wrapper, m.data_ptr(), B, H, W, rast.data_ptr(), L.stream_ptr()), "rasterize")
    else:
        L.check(L.lib().mcs_rasterize_peel(optix_ctx.cpp_wrapper, m.data_ptr(), B, H, W, t_state.data_ptr(), rast.data_ptr(), L.stream_ptr()),
                "rasterize_peel")
    return rast


def _pos_args(pos):
    V = pos.shape[-2]
    return pos.data_ptr(), V * 4 if pos.dim() == 3 else 0, V


def _rast_db_launch(pos, tri, rast):
    """rast_db [B,H,W,4] of `rast` from the clip-space pos (contiguous fp32) and tri (contiguous int32); no autograd."""
    B, H, W = rast.shape[0], rast.shape[1], rast.shape[2]
    db = torch.empty(B, H, W, 4, dtype=torch.float32, device=rast.device)
    L.check(L.lib().mcs_rast_db(*_pos_args(pos), tri.data_ptr(), tri.shape[0], rast.data_ptr(), B, H, W, db.data_ptr(), L.stream_ptr()), "rast_db")
    return db


class _rasterize_func(torch.autograd.Function):
    """rast of one rasterize or peel launch, or (rast, rast_db) with grad_db; the backward maps d rast and d rast_db to d pos in one
    launch."""
    @staticmethod
    def forward(ctx, pos, tri, optix_ctx, m, resolution, t_state, grad_db):
        ctx.set_materialize_grads(False)
        rast = _rasterize_launch(optix_ctx, m, resolution, t_state)
        ctx.save_for_backward(pos, tri, rast)
        return (rast, _rast_db_launch(pos, tri, rast)) if grad_db else rast

    @staticmethod
    def backward(ctx, d_rast, d_db=None):
        pos, tri, rast = ctx.saved_tensors
        if not ctx.needs_input_grad[0] or (d_rast is None and d_db is None):
            return None, None, None, None, None, None, None
        B, H, W = rast.shape[0], rast.shape[1], rast.shape[2]
        d_pos = torch.zeros_like(pos)
        g = d_rast.to(torch.float32).contiguous() if d_rast is not None else None
        if d_db is None:
            L.check(L.lib().mcs_rasterize_bwd(*_pos_args(pos), tri.data_ptr(), tri.shape[0], rast.data_ptr(), B, H, W, g.data_ptr(), d_pos.data_ptr(),
                                              L.stream_ptr()), "rasterize (backward)")
        else:
            h = d_db.to(torch.float32).contiguous()
            L.check(L.lib().mcs_rasterize_bwd_db(*_pos_args(pos), tri.data_ptr(), tri.shape[0], rast.data_ptr(), B, H, W,
                                                 g.data_ptr() if g is not None else None, h.data_ptr(), d_pos.data_ptr(), L.stream_ptr()),
                    "rasterize_db (backward)")
        return d_pos, None, None, None, None, None, None


def _rasterize_layer(optix_ctx, m, resolution, pos, tri, t_state, grad_db):
    """rast, or (rast, rast_db) with grad_db, of one rasterize or peel launch; differentiable with respect to pos when pos is given."""
    if pos is None:
        return _rasterize_launch(optix_ctx, m, resolution, t_state)
    return _rasterize_func.apply(pos, tri, optix_ctx, m, resolution, t_state, grad_db)


def _rasterize_args(name, mtx, pos, tri, grad_db):
    """Validated (contiguous fp32 mtx, pos, tri) of a rasterize-style call; pos and tri are None together, and grad_db needs them."""
    L.require_cuda(mtx)
    if mtx.dim() != 3 or mtx.shape[1:] != (4, 4):
        raise ValueError("%s: mtx must be [B,4,4]" % name)
    m = mtx.detach().to(torch.float32).contiguous()
    if pos is None:
        if tri is not None:
            raise ValueError("%s: tri is only used together with pos" % name)
        if grad_db:
            raise ValueError("%s: grad_db=True needs pos and tri (the derivatives are those of the clip-space triangle)" % name)
        return m, None, None
    if tri is None:
        raise ValueError("%s: pos needs tri" % name)
    L.require_cuda(pos, tri)
    _check_pos(pos, m.shape[0], name)
    _check_tri(tri, name)
    return m, pos.contiguous(), tri.contiguous()


def rasterize(optix_ctx, mtx, resolution, pos=None, tri=None, grad_db=False):
    """mtx: [B,4,4] clip-space transform (clip = mtx @ (p, 1), the `mtx_in` of render_mesh, render.py:289-293);
    resolution: (H, W).  Returns rast [B,H,W,4] fp32; a pixel whose ray hits nothing is all zeros.

    pos (clip-space vertices [V,4] or [B,V,4], fp32, equal to mtx @ (verts, 1) for the vertices the context's BVH was built from, e.g.
    `ru.xfm_points(v_pos[None], mtx)`) and tri (int32 [T,3]) make the result differentiable with respect to pos: the forward is the
    same ray-traced launch with a bit-identical output, and the backward maps d rast[...,0:2] to d pos through the perspective-correct
    barycentrics of the clip-space triangle.  z/w and the id channel carry no gradient.

    grad_db=True returns (rast, rast_db): rast_db [B,H,W,4] = (du/dX, du/dY, dv/dX, dv/dY) in pixels at each pixel centre, for the
    triangle in rast, from the clip-space triangle (so it needs pos and tri), differentiable with respect to pos."""
    m, pos, tri = _rasterize_args("rasterize", mtx, pos, tri, grad_db)
    return _rasterize_layer(optix_ctx, m, resolution, pos, tri, None, bool(grad_db))


class DepthPeeler:
    """Depth peeling, the stand-in for nvdiffrast's `dr.DepthPeeler` in render_mesh (render/render.py:308-311).  Arguments as
    `rasterize`; use it as a context manager:

        with DepthPeeler(optix_ctx, mtx, (H, W), pos, tri) as peeler:
            for _ in range(num_layers):
                rast, _ = peeler.rasterize_next_layer()

    Each layer is the next surface along every pixel's primary ray: the closest hit with t > t_prev * (1 + 2^-16) in fp32, where
    t_prev is the previous layer's hit (semantics in csrc/raster.cu).  Surfaces closer than that along the ray merge into one layer,
    so a ray through an edge shared by two triangles does not return the same surface twice.  Layer 0 equals `rasterize`; a pixel
    with no further surface is all zeros.  Every layer is an ordinary `rast`: given pos and tri it is differentiable with respect to
    pos exactly like `rasterize`, and `interpolate` and `antialias` take it.  The peeler keeps one fp32 per pixel, zeroed on entry.
    Rebuilding or refitting the context's BVH between layers is an error, as it is for nvdiffrast's peeler to change the geometry.
    grad_db=True (needs pos and tri) makes every layer return (rast, rast_db) with that layer's screen-space derivatives, as
    `rasterize(grad_db=True)`."""

    def __init__(self, optix_ctx, mtx, resolution, pos=None, tri=None, grad_db=False):
        self._m, self._pos, self._tri = _rasterize_args("DepthPeeler", mtx, pos, tri, grad_db)
        self._ctx, self._res = optix_ctx, tuple(resolution)
        self._grad_db = bool(grad_db)
        self._state = None
        self._version = None

    def __enter__(self):
        H, W = self._res
        self._state = torch.zeros(self._m.shape[0], H, W, dtype=torch.float32, device=self._m.device)
        self._version = self._ctx._version
        return self

    def __exit__(self, *exc):
        self._state = None
        return False

    def rasterize_next_layer(self):
        """Returns (rast [B,H,W,4], rast_db [B,H,W,4]) with grad_db=True, else (rast, None), like dr.DepthPeeler.rasterize_next_layer."""
        if self._state is None:
            raise RuntimeError("DepthPeeler.rasterize_next_layer: only inside the peeler's `with` block")
        if self._ctx._version != self._version:
            raise RuntimeError("DepthPeeler.rasterize_next_layer: the BVH was rebuilt or refitted since the peeler started")
        out = _rasterize_layer(self._ctx, self._m, self._res, self._pos, self._tri, self._state, self._grad_db)
        return out if self._grad_db else (out, None)


class _interpolate_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attr, rast, tri):
        a = attr.to(torch.float32).contiguous(); r = rast.to(torch.float32).contiguous(); t = tri.contiguous()
        batched = a.dim() == 3
        V, Cn = a.shape[-2], a.shape[-1]
        B, H, W = r.shape[0], r.shape[1], r.shape[2]
        out = torch.empty(B, H, W, Cn, dtype=torch.float32, device=a.device)
        L.check(L.lib().mcs_interpolate_fwd(a.data_ptr(), V * Cn if batched else 0, V, Cn, t.data_ptr(), t.shape[0], r.data_ptr(), B, H, W,
                                            out.data_ptr(), L.stream_ptr()), "interpolate (forward)")
        ctx.save_for_backward(a, r, t)
        return out

    @staticmethod
    def backward(ctx, dout):
        a, r, t = ctx.saved_tensors
        batched = a.dim() == 3
        V, Cn = a.shape[-2], a.shape[-1]
        B, H, W = r.shape[0], r.shape[1], r.shape[2]
        g = dout.to(torch.float32).contiguous()
        if ctx.needs_input_grad[1]:
            d_attr = torch.zeros_like(a) if ctx.needs_input_grad[0] else None
            d_rast = torch.empty_like(r)
            L.check(L.lib().mcs_interpolate_bwd_rast(a.data_ptr(), V * Cn if batched else 0, V, Cn, t.data_ptr(), t.shape[0], r.data_ptr(), B, H, W,
                                                     g.data_ptr(), d_attr.data_ptr() if d_attr is not None else None, d_rast.data_ptr(),
                                                     L.stream_ptr()), "interpolate (backward)")
            return d_attr, d_rast, None
        d_attr = torch.zeros_like(a)
        L.check(L.lib().mcs_interpolate_bwd(a.data_ptr(), V * Cn if batched else 0, V, Cn, t.data_ptr(), t.shape[0], r.data_ptr(), B, H, W,
                                            g.data_ptr(), d_attr.data_ptr(), L.stream_ptr()), "interpolate (backward)")
        return d_attr, None, None


def _da_args(a, r, db, t, idx):
    batched = a.dim() == 3
    V, Cn = a.shape[-2], a.shape[-1]
    n = Cn if idx is None else len(idx)
    arr = None if idx is None else (ctypes.c_int32 * n)(*idx)       # passed by value into the kernel's parameters (no device tensor)
    return (a.data_ptr(), V * Cn if batched else 0, V, Cn, t.data_ptr(), t.shape[0], r.data_ptr(), db.data_ptr(), r.shape[0], r.shape[1], r.shape[2],
            n, arr), n


class _interpolate_da_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attr, rast_db, rast, tri, idx):
        a = attr.to(torch.float32).contiguous(); db = rast_db.to(torch.float32).contiguous(); r = rast.to(torch.float32).contiguous()
        t = tri.contiguous()
        args, n = _da_args(a, r, db, t, idx)
        out_da = torch.empty(r.shape[0], r.shape[1], r.shape[2], 2 * n, dtype=torch.float32, device=a.device)
        L.check(L.lib().mcs_interpolate_da_fwd(*args, out_da.data_ptr(), L.stream_ptr()), "interpolate_da (forward)")
        ctx.save_for_backward(a, db, r, t)
        ctx.idx = idx
        return out_da

    @staticmethod
    def backward(ctx, d_out_da):
        a, db, r, t = ctx.saved_tensors
        need_a, need_db = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_a or need_db):
            return None, None, None, None, None
        d_attr = torch.zeros_like(a) if need_a else None
        d_db = torch.empty_like(db) if need_db else None
        g = d_out_da.to(torch.float32).contiguous()
        args, _ = _da_args(a, r, db, t, ctx.idx)
        L.check(L.lib().mcs_interpolate_da_bwd(*args, g.data_ptr(), d_attr.data_ptr() if need_a else None, d_db.data_ptr() if need_db else None,
                                               L.stream_ptr()), "interpolate_da (backward)")
        return d_attr, d_db, None, None, None


def _diff_attr_list(diff_attrs, C):
    """None for 'all', else the validated tuple of attribute indices."""
    if isinstance(diff_attrs, str):
        if diff_attrs != "all":
            raise ValueError("interpolate: diff_attrs must be 'all' or a list of attribute indices, got %r" % diff_attrs)
        return None
    idx = tuple(int(k) for k in diff_attrs)
    if not idx or len(idx) > 32:
        raise ValueError("interpolate: diff_attrs lists %d indices; 1 to 32 are allowed" % len(idx))
    bad = [k for k in idx if not 0 <= k < C]
    if bad:
        raise ValueError("interpolate: diff_attrs index %d is outside [0, %d)" % (bad[0], C))
    return idx


def interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
    """attr [V,C] or [B,V,C], rast from `rasterize`, tri int32 [T,3].  Returns (out [B,H,W,C], out_da) like dr.interpolate.

    out_da is None unless diff_attrs is given: 'all', or a list of up to 32 attribute indices (order kept, repeats allowed).  It then
    needs rast_db [B,H,W,4] (from `rasterize(grad_db=True)` or a `DepthPeeler(grad_db=True)` layer) and is [B,H,W,2n] in nvdiffrast's
    layout: channels 2k and 2k+1 hold (dA/dX, dA/dY) of the k-th selected attribute A, zero where rast has no triangle.  out_da is
    differentiable with respect to attr and rast_db (not rast: it does not depend on the barycentrics).  Semantics: csrc/raster.cu."""
    da = diff_attrs is not None
    if da and rast_db is None:
        raise ValueError("interpolate: diff_attrs needs rast_db")
    L.require_cuda(attr, rast, tri, *((rast_db,) if da else ()))
    if tri.dtype != torch.int32:
        raise TypeError("interpolate: tri must be int32 [T,3]")
    if da:
        if rast.dim() != 4 or rast.shape[3] != 4:
            raise ValueError("interpolate: rast must be [B,H,W,4], got %s" % (tuple(rast.shape),))
        if tuple(rast_db.shape) != tuple(rast.shape):
            raise ValueError("interpolate: rast_db must be [B,H,W,4] like rast %s, got %s" % (tuple(rast.shape), tuple(rast_db.shape)))
        if attr.dim() not in (2, 3):
            raise ValueError("interpolate: attr must be [V,C] or [B,V,C], got %s" % (tuple(attr.shape),))
        idx = _diff_attr_list(diff_attrs, attr.shape[-1])
    if attr.dim() == 3 and attr.shape[0] != rast.shape[0]:
        raise ValueError("interpolate: attribute batch %d does not match rast batch %d" % (attr.shape[0], rast.shape[0]))
    out = _interpolate_func.apply(attr, rast, tri)
    return out, (_interpolate_da_func.apply(attr, rast_db, rast.detach(), tri, idx) if da else None)


def antialias_topology(tri):
    """Edge adjacency of a triangle list: int32 [T,3], entry k of triangle t is the triangle across edge (tri[t,k], tri[t,(k+1)%3]),
    -1 on a boundary edge, -2 on an edge shared by three or more triangles.  Built on the device (hash of the undirected edge keys)
    without a host sync; the result depends only on which triangles share each edge, not on the order they are inserted."""
    L.require_cuda(tri)
    _check_tri(tri, "antialias_topology")
    t = tri.contiguous()
    T = t.shape[0]
    ws = torch.empty(int(L.lib().mcs_aa_topology_workspace_bytes(T)), dtype=torch.uint8, device=t.device)
    adj = torch.empty(T, 3, dtype=torch.int32, device=t.device)
    L.check(L.lib().mcs_aa_topology(t.data_ptr(), T, ws.data_ptr(), adj.data_ptr(), L.stream_ptr()), "antialias_topology")
    return adj


def _aa_args(color, rast, pos, tri, topology):
    return (color.data_ptr(), color.shape[3], rast.data_ptr(), rast.shape[0], rast.shape[1], rast.shape[2], *_pos_args(pos), tri.data_ptr(),
            tri.shape[0], topology.data_ptr())


class _antialias_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, color, pos, rast, tri, topology):
        out = torch.empty_like(color)
        L.check(L.lib().mcs_antialias_fwd(*_aa_args(color, rast, pos, tri, topology), out.data_ptr(), L.stream_ptr()), "antialias (forward)")
        ctx.save_for_backward(color, pos, rast, tri, topology)
        return out

    @staticmethod
    def backward(ctx, dout):
        color, pos, rast, tri, topology = ctx.saved_tensors
        g = dout.to(torch.float32).contiguous()
        d_color = torch.empty_like(color) if ctx.needs_input_grad[0] else None
        d_pos = torch.zeros_like(pos) if ctx.needs_input_grad[1] else None
        if d_color is None and d_pos is None:
            return None, None, None, None, None
        L.check(L.lib().mcs_antialias_bwd(*_aa_args(color, rast, pos, tri, topology), g.data_ptr(), d_color.data_ptr() if d_color is not None else None,
                                          d_pos.data_ptr() if d_pos is not None else None, L.stream_ptr()), "antialias (backward)")
        return d_color, d_pos, None, None, None


def antialias(color, rast, pos, tri, topology=None):
    """Analytic antialiasing of `color` [B,H,W,C] (any C >= 1) along silhouette edges, the stand-in for dr.antialias in render_mesh's
    composite_buffer (render/render.py:290).  rast from `rasterize` or a `DepthPeeler` layer, pos the clip-space vertices [V,4] or [B,V,4] it was made from,
    tri int32 [T,3], topology from `antialias_topology(tri)` (built inside the call when None; pass it to share one build between
    the buffers of a frame).  Differentiable with respect to color and pos; rast carries no gradient.  The output is a
    deterministic per-pixel gather and antialias is linear in color for fixed geometry, so channels of several buffers may be
    concatenated into one call.  Semantics: csrc/raster.cu."""
    L.require_cuda(color, rast, pos, tri)
    if color.dim() != 4 or color.shape[3] < 1:
        raise ValueError("antialias: color must be [B,H,W,C], got %s" % (tuple(color.shape),))
    if not color.is_floating_point() or rast.dtype != torch.float32:
        raise TypeError("antialias: color must be floating point and rast fp32")
    if rast.dim() != 4 or rast.shape[3] != 4 or rast.shape[:3] != color.shape[:3]:
        raise ValueError("antialias: rast must be [B,H,W,4] matching color %s, got %s" % (tuple(color.shape), tuple(rast.shape)))
    _check_pos(pos, color.shape[0], "antialias")
    _check_tri(tri, "antialias")
    if topology is None:
        topology = antialias_topology(tri)
    else:
        L.require_cuda(topology)
        _check_tri(topology, "antialias", "topology")
        if topology.shape[0] != tri.shape[0]:
            raise ValueError("antialias: topology has %d rows for %d triangles" % (topology.shape[0], tri.shape[0]))
    return _antialias_func.apply(color.to(torch.float32).contiguous(), pos.contiguous(), rast.detach().contiguous(), tri.contiguous(),
                                 topology.contiguous())


_TEX_FILTERS = {"linear": 0, "linear-mipmap-linear": 1}
_TEX_BOUNDARIES = {"wrap": 0, "clamp": 1}
_TEX_MAX_LEVELS = 16


def _tex_levels(levels):
    lv = L.mcs_texture_levels()
    lv.n_levels, lv.C = len(levels), levels[0].shape[3]
    for k, t in enumerate(levels):
        lv.ptr[k], lv.h[k], lv.w[k] = t.data_ptr(), t.shape[1], t.shape[2]
        lv.batch_stride[k] = 0 if t.shape[0] == 1 else t.shape[1] * t.shape[2] * t.shape[3]
    return lv


class _texture_func(torch.autograd.Function):
    """inputs: filter and boundary codes, uv, uv_da (None in 'linear'), then the levels (level 0 first); one launch each way."""
    @staticmethod
    def forward(ctx, filt, bnd, uv, uv_da, *levels):
        B, H, W = uv.shape[0], uv.shape[1], uv.shape[2]
        out = torch.empty(B, H, W, levels[0].shape[3], dtype=torch.float32, device=uv.device)
        L.check(L.lib().mcs_texture_fwd(ctypes.byref(_tex_levels(levels)), uv.data_ptr(), uv_da.data_ptr() if uv_da is not None else None, B, H, W,
                                        filt, bnd, out.data_ptr(), L.stream_ptr()), "texture_fwd")
        ctx.save_for_backward(uv, uv_da, *levels)
        ctx.codes = (filt, bnd)
        return out

    @staticmethod
    def backward(ctx, dout):
        uv, uv_da, *levels = ctx.saved_tensors
        need = ctx.needs_input_grad
        if not any(need[2:]):
            return (None,) * len(need)
        filt, bnd = ctx.codes
        d_uv = torch.empty_like(uv) if need[2] else None
        d_uv_da = torch.empty_like(uv_da) if need[3] else None
        d_levels = [torch.zeros_like(t) if need[4 + k] else None for k, t in enumerate(levels)]
        ptrs = (ctypes.c_void_p * len(levels))(*[t.data_ptr() if t is not None else None for t in d_levels])
        g = dout.to(torch.float32).contiguous()
        B, H, W = uv.shape[0], uv.shape[1], uv.shape[2]
        L.check(L.lib().mcs_texture_bwd(ctypes.byref(_tex_levels(levels)), uv.data_ptr(), uv_da.data_ptr() if uv_da is not None else None, B, H, W,
                                        filt, bnd, g.data_ptr(), ptrs, d_uv.data_ptr() if d_uv is not None else None,
                                        d_uv_da.data_ptr() if d_uv_da is not None else None, L.stream_ptr()), "texture_bwd")
        return (None, None, d_uv, d_uv_da, *d_levels)


def _check_tex(t, what, Bt=None, C=None):
    if not isinstance(t, torch.Tensor) or t.dim() != 4:
        raise ValueError("texture: %s must be a [Bt,H,W,C] tensor, got %s" % (what, tuple(t.shape) if isinstance(t, torch.Tensor) else type(t)))
    if t.dtype != torch.float32:
        raise ValueError("texture: %s must be fp32, got %s" % (what, t.dtype))
    if t.shape[1] < 1 or t.shape[2] < 1 or t.shape[3] < 1:
        raise ValueError("texture: %s has an empty dimension %s" % (what, tuple(t.shape)))
    if Bt is not None and (t.shape[0] != Bt or t.shape[3] != C):
        raise ValueError("texture: %s is %s; its minibatch and channels must be those of tex (%d, %d)" % (what, tuple(t.shape), Bt, C))


def texture(tex, uv, uv_da=None, mip_level_bias=None, mip=None, filter_mode='auto', boundary_mode='wrap', max_mip_level=None):
    """Filtered texture look-up with nvdiffrast's signature, the stand-in for `dr.texture` in the modes the reference calls.

    tex [Bt,H,W,C] fp32 (any C >= 1; Bt = 1 is shared by the whole minibatch, else Bt = B), uv [B,h,w,2], uv_da [B,h,w,4] =
    (du/dX, du/dY, dv/dX, dv/dY) as `interpolate(..., diff_attrs='all')` returns them for a 2-channel texture coordinate.  Returns
    [B,h,w,C] fp32.  filter_mode 'linear' (level 0 only) or 'linear-mipmap-linear' (trilinear on the chain tex, mip[0], mip[1], ...,
    level k of max(1, H >> k) x max(1, W >> k), up to 16 levels; the chain may stop early); 'auto' is the latter when uv_da is given.
    mip=None in a mipmap mode is accepted for a 1x1 tex only (a one-level chain); build the chain of a larger texture and pass it.
    boundary_mode 'wrap' or 'clamp'.  Differentiable with respect to tex, every mip level, uv and uv_da ('linear' ignores mip and uv_da).
    Not provided (ValueError): 'nearest', 'linear-mipmap-nearest', 'zero', 'cube', mip_level_bias, max_mip_level.  Semantics,
    including the level of detail: csrc/texture.cu."""
    if filter_mode == 'auto':
        filter_mode = 'linear-mipmap-linear' if uv_da is not None else 'linear'
    if filter_mode not in _TEX_FILTERS:
        raise ValueError("texture: filter_mode %r is not provided (only 'linear' and 'linear-mipmap-linear')" % (filter_mode,))
    if boundary_mode not in _TEX_BOUNDARIES:
        raise ValueError("texture: boundary_mode %r is not provided (only 'wrap' and 'clamp')" % (boundary_mode,))
    if mip_level_bias is not None or max_mip_level is not None:
        raise ValueError("texture: mip_level_bias and max_mip_level are not provided")
    mipmap = filter_mode == 'linear-mipmap-linear'
    _check_tex(tex, "tex")
    Bt, H0, W0, C = tex.shape
    if not isinstance(uv, torch.Tensor) or uv.dim() != 4 or uv.shape[3] != 2:
        raise ValueError("texture: uv must be [B,h,w,2], got %s" % (tuple(uv.shape) if isinstance(uv, torch.Tensor) else type(uv),))
    if uv.dtype != torch.float32:
        raise ValueError("texture: uv must be fp32, got %s" % uv.dtype)
    B = uv.shape[0]
    if Bt not in (1, B):
        raise ValueError("texture: tex minibatch %d must be 1 or that of uv (%d)" % (Bt, B))
    levels = [tex]
    if mipmap:
        if uv_da is None:
            raise ValueError("texture: filter_mode 'linear-mipmap-linear' needs uv_da")
        if not isinstance(uv_da, torch.Tensor) or tuple(uv_da.shape) != tuple(uv.shape[:3]) + (4,):
            raise ValueError("texture: uv_da must be [B,h,w,4] like uv %s, got %s" % (tuple(uv.shape), tuple(uv_da.shape) if isinstance(uv_da, torch.Tensor) else type(uv_da)))
        if uv_da.dtype != torch.float32:
            raise ValueError("texture: uv_da must be fp32, got %s" % uv_da.dtype)
        if mip is None:
            if (H0, W0) != (1, 1):
                raise ValueError("texture: filter_mode 'linear-mipmap-linear' on a %d x %d texture needs its chain: pass mip=[level 1, ...]" % (H0, W0))
        else:
            mip = list(mip)
            if len(mip) + 1 > _TEX_MAX_LEVELS:
                raise ValueError("texture: %d levels; at most %d are supported" % (len(mip) + 1, _TEX_MAX_LEVELS))
            for k, m in enumerate(mip, 1):
                _check_tex(m, "mip[%d]" % (k - 1), Bt, C)
                want = (max(1, H0 >> k), max(1, W0 >> k))
                if tuple(m.shape[1:3]) != want:
                    raise ValueError("texture: mip[%d] (level %d) is %d x %d, expected %d x %d" % (k - 1, k, m.shape[1], m.shape[2], *want))
            levels += mip
    else:
        uv_da = None
    L.require_cuda(uv, *levels)
    if uv_da is not None:
        L.require_cuda(uv_da)
        uv_da = uv_da.contiguous()
    return _texture_func.apply(_TEX_FILTERS[filter_mode], _TEX_BOUNDARIES[boundary_mode], uv.contiguous(), uv_da,
                               *[t.contiguous() for t in levels])


class _texel_fetch_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tex, idx):
        L.require_cuda(tex, idx)
        if idx.dtype != torch.int64:
            raise TypeError("texel_fetch: idx must be int64")
        t = tex.to(torch.float32).contiguous(); ix = idx.contiguous()
        T, Cn = t.shape[0], t.shape[1]
        out = torch.empty(*ix.shape, Cn, dtype=torch.float32, device=t.device)
        L.check(L.lib().mcs_texel_fetch_fwd(t.data_ptr(), T, Cn, ix.data_ptr(), ix.numel(), out.data_ptr(), L.stream_ptr()), "texel_fetch (forward)")
        ctx.save_for_backward(ix)
        ctx.shape = (T, Cn)
        return out

    @staticmethod
    def backward(ctx, dout):
        (ix,) = ctx.saved_tensors
        T, Cn = ctx.shape
        d_tex = torch.zeros(T, Cn, dtype=torch.float32, device=ix.device)
        g = dout.to(torch.float32).contiguous()
        L.check(L.lib().mcs_texel_fetch_bwd(T, Cn, ix.data_ptr(), ix.numel(), g.data_ptr(), d_tex.data_ptr(), L.stream_ptr()), "texel_fetch (backward)")
        return d_tex, None


def texel_fetch(tex, idx):
    """tex [T,C] fp32, idx int64 [...] -> [..., C]; `tex[idx]` with an atomic scatter-add backward (nearest-filter material look-up)."""
    return _texel_fetch_func.apply(tex, idx)
