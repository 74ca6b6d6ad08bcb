"""GPU: rasterize and every depth-peel layer (k_invert4 + k_rasterize) bit for bit against the fp32 oracle (oracle/mcoracle.c
orc_rasterize), from the clip matrix to z/w: all four rast channels and the per-pixel peel state after every layer, over image shapes
that leave a partial thread block, batches with a different matrix per view, off-axis / orthographic / wide-range / inside / looking-away
/ singular cameras, meshes with exact ties (duplicated triangles, a grid on the pixel centres), zero-area triangles, one triangle, a
surface beyond the far plane, a refitted and a reused context, the training shape, and the G-buffer chain computed from (v, f, mtx)."""
import numpy as np
import pytest
import torch

from common import oracle, pixel_grid_mesh, raster_mesh, raster_mtx, RASTER_CAMERAS
from common import same_bits as _same
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _ctx(dev, v, f, ctx=None, rebuild=1):
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext() if ctx is None else ctx
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=rebuild)
    return ctx


def _gpu_layer(ctx, m, res, state):
    """One mcs_rasterize_peel launch on the caller's state buffer; rast starts as NaN so an unwritten pixel cannot pass."""
    from nvdiffrecmc_b200 import _lib as L
    B, (H, W) = m.shape[0], res
    rast = torch.full((B, H, W, 4), float("nan"), device=m.device)
    L.check(L.lib().mcs_rasterize_peel(ctx.cpp_wrapper, m.data_ptr(), B, H, W, state.data_ptr(), rast.data_ptr(), L.stream_ptr()), "rasterize_peel")
    return rast


def _check(dev, ctx, sc, mtx, res, max_layers=16):
    """rasterize and then every peel layer until the image is empty, on the GPU and in the oracle; each rast and each state equal bit
    for bit.  Returns the covered-pixel count per layer (the last one 0 unless max_layers ran out)."""
    from nvdiffrecmc_b200.raster import rasterize
    m = torch.tensor(mtx, device=dev)
    r0 = rasterize(ctx, m, res).cpu().numpy()
    ref0, _ = sc.rasterize(mtx, res)
    assert _same(r0, ref0), "rasterize: %d of %d pixels differ" % ((r0 != ref0).any(-1).sum(), r0[..., 0].size)
    state = torch.zeros(mtx.shape[0], *res, device=dev)
    t_ref, cov = None, []
    for k in range(max_layers):
        got = _gpu_layer(ctx, m, res, state).cpu().numpy()
        ref, t_ref = sc.rasterize(mtx, res, t_ref)
        assert _same(got, ref), "layer %d: %d of %d pixels differ" % (k, (got != ref).any(-1).sum(), got[..., 0].size)
        assert _same(state.cpu().numpy(), t_ref), "layer %d: peel state differs" % k
        if k == 0:
            assert _same(got, r0)                                     # layer 0 is rasterize
        cov.append(int((ref[..., 3] > 0).sum()))
        if cov[-1] == 0:
            break
    return cov


SHAPES = [(1, 1), (1, 37), (37, 1), (48, 64), (129, 257)]


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("res", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_shapes_and_batches(dev, res, B):
    v, f = raster_mesh("blob+torus")
    cov = _check(dev, _ctx(dev, v, f), oracle().scene(v, f), raster_mtx("persp", B, aspect=res[1] / res[0]), res)
    if res[0] * res[1] > 1000:
        assert cov[0] > 0.1 * B * res[0] * res[1] and cov[1] > 0 and cov[-1] == 0


@pytest.mark.parametrize("cam", RASTER_CAMERAS)
def test_cameras(dev, cam):
    v, f = raster_mesh("blob+torus")
    res = (48, 64)
    mtx = raster_mtx(cam, 3, aspect=res[1] / res[0])
    cov = _check(dev, _ctx(dev, v, f), oracle().scene(v, f), mtx, res)
    print("%s: covered pixels per layer %s" % (cam, cov))
    if cam in ("away", "singular"):
        assert cov == [0]
    else:
        assert cov[0] > 500 and cov[-1] == 0


def test_singular_and_looking_away_leave_the_state_infinite(dev):
    from nvdiffrecmc_b200.raster import rasterize
    v, f = raster_mesh("blob+torus")
    ctx = _ctx(dev, v, f)
    for cam in ("away", "singular"):
        m = torch.tensor(raster_mtx(cam, 3), device=dev)
        assert (rasterize(ctx, m, (20, 24)) == 0).all()
        state = torch.zeros(3, 20, 24, device=dev)
        assert (_gpu_layer(ctx, m, (20, 24), state) == 0).all() and torch.isinf(state).all() and (state > 0).all()


MESHES = ["blob+torus", "icosphere", "dup", "degenerate", "single", "far"]


@pytest.mark.parametrize("mesh", MESHES)
def test_meshes(dev, mesh):
    v, f = raster_mesh(mesh)
    res = (48, 64)
    mtx = raster_mtx("front" if mesh == "far" else "persp", 3, aspect=res[1] / res[0])
    sc = oracle().scene(v, f)
    cov = _check(dev, _ctx(dev, v, f), sc, mtx, res)
    print("%s: covered pixels per layer %s" % (mesh, cov))
    assert cov[0] > 200 and cov[-1] == 0
    if mesh == "icosphere":
        assert len(cov) == 3                      # front and back, then nothing
    if mesh == "far":                             # the quad beyond the far plane is returned, with z/w > 1 (no far clipping)
        r, _ = sc.rasterize(mtx, res)
        beyond = (r[..., 3] > f.shape[0] - 2) & (r[..., 2] > 1)
        assert beyond.sum() > 1000


@pytest.mark.parametrize("tilt", [0.0, 0.3])
def test_pixel_aligned_grid(dev, tilt):
    """Vertices on pixel centres, so rays run through vertices and along edges: closed Moeller-Trumbore bounds and ties to the lower id."""
    res = (37, 53)
    v, f = pixel_grid_mesh(*res, tilt=tilt)
    mtx = np.stack([np.eye(4), np.eye(4)]).astype(np.float32)
    mtx[1, 2, 3] = 0.25                           # view 1: the same grid, shifted in depth
    cov = _check(dev, _ctx(dev, v, f), oracle().scene(v, f), mtx, res)
    assert cov[0] > 0.8 * 2 * (res[0] - 1) * (res[1] - 1) and len(cov) == 2


def test_refit_then_rasterize_the_moved_mesh(dev):
    v, f = raster_mesh("blob+torus")
    ctx = _ctx(dev, v, f)
    rng = np.random.default_rng(5)
    v2 = (v * np.float32(1.07) + rng.normal(scale=0.01, size=v.shape)).astype(np.float32)
    _ctx(dev, v2, f, ctx=ctx, rebuild=0)
    cov = _check(dev, ctx, oracle().scene(v2, f), raster_mtx("persp", 3), (40, 40))
    assert cov[0] > 300


def test_one_context_across_mesh_sizes(dev):
    ctx = None
    for mesh in ["blob+torus", "single", "dup", "icosphere", "single"]:
        v, f = raster_mesh(mesh)
        ctx = _ctx(dev, v, f, ctx=ctx)
        cov = _check(dev, ctx, oracle().scene(v, f), raster_mtx("persp", 2), (33, 41))
        assert cov[0] > 50, mesh


def _train_pixels(B, H, W, n, seed):
    """flat pixel indices: a 64^2 centre crop of view 0 and n random pixels of all views"""
    ys, xs = np.meshgrid(np.arange(H // 2 - 32, H // 2 + 32), np.arange(W // 2 - 32, W // 2 + 32), indexing="ij")
    crop = (ys * W + xs).reshape(-1)
    rnd = np.random.default_rng(seed).integers(0, B * H * W, n)
    return np.unique(np.concatenate([crop, rnd]))


def test_training_shape(dev):
    """8 x 512^2 on the bench mesh, every peel layer.  The oracle is brute force, so it evaluates a 64^2 crop of view 0 plus 16 k
    random pixels: each pixel's result depends on that pixel's ray and state alone, so a subset is compared exactly."""
    import time
    import bench
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    ctx = _ctx(dev, v, f)
    B, res = 8, (512, 512)
    mtx = np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32)
    from nvdiffrecmc_b200.raster import rasterize
    m = torch.tensor(mtx, device=dev)
    px = _train_pixels(B, *res, 16384, 0)
    sc = oracle().scene(v, f)
    t0 = time.time()
    r0 = rasterize(ctx, m, res).cpu().numpy().reshape(-1, 4)
    ref, t_ref = sc.rasterize(mtx, res, px=px)
    assert _same(r0[px], ref)
    state = torch.zeros(B, *res, device=dev)
    for k in range(8):
        got = _gpu_layer(ctx, m, res, state).cpu().numpy().reshape(-1, 4)
        if k > 0:
            ref, t_ref = sc.rasterize(mtx, res, t_ref, px=px)
        assert _same(got[px], ref), "layer %d: %d of %d pixels differ" % (k, (got[px] != ref).any(-1).sum(), px.size)
        assert _same(state.cpu().numpy().reshape(-1)[px], t_ref), "layer %d: peel state" % k
        assert not np.isnan(got).any()
    assert (ref[:, 3] > 0).sum() < (r0[px, 3] > 0).sum()
    print("8 x 512^2, %d pixels x 8 layers: %.1f s" % (px.size, time.time() - t0))


def test_grid1m_pixels(dev):
    v, f = synth.grid1m_mesh()
    ctx = _ctx(dev, v, f)
    B, res = 2, (512, 512)
    mtx = raster_mtx("persp", B)
    from nvdiffrecmc_b200.raster import rasterize
    got = rasterize(ctx, torch.tensor(mtx, device=dev), res).cpu().numpy().reshape(-1, 4)
    px = np.random.default_rng(1).choice(B * res[0] * res[1], 1024, replace=False)
    ref, _ = oracle().scene(v, f).rasterize(mtx, res, px=px)
    assert _same(got[px], ref) and (ref[:, 3] > 0).sum() > 200


def test_gbuffer_chain_from_the_mesh_and_matrix(dev):
    """rasterize(grad_db=True) -> interpolate(v_tex, diff_attrs='all') -> texture('linear-mipmap-linear'), each output bit for bit
    against the same chain of CPU oracles started from (v, f, mtx) alone, and antialias of the result."""
    from oracle.geometry import geometry_oracle
    from oracle.texture import chain_shapes, texture_oracle
    from nvdiffrecmc_b200.raster import antialias, antialias_topology, interpolate, rasterize, texture
    LML = "linear-mipmap-linear"
    v, f = raster_mesh("blob+torus")
    c = v - v.mean(0)
    v_tex = np.stack([0.5 + np.arctan2(c[:, 2], c[:, 0]) / (2 * np.pi), 0.5 + 0.4 * c[:, 1] / np.abs(c[:, 1]).max()], -1).astype(np.float32)
    B, res = 2, (64, 96)
    mtx = raster_mtx("offaxis", B, aspect=res[1] / res[0])
    o, g, tx = oracle(), geometry_oracle(), texture_oracle()
    pos = o.xfm(v[None], mtx)                                          # clip-space vertices [B,V,4]
    levels = [np.random.default_rng(7).uniform(0, 1, (1, h, w, 3)).astype(np.float32) for h, w in chain_shapes(64, 128, 7)]
    # CPU
    rast, _ = o.scene(v, f).rasterize(mtx, res)
    db = g.rast_db(pos, f, rast)
    uv = g.interpolate(v_tex, f, rast)
    uv_da = g.interpolate_da(v_tex, f, rast, db, "all")
    col = tx.forward(levels, uv, uv_da, filter_mode=LML, boundary_mode="wrap")
    # GPU
    T = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)
    ctx, ft = _ctx(dev, v, f), T(f)
    grast, gdb = rasterize(ctx, T(mtx), res, pos=T(pos), tri=ft, grad_db=True)
    guv, guv_da = interpolate(T(v_tex), grast, ft, rast_db=gdb, diff_attrs="all")
    gcol = texture(T(levels[0]), guv, guv_da, mip=[T(x) for x in levels[1:]], filter_mode=LML, boundary_mode="wrap")
    for name, a, b in [("rast", grast, rast), ("rast_db", gdb, db), ("out", guv, uv), ("out_da", guv_da, uv_da), ("texture", gcol, col)]:
        a = a.detach().cpu().numpy()
        assert _same(a, b), "%s: %d values differ" % (name, (a != b).sum())
    assert (rast[..., 3] > 0).sum() > 1000 and np.abs(uv_da).max() > 0
    aa = antialias(gcol, grast, T(pos), ft, antialias_topology(ft)).cpu().numpy()
    ref = g.antialias(col, rast, pos, f)
    assert (np.abs(ref - col) > 1e-3).sum() > 50
    assert _same(aa, ref), "antialias: %d values differ" % (aa != ref).sum()
