"""GPU: the stage that gives the geometry its gradient, against the oracle (oracle/geometry.c) on the inputs where it can go wrong.
antialias forward and d color, and interpolate forward and d rast, have one writer per output and equal the fp32 oracle bit for bit;
antialias d pos, rasterize d pos (with and without rast_db) and interpolate d attr are float-atomic sums, held per element to the fp64
oracle run on the same fp32 inputs, with the reduction floor n 2^-24 A of their terms (tests/common.py: check_scatter_fp64).  Every case
starts from (v, f, mtx): rast comes from the GPU rasterize (bit-identical to the oracle's), pos from the oracle's xfm.  Cases: image shapes
from 1x1 to 129x257 with B in {1, 3, 8}; every test camera (w <= 0 vertices, empty images); duplicated (non-manifold edges, z ties),
zero-area, single-triangle, beyond-the-far-plane and holed meshes; grids whose edges run through pixel centres or midway between them
(t = 1/2); every peel layer; ids >= T; one [V,4] shared by the batch; C from 1 to 12 with NaN and +-inf colours; the training shape."""
import time

import numpy as np
import pytest
import torch

from common import RASTER_CAMERAS, check_scatter_fp64, nan_bits, oracle, pixel_grid_mesh, raster_mesh, raster_mtx, same_bits
from oracle.geometry import geometry_oracle
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _t(dev, a):
    return torch.tensor(np.ascontiguousarray(a), device=dev)


def _ctx(dev, v, f):
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, _t(dev, v), _t(dev, f), rebuild=1)
    return ctx


def _layer(ctx, m, res, k, pos=None, tri=None, grad_db=False):
    """G-buffer layer k (0: rasterize, else the k-th DepthPeeler layer), differentiable in pos when pos is given"""
    from nvdiffrecmc_b200.raster import DepthPeeler, rasterize
    if k == 0:
        return rasterize(ctx, m, res, pos=pos, tri=tri, grad_db=grad_db)
    with DepthPeeler(ctx, m, res, pos, tri, grad_db=grad_db) as p:
        for _ in range(k + 1):
            out = p.rasterize_next_layer()
    return out if grad_db else out[0]


def _geo(f64):
    return geometry_oracle(f64=f64)


def _bar(what, got, fn, ins, seed=0):
    """check_scatter_fp64 of one scatter: fn(o, ins, terms) is the oracle o's output on the inputs ins (pos or rast_db, and the
    upstream gradients, which Delta perturbs) in the mode `terms`"""
    return check_scatter_fp64(what, got, lambda x: [fn(_geo(True), x, "sum")], lambda x: [fn(_geo(False), x, "sum")], ins,
                              lambda f64: (fn(_geo(f64), ins, "count"), fn(_geo(f64), ins, "abs")), seed=seed, tag="geometry")


def _poison(color, rast):
    """NaN, +inf and -inf in a few silhouette pixels (a pixel whose right neighbour has another triangle)"""
    c = color.copy()
    sil = np.argwhere(rast[:, :, :-1, 3] != rast[:, :, 1:, 3])
    for k, (b, y, x) in enumerate(sil[::max(1, len(sil) // 6)][:6]):
        c[b, y, x + k % 2, k % c.shape[3]] = [np.nan, np.inf, -np.inf][k % 3]
    return c


def _check_antialias(dev, f, pos, rast, C, seed, poison=False):
    """antialias_topology equal to the oracle's; forward and d color bit for bit (d color the same with and without pos requiring grad);
    d pos per element against the fp64 oracle, exactly 0 on vertices with w <= 0, and the same without color requiring grad."""
    from nvdiffrecmc_b200.raster import antialias, antialias_topology
    g32, g64 = geometry_oracle(), geometry_oracle(f64=True)
    rng = np.random.default_rng(seed)
    color = rng.uniform(-1, 2, rast.shape[:3] + (C,)).astype(np.float32)
    g = rng.standard_normal(color.shape).astype(np.float32)
    ft, rt, gt = _t(dev, f), _t(dev, rast), _t(dev, g)
    topo = antialias_topology(ft)
    adj = g32.aa_topology(f)
    assert np.array_equal(topo.cpu().numpy(), adj)

    col, p = _t(dev, color).requires_grad_(True), _t(dev, pos).requires_grad_(True)
    out = antialias(col, rt, p, ft, topo)
    got, ref = out.detach().cpu().numpy(), g32.antialias(color, rast, pos, f, adj)
    assert same_bits(got, ref), "antialias: %d of %d values differ" % ((got != ref).sum(), got.size)
    out.backward(gt)
    dc32, dp32 = g32.antialias_bwd(color, rast, pos, f, g, adj)
    dc, dp = col.grad.cpu().numpy(), p.grad.cpu().numpy()
    assert same_bits(dc, dc32), "antialias d color: %d of %d values differ" % ((dc != dc32).sum(), dc.size)
    _, dp64 = g64.antialias_bwd(color, rast, pos, f, g, adj, scatter=True)
    _bar("antialias d pos", dp, lambda o, x, t: o.antialias_bwd(color, rast, x[0], f, x[1], adj, scatter=True, terms=t)[1], [pos, g], seed)
    assert (dp[pos[..., 3] <= 0] == 0).all()

    c1, p1 = _t(dev, color).requires_grad_(True), _t(dev, pos)
    antialias(c1, rt, p1, ft, topo).backward(gt)                         # d color alone
    assert same_bits(c1.grad.cpu().numpy(), dc32)
    c2, p2 = _t(dev, color), _t(dev, pos).requires_grad_(True)
    antialias(c2, rt, p2, ft, topo).backward(gt)                         # d pos alone
    aa_bwd = lambda o, x, t: o.antialias_bwd(color, rast, x[0], f, x[1], adj, scatter=True, terms=t)[1]
    _bar("antialias d pos (d pos alone)", p2.grad.cpu().numpy(), aa_bwd, [pos, g], seed)
    if not (rast[..., 3] > 0).any():                                     # an empty image passes through untouched
        assert same_bits(got, color) and same_bits(dc, g) and (dp == 0).all()
    if poison:
        bad = _poison(color, rast)
        got = antialias(_t(dev, bad), rt, _t(dev, pos), ft, topo).cpu().numpy()
        ref = g32.antialias(bad, rast, pos, f, adj)
        assert np.array_equal(nan_bits(got), nan_bits(ref)), "antialias of non-finite colours: %d values differ" % (nan_bits(got) != nan_bits(ref)).sum()
        assert (~np.isfinite(ref)).sum() >= 6
    return ref, dp64


def _check_rasterize_bwd(dev, ctx, m, res, k, pos, f, rast, seed):
    """d pos of layer k from d rast alone, from d rast + d rast_db and from d rast_db alone, per element against raster_bwd and
    rast_db_bwd of the fp64 oracle; random z/w and id channels in d rast change nothing; an upstream gradient zero on a checkerboard of
    pixels.  With both upstream gradients the statistics of the two scatters add."""
    rng = np.random.default_rng(seed)
    B, H, W = rast.shape[:3]
    g_any = rng.standard_normal((B, H, W, 4)).astype(np.float32)
    g = g_any.copy()
    g[..., 2:] = 0
    g_chk = g.copy()
    g_chk[:, (np.arange(H)[:, None] + np.arange(W)[None]) % 2 == 0] = 0
    h = rng.standard_normal((B, H, W, 4)).astype(np.float32)
    ft = _t(dev, f)

    def run(g=None, h=None):
        p = _t(dev, pos).requires_grad_(True)
        if h is None:
            r = _layer(ctx, m, res, k, p, ft)
            assert same_bits(r.detach().cpu().numpy(), rast)
            r.backward(_t(dev, g))
        else:
            r, db = _layer(ctx, m, res, k, p, ft, grad_db=True)
            ts, gs = ([r, db], [_t(dev, g), _t(dev, h)]) if g is not None else ([db], [_t(dev, h)])
            torch.autograd.backward(ts, gs)
        return p.grad.cpu().numpy()

    r_bwd = lambda o, x, t: o.raster_bwd(x[0], f, rast, x[1], terms=t)
    db_bwd = lambda o, x, t: o.rast_db_bwd(x[0], f, rast, x[1], terms=t)
    for gg, what in ((g, "rasterize d pos"), (g_chk, "rasterize d pos (checkerboard)")):
        _bar(what, run(gg), r_bwd, [pos, gg], seed)
    _bar("rasterize d pos (random z/w, id)", run(g_any), r_bwd, [pos, g], seed)
    _bar("rasterize_db d pos", run(g, h), lambda o, x, t: r_bwd(o, x[:2], t) + db_bwd(o, [x[0], x[2]], t), [pos, g, h], seed)
    _bar("rasterize_db d pos (rast_db only)", run(None, h), db_bwd, [pos, h], seed)


def _check_interpolate(dev, f, rast, V, seed, chans=(1, 5, 9)):
    """forward and d rast bit for bit against the fp32 oracle for [V,C] and [B,V,C] attributes (d rast the same without attr requiring
    grad), d attr per element against the fp64 oracle"""
    from nvdiffrecmc_b200.raster import interpolate
    g32 = geometry_oracle()
    rng = np.random.default_rng(seed)
    ft, rt = _t(dev, f), _t(dev, rast)
    for Cn in chans:
        for batched in (False, True):
            attr = rng.uniform(-1, 1, ((rast.shape[0],) if batched else ()) + (V, Cn)).astype(np.float32)
            g = rng.standard_normal(rast.shape[:3] + (Cn,)).astype(np.float32)
            a, r = _t(dev, attr).requires_grad_(True), rt.clone().requires_grad_(True)
            out, _ = interpolate(a, r, ft)
            assert same_bits(out.detach().cpu().numpy(), g32.interpolate(attr, f, rast)), "interpolate C=%d" % Cn
            out.backward(_t(dev, g))
            dr = g32.interpolate_bwd_rast(attr, f, rast, g)
            got = r.grad.cpu().numpy()
            assert same_bits(got, dr), "interpolate d rast C=%d: %d values differ" % (Cn, (got != dr).sum())
            r2 = rt.clone().requires_grad_(True)
            interpolate(_t(dev, attr), r2, ft)[0].backward(_t(dev, g))
            assert same_bits(r2.grad.cpu().numpy(), dr)
            _bar("interpolate d attr C=%d%s" % (Cn, " [B,V,C]" if batched else ""), a.grad.cpu().numpy(),
                 lambda o, x, t: o.interpolate_bwd_attr(attr.shape, f, rast, x[0], terms=t), [g], seed)


def _run(dev, v, f, mtx, res, layers=(0,), C=4, T=None, pos=None, seed=0, chans=(1, 5, 9), poison=False):
    """Every check on the given layers of the G-buffer of (v, f, mtx); the ops see only f[:T].  Returns the rast of each layer."""
    ctx, m = _ctx(dev, v, f), _t(dev, mtx)
    pos = oracle().xfm(v[None], mtx) if pos is None else pos
    f = f[:T] if T is not None else f
    out = []
    for k in layers:
        rast = _layer(ctx, m, res, k).cpu().numpy()
        _check_antialias(dev, f, pos, rast, C, seed + k, poison)
        _check_rasterize_bwd(dev, ctx, m, res, k, pos, f, rast, seed + k)
        _check_interpolate(dev, f, rast, v.shape[0], seed + k, chans)
        out.append(rast)
    return out


SHAPES = [(1, 1), (1, 37), (37, 1), (48, 64), (129, 257)]


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("res", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_shapes_and_batches(dev, res, B):
    v, f = raster_mesh("blob+torus")
    (rast,) = _run(dev, v, f, raster_mtx("persp", B, aspect=res[1] / res[0]), res)
    if res[0] * res[1] > 1000:
        assert (rast[..., 3] > 0).sum() > 0.1 * rast[..., 0].size


@pytest.mark.parametrize("cam", RASTER_CAMERAS)
def test_cameras(dev, cam):
    v, f = raster_mesh("blob+torus")
    res = (48, 64)
    mtx = raster_mtx(cam, 3, aspect=res[1] / res[0])
    (rast,) = _run(dev, v, f, mtx, res)
    if cam in ("away", "singular"):
        assert (rast == 0).all()
        return
    assert (rast[..., 3] > 0).sum() > 500
    if cam == "behind":                        # covered pixels whose triangle has a vertex with w <= 0
        pos = oracle().xfm(v[None], mtx)
        b, y, x = np.nonzero(rast[..., 3] > 0)
        ids = rast[b, y, x, 3].astype(np.int64) - 1
        assert (pos[b[:, None], f[ids], 3] <= 0).any(-1).sum() > 50


def _holes(f, seed=0):
    return f[np.random.default_rng(seed).random(f.shape[0]) > 0.1]


@pytest.mark.parametrize("mesh", ["dup", "degenerate", "single", "far", "holes"])
def test_meshes(dev, mesh):
    res = (48, 64)
    v, f = raster_mesh("blob+torus" if mesh == "holes" else mesh)
    if mesh == "holes":
        f = _holes(f)
    mtx = raster_mtx("front" if mesh == "far" else "persp", 3, aspect=res[1] / res[0])
    pos = oracle().xfm(v[None], mtx)
    if mesh == "degenerate":
        # Collapse one edge of a third of the visible triangles in pos: their pixels have S == 0 exactly
        rast = oracle().scene(v, f).rasterize(mtx, res)[0]
        b, y, x = np.nonzero(rast[..., 3] > 0)
        ids = rast[b, y, x, 3].astype(np.int64) - 1
        pos[:, f[np.unique(ids)[::3], 1]] = pos[:, f[np.unique(ids)[::3], 0]]
        assert (pos[:, f[:, 0]] == pos[:, f[:, 1]]).all(-1)[b, ids].sum() > 100
    (rast,) = _run(dev, v, f, mtx, res, pos=pos)
    adj = geometry_oracle().aa_topology(f)
    assert (rast[..., 3] > 0).sum() > 200
    if mesh == "dup":
        assert (adj == -2).all()
    if mesh in ("single", "holes"):
        assert (adj == -1).any()
    if mesh == "far":
        assert ((rast[..., 3] > f.shape[0] - 2) & (rast[..., 2] > 1)).sum() > 1000


@pytest.mark.parametrize("offset", [0.5, 1.0], ids=["on-centres", "midway"])
def test_pixel_grids(dev, offset):
    """A holed planar grid for the identity matrix.  on-centres: vertices on pixel centres, so the rim runs through centres (e = 0, no
    crossing).  midway: vertices on pixel corners of a power-of-two image, so the rim lies exactly midway between centres (t = 1/2 in
    fp32, no blend)."""
    res = (37, 53) if offset == 0.5 else (32, 64)
    v, f = pixel_grid_mesh(*res, offset=offset)
    f = _holes(f, 1)
    mtx = np.stack([np.eye(4), np.eye(4)]).astype(np.float32)
    mtx[1, 2, 3] = 0.25
    (rast,) = _run(dev, v, f, mtx, res)
    t = geometry_oracle().antialias_pair_t(rast, oracle().xfm(v[None], mtx), f)
    ids = rast[..., 3]
    differ = np.stack([np.pad(ids[:, :, :-1] != ids[:, :, 1:], ((0, 0), (0, 0), (0, 1))),
                       np.pad(ids[:, :-1] != ids[:, 1:], ((0, 0), (0, 1), (0, 0)))], -1)
    if offset == 1.0:
        assert (t == 0.5).sum() > 100
    else:
        assert (differ & np.isnan(t)).sum() > 100


@pytest.mark.parametrize("mesh", ["blob+torus", "dup"])
def test_peel_layers(dev, mesh):
    v, f = raster_mesh(mesh)
    res = (48, 64)
    mtx = raster_mtx("persp", 2, aspect=res[1] / res[0])
    n = 0
    t = None
    while True:                                # the layer count, from the oracle
        r, t = oracle().scene(v, f).rasterize(mtx, res, t)
        n += 1
        if not (r[..., 3] > 0).any():
            break
    rasts = _run(dev, v, f, mtx, res, layers=range(n))
    assert n >= 4 and (rasts[1][..., 3] > 0).sum() > 300 and not (rasts[-1][..., 3] > 0).any()


def test_ids_at_or_above_T(dev):
    """rast of the whole mesh, ops given its first half: pixels with ids >= T are background everywhere"""
    v, f = raster_mesh("blob+torus")
    T = f.shape[0] // 2
    res = (48, 64)
    (rast,) = _run(dev, v, f, raster_mtx("persp", 3, aspect=res[1] / res[0]), res, T=T)
    assert (rast[..., 3] > T).sum() > 500 and ((rast[..., 3] > 0) & (rast[..., 3] <= T)).sum() > 500


@pytest.mark.parametrize("B", [3, 8])
def test_shared_pos(dev, B):
    """one [V,4] pos for a batch of one repeated matrix (different colours per view): every view scatters into the same rows"""
    v, f = raster_mesh("blob+torus")
    res = (48, 64)
    mtx = np.repeat(raster_mtx("offaxis", 1, aspect=res[1] / res[0]), B, 0)
    _run(dev, v, f, mtx, res, pos=oracle().xfm(v[None], mtx[:1])[0])


@pytest.mark.parametrize("C", [1, 3, 4, 7, 12])
def test_colours(dev, C):
    v, f = raster_mesh("blob+torus")
    res = (48, 64)
    _run(dev, v, f, raster_mtx("persp", 2, aspect=res[1] / res[0]), res, C=C, seed=C, chans=(), poison=True)


def test_training_shape(dev):
    """8 x 512^2 on the bench mesh, C = 4, the whole image"""
    import bench
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    B, res = 8, (512, 512)
    mtx = np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32)
    t0 = time.time()
    (rast,) = _run(dev, v, f, mtx, res, chans=(4,))
    print("8 x 512^2: %.1f s" % (time.time() - t0))
    assert (rast[..., 3] > 0).sum() > 100000
