"""GPU, row f2 screen-space derivatives: rast_db from rasterize and peel layers and interpolate's out_da bit for bit against the fp32
oracle, the NDC invariant, the backward passes, errors, CUDA-graph capture, the full 8 x 512^2 size and the render_layer golden."""
import os

import numpy as np
import pytest
import torch

from common import check_scatter_fp64, rel_l2
from oracle.geometry import geometry_oracle
from test_gpu_raster import _scene
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu
RES = (48, 64)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_render_layer_db.npz")


def _setup(dev):
    import nvdiffrecmc_b200.renderutils as ru
    ctx, v, f, vt, ft, mtx = _scene(dev, res=RES)
    m = torch.tensor(mtx, device=dev)
    pos = ru.xfm_points(vt[None], m).detach().contiguous()
    return ctx, v, f, vt, ft, m, pos


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("batched", [False, True])
def test_rast_db_bit_identical_on_rasterize_and_peel_layers(dev, batched):
    from nvdiffrecmc_b200.raster import DepthPeeler, rasterize
    ctx, v, f, vt, ft, m, pos = _setup(dev)
    p = pos if batched else pos[0].contiguous()            # [V,4]: one clip-space triangle set for both images (still well defined)
    o = geometry_oracle()
    rast, db = rasterize(ctx, m, RES, p, ft, grad_db=True)
    assert torch.equal(rast, rasterize(ctx, m, RES))
    r = _np(rast)
    assert (r[..., 3] > 0).sum() > 1000
    ref = o.rast_db(_np(p), f, r)
    assert np.abs(ref).max() > 0 and np.array_equal(_np(db), ref)
    with DepthPeeler(ctx, m, RES, p, ft, grad_db=True) as peeler:
        layers = [peeler.rasterize_next_layer() for _ in range(4)]
    assert torch.equal(layers[0][0], rast) and torch.equal(layers[0][1], db)
    for k, (rk, dk) in enumerate(layers):
        assert np.array_equal(_np(dk), o.rast_db(_np(p), f, _np(rk))), k
    assert (_np(layers[1][0])[..., 3] > 0).sum() > 300
    with DepthPeeler(ctx, m, RES, p, ft) as peeler:
        assert peeler.rasterize_next_layer()[1] is None


@pytest.mark.parametrize("Cn", [1, 4, 7])
@pytest.mark.parametrize("batched", [False, True])
def test_out_da_bit_identical(dev, Cn, batched):
    from nvdiffrecmc_b200.raster import interpolate, rasterize
    ctx, v, f, vt, ft, m, pos = _setup(dev)
    rast, db = rasterize(ctx, m, RES, pos, ft, grad_db=True)
    g = torch.Generator().manual_seed(Cn)
    attr = torch.randn((2, v.shape[0], Cn) if batched else (v.shape[0], Cn), generator=g).to(dev)
    o = geometry_oracle()
    for sel in ("all", [min(2, Cn - 1), 0]):
        out, da = interpolate(attr, rast, ft, rast_db=db, diff_attrs=sel)
        n = Cn if sel == "all" else 2
        assert da.shape == (2, *RES, 2 * n)
        ref = o.interpolate_da(_np(attr), f, _np(rast), _np(db), sel)
        assert np.abs(ref).max() > 0 and np.array_equal(_np(da), ref), sel
        assert torch.equal(out, interpolate(attr, rast, ft)[0])
    assert interpolate(attr, rast, ft, rast_db=db)[1] is None


def test_ndc_invariant(dev):
    """d(Px/Pw)/dX = 2/W and d(Py/Pw)/dY = 2/H on covered pixels, cross terms 0: the derivatives against the pixel grid itself."""
    from nvdiffrecmc_b200.raster import interpolate, rasterize
    ctx, v, f, vt, ft, m, pos = _setup(dev)
    rast, db = rasterize(ctx, m, RES, pos, ft, grad_db=True)
    P, dP = interpolate(pos, rast, ft, rast_db=db, diff_attrs="all")
    P, dP = _np(P).astype(np.float64), _np(dP).astype(np.float64).reshape(2, *RES, 4, 2)
    cov = _np(rast)[..., 3] > 0
    w = np.where(cov, P[..., 3], 1.0)                  # background: w = 0, not evaluated
    q = lambda c, d: (dP[..., c, d] * w - P[..., c] * dP[..., 3, d]) / w ** 2          # d(P_c / P_w) / d(X, Y)[d]
    H, W = RES
    # errors relative to 2/W and 2/H (fp32 barycentrics of the ray tracer, fp32 derivatives): 99.5 % of the covered pixels within 1e-4,
    # every one within 1e-2 (grazing triangles have large derivatives whose fp32 sums cancel)
    err = np.stack([np.abs(q(0, 0) - 2 / W) * W / 2, np.abs(q(1, 1) - 2 / H) * H / 2, np.abs(q(0, 1)) * H / 2, np.abs(q(1, 0)) * W / 2])[:, cov]
    print("NDC invariant, relative error: median %.2e, 99.5%% %.2e, max %.2e" % (np.median(err), np.quantile(err, 0.995), err.max()))
    assert np.quantile(err, 0.995) < 1e-4 and err.max() < 1e-2


def _scatter_bar(what, got, fn, ins):
    """got per element against the fp64 oracle (tests/common.py: check_scatter_fp64); fn(o, ins, terms) is the oracle o's scatter"""
    o = lambda f64: geometry_oracle(f64=f64)
    check_scatter_fp64(what, got, lambda x: [fn(o(True), x, "sum")], lambda x: [fn(o(False), x, "sum")], ins,
                       lambda f64: (fn(o(f64), ins, "count"), fn(o(f64), ins, "abs")), tag="raster_db")


def test_backward(dev):
    from nvdiffrecmc_b200.raster import interpolate, rasterize
    ctx, v, f, vt, ft, m, pos0 = _setup(dev)
    o = geometry_oracle()
    gen = torch.Generator().manual_seed(7)
    # interpolate: d rast_db bit for bit, d attr per element against the fp64 oracle (Delta from rast_db and d out_da)
    rast, db0 = rasterize(ctx, m, RES, pos0, ft, grad_db=True)
    attr = torch.randn(v.shape[0], 3, generator=gen).to(dev).requires_grad_(True)
    db = db0.clone().requires_grad_(True)
    _, da = interpolate(attr, rast, ft, rast_db=db, diff_attrs=[2, 0, 2])
    g = torch.randn(da.shape, generator=gen).to(dev)
    da.backward(g)
    ref_a, ref_db = o.interpolate_da_bwd(_np(attr), f, _np(rast), _np(db0), _np(g), [2, 0, 2])
    assert np.array_equal(_np(db.grad), ref_db) and np.abs(ref_db).max() > 0 and np.abs(ref_a).max() > 0
    da_bwd = lambda o, x, t: o.interpolate_da_bwd(_np(attr), f, _np(rast), x[0], x[1], [2, 0, 2], terms=t)[0]
    _scatter_bar("interpolate_da d attr", _np(attr.grad), da_bwd, [_np(db0), _np(g)])
    # only attr needs a gradient / only rast_db does
    a2 = attr.detach().clone().requires_grad_(True)
    interpolate(a2, rast, ft, rast_db=db0, diff_attrs=[2, 0, 2])[1].backward(g)
    _scatter_bar("interpolate_da d attr (attr alone)", _np(a2.grad), da_bwd, [_np(db0), _np(g)])
    db2 = db0.clone().requires_grad_(True)
    interpolate(attr.detach(), rast, ft, rast_db=db2, diff_attrs=[2, 0, 2])[1].backward(g)
    assert torch.equal(db2.grad, db.grad)
    # rasterize: d pos from d rast_db, from d rast, and from both
    g_db = torch.randn(rast.shape, generator=gen).to(dev)
    g_r = torch.randn(rast.shape, generator=gen).to(dev)

    def dpos(use_r, use_db):
        p = pos0.clone().requires_grad_(True)
        r, d = rasterize(ctx, m, RES, p, ft, grad_db=True)
        loss = (r * g_r).sum() * use_r + (d * g_db).sum() * use_db
        loss.backward()
        return _np(p.grad)

    ref_db_pos = o.rast_db_bwd(_np(pos0), f, _np(rast), _np(g_db))
    assert np.abs(ref_db_pos).max() > 0
    only_db, only_r, both = dpos(0.0, 1.0), dpos(1.0, 0.0), dpos(1.0, 1.0)
    r_bwd = lambda o, x, t: o.raster_bwd(x[0], f, _np(rast), x[1], terms=t)
    db_bwd = lambda o, x, t: o.rast_db_bwd(x[0], f, _np(rast), x[1], terms=t)
    both_bwd = lambda o, x, t: r_bwd(o, x[:2], t) + db_bwd(o, [x[0], x[2]], t)
    _scatter_bar("rasterize d pos (rast_db only)", only_db, db_bwd, [_np(pos0), _np(g_db)])
    _scatter_bar("rasterize d pos (rast only)", only_r, r_bwd, [_np(pos0), _np(g_r)])
    _scatter_bar("rasterize d pos (both)", both, both_bwd, [_np(pos0), _np(g_r), _np(g_db)])
    # the C entry point with both gradients in one launch equals the sum of the two single-input launches
    from nvdiffrecmc_b200 import _lib as L
    args = lambda d_r, d_db, out: (pos0.data_ptr(), pos0.shape[1] * 4, pos0.shape[1], ft.data_ptr(), ft.shape[0], rast.data_ptr(), 2, *RES,
                                   d_r, d_db, out.data_ptr(), L.stream_ptr())
    one, a, b = (torch.zeros_like(pos0) for _ in range(3))
    L.check(L.lib().mcs_rasterize_bwd_db(*args(g_r.data_ptr(), g_db.data_ptr(), one)), "t")
    L.check(L.lib().mcs_rasterize_bwd_db(*args(None, g_db.data_ptr(), a)), "t")
    L.check(L.lib().mcs_rasterize_bwd(pos0.data_ptr(), pos0.shape[1] * 4, pos0.shape[1], ft.data_ptr(), ft.shape[0], rast.data_ptr(), 2, *RES,
                                      g_r.data_ptr(), b.data_ptr(), L.stream_ptr()), "t")
    _scatter_bar("mcs_rasterize_bwd_db, both in one launch", _np(one), both_bwd, [_np(pos0), _np(g_r), _np(g_db)])
    _scatter_bar("mcs_rasterize_bwd_db, rast_db only", _np(a), db_bwd, [_np(pos0), _np(g_db)])
    _scatter_bar("mcs_rasterize_bwd", _np(b), r_bwd, [_np(pos0), _np(g_r)])


def test_errors(dev):
    from nvdiffrecmc_b200.raster import DepthPeeler, interpolate, rasterize
    ctx, v, f, vt, ft, m, pos = _setup(dev)
    with pytest.raises(ValueError):
        rasterize(ctx, m, RES, grad_db=True)
    with pytest.raises(ValueError):
        DepthPeeler(ctx, m, RES, grad_db=True)
    rast, db = rasterize(ctx, m, RES, pos, ft, grad_db=True)
    attr = torch.rand(v.shape[0], 3, device=dev)
    with pytest.raises(ValueError):
        interpolate(attr, rast, ft, diff_attrs="all")                       # no rast_db
    for bad in ([3], [-1], [0, 5], "some", []):
        with pytest.raises(ValueError):
            interpolate(attr, rast, ft, rast_db=db, diff_attrs=bad)
    with pytest.raises(ValueError):
        interpolate(attr, rast, ft, rast_db=db, diff_attrs=[0] * 33)
    assert interpolate(attr, rast, ft, rast_db=db, diff_attrs=[1] * 32)[1].shape[-1] == 64
    with pytest.raises(ValueError):
        interpolate(attr, rast, ft, rast_db=db[:1], diff_attrs="all")
    with pytest.raises(ValueError):
        interpolate(attr, rast, ft, rast_db=db[..., :2], diff_attrs="all")


def test_cuda_graph_replay_equals_eager(dev):
    from nvdiffrecmc_b200.raster import DepthPeeler, interpolate
    ctx, v, f, vt, ft, m, pos = _setup(dev)
    tex = torch.rand(v.shape[0], 2, device=dev)

    def run():
        outs = []
        with DepthPeeler(ctx, m, RES, pos, ft, grad_db=True) as p:
            for _ in range(3):
                r, d = p.rasterize_next_layer()
                outs += [r, d, interpolate(pos, r, ft, rast_db=d, diff_attrs="all")[1], interpolate(tex, r, ft, rast_db=d, diff_attrs=[1, 0])[1]]
        return outs

    eager = [t.clone() for t in run()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    for t in captured:
        t.fill_(-1.0)
    graph.replay()
    torch.cuda.synchronize()
    assert (eager[5] != 0).any()
    for a, b in zip(captured, eager):
        assert torch.equal(a, b)


def test_full_size_bench_mesh(dev):
    """8 x 512^2 on the bench mesh: rast_db and out_da of the clip-space positions bit for bit."""
    import bench
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.raster import interpolate, rasterize
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    ctx = ou.OptiXContext()
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    B, res = 8, (512, 512)
    m = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32), device=dev)
    pos = ru.xfm_points(vt[None], m).contiguous()
    rast, db = rasterize(ctx, m, res, pos, ft, grad_db=True)
    _, da = interpolate(pos, rast, ft, rast_db=db, diff_attrs="all")
    o = geometry_oracle()
    r = _np(rast)
    assert (r[..., 3] > 0).sum() > 100000
    ref = o.rast_db(_np(pos), f, r)
    assert np.array_equal(_np(db), ref)
    assert np.array_equal(_np(da), o.interpolate_da(_np(pos), f, r, ref))


def test_render_layer_golden(dev):
    """The product, fed the golden's rast and pos, reproduces what the reference's render_layer computed under nvdiffrast's signature."""
    from nvdiffrecmc_b200.raster import _rast_db_launch, interpolate
    g = np.load(GOLDEN)
    t = lambda k: torch.tensor(g[k], device=dev)
    pos, rast, tri = t("pos"), t("rast"), t("tris")
    db = _rast_db_launch(pos, tri, rast)
    assert np.array_equal(_np(db), g["rast_deriv"])
    texc, texc_deriv = interpolate(t("v_tex"), rast, t("uv_idx"), rast_db=db, diff_attrs="all")
    assert np.array_equal(_np(texc_deriv), g["gb_texc_deriv"])
    assert rel_l2(_np(texc), g["gb_texc"]) < 1e-6
    # render.py:228-234, as written there
    with torch.no_grad():
        eps = 0.00001
        clip_pos, clip_pos_deriv = interpolate(pos, rast, tri, rast_db=db, diff_attrs="all")
        z0 = torch.clamp(clip_pos[..., 2:3], min=eps) / torch.clamp(clip_pos[..., 3:4], min=eps)
        z1 = torch.clamp(clip_pos[..., 2:3] + torch.abs(clip_pos_deriv[..., 2:3]), min=eps) / torch.clamp(clip_pos[..., 3:4] + torch.abs(clip_pos_deriv[..., 3:4]), min=eps)
        gb_depth = torch.cat((z0, torch.abs(z1 - z0)), dim=-1)
    assert rel_l2(_np(gb_depth), g["gb_depth"]) <= 1e-6
