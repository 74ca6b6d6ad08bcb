"""GPU, row f2 depth peeling: trace_closest(t_after=) bit for bit against the brute-force fp32 twin, DepthPeeler layers against the
twin on host-rebuilt rays, no duplicate layers on a closed mesh, gradients through peeled layers, back-to-front compositing, a
silhouette fit that only sees the second layer, CUDA-graph capture, errors, and the full 8 x 512^2 size."""
import numpy as np
import pytest
import torch

from common import rel_l2
from oracle.geometry import geometry_oracle
from peel_oracle import PeelScene
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _rot(ang, tilt=0.0):
    ry = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    rx = np.array([[1, 0, 0], [0, np.cos(tilt), -np.sin(tilt)], [0, np.sin(tilt), np.cos(tilt)]])
    return rx @ ry


def _mtx(views, aspect=1.0, dist=3.0):
    proj = synth.perspective(aspect=aspect, n=0.1, f=10.0).astype(np.float64)
    out = []
    for ang, tilt in views:
        mv = np.eye(4)
        mv[:3, :3] = _rot(ang, tilt)
        mv[2, 3] = -dist
        out.append(proj @ mv)
    return np.stack(out).astype(np.float32)


def _ctx(dev, v, f):
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext()
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    return ctx, vt, ft


def _scene(dev, B=2, res=(48, 64), kind="blob+torus", level=2):
    v, f = synth.scene_mesh(kind, level=level)
    ctx, vt, ft = _ctx(dev, v, f)
    mtx = torch.tensor(_mtx([(0.7 * b + 0.3, 0.2 * b - 0.1) for b in range(B)], aspect=res[1] / res[0]), device=dev)
    return ctx, v, f, vt, ft, mtx


def _host_rays(mtx, res):
    """The pixel rays of k_rasterize rebuilt in float64 through the fp32-rounded inverse: (o [B,H*W,3], d [B,H*W,3])."""
    H, W = res
    ys, xs = np.meshgrid((np.arange(H, dtype=np.float32) + 0.5) / H * 2 - 1, (np.arange(W, dtype=np.float32) + 0.5) / W * 2 - 1, indexing="ij")
    os_, ds = [], []
    for m in mtx:
        inv = np.linalg.inv(m.astype(np.float64)).astype(np.float32).astype(np.float64)
        near = np.stack([xs, ys, -np.ones_like(xs), np.ones_like(xs)], -1) @ inv.T
        far = np.stack([xs, ys, np.ones_like(xs), np.ones_like(xs)], -1) @ inv.T
        o = (near[..., :3] / near[..., 3:]).reshape(-1, 3).astype(np.float32); e = (far[..., :3] / far[..., 3:]).reshape(-1, 3).astype(np.float32)
        os_.append(o); ds.append(e - o)
    return np.stack(os_), np.stack(ds)


def _peel(ctx, mtx, res, n, pos=None, tri=None):
    from nvdiffrecmc_b200.raster import DepthPeeler
    with DepthPeeler(ctx, mtx, res, pos, tri) as p:
        return [p.rasterize_next_layer()[0] for _ in range(n)]


def _random_rays(n, seed, v):
    rng = np.random.default_rng(seed)
    c = v.mean(0); ext = (v.max(0) - v.min(0)).max()
    ro = (c + rng.normal(size=(n, 3)) * ext * 0.7).astype(np.float32)
    rd = (c + rng.normal(size=(n, 3)) * ext * 0.3).astype(np.float32) - ro
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    k = n // 8            # axis-aligned directions (slab-test corner cases)
    rd[:k] = np.eye(3, dtype=np.float32)[rng.integers(0, 3, k)] * rng.choice([-1.0, 1.0], (k, 1)).astype(np.float32)
    return ro, rd.astype(np.float32)


def _ray_parity(dev, ctx, sc, ro, rd, layers):
    """Iterates trace_closest(t_after=) and the twin; every layer must agree bit for bit.  Returns the hit count per layer."""
    import nvdiffrecmc_b200.optixutils as ou
    rot, rdt = torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)
    ta = np.zeros(ro.shape[0], np.float32)
    hits = []
    for k in range(layers):
        tid, tuv = ou.trace_closest(ctx, rot, rdt, t_after=torch.tensor(ta, device=dev))
        rid, rtuv = sc.closest_hit(ro, rd, ta)
        tid, tuv = tid.cpu().numpy(), tuv.cpu().numpy()
        assert np.array_equal(tid, rid), "layer %d: %d of %d rays differ" % (k, (tid != rid).sum(), ro.shape[0])
        assert np.array_equal(tuv, rtuv), "layer %d" % k
        hits.append(int((rid >= 0).sum()))
        ta = np.where(rid >= 0, rtuv[:, 0], np.float32(np.inf)).astype(np.float32)
    return hits


@pytest.mark.parametrize("kind,level", [("blob+torus", 2), ("full", 3)])
def test_trace_closest_after_bit_exact(dev, kind, level):
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh(kind, level=level)
    ctx, _, _ = _ctx(dev, v, f)
    ro, rd = _random_rays(30000, 2, v)
    hits = _ray_parity(dev, ctx, PeelScene(v, f), ro, rd, 6)
    print("%s: hits per layer %s" % (kind, hits))
    assert hits[0] > 5000 and hits[1] > 1000 and hits[2] > 100
    # without t_after, and with t_after = 0: the plain closest-hit query
    rot, rdt = torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)
    a, b = ou.trace_closest(ctx, rot, rdt), ou.trace_closest(ctx, rot, rdt, t_after=torch.zeros(ro.shape[0], device=dev))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_peeled_layers_match_oracle(dev):
    from nvdiffrecmc_b200.raster import rasterize
    res = (48, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    layers = _peel(ctx, mtx, res, 12)
    assert torch.equal(layers[0], rasterize(ctx, mtx, res))
    L = [r.cpu().numpy() for r in layers]
    assert (L[-1] == 0).all()                                          # beyond the scene's depth: all zeros
    assert (L[1][..., 3] > 0).sum() > 500
    for k in range(len(L) - 1):
        c0, c1 = L[k][..., 3] > 0, L[k + 1][..., 3] > 0
        assert not (c1 & ~c0).any()                                    # coverage of layer k+1 within that of layer k
        both = c0 & c1
        assert (L[k + 1][..., 2][both] >= L[k][..., 2][both]).all()     # z/w never decreases
    sc = PeelScene(v, f)
    o, d = _host_rays(mtx.cpu().numpy(), res)
    for b in range(2):
        ref = sc.peel(o[b], d[b], 4)
        for k in range(1, 4):
            got = L[k][b].reshape(-1, 4)
            gid = got[:, 3].astype(np.int64) - 1
            rid, rtuv = ref[k]
            agree = gid == rid
            assert agree.mean() > 0.995, (b, k, agree.mean())          # host-rebuilt rays: a few silhouette pixels may differ
            hit = agree & (rid >= 0)
            assert np.abs(got[hit, 1] - rtuv[hit, 1]).max() < 1e-3 and np.abs(got[hit, 0] - (1 - rtuv[hit, 1] - rtuv[hit, 2])).max() < 1e-3
            assert (got[gid < 0] == 0).all()


def test_closed_convex_mesh_has_two_layers(dev):
    """An icosphere fills the view's centre: every pixel it covers has exactly its front and back, so layer 2 is empty.  Shared
    edges would come back as extra layers without the separation."""
    v, f = synth.icosphere(3)
    v, f = v.astype(np.float32), f.astype(np.int32)
    ctx, _, _ = _ctx(dev, v, f)
    mtx = torch.tensor(_mtx([(0.3, 0.2), (1.9, -0.6)]), device=dev)
    L = [r.cpu().numpy() for r in _peel(ctx, mtx, (256, 256), 3)]
    c0, c1 = L[0][..., 3] > 0, L[1][..., 3] > 0
    assert (L[2] == 0).all()
    rim = int((c0 & ~c1).sum())
    print("icosphere 2 x 256^2: %d covered pixels, %d without a second layer" % (c0.sum(), rim))
    assert c0.sum() > 50000 and not (c1 & ~c0).any()
    assert rim <= 0.005 * c0.sum()


def test_gradients_through_peeled_layers(dev):
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.raster import antialias, antialias_topology
    res = (64, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    pos0 = ru.xfm_points(vt[None], mtx).detach()
    plain = [r.cpu().numpy() for r in _peel(ctx, mtx, res, 3)]
    for k in (1, 2):
        pos = pos0.clone().requires_grad_(True)
        rast = _peel(ctx, mtx, res, k + 1, pos, ft)[k]
        assert rast.grad_fn is not None and np.array_equal(rast.detach().cpu().numpy(), plain[k])
        r = rast.detach().cpu().numpy()
        assert (r[..., 3] > 0).sum() > 300
        g = torch.randn(rast.shape, generator=torch.Generator().manual_seed(3 + k)).to(dev)
        rast.backward(g)
        ref = geometry_oracle().raster_bwd(pos0.cpu().numpy(), f, r, g.cpu().numpy())
        assert np.abs(ref).max() > 0
        assert rel_l2(pos.grad.cpu().numpy(), ref) < 1e-5
    # antialias of a peeled layer, forward and backward
    rast = torch.tensor(plain[1], device=dev)
    color = torch.rand(2, 64, 64, 4, generator=torch.Generator().manual_seed(9)).to(dev)
    col, p = color.clone().requires_grad_(True), pos0.clone().requires_grad_(True)
    out = antialias(col, rast, p, ft, antialias_topology(ft))
    o = geometry_oracle()
    args = (color.cpu().numpy(), plain[1], pos0.cpu().numpy(), f)
    ref = o.antialias(*args)
    assert (np.abs(ref - args[0]) > 1e-3).sum() > 50
    assert rel_l2(out.detach().cpu().numpy(), ref) < 1e-6
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(11)).to(dev)
    out.backward(g)
    dc, dp = o.antialias_bwd(*args, g.cpu().numpy())
    assert np.abs(dp).max() > 0
    assert rel_l2(col.grad.cpu().numpy(), dc) < 1e-6 and rel_l2(p.grad.cpu().numpy(), dp) < 1e-5


def test_back_to_front_compositing(dev):
    """composite_buffer (render/render.py:284-291) without antialias: layers lerped back to front with a constant alpha, against
    the same compositing of the twin's per-ray hit lists."""
    res = (48, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    palette = torch.rand(f.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(dev)
    alpha = 0.4
    layers = _peel(ctx, mtx, res, 4)
    accum = torch.zeros(2, *res, 4, device=dev)
    for rast in reversed(layers):
        tid = rast[..., 3].long() - 1
        col = torch.cat([palette[tid.clamp(min=0)], torch.ones_like(rast[..., :1])], -1)
        accum = torch.lerp(accum, col, (rast[..., 3:4] > 0).float() * alpha)
    got = accum.cpu().numpy().reshape(2, -1, 4)
    sc = PeelScene(v, f)
    o, d = _host_rays(mtx.cpu().numpy(), res)
    pal = palette.cpu().numpy().astype(np.float64)
    for b in range(2):
        ref_layers = sc.peel(o[b], d[b], 4)
        acc = np.zeros((o.shape[1], 4))
        for rid, _ in reversed(ref_layers):
            col = np.concatenate([pal[np.maximum(rid, 0)], np.ones((rid.shape[0], 1))], -1)
            w = (rid >= 0)[:, None] * alpha
            acc = acc + w * (col - acc)
        agree = np.ones(o.shape[1], bool)
        for rast, (rid, _) in zip(layers, ref_layers):
            agree &= rast[b].reshape(-1, 4)[:, 3].cpu().numpy().astype(np.int64) - 1 == rid
        assert agree.mean() > 0.99
        assert (got[b][agree, 3] > alpha + 0.1).sum() > 200                      # pixels with two or more layers blended
        assert np.abs(got[b][agree] - acc[agree]).max() < 1e-5


def test_silhouette_fit_through_the_second_layer(dev):
    """A radius-0.5 sphere inside a fixed radius-1.2 shell, fitted to a radius-0.6 target from four views.  Layer 0 is the shell
    everywhere; the loss sees only layer 1, through antialias of an indicator of the inner sphere's triangles."""
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.raster import DepthPeeler, antialias, antialias_topology
    d, fi = synth.icosphere(3)
    n_in = d.shape[0]
    dirs = torch.tensor(d, dtype=torch.float32, device=dev)
    shell = torch.tensor(d * 1.2, dtype=torch.float32, device=dev)
    ft = torch.tensor(np.concatenate([fi, fi + n_in]).astype(np.int32), device=dev)
    T_in = fi.shape[0]
    topo = antialias_topology(ft)
    e = torch.tensor(np.concatenate([fi[:, [0, 1]], fi[:, [1, 2]], fi[:, [2, 0]]]), device=dev).long()
    res = (128, 128)
    mtx = torch.tensor(_mtx([(0.0, 0.5), (1.6, -0.5), (3.1, 0.6), (4.7, -0.4)]), device=dev)
    ctx = ou.OptiXContext()

    def inner(r, aa=True):
        v = torch.cat([dirs * r[:, None], shell])
        ou.optix_build_bvh(ctx, v.detach(), ft, rebuild=1)
        pos = ru.xfm_points(v[None], mtx)
        with DepthPeeler(ctx, mtx, res, pos, ft) as p:
            p.rasterize_next_layer()
            rast, _ = p.rasterize_next_layer()
        ind = rast[..., 3:4].clamp(0, 1) * (rast[..., 3:4] <= T_in)       # 1 on the inner sphere's triangles (ids 1..T_in)
        return antialias(ind, rast, pos, ft, topo) if aa else ind

    with torch.no_grad():
        target = inner(torch.full((n_in,), 0.6, device=dev))
    r = torch.full((n_in,), 0.5, device=dev, requires_grad=True)
    # control: without antialias the loss gives the vertices no gradient at all
    (g0,) = torch.autograd.grad(torch.nn.functional.mse_loss(inner(r, aa=False), target), r)
    assert (g0 == 0).all()
    opt = torch.optim.Adam([r], lr=0.01)
    losses = []
    for it in range(150):
        img = torch.nn.functional.mse_loss(inner(r), target)
        loss = img + 10.0 * ((r[e[:, 0]] - r[e[:, 1]]) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        if it == 0:
            assert r.grad.abs().max() > 0
        opt.step()
        losses.append(float(img.detach()))
    mean_r = float(r.detach().mean())
    print("peeled silhouette fit: image loss %.3e -> %.3e, mean radius %.4f" % (losses[0], losses[-1], mean_r))
    assert losses[-1] * 10 <= losses[0]
    assert abs(mean_r - 0.6) < 0.05


def test_cuda_graph_replay_equals_eager(dev):
    res = (64, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    eager = [r.clone() for r in _peel(ctx, mtx, res, 4)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _peel(ctx, mtx, res, 4)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _peel(ctx, mtx, res, 4)
    for r in captured:
        r.fill_(-1.0)
    graph.replay()
    torch.cuda.synchronize()
    assert (eager[1][..., 3] > 0).any()
    for a, b in zip(captured, eager):
        assert torch.equal(a, b)


def test_errors(dev):
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.raster import DepthPeeler
    ctx, v, f, vt, ft, mtx = _scene(dev, res=(16, 16))
    pos = torch.rand(2, v.shape[0], 4, device=dev)
    p = DepthPeeler(ctx, mtx, (16, 16))
    with pytest.raises(RuntimeError):
        p.rasterize_next_layer()                                       # outside `with`
    with p:
        p.rasterize_next_layer()
    with pytest.raises(RuntimeError):
        p.rasterize_next_layer()                                       # after the block
    with pytest.raises(RuntimeError):
        with DepthPeeler(ctx, mtx, (16, 16)) as q:
            q.rasterize_next_layer()
            ou.optix_build_bvh(ctx, vt, ft, rebuild=0)                 # refit between layers
            q.rasterize_next_layer()
    with pytest.raises(ValueError):
        DepthPeeler(ctx, mtx[0], (16, 16))
    with pytest.raises(ValueError):
        DepthPeeler(ctx, mtx, (16, 16), pos=pos[..., :3], tri=ft)
    with pytest.raises(ValueError):
        DepthPeeler(ctx, mtx, (16, 16), pos=pos[:1].repeat(3, 1, 1), tri=ft)
    with pytest.raises(TypeError):
        DepthPeeler(ctx, mtx, (16, 16), pos=pos, tri=ft.long())
    with pytest.raises(TypeError):
        DepthPeeler(ctx, mtx, (16, 16), pos=pos.double(), tri=ft)
    with pytest.raises(ValueError):
        DepthPeeler(ctx, mtx, (16, 16), pos=pos)
    with pytest.raises(ValueError):
        DepthPeeler(ctx, mtx, (16, 16), tri=ft)
    with pytest.raises(RuntimeError):
        with DepthPeeler(ou.OptiXContext(), mtx, (16, 16)) as q:     # no BVH built
            q.rasterize_next_layer()
    with pytest.raises(ValueError):
        ou.trace_closest(ctx, vt, vt, t_after=torch.zeros(3, device=dev))


def test_full_size_peel(dev):
    """8 x 512^2, 8 layers on the bench mesh; the ray query is bit-exact on 4 k random pixels' rays per layer, and the peeled
    layers agree with it on those pixels."""
    import bench
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    ctx, vt, ft = _ctx(dev, v, f)
    B, res = 8, (512, 512)
    mtx_np = np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32)
    layers = [r.cpu().numpy() for r in _peel(ctx, torch.tensor(mtx_np, device=dev), res, 8)]
    cov = [int((r[..., 3] > 0).sum()) for r in layers]
    print("8 x 512^2 covered pixels per layer:", cov)
    assert cov[0] > 100000 and cov[1] > 10000 and all(a >= b for a, b in zip(cov, cov[1:]))
    o, d = _host_rays(mtx_np, res)
    rng = np.random.default_rng(0)
    b = rng.integers(0, B, 4096); px = rng.integers(0, res[0] * res[1], 4096)
    ro, rd = o[b, px], d[b, px]
    sc = PeelScene(v, f)
    hits = _ray_parity(dev, ctx, sc, ro, rd, 8)
    assert hits[1] > 200
    ref = sc.peel(ro, rd, 8)
    for k in range(8):
        gid = layers[k].reshape(B, -1, 4)[b, px, 3].astype(np.int64) - 1
        assert (gid == ref[k][0]).mean() > 0.995, k
