"""GPU, row f2 geometry gradients: rasterize / interpolate backward to positions and barycentrics, the device edge adjacency and the
analytic antialias, against the CPU oracle; a silhouette fit that moves a mesh only through antialias; CUDA-graph capture; errors."""
import numpy as np
import pytest
import torch

from common import rel_l2, same_bits
from oracle.geometry import geometry_oracle
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


def _scene(dev, B=2, res=(48, 64), kind="blob+torus", level=2):
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh(kind, level=level)
    ctx = ou.OptiXContext()
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    mtx = torch.tensor(_mtx([(0.7 * b + 0.3, 0.2 * b - 0.1) for b in range(B)], aspect=res[1] / res[0]), device=dev)
    return ctx, v, f, vt, ft, mtx


@pytest.mark.parametrize("shared", [False, True])
def test_rasterize_pos_gradient(dev, shared):
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.raster import rasterize
    res = (48, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    if shared:                                    # one [V,4] for a batch of identical views: the gradient sums over the batch
        mtx = mtx[:1].repeat(2, 1, 1)
    pos = ru.xfm_points(vt[None], mtx).detach()
    if shared:
        pos = pos[0].contiguous()
    pos.requires_grad_(True)
    plain = rasterize(ctx, mtx, res)
    rast = rasterize(ctx, mtx, res, pos=pos, tri=ft)
    assert plain.grad_fn is None and rast.grad_fn is not None
    assert torch.equal(plain, rast.detach())                                   # same launch, bit-identical output
    r = rast.detach().cpu().numpy(); p = pos.detach().cpu().numpy()
    uv = geometry_oracle(f64=True).raster_bary(p, f, r)
    m = r[..., 3] > 0
    assert m.sum() > 1000
    # ray-traced barycentrics = clip-space barycentrics of pos.  The ray is rebuilt through the fp32 inverse clip matrix, so grazing
    # triangles differ by more than the bulk: measured on an H100, max 2.3e-4 over ~2 k covered pixels, so 1e-4 holds for the 99th
    # percentile and the maximum is checked at 5e-4.
    err = np.abs(r[..., :2] - uv)[m]
    assert np.quantile(err, 0.99) < 1e-4 and err.max() < 5e-4, (float(np.quantile(err, 0.99)), float(err.max()))
    g = torch.randn(rast.shape, generator=torch.Generator().manual_seed(3)).to(dev)
    rast.backward(g)
    ref = geometry_oracle().raster_bwd(p, f, r, g.cpu().numpy())
    assert np.abs(ref).max() > 0
    assert rel_l2(pos.grad.cpu().numpy(), ref) < 1e-5


@pytest.mark.parametrize("batched", [False, True])
def test_interpolate_rast_gradient(dev, batched):
    from nvdiffrecmc_b200.raster import rasterize, interpolate
    res = (40, 40)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    rast = rasterize(ctx, mtx, res)
    gen = torch.Generator().manual_seed(5)
    V = v.shape[0]
    a0 = torch.rand((2, V, 5) if batched else (V, 5), generator=gen).to(dev)
    gout = torch.randn(2, 40, 40, 5, generator=gen).to(dev)
    attr, attr_ref = a0.clone().requires_grad_(True), a0.clone().requires_grad_(True)
    rg = rast.clone().requires_grad_(True)
    interpolate(attr, rg, ft)[0].backward(gout)
    interpolate(attr_ref, rast, ft)[0].backward(gout)                          # the attribute-only path
    assert rel_l2(attr.grad.cpu().numpy(), attr_ref.grad.cpu().numpy()) < 1e-6
    r = rast.cpu().numpy(); A = a0.cpu().numpy(); go = gout.cpu().numpy()
    ids = r[..., 3].astype(np.int64) - 1
    ref = np.zeros((2, 40, 40, 4), np.float64)
    for b in range(2):
        Ab = A[b] if batched else A
        m = ids[b] >= 0
        tri = f[ids[b][m]]
        ref[b][m, 0] = ((Ab[tri[:, 0]] - Ab[tri[:, 2]]) * go[b][m]).sum(-1)
        ref[b][m, 1] = ((Ab[tri[:, 1]] - Ab[tri[:, 2]]) * go[b][m]).sum(-1)
    assert rel_l2(rg.grad.cpu().numpy(), ref) < 1e-6
    rg2 = rast.clone().requires_grad_(True)                                    # attributes without grad: d_rast only
    interpolate(a0, rg2, ft)[0].backward(gout)
    assert torch.equal(rg2.grad, rg.grad)


@pytest.mark.parametrize("kind", ["blob+torus", "holes", "grid1m"])
def test_topology_matches_oracle(dev, kind):
    from nvdiffrecmc_b200.raster import antialias_topology
    v, f = synth.scene_mesh("grid1m" if kind == "grid1m" else "blob+torus", level=3)
    if kind == "holes":
        f = f[np.random.default_rng(0).random(f.shape[0]) > 0.1]
    ft = torch.tensor(f, device=dev)
    a1 = antialias_topology(ft)
    a2 = antialias_topology(ft)
    assert torch.equal(a1, a2)
    ref = geometry_oracle().aa_topology(f)
    assert np.array_equal(a1.cpu().numpy(), ref)
    if kind == "grid1m":
        assert f.shape[0] > 1_000_000 and (ref == -1).any()


def _aa_case(dev, C, res=256):
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.raster import rasterize, antialias_topology
    ctx, v, f, vt, ft, mtx = _scene(dev, res=(res, res))
    pos = ru.xfm_points(vt[None], mtx).detach()
    rast = rasterize(ctx, mtx, (res, res), pos=pos, tri=ft).detach()
    color = torch.rand(2, res, res, C, generator=torch.Generator().manual_seed(C)).to(dev)
    return f, ft, pos, rast, color, antialias_topology(ft)


@pytest.mark.parametrize("C", [1, 4, 7])
def test_antialias_matches_oracle(dev, C):
    from nvdiffrecmc_b200.raster import antialias
    f, ft, pos, rast, color, topo = _aa_case(dev, C)
    col = color.clone().requires_grad_(True); p = pos.clone().requires_grad_(True)
    out = antialias(col, rast, p, ft, topo)
    out2 = antialias(color, rast, pos, ft)                                     # topology built inside the call
    assert torch.equal(out.detach(), out2)                                     # bit-deterministic
    o = geometry_oracle()
    args = (color.cpu().numpy(), rast.cpu().numpy(), pos.cpu().numpy(), f)
    ref = o.antialias(*args)
    assert (np.abs(ref - args[0]) > 1e-3).sum() > 200                         # the silhouettes are blended
    assert same_bits(out.detach().cpu().numpy(), ref)
    g = torch.randn(out.shape, generator=torch.Generator().manual_seed(11)).to(dev)
    out.backward(g)
    dc, dp = o.antialias_bwd(*args, g.cpu().numpy())
    assert same_bits(col.grad.cpu().numpy(), dc)
    assert np.abs(dp).max() > 0
    assert rel_l2(p.grad.cpu().numpy(), dp) < 1e-5
    if C == 4:                                                                 # shared [V,4] positions, one image
        p1 = pos[0].clone().requires_grad_(True)
        o1 = antialias(color[:1], rast[:1], p1, ft, topo)
        o1.backward(g[:1])
        ref1 = o.antialias(args[0][:1], args[1][:1], args[2][0], f)
        _, dp1 = o.antialias_bwd(args[0][:1], args[1][:1], args[2][0], f, g[:1].cpu().numpy())
        assert same_bits(o1.detach().cpu().numpy(), ref1) and rel_l2(p1.grad.cpu().numpy(), dp1) < 1e-5


def test_antialias_is_channelwise(dev):
    from nvdiffrecmc_b200.raster import antialias
    f, ft, pos, rast, color, topo = _aa_case(dev, 7)
    a, b = color[..., :3].contiguous(), color[..., 3:].contiguous()
    assert torch.equal(antialias(color, rast, pos, ft, topo), torch.cat([antialias(a, rast, pos, ft, topo), antialias(b, rast, pos, ft, topo)], -1))


def test_silhouette_fit(dev):
    """A radius-0.8 sphere fitted to the alpha of a radius-1.0 one from four views, alpha = antialias(coverage): the only path from the
    loss to the vertices is antialias (the coverage itself is a step function of the geometry).  The BVH is rebuilt every iteration, as
    in geometry/dlmesh.py:50.  Parameters: one radius per vertex along fixed directions, with an edge smoothness term that carries
    the motion from the silhouette bands to the vertices no view sees on a silhouette."""
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.raster import rasterize, antialias, antialias_topology
    d, f = synth.icosphere(3)
    dirs = torch.tensor(d, dtype=torch.float32, device=dev)
    ft = torch.tensor(f.astype(np.int32), device=dev)
    topo = antialias_topology(ft)
    e = torch.cat([ft[:, [0, 1]], ft[:, [1, 2]], ft[:, [2, 0]]]).long()
    res = (128, 128)
    mtx = torch.tensor(_mtx([(0.0, 0.5), (1.6, -0.5), (3.1, 0.6), (4.7, -0.4)]), device=dev)
    ctx = ou.OptiXContext()

    def alpha(r, aa=True):
        v = dirs * r[:, None]
        ou.optix_build_bvh(ctx, v.detach(), ft, rebuild=1)
        pos = ru.xfm_points(v[None], mtx)
        rast = rasterize(ctx, mtx, res, pos=pos, tri=ft)
        cov = rast[..., 3:4].clamp(0, 1)
        return antialias(cov, rast, pos, ft, topo) if aa else cov

    with torch.no_grad():
        target = alpha(torch.ones(dirs.shape[0], device=dev))
    r = torch.full((dirs.shape[0],), 0.8, device=dev, requires_grad=True)
    # control: without antialias the silhouette loss gives the vertices no gradient at all
    (g0,) = torch.autograd.grad(torch.nn.functional.mse_loss(alpha(r, aa=False), target), r)
    assert (g0 == 0).all()
    opt = torch.optim.Adam([r], lr=0.01)
    losses = []
    for it in range(150):
        img = torch.nn.functional.mse_loss(alpha(r), target)
        loss = img + 10.0 * ((r[e[:, 0]] - r[e[:, 1]]) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        if it == 0:
            assert r.grad.abs().max() > 0
        opt.step()
        losses.append(float(img.detach()))
    mean_r = float(r.detach().mean())
    print("silhouette fit: image loss %.3e -> %.3e, mean radius %.4f" % (losses[0], losses[-1], mean_r))
    assert losses[-1] * 10 <= losses[0]
    assert abs(mean_r - 1.0) < 0.05


def test_cuda_graph_replay_equals_eager(dev):
    from nvdiffrecmc_b200.raster import rasterize, antialias
    import nvdiffrecmc_b200.renderutils as ru
    res = (64, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    from nvdiffrecmc_b200.raster import antialias_topology
    topo = antialias_topology(ft)
    pos0 = ru.xfm_points(vt[None], mtx).detach()
    color = torch.rand(2, 64, 64, 4, generator=torch.Generator().manual_seed(4)).to(dev)
    gout = torch.randn(2, 64, 64, 4, generator=torch.Generator().manual_seed(5)).to(dev)

    def step(p):
        rast = rasterize(ctx, mtx, res, pos=p, tri=ft)
        out = antialias(color, rast, p, ft, topo)
        out.backward(gout)
        return out

    pe = pos0.clone().requires_grad_(True)
    out_e = step(pe).detach().clone()
    ps = pos0.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            ps.grad = None
            step(ps)
    torch.cuda.current_stream().wait_stream(s)
    ps.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_s = step(ps)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_s, out_e)
    assert rel_l2(ps.grad.cpu().numpy(), pe.grad.cpu().numpy()) < 1e-6


def test_errors(dev):
    from nvdiffrecmc_b200.raster import rasterize, antialias, antialias_topology, interpolate
    ctx, v, f, vt, ft, mtx = _scene(dev, res=(16, 16))
    pos = torch.rand(2, v.shape[0], 4, device=dev)
    rast = rasterize(ctx, mtx, (16, 16))
    col = torch.rand(2, 16, 16, 3, device=dev)
    with pytest.raises(TypeError):
        rasterize(ctx, mtx, (16, 16), pos=pos, tri=ft.long())
    with pytest.raises(TypeError):
        rasterize(ctx, mtx, (16, 16), pos=pos.double(), tri=ft)
    with pytest.raises(ValueError):
        rasterize(ctx, mtx, (16, 16), pos=pos[..., :3], tri=ft)
    with pytest.raises(ValueError):
        rasterize(ctx, mtx, (16, 16), pos=pos[:1].repeat(3, 1, 1), tri=ft)           # batch 3 for 2 views
    with pytest.raises(ValueError):
        rasterize(ctx, mtx, (16, 16), pos=pos)
    with pytest.raises(TypeError):
        antialias_topology(ft.long())
    with pytest.raises(ValueError):
        antialias_topology(ft[:, :2].contiguous())
    with pytest.raises(TypeError):
        antialias(col, rast, pos, ft.long())
    with pytest.raises(ValueError):
        antialias(col, rast[:, :8], pos, ft)
    with pytest.raises(ValueError):
        antialias(col, rast, pos[:1].repeat(3, 1, 1), ft)
    with pytest.raises(ValueError):
        antialias(col[0], rast, pos, ft)
    with pytest.raises(ValueError):
        antialias(col, rast, pos, ft, antialias_topology(ft)[:5])
    with pytest.raises(RuntimeError):
        antialias(col.cpu(), rast, pos, ft)
    with pytest.raises(RuntimeError):
        antialias_topology(ft.cpu())
    with pytest.raises(RuntimeError):
        rasterize(ctx, mtx, (16, 16), pos=pos.cpu(), tri=ft)
    with pytest.raises(RuntimeError):
        interpolate(torch.rand(v.shape[0], 3), rast, ft)
