"""GPU parity, row f2: ray-traced rasterize vs the CPU oracle's restatement, interpolate vs numpy interpolation."""
import numpy as np
import pytest
import torch

from common import check_scatter_fp32, oracle, rel_l2, texel_fetch_stats
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _perspective(fovy=0.7854, aspect=1.0, n=0.1, f=10.0):
    y = np.tan(fovy / 2)
    return np.array([[1 / (y * aspect), 0, 0, 0], [0, 1 / -y, 0, 0], [0, 0, -(f + n) / (f - n), -(2 * f * n) / (f - n)], [0, 0, -1, 0]], np.float32)


def _scene(dev, B=2, res=(48, 64)):
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh("blob+torus", level=2)
    ctx = ou.OptiXContext()
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    proj = _perspective(aspect=res[1] / res[0])
    mvs = []
    for b in range(B):
        mv = np.eye(4, dtype=np.float32)
        a = 0.7 * b + 0.3
        mv[:3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32)
        mv[2, 3] = -3.0
        mvs.append(proj @ mv)
    mtx = np.stack(mvs).astype(np.float32)
    return ctx, v, f, vt, ft, mtx


def test_rasterize_matches_oracle_closest_hit(dev):
    """rast bit for bit against the oracle's restatement of k_invert4 + k_rasterize (tests/test_gpu_rasterize_exact.py covers the
    edge cases)."""
    from nvdiffrecmc_b200.raster import rasterize
    res = (48, 64)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    rast = rasterize(ctx, torch.tensor(mtx, device=dev), res).cpu().numpy()
    assert rast.shape == (2, 48, 64, 4)
    ref, t = oracle().scene(v, f).rasterize(mtx, res)
    assert np.array_equal(rast.view(np.uint32), ref.view(np.uint32))
    hit = ref[..., 3] > 0
    assert hit.sum() > 500 and (rast[~hit] == 0).all() and np.isinf(t[~hit]).all()


@pytest.mark.parametrize("batched", [False, True])
def test_interpolate_forward_backward(dev, batched):
    from nvdiffrecmc_b200.raster import rasterize, interpolate
    res = (40, 40)
    ctx, v, f, vt, ft, mtx = _scene(dev, res=res)
    rast = rasterize(ctx, torch.tensor(mtx, device=dev), res)
    g = torch.Generator().manual_seed(5)
    V = v.shape[0]
    attr = torch.rand((2, V, 5) if batched else (V, 5), generator=g).to(dev).requires_grad_(True)
    out, _ = interpolate(attr, rast, ft)
    r = rast.cpu().numpy(); a = attr.detach().cpu().numpy()
    ids = r[..., 3].astype(np.int64) - 1
    ref = np.zeros((2, 40, 40, 5), np.float32)
    for b in range(2):
        A = a[b] if batched else a
        m = ids[b] >= 0
        tri = f[ids[b][m]]
        w0, w1 = r[b][m][:, 0:1], r[b][m][:, 1:2]
        ref[b][m] = w0 * A[tri[:, 0]] + w1 * A[tri[:, 1]] + (1 - w0 - w1) * A[tri[:, 2]]
    assert rel_l2(out.detach().cpu().numpy(), ref) < 1e-6
    # interpolating the positions reproduces the hit points: round trip through the clip matrix gives the pixel centre back
    pos, _ = interpolate(vt, rast, ft)
    hp = torch.cat([pos, torch.ones_like(pos[..., :1])], -1) @ torch.tensor(mtx, device=dev).transpose(1, 2)[:, None]
    ndc = (hp[..., :2] / hp[..., 3:]).cpu().numpy()
    m = ids >= 0
    xs = (np.arange(40, dtype=np.float32) + 0.5) / 40 * 2 - 1
    assert np.abs(ndc[..., 0] - xs[None, None, :])[m].max() < 1e-3 and np.abs(ndc[..., 1] - xs[None, :, None])[m].max() < 1e-3
    # backward = transpose of the (linear) forward
    gout = torch.rand(out.shape, generator=g).to(dev)
    out.backward(gout)
    d = np.zeros_like(a)
    go = gout.cpu().numpy()
    for b in range(2):
        D = d[b] if batched else d
        m = ids[b] >= 0
        tri = f[ids[b][m]]
        w0, w1 = r[b][m][:, 0:1], r[b][m][:, 1:2]
        for k, w in enumerate((w0, w1, 1 - w0 - w1)):
            np.add.at(D, tri[:, k], w * go[b][m])
    assert rel_l2(attr.grad.cpu().numpy(), d) < 1e-5


def test_raster_errors(dev):
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.raster import rasterize, interpolate
    with pytest.raises(RuntimeError):
        rasterize(ou.OptiXContext(), torch.eye(4, device=dev)[None], (8, 8))            # no BVH built
    with pytest.raises(ValueError):
        rasterize(ou.OptiXContext(), torch.eye(4, device=dev), (8, 8))
    with pytest.raises(TypeError):
        interpolate(torch.rand(4, 3, device=dev), torch.zeros(1, 2, 2, 4, device=dev), torch.zeros(2, 3, dtype=torch.int64, device=dev))


def test_texel_fetch_equals_indexing(dev):
    from nvdiffrecmc_b200.raster import texel_fetch
    g = torch.Generator().manual_seed(2)
    tex = torch.rand(1000, 3, generator=g).to(dev).requires_grad_(True)
    ref = tex.detach().clone().requires_grad_(True)
    idx = torch.randint(0, 1000, (2, 33, 17), generator=g).to(dev)
    out = texel_fetch(tex, idx)
    assert torch.equal(out, ref[idx])
    gout = torch.rand(out.shape, generator=g).to(dev)
    out.backward(gout); ref[idx].backward(gout)
    s, a, n = texel_fetch_stats(1000, idx.cpu().numpy(), gout.cpu().numpy())
    check_scatter_fp32("texel_fetch d tex", tex.grad.cpu().numpy(), s, a, n, tag="texel_fetch")
    with pytest.raises(TypeError):
        texel_fetch(tex, idx.int())
