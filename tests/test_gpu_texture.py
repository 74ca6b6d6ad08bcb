"""GPU: the filtered texture look-up (csrc/texture.cu) against the fp32 CPU oracle -- forward, d uv and d uv_da bit for bit, d tex per
level to the atomics' summation order -- over both filter and boundary modes, channel counts, shared and per-batch textures, chain
shapes and edge uv / uv_da; plus the frozen output of the reference's Texture2D / EnvironmentLight, the regulariser taps against
grid_sample, needs_input_grad, CUDA-graph replay, composition with rasterize / interpolate, and a texture fit."""
import os
import zlib

import numpy as np
import pytest
import torch

from common import rel_l2
from oracle.texture import chain_shapes, texture_oracle
from nvdiffrecmc_b200 import _lib as L
from nvdiffrecmc_b200.raster import texture

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LML = "linear-mipmap-linear"


def _uv(rng, B, h, w, H0, W0):
    """uv mixing uniform values in [-0.5, 1.5], texel centres and edges of level 0, exact 0 / 1, negative, above 1 and huge"""
    uv = rng.uniform(-0.5, 1.5, (B, h, w, 2)).astype(np.float32)
    k = rng.integers(0, 6, (B, h, w, 2))
    cen = np.stack([(rng.integers(0, W0, (B, h, w)) + 0.5) / W0, (rng.integers(0, H0, (B, h, w)) + 0.5) / H0], -1)
    edge = np.stack([rng.integers(-W0, 2 * W0, (B, h, w)) / W0, rng.integers(-H0, 2 * H0, (B, h, w)) / H0], -1)
    uv[k == 1] = cen[k == 1]
    uv[k == 2] = edge[k == 2]
    uv[k == 3] = rng.choice(np.array([0.0, 1.0, -1.0, 2.0, 1e5, -3e7, 4e9], np.float32), int((k == 3).sum()))
    return uv.astype(np.float32)


def _uv_da(rng, B, h, w, H0, W0, L):
    """zero, isotropic, anisotropic and beyond-the-last-level footprints (major axis 2^s texels, s in [-2, L + 2])"""
    s = rng.uniform(-2, L + 2, (B, h, w, 1))
    J = rng.normal(size=(B, h, w, 4)) * 2.0 ** s
    iso = rng.random((B, h, w)) < 0.25
    J[iso] = np.stack([J[iso][:, 0], np.zeros(iso.sum()), np.zeros(iso.sum()), J[iso][:, 0]], -1)
    J[rng.random((B, h, w)) < 0.15] = 0.0
    return (J / np.array([W0, W0, H0, H0])).astype(np.float32)


def _run(dev, levels, uv, da, g, filt, bnd, mip_passed=True):
    t = [torch.from_numpy(x).to(dev).requires_grad_(True) for x in levels]
    uvt = torch.from_numpy(uv).to(dev).requires_grad_(True)
    dat = torch.from_numpy(da).to(dev).requires_grad_(True) if da is not None else None
    y = texture(t[0], uvt, dat, mip=t[1:] if (filt == LML and mip_passed) else None, filter_mode=filt, boundary_mode=bnd)
    y.backward(torch.from_numpy(g).to(dev))
    n = lambda x: None if x is None or x.grad is None else x.grad.cpu().numpy()
    return y.detach().cpu().numpy(), [n(x) for x in t], n(uvt), n(dat)


def _check_dtex(got, ref):
    assert np.array_equal(got == 0, ref == 0)
    if np.any(ref):
        assert rel_l2(got, ref) <= 1e-5


CHAINS = {"square": (32, 32, 6), "non_square": (24, 40, 6), "odd": (13, 29, 5), "stops_early": (64, 16, 3), "one_level": (9, 7, 1),
          "1x1": (1, 1, 1)}


@pytest.mark.parametrize("bnd", ["wrap", "clamp"])
@pytest.mark.parametrize("filt", ["linear", LML])
@pytest.mark.parametrize("C", [1, 3, 4, 7])
@pytest.mark.parametrize("Bt", [1, 2])
@pytest.mark.parametrize("chain", list(CHAINS))
def test_bit_identical_to_the_oracle(dev, chain, Bt, C, filt, bnd):
    H0, W0, n = CHAINS[chain]
    rng = np.random.default_rng(zlib.crc32(repr((chain, Bt, C, filt, bnd)).encode()))
    levels = [rng.normal(size=(Bt, h, w, C)).astype(np.float32) for h, w in chain_shapes(H0, W0, n)]
    B, h, w = 2, 19, 23
    uv = _uv(rng, B, h, w, H0, W0)
    da = _uv_da(rng, B, h, w, H0, W0, n - 1) if filt == LML else None
    # non-negative upstream gradients: the coarse levels sum hundreds of them into one texel, and a zero-mean sum would cancel down to the
    # float atomics' order noise, which a relative bar cannot measure
    g = rng.uniform(0.1, 1.0, size=(B, h, w, C)).astype(np.float32) * rng.choice([-1.0, 1.0], size=(1, 1, 1, C)).astype(np.float32)
    g[0, ::3] = 0.0
    o = texture_oracle()
    y, dt, duv, dda = _run(dev, levels, uv, da, g, filt, bnd, mip_passed=chain != "1x1")      # the 1x1 texture goes without mip=
    assert np.array_equal(y, o.forward(levels, uv, da, filt, bnd), equal_nan=True)
    rt, ruv, rda = o.backward(levels, uv, da, g, filt, bnd)
    assert np.array_equal(duv, ruv, equal_nan=True)
    if filt == LML:
        assert np.array_equal(dda, rda, equal_nan=True)
    else:
        assert dda is None and all(x is None for x in dt[1:])
    finite = np.isfinite(uv).all() and (np.abs(uv) < 1e9).all()
    for k in range(len(rt)):
        if finite or np.isfinite(rt[k]).all():
            _check_dtex(dt[k], rt[k])


def test_magnified_hot_spot(dev):
    """Many pixels on a few texels (magnification: a 4 x 4 texture under 256 x 256 pixels), the case the warp aggregation is for."""
    rng = np.random.default_rng(3)
    levels = [rng.normal(size=(1, h, w, 4)).astype(np.float32) for h, w in chain_shapes(4, 4, 3)]
    ys, xs = np.meshgrid((np.arange(256) + 0.5) / 256, (np.arange(256) + 0.5) / 256, indexing="ij")
    uv = np.broadcast_to(np.stack([xs, ys], -1), (2, 256, 256, 2)).astype(np.float32).copy()
    da = np.zeros((2, 256, 256, 4), np.float32)
    da[1, ..., 0] = da[1, ..., 3] = 1.5 / 4            # lambda = log2(1.5): levels 0 and 1
    g = rng.normal(size=(2, 256, 256, 4)).astype(np.float32)
    g[:, :, :100] = 0.0
    o = texture_oracle()
    for bnd in ("wrap", "clamp"):
        y, dt, duv, dda = _run(dev, levels, uv, da, g, LML, bnd)
        assert np.array_equal(y, o.forward(levels, uv, da, LML, bnd))
        rt, ruv, rda = o.backward(levels, uv, da, g, LML, bnd)
        assert np.array_equal(duv, ruv) and np.array_equal(dda, rda)
        for k in range(3):
            _check_dtex(dt[k], rt[k])


def test_reproduces_the_reference_texture2d(dev):
    """Texture2D.sample (render/texture.py:57-68) restated on the product: the automatic chain pools by 2 x 2 averages and its backward is
    the clamped bilinear look-up of dout / 4 at the centres of the finer level's texels; a custom chain; a 1x1 constant; the probe image."""
    d = np.load(os.path.join(HERE, "golden", "ref_texture2d.npz"))
    t = lambda k: torch.from_numpy(d[k]).to(dev)

    class Pool(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x):
            return torch.nn.functional.avg_pool2d(x.permute(0, 3, 1, 2), (2, 2)).permute(0, 2, 3, 1).contiguous()

        @staticmethod
        def backward(ctx, dout):
            h, w = dout.shape[1], dout.shape[2]
            gy, gx = torch.meshgrid(torch.linspace(0.25 / h, 1 - 0.25 / h, 2 * h, device=dev), torch.linspace(0.25 / w, 1 - 0.25 / w, 2 * w, device=dev),
                                    indexing="ij")
            return texture(dout * 0.25, torch.stack((gx, gy), -1)[None].contiguous(), filter_mode="linear", boundary_mode="clamp")

    def check(case, y, uv, da, mips):
        y.backward(t("dout_" + case))
        assert rel_l2(y.detach().cpu().numpy(), d["out_" + case]) <= 1e-6, case
        assert rel_l2(uv.grad.cpu().numpy(), d["d_texc_" + case]) <= 1e-5, case
        ref = d["d_texc_deriv_" + case]
        got = da.grad.cpu().numpy()
        assert (not ref.any() and not got.any()) or rel_l2(got, ref) <= 1e-5, case
        for k, m in enumerate(mips):
            assert rel_l2(m.grad.cpu().numpy(), d["d_level%d_%s" % (k, case)]) <= 1e-5, (case, k)

    new = lambda: (t("texc").requires_grad_(True), t("texc_deriv").requires_grad_(True))
    uv, da = new()
    base = t("auto_base")[None].requires_grad_(True)
    chain = [base]
    while chain[-1].shape[1] > 1 and chain[-1].shape[2] > 1:
        chain.append(Pool.apply(chain[-1]))
    check("auto", texture(chain[0], uv, da, mip=chain[1:], filter_mode=LML), uv, da, [base])
    uv, da = new()
    custom = [t("level%d_custom" % k).requires_grad_(True) for k in range(7)]
    check("custom", texture(custom[0], uv, da, mip=custom[1:], filter_mode=LML), uv, da, custom)
    uv, da = new()
    const = t("const")[None, None, None, :].requires_grad_(True)
    check("const", texture(const, uv, da, filter_mode=LML), uv, da, [const])
    Hr, Wr = d["out_env"].shape[:2]
    ys, xs = torch.meshgrid((torch.arange(Hr, device=dev, dtype=torch.float32) + 0.5) / Hr, (torch.arange(Wr, device=dev, dtype=torch.float32) + 0.5) / Wr,
                            indexing="ij")
    env = texture(t("env_base")[None].contiguous(), torch.stack((xs, ys), -1)[None].contiguous(), filter_mode="linear")[0]
    assert rel_l2(env.cpu().numpy(), d["out_env"]) <= 1e-6


def test_regulariser_taps_match_grid_sample(dev):
    """render.py's five jittered taps ('linear', 'clamp') at 8 x 512^2 against grid_sample(bilinear, border, align_corners=False)."""
    g = torch.Generator(device=dev).manual_seed(0)
    B, H, W = 8, 512, 512
    ys, xs = torch.meshgrid((torch.arange(H, device=dev) + 0.5) / H, (torch.arange(W, device=dev) + 0.5) / W, indexing="ij")
    jitter = (torch.stack((xs, ys), -1)[None] + torch.randn(B, H, W, 2, device=dev, generator=g) * 0.005).contiguous()
    for C in (1, 4, 3, 3, 3):
        img = torch.rand(B, H, W, C, device=dev, generator=g).requires_grad_(True)
        y = texture(img, jitter, filter_mode="linear", boundary_mode="clamp")
        ref = torch.nn.functional.grid_sample(img.permute(0, 3, 1, 2), jitter * 2 - 1, mode="bilinear", padding_mode="border",
                                              align_corners=False).permute(0, 2, 3, 1)
        # grid_sample takes 2u - 1 (rounded) and un-normalises it with its own roundings: single pixels differ by up to ~1.4e-5 and the
        # relative L2 is ~2e-6; the bit-exact check of these taps is the one against the oracle above
        assert rel_l2(y.detach().cpu().numpy(), ref.detach().cpu().numpy()) <= 5e-6
        dy = torch.randn(B, H, W, C, device=dev, generator=g)
        (gi,) = torch.autograd.grad(y, img, dy)
        (gr,) = torch.autograd.grad(ref, img, dy)
        assert rel_l2(gi.cpu().numpy(), gr.cpu().numpy()) <= 1e-5


def test_needs_input_grad_and_no_grad(dev):
    rng = np.random.default_rng(5)
    levels = [torch.from_numpy(rng.normal(size=(1, h, w, 4)).astype(np.float32)).to(dev) for h, w in chain_shapes(16, 16, 5)]
    uv = torch.from_numpy(_uv(rng, 1, 8, 8, 16, 16)).to(dev)
    da = torch.from_numpy(_uv_da(rng, 1, 8, 8, 16, 16, 4)).to(dev)
    o = texture_oracle()
    n = [x.cpu().numpy() for x in levels]
    g = rng.normal(size=(1, 8, 8, 4)).astype(np.float32)
    rt, ruv, rda = o.backward(n, uv.cpu().numpy(), da.cpu().numpy(), g, LML, "wrap")
    gt = torch.from_numpy(g).to(dev)
    # only uv_da
    L.LAUNCHES.clear()
    dag = da.clone().requires_grad_(True)
    texture(levels[0], uv, dag, mip=levels[1:]).backward(gt)
    assert L.LAUNCHES == {"texture_fwd": 1, "texture_bwd": 1} and np.array_equal(dag.grad.cpu().numpy(), rda)
    # only the mip level 2
    m2 = levels[2].clone().requires_grad_(True)
    texture(levels[0], uv, da, mip=[levels[1], m2, levels[3], levels[4]]).backward(gt)
    _check_dtex(m2.grad.cpu().numpy(), rt[2])
    # nothing needs a gradient, and no_grad: the forward only
    L.LAUNCHES.clear()
    y = texture(levels[0], uv, da, mip=levels[1:])
    with torch.no_grad():
        y2 = texture(levels[0], uv.requires_grad_(True), da, mip=levels[1:])
    assert not y.requires_grad and not y2.requires_grad and L.LAUNCHES == {"texture_fwd": 2}
    # 'linear' ignores uv_da and mip: they get no gradient
    dag = da.clone().requires_grad_(True)
    m1 = levels[1].clone().requires_grad_(True)
    uvg = uv.detach().clone().requires_grad_(True)
    texture(levels[0], uvg, dag, mip=[m1], filter_mode="linear").sum().backward()
    assert dag.grad is None and m1.grad is None and uvg.grad is not None


def test_cuda_graph_replay_matches_eager(dev):
    rng = np.random.default_rng(6)
    lv = [torch.from_numpy(rng.normal(size=(1, h, w, 4)).astype(np.float32)).to(dev) for h, w in chain_shapes(128, 256, 8)]
    uv = torch.from_numpy(_uv(rng, 2, 96, 96, 128, 256)).to(dev)
    da = torch.from_numpy(_uv_da(rng, 2, 96, 96, 128, 256, 7)).to(dev)
    dy = torch.rand(2, 96, 96, 4, device=dev, generator=torch.Generator(device=dev).manual_seed(0))      # non-negative: see above
    params = [x.clone().requires_grad_(True) for x in lv]

    def step():
        uvg, dag = uv.clone().requires_grad_(True), da.clone().requires_grad_(True)
        for p in params:
            p.grad = None
        y = texture(params[0], uvg, dag, mip=params[1:])
        y.backward(dy)
        return [y.detach(), uvg.grad, dag.grad] + [p.grad for p in params]

    ref = [x.clone() for x in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out = step()
    for _ in range(2):
        gr.replay()
    torch.cuda.synchronize()
    for k in range(3):
        assert torch.equal(out[k], ref[k]), k
    for a, b in zip(out[3:], ref[3:]):          # d tex: float atomics in another order (the coarse levels sum ~18k terms per texel)
        assert torch.equal(a == 0, b == 0) and rel_l2(a.cpu().numpy(), b.cpu().numpy()) <= 1e-5


def test_composition_with_rasterize_and_interpolate(dev):
    """rasterize(grad_db=True) -> interpolate(diff_attrs='all') -> texture('linear-mipmap-linear') -> backward gives a finite d pos equal to
    the raster backward applied to the texture op's d uv and d uv_da."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200 import renderutils as ru, synth
    from nvdiffrecmc_b200.raster import interpolate, rasterize
    v, f = synth.scene_mesh("blob+torus", level=1)
    v, f = torch.tensor(v, dtype=torch.float32, device=dev), torch.tensor(f, dtype=torch.int32, device=dev)
    c = v - v.mean(0)
    v_tex = torch.stack([0.5 + torch.atan2(c[:, 2], c[:, 0]) / (2 * np.pi), 0.5 + 0.4 * c[:, 1] / c[:, 1].abs().max()], -1).contiguous()
    proj = torch.tensor(synth.perspective(aspect=1.0, n=0.1, f=10.0), dtype=torch.float32, device=dev)
    mv = torch.eye(4, device=dev); mv[2, 3] = -2.6
    mtx = (proj @ mv)[None].repeat(2, 1, 1)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, v, f, rebuild=1)
    rng = np.random.default_rng(7)
    tex = [torch.from_numpy(rng.uniform(0, 1, (1, h, w, 3)).astype(np.float32)).to(dev) for h, w in chain_shapes(64, 128, 7)]
    dy = torch.randn(2, 64, 64, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(1))

    def run():
        pos = ru.xfm_points(v[None], mtx).detach().requires_grad_(True)
        rast, db = rasterize(ctx, mtx, (64, 64), pos=pos, tri=f, grad_db=True)
        uv, uv_da = interpolate(v_tex, rast, f, rast_db=db, diff_attrs="all")
        uv.retain_grad()
        uv_da.retain_grad()
        return pos, uv, uv_da

    pos, uv, uv_da = run()
    texture(tex[0], uv, uv_da, mip=tex[1:], filter_mode=LML).backward(dy)
    assert torch.isfinite(pos.grad).all() and float(pos.grad.abs().max()) > 0 and float(uv_da.grad.abs().max()) > 0
    pos2, uv2, uv_da2 = run()
    torch.autograd.backward([uv2, uv_da2], [uv.grad, uv_da.grad])
    assert torch.equal(pos.grad == 0, pos2.grad == 0) and rel_l2(pos.grad.cpu().numpy(), pos2.grad.cpu().numpy()) <= 1e-5


def test_fit_a_texture(dev):
    """A 256^2 texture with its full chain, fitted through fixed uv / uv_da to a target rendered from a known texture."""
    g = torch.Generator(device=dev).manual_seed(2)
    ys, xs = torch.meshgrid(torch.linspace(0, 1, 256, device=dev), torch.linspace(0, 1, 256, device=dev), indexing="ij")
    known = torch.stack([0.5 + 0.5 * torch.sin(12 * xs), 0.5 + 0.5 * torch.cos(9 * ys + 3 * xs), (xs + ys) / 2], -1)[None]
    chain = [known]
    while chain[-1].shape[1] > 1:
        chain.append(torch.nn.functional.avg_pool2d(chain[-1].permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).contiguous())
    uv = torch.rand(4, 128, 128, 2, device=dev, generator=g)
    da = (torch.randn(4, 128, 128, 4, device=dev, generator=g) * 2.0 ** (torch.rand(4, 128, 128, 1, device=dev, generator=g) * 8 - 1) / 256).contiguous()
    target = texture(chain[0], uv, da, mip=chain[1:])
    params = [torch.full_like(x, 0.5).requires_grad_(True) for x in chain]
    opt = torch.optim.Adam(params, lr=0.05)
    losses = []
    for _ in range(200):
        loss = torch.mean((texture(params[0], uv, da, mip=params[1:]) - target) ** 2)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print("texture fit: loss %.3e -> %.3e" % (losses[0], losses[-1]))
    assert losses[-1] * 10 <= losses[0]
