"""GPU: Texture2D's automatic mip chain (csrc/texture.cu) -- the chain forward bit for bit against the oracle and the device's avg_pool2d,
the fold against the oracle and the reference's per-level composition (a torch avg_pool2d Function whose backward is the clamped bilinear
look-up of a quarter of the gradient), clamp_ / normalize_ against the reference's loops, the frozen output of the reference's Texture2D,
and CUDA-graph replay."""
import os

import numpy as np
import pytest
import torch

from common import rel_l2
from oracle.mipchain import mipchain_oracle
from nvdiffrecmc_b200 import _lib as L
from nvdiffrecmc_b200.raster import texture
from nvdiffrecmc_b200.texture import Texture2D, chain_shapes, mip_chain

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LML = "linear-mipmap-linear"
SHAPES = [(1024, 1024, 4), (32, 96, 4), (24, 40, 3), (13, 29, 1), (64, 16, 7), (2, 2, 1)]
EVEN = [(1024, 1024, 4, True), (64, 16, 7, True), (32, 96, 4, False)]         # (H, W, C, power of two)


def same_bits(a, b):
    """equal bit for bit, every NaN equal to every other"""
    a, b = (x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x for x in (a, b))
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def _base(rng, Bt, H, W, C, specials=True):
    x = rng.normal(size=(Bt, H, W, C)).astype(np.float32)
    if specials:
        m = rng.random(x.shape)
        x[m < 0.002] = np.nan
        x[(m >= 0.002) & (m < 0.004)] = np.inf
        x[(m >= 0.004) & (m < 0.006)] = -np.inf
    return x


class Pool(torch.autograd.Function):
    """The reference's texture2d_mip (render/texture.py:20-30) on this project's texture."""
    @staticmethod
    def forward(ctx, x):
        return torch.nn.functional.avg_pool2d(x.permute(0, 3, 1, 2), (2, 2)).permute(0, 2, 3, 1).contiguous()

    @staticmethod
    def backward(ctx, dout):
        h, w = dout.shape[1], dout.shape[2]
        gy, gx = torch.meshgrid(torch.linspace(0.25 / h, 1 - 0.25 / h, 2 * h, device=dout.device),
                                torch.linspace(0.25 / w, 1 - 0.25 / w, 2 * w, device=dout.device), indexing="ij")
        return texture(dout * 0.25, torch.stack((gx, gy), -1)[None].contiguous(), filter_mode="linear", boundary_mode="clamp")


@pytest.mark.parametrize("Bt", [1, 2])
@pytest.mark.parametrize("H,W,C", SHAPES)
def test_chain_forward_is_avg_pool2d_and_the_oracle(dev, H, W, C, Bt):
    base = _base(np.random.default_rng(H * W * C + Bt), Bt, H, W, C)
    L.LAUNCHES.clear()
    got = mip_chain(torch.from_numpy(base).to(dev))
    n = len(chain_shapes(H, W)) - 1
    assert len(got) == n and L.LAUNCHES == {"mip_chain_fwd": (n + 4) // 5}
    for k, (g, r) in enumerate(zip(got, mipchain_oracle().forward(base)), 1):
        ref = torch.nn.functional.avg_pool2d((got[k - 2] if k > 1 else torch.from_numpy(base).to(dev)).permute(0, 3, 1, 2), (2, 2)).permute(0, 2, 3, 1)
        assert same_bits(g, r), k
        assert same_bits(g, ref), k


def _grads(rng, Bt, H, W, C, absent):
    return [None if k in absent else rng.normal(size=(Bt, h, w, C)).astype(np.float32) for k, (h, w) in enumerate(chain_shapes(H, W))][1:]


def _fold(dev, base, grads, chain=mip_chain):
    tex = torch.from_numpy(base).to(dev).requires_grad_(True)
    levels = chain(tex)
    outs = [(lv, torch.from_numpy(g).to(dev)) for lv, g in zip(levels, grads) if g is not None]
    return torch.autograd.grad([a for a, _ in outs], tex, [b for _, b in outs])[0]


def _pool_chain(tex):
    levels = [tex]
    while levels[-1].shape[1] > 1 and levels[-1].shape[2] > 1:
        levels.append(Pool.apply(levels[-1]))
    return levels[1:]


@pytest.mark.parametrize("absent", [(), (1, 3), (2, 4, 5, 6, 7, 8, 9, 10)], ids=["all", "some", "fine_only"])
@pytest.mark.parametrize("H,W,C,pow2", EVEN)
def test_fold_matches_the_oracle_and_the_reference_composition(dev, H, W, C, pow2, absent):
    rng = np.random.default_rng(H + W + C + len(absent))
    for Bt in (1, 2):
        base = rng.normal(size=(Bt, H, W, C)).astype(np.float32)
        grads = _grads(rng, Bt, H, W, C, absent)
        L.LAUNCHES.clear()
        d = _fold(dev, base, grads)
        assert L.LAUNCHES["mip_chain_bwd"] == 1 and "texture_fwd" not in L.LAUNCHES
        assert same_bits(d, mipchain_oracle().fold([None] + grads, base.shape))
        assert same_bits(d, _fold(dev, base, grads)), "two runs differ"
        if Bt == 1:                         # the composition samples with a one-image grid
            ref = _fold(dev, base, grads, _pool_chain)
            if pow2:
                assert same_bits(d, ref)
            else:
                assert rel_l2(d.cpu().numpy(), ref.cpu().numpy()) <= 1e-6


@pytest.mark.parametrize("H,W,odd,shape", [(24, 40, 3, (3, 5)), (48, 80, 4, (3, 5)), (13, 29, 0, (13, 29))])
def test_fold_raises_past_an_odd_level(dev, H, W, odd, shape):
    rng = np.random.default_rng(0)
    base = rng.normal(size=(1, H, W, 2)).astype(np.float32)
    grads = _grads(rng, 1, H, W, 2, ())
    with pytest.raises(RuntimeError, match=r"level %d \(%d x %d\) has an odd side" % (odd, *shape)):
        _fold(dev, base, grads)
    # gradients that stop at or above the odd level fold as usual
    fine = [g if k <= odd else None for k, g in enumerate(grads, 1)]
    if any(g is not None for g in fine):
        assert same_bits(_fold(dev, base, fine), mipchain_oracle().fold([None] + fine, base.shape))


def test_reproduces_the_reference_texture2d(dev):
    """Texture2D on tests/golden/ref_texture2d.npz, the reference's own Texture2D run on the CPU, at test_gpu_texture.py's tolerances."""
    d = np.load(os.path.join(HERE, "golden", "ref_texture2d.npz"))
    t = lambda k: torch.from_numpy(d[k]).to(dev)

    def check(case, tex, grads):
        uv, da = t("texc").requires_grad_(True), t("texc_deriv").requires_grad_(True)
        y = tex.sample(uv, da)
        y.backward(t("dout_" + case))
        assert rel_l2(y.detach().cpu().numpy(), d["out_" + case]) <= 1e-6, case
        assert rel_l2(uv.grad.cpu().numpy(), d["d_texc_" + case]) <= 1e-5, case
        ref, got = d["d_texc_deriv_" + case], da.grad.cpu().numpy()
        assert (not ref.any() and not got.any()) or rel_l2(got, ref) <= 1e-5, case
        for k, g in enumerate(grads()):
            assert rel_l2(g.cpu().numpy(), d["d_level%d_%s" % (k, case)]) <= 1e-5, (case, k)

    leaf = t("auto_base").requires_grad_(True)
    check("auto", Texture2D(leaf), lambda: [leaf.grad[None]])
    custom = Texture2D([t("level%d_custom" % k).requires_grad_(True) for k in range(7)])
    check("custom", custom, lambda: [m.grad for m in custom.getMips()])
    const = Texture2D(d["const"].copy())
    const.data.requires_grad_(True)
    check("const", const, lambda: [const.data.grad])
    assert const.getRes() == (1, 1) and const.getChannels() == 3 and custom.getRes() == (48, 80) and len(custom.parameters()) == 7


def test_linear_mode_skips_the_chain(dev):
    d = np.load(os.path.join(HERE, "golden", "ref_texture2d.npz"))
    uv = torch.from_numpy(d["texc"]).to(dev)
    da = torch.from_numpy(d["texc_deriv"]).to(dev)
    dy = torch.from_numpy(d["dout_auto"]).to(dev)
    base = torch.from_numpy(d["auto_base"]).to(dev)[None].requires_grad_(True)
    y_chain = texture(base, uv, da, mip=mip_chain(base), filter_mode="linear")
    (g_chain,) = torch.autograd.grad(y_chain, base, dy)
    L.LAUNCHES.clear()
    y = Texture2D(base).sample(uv, da, filter_mode="linear")
    (g,) = torch.autograd.grad(y, base, dy)
    assert "mip_chain_fwd" not in L.LAUNCHES and "mip_chain_bwd" not in L.LAUNCHES
    assert torch.equal(y, y_chain) and torch.equal(g == 0, g_chain == 0) and rel_l2(g.cpu().numpy(), g_chain.cpu().numpy()) <= 1e-6
    with pytest.raises(ValueError, match="needs its chain"):
        Texture2D(base[:, :1]).sample(uv, da)


def _mm(dev, lo, hi):
    return [torch.tensor(lo, dtype=torch.float32, device=dev), torch.tensor(hi, dtype=torch.float32, device=dev)]


def test_clamp_is_the_reference_loop(dev):
    rng = np.random.default_rng(4)
    lo, hi = [0.0, 0.1, np.nan, 0.5, -1.0], [1.0, 0.9, 0.5, 0.25, 1.0]      # a NaN bound, lo > hi, and a fifth entry beyond C
    auto = _base(rng, 1, 64, 32, 4)
    custom = [_base(rng, 1, h, w, 4) for h, w in [(16, 8), (8, 4), (4, 2), (2, 1), (1, 1)]]
    for init in (auto, custom):
        mips = [torch.from_numpy(x).to(dev) for x in (init if isinstance(init, list) else [init])]
        ref = [m.clone() for m in mips]
        mm = _mm(dev, lo, hi)
        for m in ref:                                     # render/texture.py:89-94
            for i in range(m.shape[-1]):
                m[..., i].clamp_(min=mm[0][i], max=mm[1][i])
        tex = Texture2D(mips if len(mips) > 1 else mips[0], min_max=mm)
        L.LAUNCHES.clear()
        tex.clamp_()
        assert L.LAUNCHES == {"mip_clamp": 1}
        for m, r, x in zip(tex.getMips(), ref, mipchain_oracle().clamp([x for x in (init if isinstance(init, list) else [init])],
                                                                          np.array(lo[:4], np.float32), np.array(hi[:4], np.float32))):
            assert same_bits(m, r)
            assert same_bits(m, x)
    Texture2D(torch.zeros(1, 4, 4, 3, device=dev)).clamp_()          # no min_max: nothing to do
    with pytest.raises(ValueError, match="min_max"):
        Texture2D(torch.zeros(1, 4, 4, 3, device=dev), min_max=[[0, 0, 0], [1, 1, 1]]).clamp_()
    with pytest.raises(ValueError, match="min_max"):
        Texture2D(torch.zeros(1, 4, 4, 3, device=dev), min_max=_mm(dev, [0, 0], [1, 1])).clamp_()


def test_normalize_is_the_oracle_and_safe_normalize(dev):
    """Bit for bit the oracle; within 2 ulp of the device's util.safe_normalize, which sums the dot product in its own order (one ulp of
    the dot moves the length by half an ulp and the quotient by up to two: 2 ulp is the worst seen on an H100)."""
    rng = np.random.default_rng(5)
    init = [_base(rng, 1, h, w, 3) * np.float32(10.0) ** rng.integers(-15, 15, (1, h, w, 1)).astype(np.float32)
            for h, w in [(64, 32), (32, 16), (16, 8)]]
    init[2][0, 0, :3] = [[0, 0, 0], [1e-12, 0, 0], [-0.0, 0, 2]]
    tex = Texture2D([torch.from_numpy(x).to(dev) for x in init])
    ref = [(m / torch.sqrt(torch.clamp(torch.sum(m * m, -1, keepdim=True), min=1e-20))).cpu().numpy() for m in tex.getMips()]  # util.py:29-30
    L.LAUNCHES.clear()
    tex.normalize_()
    assert L.LAUNCHES == {"mip_normalize": 1}
    worst = 0
    for m, r, o in zip(tex.getMips(), ref, mipchain_oracle().normalize(init)):
        g = m.cpu().numpy()
        assert same_bits(g, o)
        assert np.array_equal(np.isnan(g), np.isnan(r))
        fin = np.isfinite(g) & np.isfinite(r)
        worst = max(worst, int(np.abs(g[fin].view(np.int32).astype(np.int64) - r[fin].view(np.int32).astype(np.int64)).max()))
        assert same_bits(g[~fin], r[~fin])
    print("normalize_: worst difference to safe_normalize %d ulp" % worst)
    assert worst <= 2
    with pytest.raises(ValueError, match="3 channels"):
        Texture2D(torch.ones(1, 4, 4, 4, device=dev)).normalize_()


def test_cuda_graph_replay_matches_eager(dev):
    """Three samples forward and backward, then clamp_ and normalize_, as one training step of pass 2 runs them."""
    d = np.load(os.path.join(HERE, "golden", "ref_texture2d.npz"))
    uv = torch.from_numpy(d["texc"]).to(dev)
    da = torch.from_numpy(d["texc_deriv"]).to(dev)
    rng = np.random.default_rng(6)
    init = {"kd": rng.uniform(0, 1, (1, 128, 128, 4)), "ks": rng.uniform(0, 1, (1, 128, 128, 3)), "normal": rng.normal(size=(1, 128, 128, 3))}
    init = {k: torch.from_numpy(v.astype(np.float32)).to(dev) for k, v in init.items()}
    mm = {"kd": _mm(dev, [0.1] * 4, [0.9] * 4), "ks": _mm(dev, [0.0, 0.2, 0.0], [0.0, 0.8, 1.0]), "normal": _mm(dev, [-1, -1, 0], [1, 1, 1])}
    texs = {k: Texture2D(v.clone().requires_grad_(True), min_max=mm[k]) for k, v in init.items()}
    dys = {k: torch.from_numpy(rng.uniform(0.1, 1, (2, 24, 32, v.shape[3])).astype(np.float32)).to(dev) for k, v in init.items()}

    def step():
        outs, grads = [], []
        for k, t in texs.items():
            with torch.no_grad():
                t.data.copy_(init[k])
            t.data.grad = None
            y = t.sample(uv, da)
            y.backward(dys[k])
            outs.append(y.detach())
            grads.append(t.data.grad)
        with torch.no_grad():
            for t in texs.values():
                t.clamp_()
            texs["normal"].normalize_()
        return outs + [t.data.detach() for t in texs.values()], grads

    ref_out, ref_grads = [[x.clone() for x in r] for r in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out, grads = step()
    for _ in range(2):
        gr.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, ref_out):
        assert same_bits(a, b)
    for a, b in zip(grads, ref_grads):          # d tex of each level: float atomics in another order, then the deterministic fold
        assert torch.equal(a == 0, b == 0) and rel_l2(a.cpu().numpy(), b.cpu().numpy()) <= 1e-5
