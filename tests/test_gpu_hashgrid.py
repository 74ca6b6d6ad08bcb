"""GPU: the hash-grid encoding (csrc/hashgrid.cu) against the fp32 CPU oracle -- forward and d x bit for bit, d params to the atomics'
summation order -- plus autograd's needs_input_grad, CUDA-graph replay, the frozen output of the reference's MLPTexture3D and a small
training run."""
import os

import numpy as np
import pytest
import torch

from common import rel_l2
from oracle.hashgrid import REF_CONFIG, hashgrid_oracle
from nvdiffrecmc_b200 import _lib as L
from nvdiffrecmc_b200.tinycudann import Encoding

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
EDGE = {"otype": "HashGrid", "n_levels": 5, "log2_hashmap_size": 9, "base_resolution": 4, "per_level_scale": 2.0}
PADDED = {"otype": "HashGrid", "n_levels": 3, "log2_hashmap_size": 10, "base_resolution": 5, "per_level_scale": 1.5}


def _points(n, cfg, seed):
    """Uniform points mixed with exact 0, exact 1, cell faces of every level and finite out-of-range values in [-0.5, 1.5]."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    k = rng.integers(0, 5, (n, 3))
    x[k == 1] = 0.0
    x[k == 2] = 1.0
    lv = hashgrid_oracle().levels(cfg)
    faces = np.concatenate([((np.arange(int(r)) - 0.5) / float(s)).astype(np.float32) for r, s in zip(lv["res"], lv["scale"]) if s > 0])
    x[k == 3] = rng.choice(faces, int((k == 3).sum()))
    x[k == 4] = rng.uniform(-0.5, 1.5, int((k == 4).sum())).astype(np.float32)
    return x, lv


def _enc(dev, cfg, params=None):
    enc = Encoding(3, cfg)
    if params is not None:
        with torch.no_grad():
            enc.params.copy_(torch.from_numpy(params))
    return enc


def _random_params(enc, seed):
    return np.random.default_rng(seed).uniform(-1, 1, enc.params.numel()).astype(np.float32)


@pytest.mark.parametrize("cfg", [REF_CONFIG, EDGE, PADDED], ids=["ref", "edge", "padded"])
@pytest.mark.parametrize("n", [1, 31, 33, 4097, 1048576])
def test_forward_and_dx_are_bit_identical_to_the_oracle(dev, cfg, n):
    o = hashgrid_oracle()
    x, lv = _points(n, cfg, seed=n)
    enc = _enc(dev, cfg)
    p = _random_params(enc, 3)
    enc = _enc(dev, cfg, p)
    xt = torch.from_numpy(x).to(dev).requires_grad_(True)
    y = enc(xt)
    assert y.shape == (n, 2 * lv["n_levels"]) and y.dtype == torch.float32
    assert np.array_equal(y.detach().cpu().numpy(), o.forward(x, p, lv))
    dy = np.random.default_rng(n + 1).normal(size=y.shape).astype(np.float32)
    dy[::4] = 0.0
    dy[1::4, ::3] = 0.0
    y.backward(torch.from_numpy(dy).to(dev))
    dp_ref, dx_ref = o.backward(x, p, lv, dy)
    assert np.array_equal(xt.grad.cpu().numpy(), dx_ref)
    _check_dparams(enc.params.grad.cpu().numpy(), dp_ref, lv)


def _check_dparams(dp, ref, lv):
    assert np.array_equal(dp == 0, ref == 0)
    for l in range(lv["n_levels"]):
        a, b = 2 * int(lv["offset"][l]), 2 * int(lv["offset"][l + 1])
        if np.any(ref[a:b]):
            assert rel_l2(dp[a:b], ref[a:b]) <= 1e-5, l


@pytest.mark.parametrize("cfg", [REF_CONFIG, EDGE], ids=["ref", "edge"])
def test_dparams_with_a_zero_gradient_hot_spot(dev, cfg):
    """Half the points coincide at one spot with a zero upstream gradient, as uncovered pixels do after the AABB normalisation."""
    o = hashgrid_oracle()
    n = 1 << 18
    x, lv = _points(n, cfg, seed=11)
    x[::2] = np.float32(0.5)
    enc = _enc(dev, cfg)
    p = _random_params(enc, 5)
    enc = _enc(dev, cfg, p)
    dy = np.random.default_rng(12).normal(size=(n, 2 * lv["n_levels"])).astype(np.float32)
    dy[::2] = 0.0
    y = enc(torch.from_numpy(x).to(dev))
    y.backward(torch.from_numpy(dy).to(dev))
    dp_ref, _ = o.backward(x, p, lv, dy, want_x=False)
    _check_dparams(enc.params.grad.cpu().numpy(), dp_ref, lv)


def test_needs_input_grad_and_no_grad(dev):
    o = hashgrid_oracle()
    x, lv = _points(5000, EDGE, seed=2)
    enc = _enc(dev, EDGE)
    p = _random_params(enc, 1)
    enc = _enc(dev, EDGE, p)
    xt = torch.from_numpy(x).to(dev)
    dy = np.random.default_rng(3).normal(size=(5000, 10)).astype(np.float32)
    dp_ref, dx_ref = o.backward(x, p, lv, dy)
    # x without grad: only d params (one kernel, no d x pass)
    L.LAUNCHES.clear()
    enc(xt).backward(torch.from_numpy(dy).to(dev))
    assert L.LAUNCHES == {"hashgrid_fwd": 1, "hashgrid_bwd": 1}
    _check_dparams(enc.params.grad.cpu().numpy(), dp_ref, lv)
    # params frozen: only d x
    enc.params.grad = None
    enc.params.requires_grad_(False)
    xg = xt.clone().requires_grad_(True)
    enc(xg).backward(torch.from_numpy(dy).to(dev))
    assert enc.params.grad is None and np.array_equal(xg.grad.cpu().numpy(), dx_ref)
    enc.params.requires_grad_(True)
    # no_grad: forward only
    L.LAUNCHES.clear()
    with torch.no_grad():
        y = enc(xg)
    assert y.grad_fn is None and not y.requires_grad and L.LAUNCHES == {"hashgrid_fwd": 1}
    # fp64 / non-contiguous input is cast to contiguous fp32
    xs = torch.from_numpy(np.ascontiguousarray(x.T)).to(dev).double().t()
    assert np.array_equal(enc(xs).detach().cpu().numpy(), o.forward(x, p, lv))


def test_rejects_bad_inputs(dev):
    enc = _enc(dev, EDGE)
    with pytest.raises(RuntimeError, match="CUDA"):
        enc(torch.rand(4, 3))
    with pytest.raises(ValueError, match=r"\[N,3\]"):
        enc(torch.rand(4, 2, device=dev))
    with pytest.raises(TypeError):
        enc(torch.ones(4, 3, dtype=torch.int32, device=dev))
    x0 = torch.rand(0, 3, device=dev, requires_grad=True)
    y = enc(x0)
    assert y.shape == (0, 10)
    y.sum().backward()
    assert x0.grad.shape == (0, 3) and not enc.params.grad.any()


def test_cuda_graph_replay_matches_eager(dev):
    x, lv = _points(100000, REF_CONFIG, seed=4)
    enc = _enc(dev, REF_CONFIG)
    enc = _enc(dev, REF_CONFIG, _random_params(enc, 2))
    xs = torch.from_numpy(x).to(dev)
    dy = torch.randn(100000, 32, device=dev, generator=torch.Generator(device=dev).manual_seed(0))

    def step():
        xg = xs.clone().requires_grad_(True)
        enc.params.grad = None
        y = enc(xg)
        y.backward(dy)
        return y.detach(), xg.grad, enc.params.grad

    y0, dx0, dp0 = [t.clone() for t in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], y0) and torch.equal(out[1], dx0)
    assert torch.equal(out[2] == 0, dp0 == 0) and float(rel_l2(out[2].cpu().numpy(), dp0.cpu().numpy())) <= 1e-6


def test_product_reproduces_the_reference_mlptexture(dev):
    """MLPTexture3D.sample (render/mlptexture.py:87-99) restated on the product: normalise into the AABB, clamp, encode, three bias-free
    Linear layers with ReLU, sigmoid scaled into min_max; with the reference's hooks (x128 on the MLP's input gradient, /128 on the
    encoder's)."""
    d = np.load(os.path.join(HERE, "golden", "ref_mlptexture.npz"))
    t = lambda k: torch.from_numpy(d[k]).to(dev)
    enc = Encoding(3, REF_CONFIG)
    assert np.array_equal(enc.params[:8].detach().cpu().numpy(), d["params_head"])
    enc.register_full_backward_hook(lambda m, gi, go: (gi[0] / 128.0,))
    lin = [torch.nn.Linear(32, 32, bias=False), torch.nn.Linear(32, 32, bias=False), torch.nn.Linear(32, 6, bias=False)]
    net = torch.nn.Sequential(lin[0], torch.nn.ReLU(), lin[1], torch.nn.ReLU(), lin[2]).to(dev)
    with torch.no_grad():
        for k, m in enumerate(lin):
            m.weight.copy_(t("w%d" % k))
    net.register_full_backward_hook(lambda m, gi, go: (gi[0] * 128.0,))
    aabb, mm = t("aabb"), t("min_max")
    pts = t("points").requires_grad_(True)
    x = torch.clamp((pts.view(-1, 3) - aabb[0][None]) / (aabb[1] - aabb[0])[None], min=0, max=1)
    out = torch.sigmoid(net(enc(x.contiguous()))) * (mm[1] - mm[0])[None] + mm[0][None]
    out = out.view(*pts.shape[:-1], 6)
    out.backward(t("dout"))
    n = lambda v: v.detach().cpu().numpy()
    assert rel_l2(n(out), d["out"]) <= 1e-5
    assert rel_l2(n(pts.grad), d["d_points"]) <= 1e-4
    for k, m in enumerate(lin):
        assert rel_l2(n(m.weight.grad), d["d_w%d" % k]) <= 1e-4, k
    ref = np.zeros(enc.params.numel(), np.float32)
    ref[d["params_grad_idx"]] = d["params_grad_val"]
    assert rel_l2(n(enc.params.grad), ref) <= 1e-4


def test_training_fits_a_colour_field(dev):
    """The encoding plus a 3-layer torch MLP, fitted with Adam to a procedural 3-D colour field, at 64k points per step."""
    torch.manual_seed(0)
    enc = Encoding(3, REF_CONFIG)
    net = torch.nn.Sequential(torch.nn.Linear(32, 32, bias=False), torch.nn.ReLU(), torch.nn.Linear(32, 32, bias=False), torch.nn.ReLU(),
                              torch.nn.Linear(32, 3, bias=False)).to(dev)
    opt = torch.optim.Adam([{"params": enc.parameters(), "lr": 1e-2}, {"params": net.parameters(), "lr": 1e-2}], betas=(0.9, 0.99), eps=1e-15)
    g = torch.Generator(device=dev).manual_seed(1)

    def field(x):
        return torch.stack([0.5 + 0.5 * torch.sin(6.0 * x[:, 0] + 3.0 * x[:, 1]), 0.5 + 0.5 * torch.cos(9.0 * x[:, 1] * x[:, 2]),
                            (x[:, 0] + x[:, 2]) * 0.5 + 0.2 * torch.sin(20.0 * x[:, 1])], -1)

    losses = []
    for it in range(300):
        x = torch.rand(65536, 3, device=dev, generator=g)
        loss = torch.mean((torch.sigmoid(net(enc(x))) - field(x)) ** 2)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    first, last = np.mean(losses[:5]), np.mean(losses[-10:])
    print("hash-grid fit: loss %.3e -> %.3e" % (first, last))
    assert last * 10 <= first
