"""GPU: the fused MLP texture (csrc/mlptexture.cu, nvdiffrecmc_b200.mlptexture.MLPTexture3D) against the fp32 CPU oracle -- output, saved
encoding, d texc and d W bit for bit, d params per element within the bound of two summation orders of the same fp32 terms -- on edge
inputs and at the chunk boundaries of d W; plus the drop-in's reproduction of the reference's MLPTexture3D, its initialisation,
needs_input_grad, no_grad, CUDA-graph replay and a small training run."""
import os

import numpy as np
import pytest
import torch

from common import check_scatter_fp32, rel_l2
from oracle.hashgrid import REF_CONFIG
from oracle.mlptexture import MLPTEX_CHUNK, mlptexture_oracle
from nvdiffrecmc_b200 import _lib as L
from nvdiffrecmc_b200.mlptexture import MLPTexture3D

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
K = MLPTEX_CHUNK
AABB = np.array([[-1.0, -0.5, -0.8], [1.1, 0.9, 0.7]], np.float32)


def _points(n, seed, nonfinite=False):
    """Points inside the AABB, outside it, exactly on its faces (and, with nonfinite, +-inf and NaN coordinates)."""
    rng = np.random.default_rng(seed)
    u = rng.uniform(-0.2, 1.2, (n, 3)).astype(np.float32)
    t = (AABB[0] + u * (AABB[1] - AABB[0])).astype(np.float32)
    k = rng.integers(0, 8, (n, 3))
    lo, hi = np.broadcast_to(AABB[0], (n, 3)), np.broadcast_to(AABB[1], (n, 3))
    t[k == 1] = lo[k == 1]
    t[k == 2] = hi[k == 2]
    if nonfinite:
        t[k == 3] = np.inf
        t[k == 4] = -np.inf
        t[k == 5] = np.nan
    return t


def _texture(dev, C, hidden, seed, zero_weights=False):
    torch.manual_seed(seed)
    tex = MLPTexture3D(torch.tensor(AABB, device=dev), channels=C, hidden=hidden,
                       min_max=[torch.linspace(-0.2, 0.1, C, device=dev), torch.linspace(0.8, 1.3, C, device=dev)])
    rng = np.random.default_rng(seed)
    with torch.no_grad():
        tex.encoder.params.copy_(torch.from_numpy(rng.uniform(-1, 1, tex.encoder.params.numel()).astype(np.float32)))
        for w in tex.net.weights():
            w.copy_(torch.zeros_like(w) if zero_weights else torch.from_numpy(rng.normal(0, 0.4, tuple(w.shape)).astype(np.float32)))
    return tex


def _np(v):
    return v.detach().cpu().numpy()


def _mm(tex):
    return np.stack([_np(tex.min_max[0]), _np(tex.min_max[1])])


def _run(tex, t, g, dev):
    tt = torch.from_numpy(t).to(dev).requires_grad_(True)
    for p in tex.parameters():
        p.grad = None
    out = tex.sample(tt)
    _run.enc = out.grad_fn.next_functions[0][0].saved_tensors[4].clone() if out.numel() else None   # out: a view of the [n, C] output
    out.backward(torch.from_numpy(g).to(dev))
    return out, tt.grad, tex.encoder.params.grad, [w.grad for w in tex.net.weights()]


def _oracle(tex, t, g):
    o = mlptexture_oracle()
    lv = o.levels(REF_CONFIG)
    ws = [_np(w) for w in tex.net.weights()]
    p = _np(tex.encoder.params)
    out, enc = o.mlptex_forward(t, AABB, _mm(tex), p, lv, ws)
    dp, dt, dw = o.mlptex_backward(t, AABB, _mm(tex), p, lv, ws, g)
    return out, enc, dt, dp * 128, dw, lv


def _dp_stats(tex, t, g):
    """(abs sum x 128, count) of the fp32 oracle's d params terms, in the units of the kernel's gradient (the reference's x128)"""
    o = mlptexture_oracle()
    lv = o.levels(REF_CONFIG)
    ws = [_np(w) for w in tex.net.weights()]
    p = _np(tex.encoder.params)
    a = o.mlptex_backward(t, AABB, _mm(tex), p, lv, ws, g, want_t=False, want_w=False, terms="abs")[0]
    n = o.mlptex_backward(t, AABB, _mm(tex), p, lv, ws, g, want_t=False, want_w=False, terms="count")[0]
    return a * 128, n


def _check_dparams(dp, ref, stats, what="d params"):
    """d params per element: the kernel adds the fp32 oracle's terms w_c d e (x128) in another order"""
    check_scatter_fp32(what, dp, ref, stats[0], stats[1], tag="mlptexture")


def _saved_encoding(out):
    """The encoding the forward saved for the backward, in the last _run."""
    return _run.enc


@pytest.mark.parametrize("C,hidden", [(1, 1), (3, 2), (6, 2), (8, 4)])
@pytest.mark.parametrize("n", [0, 1, 31, 255, 256, 257, K - 1, K, K + 1, 3 * K + 5, 65537])
def test_bit_identical_to_the_oracle(dev, n, C, hidden):
    tex = _texture(dev, C, hidden, seed=n + C)
    t = _points(n, seed=n)
    g = np.random.default_rng(n + 1).normal(size=(n, C)).astype(np.float32)
    g[::5] = 0.0
    out, dt, dp, dw = _run(tex, t, g, dev)
    r_out, r_enc, r_dt, r_dp, r_dw, lv = _oracle(tex, t, g)
    assert out.shape == (n, C)
    assert np.array_equal(_np(out), r_out)
    if n > 0:
        assert np.array_equal(_np(_saved_encoding(out)), r_enc)
    assert np.array_equal(_np(dt), r_dt)
    for a, b in zip(dw, r_dw):
        assert np.array_equal(_np(a), b)
    _check_dparams(_np(dp), r_dp, _dp_stats(tex, t, g), "d params n=%d C=%d hidden=%d" % (n, C, hidden))


def test_nonfinite_points_match_the_oracle_where_finite(dev):
    n = 20000
    tex = _texture(dev, 6, 2, seed=3)
    t = _points(n, seed=5, nonfinite=True)
    g = np.random.default_rng(6).normal(size=(n, 6)).astype(np.float32)
    out, dt, dp, dw = _run(tex, t, g, dev)
    torch.cuda.synchronize()
    r_out, r_enc, r_dt, r_dp, r_dw, lv = _oracle(tex, t, g)
    assert np.isnan(_np(out)).any()
    assert np.array_equal(_np(out), r_out, equal_nan=True)
    assert np.array_equal(_np(_saved_encoding(out)), r_enc, equal_nan=True)
    assert np.array_equal(_np(dt), r_dt, equal_nan=True)
    for a, b in zip(dw, r_dw):
        assert np.array_equal(_np(a), b, equal_nan=True)
    fin = np.isfinite(r_dp)
    assert np.array_equal(np.isfinite(_np(dp)), fin)
    a, cnt = _dp_stats(tex, t, g)
    _check_dparams(np.where(fin, _np(dp), 0), np.where(fin, r_dp, 0), (np.where(fin, a, 0), np.where(fin, cnt, 0)),
                   "d params, non-finite points")


def test_dead_relus_give_exactly_zero_gradients(dev):
    tex = _texture(dev, 6, 2, seed=1, zero_weights=True)
    t = _points(5000, seed=2)
    g = np.random.default_rng(3).normal(size=(5000, 6)).astype(np.float32)
    out, dt, dp, dw = _run(tex, t, g, dev)
    assert not dt.any() and not dp.any() and not any(w.any() for w in dw)


def test_zero_upstream_gradient_points_add_nothing(dev):
    """A checkerboard of points with zero upstream gradient, all parked on one spot: the table entries only that spot touches get no
    gradient and those points' d texc is exactly zero."""
    n = 1 << 16
    tex = _texture(dev, 6, 2, seed=4)
    t = _points(n, seed=7)
    t[::2] = (AABB[0] + 0.37 * (AABB[1] - AABB[0])).astype(np.float32)
    g = np.random.default_rng(8).normal(size=(n, 6)).astype(np.float32)
    g[::2] = 0.0
    out, dt, dp, dw = _run(tex, t, g, dev)
    r_out, r_enc, r_dt, r_dp, r_dw, lv = _oracle(tex, t, g)
    assert not dt[::2].any()
    _check_dparams(_np(dp), r_dp, _dp_stats(tex, t, g), "d params, zero-gradient spot")
    only_spot = (_oracle(tex, t[:1], np.ones((1, 6), np.float32))[3] != 0) & (_oracle(tex, t[1::2], g[1::2])[3] == 0)
    assert only_spot.any() and not _np(dp)[only_spot].any()


def test_weight_gradients_are_bit_identical_across_calls(dev):
    tex = _texture(dev, 6, 2, seed=9)
    t = _points(300000, seed=10)
    g = np.random.default_rng(11).normal(size=(300000, 6)).astype(np.float32)
    a = [w.clone() for w in _run(tex, t, g, dev)[3]]
    b = _run(tex, t, g, dev)[3]
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_dropin_reproduces_the_reference_mlptexture(dev):
    d = np.load(os.path.join(HERE, "golden", "ref_mlptexture.npz"))
    t = lambda k: torch.from_numpy(d[k]).to(dev)
    tex = MLPTexture3D(t("aabb"), channels=6, min_max=[t("min_max")[0], t("min_max")[1]])
    assert np.array_equal(_np(tex.encoder.params[:8]), d["params_head"])
    assert {k: tuple(v.shape) for k, v in tex.state_dict().items()} == {
        "encoder.params": (12599920,), "net.net.0.weight": (32, 32), "net.net.2.weight": (32, 32), "net.net.4.weight": (6, 32)}
    with torch.no_grad():
        for k, w in enumerate(tex.net.weights()):
            w.copy_(t("w%d" % k))
    pts = t("points").requires_grad_(True)
    out = tex.sample(pts)
    assert out.shape == (1, 16, 16, 6)
    out.backward(t("dout"))
    assert rel_l2(_np(out), d["out"]) <= 1e-5
    assert rel_l2(_np(pts.grad), d["d_points"]) <= 1e-4
    for k, w in enumerate(tex.net.weights()):
        assert rel_l2(_np(w.grad), d["d_w%d" % k]) <= 1e-4, k
    ref = np.zeros(tex.encoder.params.numel(), np.float32)
    ref[d["params_grad_idx"]] = d["params_grad_val"]
    assert rel_l2(_np(tex.encoder.params.grad), ref) <= 1e-4


def test_initialisation_follows_the_reference_sequence(dev):
    """render/mlptexture.py:22-29: Linear layers built on the CPU (their default init draws from the CPU generator), the Sequential moved
    to the GPU, then kaiming_uniform_(relu) on the GPU tensors in layer order."""
    torch.manual_seed(123)
    tex = MLPTexture3D(torch.tensor(AABB, device=dev), channels=6, min_max=[torch.zeros(6, device=dev), torch.ones(6, device=dev)])
    torch.manual_seed(123)
    lin = [torch.nn.Linear(32, 32, bias=False), torch.nn.Linear(32, 32, bias=False), torch.nn.Linear(32, 6, bias=False)]
    ws = [m.weight.detach().to(dev) for m in lin]
    for w in ws:
        torch.nn.init.kaiming_uniform_(w, nonlinearity="relu")
    for a, b in zip(tex.net.weights(), ws):
        assert torch.equal(a, b)


def _bench_positions(dev, res=512, B=8):
    import bench
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200 import synth
    from nvdiffrecmc_b200.raster import interpolate, rasterize
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    ctx = ou.OptiXContext()
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32),
                       device=dev)
    rast = rasterize(ctx, mtx, (res, res))
    pos, _ = interpolate(vt, rast, ft)
    return pos.detach(), torch.stack([vt.min(0).values, vt.max(0).values]), rast[..., 3] > 0


def test_matches_the_torch_composition_on_bench_positions(dev):
    """Both samples of render.py:61-64 (gb_pos and a jittered copy) at 2 x 8 x 512^2, against the torch composition of
    test_gpu_hashgrid.py's reference check (with the reference's hooks)."""
    pos, aabb, cov = _bench_positions(dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    pts = torch.stack([pos + torch.randn(pos.shape, device=dev, generator=gen) * 0.01, pos])
    g = torch.randn(pts.shape[:-1] + (6,), device=dev, generator=gen) * cov[None, ..., None]
    torch.manual_seed(0)
    tex = MLPTexture3D(aabb, channels=6, min_max=[torch.tensor([0.0, 0.0, 0.0, 0.0, 0.08, 0.0], device=dev), torch.ones(6, device=dev)])
    with torch.no_grad():
        tex.encoder.params.uniform_(-1, 1, generator=gen)
    p1 = pts.clone().requires_grad_(True)
    out = tex.sample(p1)
    out.backward(g)
    # the torch composition, on copies of the same parameters
    from nvdiffrecmc_b200.tinycudann import Encoding
    enc = Encoding(3, REF_CONFIG)
    with torch.no_grad():
        enc.params.copy_(tex.encoder.params)
    enc.register_full_backward_hook(lambda m, gi, go: (gi[0] / 128.0,))
    lin = [torch.nn.Linear(32, 32, bias=False), torch.nn.Linear(32, 32, bias=False), torch.nn.Linear(32, 6, bias=False)]
    net = torch.nn.Sequential(lin[0], torch.nn.ReLU(), lin[1], torch.nn.ReLU(), lin[2]).to(dev)
    with torch.no_grad():
        for m, w in zip(lin, tex.net.weights()):
            m.weight.copy_(w)
    net.register_full_backward_hook(lambda m, gi, go: (gi[0] * 128.0,))
    mm = torch.stack(tex.min_max)
    p2 = pts.clone().requires_grad_(True)
    x = torch.clamp((p2.view(-1, 3) - aabb[0][None]) / (aabb[1] - aabb[0])[None], min=0, max=1)
    ref = (torch.sigmoid(net(enc(x.contiguous()))) * (mm[1] - mm[0])[None] + mm[0][None]).view(*p2.shape[:-1], 6)
    ref.backward(g)
    assert rel_l2(_np(out), _np(ref)) <= 1e-5
    assert rel_l2(_np(p1.grad), _np(p2.grad)) <= 1e-4
    for a, m in zip(tex.net.weights(), lin):
        assert rel_l2(_np(a.grad), _np(m.weight.grad)) <= 1e-4
    assert rel_l2(_np(tex.encoder.params.grad), _np(enc.params.grad)) <= 1e-4


def test_needs_input_grad_and_no_grad(dev):
    n = 40000
    tex = _texture(dev, 6, 2, seed=12)
    t = _points(n, seed=13)
    g = torch.from_numpy(np.random.default_rng(14).normal(size=(n, 6)).astype(np.float32)).to(dev)
    out, dt, dp, dw = [v.clone() if isinstance(v, torch.Tensor) else [w.clone() for w in v] for v in _run(tex, t, g.cpu().numpy(), dev)]
    params = [tex.encoder.params] + tex.net.weights()
    for want_t in (False, True):
        for mask in range(1 << len(params)):
            if not want_t and mask == 0:
                continue
            for k, p in enumerate(params):
                p.grad = None
                p.requires_grad_(bool(mask >> k & 1))
            tt = torch.from_numpy(t).to(dev).requires_grad_(want_t)
            L.LAUNCHES.clear()
            tex.sample(tt).backward(g)
            want_w = any(mask >> k & 1 for k in range(1, len(params)))
            assert L.LAUNCHES == {"mlptex_fwd": 1, "mlptex_bwd_dw" if want_w else "mlptex_bwd": 2 if want_w else 1}
            assert (tt.grad is not None) == want_t and (not want_t or torch.equal(tt.grad, dt))
            if mask & 1:
                assert torch.equal(tex.encoder.params.grad == 0, dp == 0)
                assert rel_l2(_np(tex.encoder.params.grad), _np(dp)) <= 1e-6
            else:
                assert tex.encoder.params.grad is None
            for k, w in enumerate(tex.net.weights()):
                assert (w.grad is not None) == bool(mask >> (k + 1) & 1)
                if w.grad is not None:
                    assert torch.equal(w.grad, dw[k])
    for p in params:
        p.requires_grad_(True)
    L.LAUNCHES.clear()
    with torch.no_grad():
        y = tex.sample(torch.from_numpy(t).to(dev))
    assert y.grad_fn is None and L.LAUNCHES == {"mlptex_fwd": 1} and torch.equal(y, out.detach())
    # fp64, non-contiguous, batched [..., 3] input
    ts = torch.from_numpy(np.ascontiguousarray(t.T)).to(dev).double().t().reshape(200, 200, 3)
    assert torch.equal(tex.sample(ts).reshape(n, 6), out.detach())


def test_rejects_bad_inputs(dev):
    tex = _texture(dev, 6, 2, seed=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        tex.sample(torch.rand(4, 3))
    with pytest.raises(ValueError, match=r"\[\.\.\., 3\]"):
        tex.sample(torch.rand(4, 2, device=dev))
    with pytest.raises(TypeError):
        tex.sample(torch.ones(4, 3, dtype=torch.int32, device=dev))


def test_cuda_graph_replay_matches_eager(dev):
    n = 100000
    tex = _texture(dev, 6, 2, seed=15)
    ts = torch.from_numpy(_points(n, seed=16)).to(dev)
    g = torch.randn(n, 6, device=dev, generator=torch.Generator(device=dev).manual_seed(0))

    def step():
        tg = ts.clone().requires_grad_(True)
        for p in tex.parameters():
            p.grad = None
        y = tex.sample(tg)
        y.backward(g)
        return [y.detach(), tg.grad] + [w.grad for w in tex.net.weights()] + [tex.encoder.params.grad]

    eager = [v.clone() for v in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(out[:-1], eager[:-1]):
        assert torch.equal(a, b)
    assert torch.equal(out[-1] == 0, eager[-1] == 0) and rel_l2(_np(out[-1]), _np(eager[-1])) <= 1e-6


def test_training_fits_a_colour_field(dev):
    """The drop-in fitted with Adam to a procedural 3-D colour field, at 64k points per step (as test_gpu_hashgrid.py's torch-MLP fit)."""
    torch.manual_seed(0)
    tex = MLPTexture3D(torch.tensor([[0.0] * 3, [1.0] * 3], device=dev), channels=3, min_max=[torch.zeros(3, device=dev), torch.ones(3, device=dev)])
    opt = torch.optim.Adam([{"params": tex.encoder.parameters(), "lr": 1e-2}, {"params": tex.net.parameters(), "lr": 1e-2}],
                           betas=(0.9, 0.99), eps=1e-15)
    g = torch.Generator(device=dev).manual_seed(1)

    def field(x):
        return torch.stack([0.5 + 0.5 * torch.sin(6.0 * x[:, 0] + 3.0 * x[:, 1]), 0.5 + 0.5 * torch.cos(9.0 * x[:, 1] * x[:, 2]),
                            (x[:, 0] + x[:, 2]) * 0.5 + 0.2 * torch.sin(20.0 * x[:, 1])], -1)

    losses = []
    for it in range(300):
        x = torch.rand(65536, 3, device=dev, generator=g)
        loss = torch.mean((tex.sample(x) - field(x)) ** 2)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    first, last = np.mean(losses[:5]), np.mean(losses[-10:])
    print("mlp texture fit: loss %.3e -> %.3e" % (first, last))
    assert last * 10 <= first
