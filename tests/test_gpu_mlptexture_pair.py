"""GPU: MLPTexture3D.sample_pair against two `sample` calls on the same device -- both outputs, both saved encodings, d texc (autograd's
accumulation over the two calls), d offset and every d W bit for bit, d params within the fp32 oracle's two-orders bound -- at the chunk
boundaries of d W, on non-finite and coincident points, the training G-buffer's uncovered pixels, dead ReLUs and an unused jittered
output; plus the fp32 oracle, the reference fixture of render.py:63-64, jitter_taps downstream, needs_input_grad, no_grad, CUDA-graph
replay, determinism and the argument errors."""
import os

import numpy as np
import pytest
import torch

from common import check_scatter_fp32, rel_l2
from oracle.hashgrid import REF_CONFIG
from oracle.mlptexture import MLPTEX_CHUNK, mlptexture_oracle
from mlptexture_pair_oracle import pair_backward, pair_forward
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


def _noise(n, seed, nonfinite=False):
    rng = np.random.default_rng(seed)
    o = rng.normal(0, 0.01, (n, 3)).astype(np.float32)
    o[::9] = 0.0
    if nonfinite:
        k = rng.integers(0, 12, (n, 3))
        o[k == 1] = np.inf
        o[k == 2] = -np.inf
        o[k == 3] = np.nan
    return o


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


def _t(x, dev):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(x).to(dev)


def _grads(tex, tt, oo):
    return [tt.grad, oo.grad, tex.encoder.params.grad] + [w.grad for w in tex.net.weights()]


def _two_calls(tex, t, o, g, gj, dev):
    """render.py:63-64 as the reference writes it: sample(t + o) and sample(t), backward through both."""
    tt, oo = _t(t, dev).clone().requires_grad_(True), _t(o, dev).clone().requires_grad_(True)
    for p in tex.parameters():
        p.grad = None
    out_j = tex.sample(tt + oo)
    out = tex.sample(tt)
    encs = [y.grad_fn.next_functions[0][0].saved_tensors[4].clone() if y.numel() else None for y in (out, out_j)]
    torch.autograd.backward([out_j, out], [_t(gj, dev), _t(g, dev)])
    return [out.detach(), out_j.detach()] + encs + [v.clone() if v is not None else None for v in _grads(tex, tt, oo)]


def _pair(tex, t, o, g, gj, dev):
    tt, oo = _t(t, dev).clone().requires_grad_(True), _t(o, dev).clone().requires_grad_(True)
    for p in tex.parameters():
        p.grad = None
    out, out_j = tex.sample_pair(tt, oo)
    saved = out.grad_fn.next_functions[0][0].saved_tensors if out.numel() else None
    encs = [saved[5].clone(), saved[6].clone()] if saved else [None, None]
    torch.autograd.backward([out, out_j], [_t(g, dev), _t(gj, dev)])
    return [out.detach(), out_j.detach()] + encs + [v.clone() if v is not None else None for v in _grads(tex, tt, oo)]


def _same(a, b, nan=False):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and np.array_equal(_np(a), _np(b), equal_nan=nan)


def _assert_pair_is_two_calls(p, r, nan=False):
    """everything but d params bit for bit: out, out_jit, enc, enc_jit, d texc, d offset, every d W"""
    names = ["out", "out_jit", "enc", "enc_jit", "d texc", "d offset"] + ["d W%d" % k for k in range(len(p) - 7)]
    for name, a, b in zip(names, p[:6] + p[7:], r[:6] + r[7:]):
        assert _same(a, b, nan), name


def _oracle_dparams(tex, t, o, g, gj):
    """the fp32 oracle's d params (x128) with the abs-sum and count of its terms (copied from test_gpu_mlptexture.py's _dp_stats)"""
    orc = mlptexture_oracle()
    lv = orc.levels(REF_CONFIG)
    ws = [_np(w) for w in tex.net.weights()]
    p = _np(tex.encoder.params)
    run = lambda terms: pair_backward(orc, t, o, AABB, _mm(tex), p, lv, ws, g, gj, want_t=False, want_offset=False, want_w=False,
                                                 terms=terms)[0] * (128 if terms != "count" else 1)
    return run("sum"), run("abs"), run("count")


def _check_dparams(dp, tex, t, o, g, gj, what):
    r, a, n = _oracle_dparams(tex, t, o, g, gj)
    fin = np.isfinite(r)
    got = _np(dp)
    assert np.array_equal(np.isfinite(got), fin), what
    check_scatter_fp32(what, np.where(fin, got, 0), np.where(fin, r, 0), np.where(fin, a, 0), np.where(fin, n, 0), tag="mlptexture_pair")


@pytest.mark.parametrize("C,hidden", [(1, 1), (3, 2), (6, 2), (8, 4)])
@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, K - 1, K, K + 1, 3 * K + 5, 65537])
def test_pair_equals_two_sample_calls(dev, n, C, hidden):
    tex = _texture(dev, C, hidden, seed=n + C)
    t, o = _points(n, seed=n), _noise(n, seed=n + 3)
    rng = np.random.default_rng(n + 1)
    g, gj = rng.normal(size=(n, C)).astype(np.float32), rng.normal(size=(n, C)).astype(np.float32)
    g[::5] = 0.0
    gj[::7] = 0.0
    r = _two_calls(tex, t, o, g, gj, dev)
    p = _pair(tex, t, o, g, gj, dev)
    assert p[0].shape == p[1].shape == (n, C)
    _assert_pair_is_two_calls(p, r)
    _check_dparams(p[6], tex, t, o, g, gj, "d params n=%d C=%d hidden=%d" % (n, C, hidden))
    if n <= 3 * K + 5:             # the forward and d texc against the fp32 oracle, bit for bit
        orc = mlptexture_oracle()
        lv = orc.levels(REF_CONFIG)
        ws = [_np(w) for w in tex.net.weights()]
        out, enc, out_j, enc_j = pair_forward(orc, t, o, AABB, _mm(tex), _np(tex.encoder.params), lv, ws)
        for a, b in zip(p[:4], (out, out_j, enc, enc_j)):
            assert n == 0 or np.array_equal(_np(a), b)
        _, dt, do, dw = pair_backward(orc, t, o, AABB, _mm(tex), _np(tex.encoder.params), lv, ws, g, gj, want_params=False)
        assert np.array_equal(_np(p[4]), dt) and np.array_equal(_np(p[5]), do)
        for a, b in zip(p[7:], dw):
            assert np.array_equal(_np(a), b)


def test_nonfinite_texc_and_offset(dev):
    n = 20000
    tex = _texture(dev, 6, 2, seed=3)
    t, o = _points(n, seed=5, nonfinite=True), _noise(n, seed=6, nonfinite=True)
    rng = np.random.default_rng(6)
    g, gj = rng.normal(size=(n, 6)).astype(np.float32), rng.normal(size=(n, 6)).astype(np.float32)
    r = _two_calls(tex, t, o, g, gj, dev)
    p = _pair(tex, t, o, g, gj, dev)
    assert np.isnan(_np(p[0])).any() and np.isnan(_np(p[1])).any()
    _assert_pair_is_two_calls(p, r, nan=True)
    _check_dparams(p[6], tex, t, o, g, gj, "d params, non-finite points")


def test_zero_offset_gives_two_equal_samples(dev):
    n = 5000
    tex = _texture(dev, 6, 2, seed=7)
    t, o = _points(n, seed=8), np.zeros((n, 3), np.float32)
    rng = np.random.default_rng(9)
    g, gj = rng.normal(size=(n, 6)).astype(np.float32), rng.normal(size=(n, 6)).astype(np.float32)
    r = _two_calls(tex, t, o, g, gj, dev)
    p = _pair(tex, t, o, g, gj, dev)
    _assert_pair_is_two_calls(p, r)
    assert torch.equal(p[0], p[1]) and torch.equal(p[2], p[3])
    _check_dparams(p[6], tex, t, o, g, gj, "d params, offset 0")


def test_dead_relus_give_exactly_zero_gradients(dev):
    n = 5000
    tex = _texture(dev, 6, 2, seed=1, zero_weights=True)
    t, o = _points(n, seed=2), _noise(n, seed=3)
    rng = np.random.default_rng(3)
    g, gj = rng.normal(size=(n, 6)).astype(np.float32), rng.normal(size=(n, 6)).astype(np.float32)
    r = _two_calls(tex, t, o, g, gj, dev)
    p = _pair(tex, t, o, g, gj, dev)
    _assert_pair_is_two_calls(p, r)
    assert not any(v.any() for v in p[4:])


def test_unused_jittered_output_is_a_null_upstream_gradient(dev):
    """Only `out` is used: autograd hands the pair's backward no d out_jit, which reaches mcs_mlptex_pair_bwd as a null pointer; the
    result is the one of an explicit zero d out_jit."""
    n = 3 * K + 5
    tex = _texture(dev, 6, 2, seed=21)
    t, o = _points(n, seed=22), _noise(n, seed=23)
    g = np.random.default_rng(24).normal(size=(n, 6)).astype(np.float32)
    z = np.zeros_like(g)
    ref = _pair(tex, t, o, g, z, dev)
    tt, oo = _t(t, dev).clone().requires_grad_(True), _t(o, dev).clone().requires_grad_(True)
    for p in tex.parameters():
        p.grad = None
    out, _ = tex.sample_pair(tt, oo)
    out.backward(_t(g, dev))
    got = _grads(tex, tt, oo)
    assert torch.equal(got[0], ref[4]) and torch.equal(got[1], ref[5]) and not got[1].any()
    for a, b in zip(got[3:], ref[7:]):
        assert torch.equal(a, b)
    assert torch.equal(got[2] == 0, ref[6] == 0) and rel_l2(_np(got[2]), _np(ref[6])) <= 1e-6


def _bench_positions(dev, res=512, B=8):
    """The training G-buffer's positions (copied from test_gpu_mlptexture.py): the bench mesh rasterized in B views, 0 where uncovered."""
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
    return pos.detach(), torch.stack([vt.min(0).values, vt.max(0).values]), rast


def test_training_gbuffer_at_8x512(dev):
    """hashbench's workload: 8 x 512^2 pixels of the bench mesh, uncovered pixels at the origin with zero upstream gradient."""
    pos, aabb, rast = _bench_positions(dev)
    cov = rast[..., 3] > 0
    gen = torch.Generator(device=dev).manual_seed(0)
    noise = torch.normal(mean=0, std=0.01, size=pos.shape, device=dev, generator=gen)
    g = torch.randn(pos.shape[:-1] + (6,), device=dev, generator=gen) * cov[..., None]
    gj = torch.randn(pos.shape[:-1] + (6,), device=dev, generator=gen) * cov[..., None]
    torch.manual_seed(0)
    tex = MLPTexture3D(aabb, channels=6, min_max=[torch.tensor([0.0, 0.0, 0.0, 0.0, 0.08, 0.0], device=dev), torch.ones(6, device=dev)])
    with torch.no_grad():
        tex.encoder.params.uniform_(-1, 1, generator=gen)
    r = _two_calls(tex, pos, noise, g, gj, dev)
    p = _pair(tex, pos, noise, g, gj, dev)
    _assert_pair_is_two_calls(p, r)
    assert torch.equal(p[6] == 0, r[6] == 0) and rel_l2(_np(p[6]), _np(r[6])) <= 1e-6
    # jitter_taps downstream, as shade() uses the two samples (MLP path): the same outputs and gradients
    from nvdiffrecmc_b200.regularizer import jitter_taps
    B, H, W = pos.shape[:3]
    jitter = torch.rand(B, H, W, 2, device=dev, generator=gen)
    nrm = torch.nn.functional.normalize(torch.randn(B, H, W, 3, device=dev, generator=gen), dim=-1)
    res = []
    for fn in ("two", "pair"):
        tt, oo = pos.clone().requires_grad_(True), noise.clone()
        for q in tex.parameters():
            q.grad = None
        if fn == "pair":
            all_tex, all_tex_jitter = tex.sample_pair(tt, oo)
        else:
            all_tex_jitter = tex.sample(tt + oo)
            all_tex = tex.sample(tt)
        taps = jitter_taps(rast, jitter, all_tex[..., 0:3], all_tex[..., 3:6], nrm, kd_jitter=all_tex_jitter[..., 0:3],
                           ks_jitter=all_tex_jitter[..., 3:6])
        keys = sorted(taps)
        ups = [torch.randn(taps[k].shape, device=dev, generator=torch.Generator(device=dev).manual_seed(i)) for i, k in enumerate(keys)]
        torch.autograd.backward([taps[k] for k in keys], ups)
        res.append([taps[k].detach() for k in keys] + [tt.grad] + [w.grad for w in tex.net.weights()])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_dropin_reproduces_the_reference_pair(dev):
    """tests/golden/ref_mlptexture_pair.npz: render.py:63-64 on the reference's MLPTexture3D, with the bars of test_gpu_mlptexture.py's
    test_dropin_reproduces_the_reference_mlptexture."""
    d = np.load(os.path.join(HERE, "golden", "ref_mlptexture_pair.npz"))
    t = lambda k: torch.from_numpy(d[k]).to(dev)
    tex = MLPTexture3D(t("aabb"), channels=6, min_max=[t("min_max")[0], t("min_max")[1]])
    assert np.array_equal(_np(tex.encoder.params[:8]), d["params_head"])
    with torch.no_grad():
        for k, w in enumerate(tex.net.weights()):
            w.copy_(t("w%d" % k))
    gb_pos = t("gb_pos").requires_grad_(True)
    all_tex, all_tex_jitter = tex.sample_pair(gb_pos, t("noise"))
    assert all_tex.shape == all_tex_jitter.shape == (2, 13, 19, 6)
    torch.autograd.backward([all_tex, all_tex_jitter], [t("dout"), t("dout_jit")])
    assert rel_l2(_np(all_tex), d["out"]) <= 1e-5 and rel_l2(_np(all_tex_jitter), d["out_jit"]) <= 1e-5
    assert rel_l2(_np(gb_pos.grad), d["d_gb_pos"]) <= 1e-4
    for k, w in enumerate(tex.net.weights()):
        assert rel_l2(_np(w.grad), d["d_w%d" % k]) <= 1e-4, k
    ref = np.zeros(tex.encoder.params.numel(), np.float32)
    ref[d["params_grad_idx"]] = d["params_grad_val"]
    assert rel_l2(_np(tex.encoder.params.grad), ref) <= 1e-4


def test_needs_input_grad_and_no_grad(dev):
    n = 40000
    tex = _texture(dev, 6, 2, seed=12)
    t, o = _points(n, seed=13), _noise(n, seed=14)
    rng = np.random.default_rng(14)
    g = torch.from_numpy(rng.normal(size=(n, 6)).astype(np.float32)).to(dev)
    gj = torch.from_numpy(rng.normal(size=(n, 6)).astype(np.float32)).to(dev)
    full = _pair(tex, t, o, g, gj, dev)
    params = [tex.encoder.params] + tex.net.weights()
    for want_t in (False, True):
        for want_o in (False, True):
            for mask in range(1 << len(params)):
                if not want_t and not want_o and mask == 0:
                    continue
                for k, p in enumerate(params):
                    p.grad = None
                    p.requires_grad_(bool(mask >> k & 1))
                tt = torch.from_numpy(t).to(dev).requires_grad_(want_t)
                oo = torch.from_numpy(o).to(dev).requires_grad_(want_o)
                L.LAUNCHES.clear()
                torch.autograd.backward(list(tex.sample_pair(tt, oo)), [g, gj])
                want_w = any(mask >> k & 1 for k in range(1, len(params)))
                assert L.LAUNCHES == {"mlptex_pair_fwd": 1, "mlptex_pair_bwd_dw" if want_w else "mlptex_pair_bwd": 2 if want_w else 1}
                assert (tt.grad is not None) == want_t and (not want_t or torch.equal(tt.grad, full[4]))
                assert (oo.grad is not None) == want_o and (not want_o or torch.equal(oo.grad, full[5]))
                if mask & 1:
                    assert torch.equal(tex.encoder.params.grad == 0, full[6] == 0)
                    assert rel_l2(_np(tex.encoder.params.grad), _np(full[6])) <= 1e-6
                else:
                    assert tex.encoder.params.grad is None
                for k, w in enumerate(tex.net.weights()):
                    assert (w.grad is not None) == bool(mask >> (k + 1) & 1)
                    if w.grad is not None:
                        assert torch.equal(w.grad, full[7 + k])
    for p in params:
        p.requires_grad_(True)
    L.LAUNCHES.clear()
    with torch.no_grad():
        y, yj = tex.sample_pair(torch.from_numpy(t).to(dev), torch.from_numpy(o).to(dev))
    assert y.grad_fn is None and yj.grad_fn is None and L.LAUNCHES == {"mlptex_pair_fwd": 1}
    assert torch.equal(y, full[0]) and torch.equal(yj, full[1])
    # fp64, non-contiguous, batched [..., 3] inputs
    ts = torch.from_numpy(np.ascontiguousarray(t.T)).to(dev).double().t().reshape(200, 200, 3)
    os_ = torch.from_numpy(np.ascontiguousarray(o.T)).to(dev).double().t().reshape(200, 200, 3)
    y, yj = tex.sample_pair(ts, os_)
    assert y.shape == (200, 200, 6) and torch.equal(y.reshape(n, 6), full[0].detach()) and torch.equal(yj.reshape(n, 6), full[1].detach())


def test_rejects_bad_inputs_before_any_launch(dev):
    tex = _texture(dev, 6, 2, seed=0)
    x = torch.rand(4, 3, device=dev)
    L.LAUNCHES.clear()
    for texc, off, err, frag in [(x, torch.rand(5, 3, device=dev), ValueError, "differ in shape"),
                                 (torch.rand(4, 2, device=dev), torch.rand(4, 2, device=dev), ValueError, r"\[\.\.\., 3\]"),
                                 (torch.ones(4, 3, dtype=torch.int32, device=dev), x, ValueError, "floating-point"),
                                 (x, torch.ones(4, 3, dtype=torch.int32, device=dev), ValueError, "floating-point"),
                                 (x, torch.rand(4, 3), ValueError, "offset is on cpu"),
                                 (torch.rand(4, 3), torch.rand(4, 3), RuntimeError, "CUDA")]:
        with pytest.raises(err, match=frag):
            tex.sample_pair(texc, off)
    assert not L.LAUNCHES
    with pytest.raises(TypeError):                      # sample keeps its own errors
        tex.sample(torch.ones(4, 3, dtype=torch.int32, device=dev))


def test_cuda_graph_replay_matches_eager(dev):
    n = 100000
    tex = _texture(dev, 6, 2, seed=15)
    ts, os_ = torch.from_numpy(_points(n, seed=16)).to(dev), torch.from_numpy(_noise(n, seed=17)).to(dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    g, gj = torch.randn(n, 6, device=dev, generator=gen), torch.randn(n, 6, device=dev, generator=gen)

    def step():
        tg = ts.clone().requires_grad_(True)
        for p in tex.parameters():
            p.grad = None
        y, yj = tex.sample_pair(tg, os_)
        torch.autograd.backward([y, yj], [g, gj])
        return [y.detach(), yj.detach(), tg.grad] + [w.grad for w in tex.net.weights()] + [tex.encoder.params.grad]

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


def test_weight_gradients_are_bit_identical_across_runs(dev):
    n = 300000
    tex = _texture(dev, 6, 2, seed=9)
    t, o = _points(n, seed=10), _noise(n, seed=11)
    rng = np.random.default_rng(11)
    g, gj = rng.normal(size=(n, 6)).astype(np.float32), rng.normal(size=(n, 6)).astype(np.float32)
    a = _pair(tex, t, o, g, gj, dev)
    b = _pair(tex, t, o, g, gj, dev)
    assert all(torch.equal(x, y) for x, y in zip(a[7:], b[7:]))
