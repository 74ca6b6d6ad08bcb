"""GPU: regularizer.coverage_image_loss (csrc/lossmesh.cu) against the geometry passes' two lines run on the same device with the package's
renderutils.image_loss (geometry/dmtet.py:229-230, geometry/dlmesh.py:75-76): per-CTA colour partials, d shaded rgb and d shaded alpha bit
for bit, coverage partials bit for bit against the fp32 oracle's sum in the kernel's order, the loss within the two-summation-order bound of
the fp64 oracle and within 1e-6 of the chain; edge values, strided operands, autograd, determinism, no host sync, CUDA-graph capture,
argument errors, and d pos through raster.composite."""
import numpy as np
import pytest
import torch

import nvdiffrecmc_b200._lib as L
import nvdiffrecmc_b200.regularizer as R
import nvdiffrecmc_b200.renderutils as ru
from common import _ulp32, nan_bits, oracle
from coverage_loss_oracle import coverage_loss_px, cta_partials
from nvdiffrecmc_b200.renderutils.ops import _image_loss_func, _loss_ids

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LOSSES = ["l1", "mse", "relmse", "smape", "n2n"]
PAIRS = [(l, t) for l in LOSSES for t in ("none", "log_srgb")]
SHAPES = [(1, 1, 1), (3, 13, 19), (8, 33, 31)]          # one pixel; 741 pixels; 8 184 pixels, the last CTA ragged
LAYOUTS = ["dense", "sliced", "transposed"]


def _values(shape, seed, finite=False):
    """Training-like shaded / ref [B,H,W,4] (numpy fp32) with the edge values in the first pixels: ref alpha exactly 0 and 1 and
    fractional, shaded alpha the same; HDR colours above 65535, zeros and negatives (the clamps' edges); NaN / +-inf colour on pixels
    whose ref alpha is 0 and 1 (with finite, NaN becomes 0.5 and +-inf +-1e30)."""
    rng = np.random.default_rng(seed)
    B, H, W = shape
    pick = lambda: np.where(rng.random((B, H, W)) < 0.4, rng.choice([0.0, 1.0], (B, H, W)), rng.random((B, H, W)))
    s = np.concatenate([rng.uniform(-0.1, 3.0, (B, H, W, 3)), pick()[..., None]], -1).astype(np.float32)
    r = np.concatenate([rng.uniform(0.0, 2.0, (B, H, W, 3)), pick()[..., None]], -1).astype(np.float32)
    edge_s = [(0.0, 0.5, 1.0, 1.0), (70000.0, 1.0, -0.5, 0.25), (np.nan, 1.0, 2.0, 0.0), (np.inf, -np.inf, 0.5, 1.0), (np.nan, 0.2, np.inf, 0.5),
              (65535.0, 0.0, 1e-30, 0.75), (-np.inf, 3.0, 2.0, 1.0), (1.0, 1.0, 1.0, 0.0)]
    edge_r = [(0.0, 0.5, 1.0, 1.0), (80000.0, 0.0, 0.5, 1.0), (1.0, 1.0, 1.0, 0.0), (1.0, 0.2, 0.3, 0.0), (0.3, 0.2, 0.1, 1.0),
              (65535.0, 0.0, 0.0, 0.5), (1.0, 1.0, 1.0, 1.0), (70000.0, 0.5, 0.0, 0.0)]
    flat_s, flat_r = s.reshape(-1, 4), r.reshape(-1, 4)
    k = min(len(edge_s), flat_s.shape[0] - 1) if flat_s.shape[0] > 1 else 1
    flat_s[:k] = edge_s[:k]
    flat_r[:k] = edge_r[:k]
    if finite:
        s, r = [np.nan_to_num(x, nan=0.5, posinf=1e30, neginf=-1e30) for x in (s, r)]
    return s, r


def _on_device(x, layout):
    """x [B,H,W,4] as a dense tensor, channels 2..5 of an 8-channel buffer, or the transpose of a [B,W,H,4] tensor."""
    x = torch.tensor(x, device=DEV)
    if layout == "sliced":
        buf = torch.full(x.shape[:3] + (8,), float("nan"), device=DEV)
        buf[..., 2:6] = x
        return buf[..., 2:6]
    if layout == "transposed":
        return x.transpose(1, 2).contiguous().transpose(1, 2)
    return x


def _chain(shaded, ref, loss, tm):
    img_loss = torch.nn.functional.mse_loss(shaded[..., 3:], ref[..., 3:])
    img_loss += ru.image_loss(shaded[..., 0:3] * ref[..., 3:], ref[..., 0:3] * ref[..., 3:], loss, tm)
    return img_loss


def _partials(shaded, ref, loss, tm):
    B, H, W = shaded.shape[:3]
    P = L.lib().mcs_coverage_loss_num_partials(B, H, W)
    part = torch.full((2 * P,), 7.0, device=DEV)
    out = torch.empty((), device=DEV)
    L.check(L.lib().mcs_coverage_loss_fwd(L.nhwc(shaded), L.nhwc(ref), *_loss_ids(loss, tm), part.data_ptr(), out.data_ptr(), L.stream_ptr()),
            "coverage_loss_fwd")
    return part[:P], part[P:], out


def _same(a, b, what):
    a, b = [np.asarray(x.detach().cpu() if isinstance(x, torch.Tensor) else x, np.float32) for x in (a, b)]
    same = nan_bits(a) == nan_bits(b)
    assert same.all(), "%s: %d of %d differ, first %s (got %r, want %r)" % (what, int((~same).sum()), same.size, tuple(np.argwhere(~same)[0]),
                                                                           a[~same][0], b[~same][0])


def _loss_bound(s, r, loss, tm):
    """(fp64 oracle loss, bound): two summation orders of the N per-pixel terms, 2 gamma(N) A (1 + gamma(N)) with A the sum of their
    magnitudes, plus the fp32 evaluation of each term, 16 |t32 - t64| + 4 ulp per term as check_per_element bounds one element, and the
    final rounding."""
    cov64, col64 = coverage_loss_px(oracle(True), s, r, loss, tm)
    cov32, col32 = coverage_loss_px(oracle(), s, r, loss, tm)
    n = cov64.size
    terms64 = np.concatenate([cov64.reshape(-1), col64.reshape(-1)])
    terms32 = np.concatenate([cov32.reshape(-1), col32.reshape(-1)]).astype(np.float64)
    want = terms64.sum() / n
    u = 2.0 ** -24
    gam = n * u / (1 - n * u)
    ev = (16 * np.abs(terms32 - terms64) + 4 * _ulp32(terms64)).sum() / n
    return want, 2 * gam * np.abs(terms64).sum() / n * (1 + gam) + ev + _ulp32(want)


def _run(shaded, ref, loss, tm, G, fn):
    s = shaded.detach().requires_grad_(True)
    out = fn(s, ref, loss, tm)
    g, = torch.autograd.grad(out, s, G)
    return out.detach(), g


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("loss,tm", PAIRS)
def test_against_the_chain(loss, tm, shape, layout):
    s_np, r_np = _values(shape, PAIRS.index((loss, tm)) + 10 * SHAPES.index(shape))
    shaded, ref = _on_device(s_np, layout), _on_device(r_np, layout)
    cov, col, out = _partials(shaded, ref, loss, tm)
    _same(col, _image_loss_func.apply(shaded[..., 0:3] * ref[..., 3:], ref[..., 0:3] * ref[..., 3:], loss, tm), "colour partials")
    _same(cov, cta_partials(coverage_loss_px(oracle(), s_np, r_np, loss, tm)[0]), "coverage partials")
    G = torch.tensor(0.75, device=DEV)
    got, g = _run(shaded, ref, loss, tm, G, R.coverage_image_loss)
    want, g_want = _run(shaded, ref, loss, tm, G, _chain)
    _same(got, out, "loss of the entry and of the function")
    _same(g[..., :3], g_want[..., :3], "d shaded rgb")
    _same(g[..., 3], g_want[..., 3], "d shaded alpha")
    got, want = float(got), float(want)
    assert np.isnan(got) == np.isnan(want)
    if np.isfinite(want):
        assert abs(got - want) <= 1e-6 * abs(want), (got, want)


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("loss,tm", PAIRS)
def test_loss_within_the_fp64_bound(loss, tm, shape):
    """The edge values without NaN and inf (the oracle's clamp passes NaN where the kernel's fminf / fmaxf drop it)."""
    s_np, r_np = _values(shape, 50 + PAIRS.index((loss, tm)), finite=True)
    got = float(R.coverage_image_loss(_on_device(s_np, "dense"), _on_device(r_np, "dense"), loss, tm))
    r64, bound = _loss_bound(s_np, r_np, loss, tm)
    assert np.isfinite(r64) and abs(got - r64) <= bound, (got, r64, bound)


@pytest.mark.parametrize("loss,tm", PAIRS)
def test_bench_size_against_the_chain(loss, tm):
    """8 x 512^2: 8 192 partials; everything as above except the fp64 bound, which the 1e-6 check against the chain stands in for."""
    s_np, r_np = _values((8, 512, 512), 99)
    shaded, ref = _on_device(s_np, "dense"), _on_device(r_np, "sliced")
    cov, col, _ = _partials(shaded, ref, loss, tm)
    _same(col, _image_loss_func.apply(shaded[..., 0:3] * ref[..., 3:], ref[..., 0:3] * ref[..., 3:], loss, tm), "colour partials")
    _same(cov, cta_partials(coverage_loss_px(oracle(), s_np, r_np, loss, tm)[0]), "coverage partials")
    G = torch.tensor(1.25, device=DEV)
    got, g = _run(shaded, ref, loss, tm, G, R.coverage_image_loss)
    want, g_want = _run(shaded, ref, loss, tm, G, _chain)
    _same(g, g_want, "d shaded")
    assert abs(float(got) - float(want)) <= 1e-6 * abs(float(want)), (float(got), float(want))


def test_gradient_only_when_shaded_requires_it():
    s_np, r_np = _values((3, 13, 19), 1)
    shaded, ref = _on_device(s_np, "dense"), _on_device(r_np, "dense")
    nf, nb = L.LAUNCHES["coverage_loss_fwd"], L.LAUNCHES["coverage_loss_bwd"]
    plain = R.coverage_image_loss(shaded, ref, "mse", "log_srgb")
    assert plain.grad_fn is None and not plain.requires_grad
    x = shaded.clone().requires_grad_(True)
    with torch.no_grad():
        ng = R.coverage_image_loss(x, ref, "mse", "log_srgb")
    assert ng.grad_fn is None and not ng.requires_grad
    assert L.LAUNCHES["coverage_loss_fwd"] == nf + 4 and L.LAUNCHES["coverage_loss_bwd"] == nb
    w = torch.ones(3, device=DEV, requires_grad=True)                # another input needs the gradient, shaded does not
    (R.coverage_image_loss(shaded, ref, "mse", "log_srgb") + w.sum()).backward()
    assert L.LAUNCHES["coverage_loss_bwd"] == nb
    y = R.coverage_image_loss(x, ref, "mse", "log_srgb")
    _same(y, plain, "loss with and without grad")
    _same(ng, plain, "loss under no_grad")
    y.backward()
    assert L.LAUNCHES["coverage_loss_bwd"] == nb + 1 and x.grad.shape == x.shape


def _step(shaded, ref, G):
    out = R.coverage_image_loss(shaded, ref, "l1", "log_srgb")
    g, = torch.autograd.grad(out, shaded, G)
    return [out.detach().clone(), g.clone()]


def test_two_runs_are_bit_identical():
    s_np, r_np = _values((8, 512, 512), 5)
    shaded, ref = _on_device(s_np, "dense").requires_grad_(True), _on_device(r_np, "sliced")
    G = torch.tensor(1.0, device=DEV)
    a, b = _step(shaded, ref, G), _step(shaded, ref, G)
    for x, y in zip(a, b):
        _same(x, y, "second run")


def test_no_host_sync():
    s_np, r_np = _values((2, 40, 56), 6)
    shaded, ref = _on_device(s_np, "transposed").requires_grad_(True), _on_device(r_np, "dense")
    G = torch.tensor(1.5, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")         # any synchronising call raises
    try:
        out = _step(shaded, ref, G)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    _, g_want = _run(shaded, ref, "l1", "log_srgb", G, _chain)
    _same(out[1], g_want, "d shaded")


def test_cuda_graph_replay_matches_eager():
    s_np, r_np = _values((3, 37, 53), 7)
    shaded, ref = _on_device(s_np, "dense").requires_grad_(True), _on_device(r_np, "sliced")
    G = torch.tensor(0.5, device=DEV)
    eager = [x.cpu().numpy() for x in _step(shaded, ref, G)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _step(shaded, ref, G)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = _step(shaded, ref, G)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(outs, eager):
        _same(x, y, "replay")
    with torch.no_grad():                           # a new upstream gradient on the device is read by the replay
        G.fill_(2.0)
    graph.replay()
    torch.cuda.synchronize()
    _, g_want = _run(shaded, ref, "l1", "log_srgb", G, _chain)
    _same(outs[1], g_want, "replay with a new upstream gradient")


def test_argument_errors_raise_before_any_launch():
    x = torch.rand(2, 8, 9, 4, device=DEV)
    cases = [
        ("shaded must be \\[B,H,W,4\\]", lambda: R.coverage_image_loss(x[..., :3], x)),
        ("color_ref must be \\[B,H,W,4\\]", lambda: R.coverage_image_loss(x, torch.rand(2, 8, 9, 5, device=DEV))),
        ("color_ref has shape", lambda: R.coverage_image_loss(x, torch.rand(2, 8, 10, 4, device=DEV))),
        ("color_ref has shape", lambda: R.coverage_image_loss(x, x[:1])),
        ("color_ref must be a CUDA tensor", lambda: R.coverage_image_loss(x, x.cpu())),
        ("shaded is empty", lambda: R.coverage_image_loss(x[:, :0], x[:, :0])),
        ("color_ref is the constant target and must not require grad", lambda: R.coverage_image_loss(x, x.clone().requires_grad_(True))),
        ("color_ref must be float32", lambda: R.coverage_image_loss(x, x.half())),
        ("unknown loss", lambda: R.coverage_image_loss(x, x, "L1")),
        ("unknown tonemapper", lambda: R.coverage_image_loss(x, x, "l1", None)),
    ]
    for frag, call in cases:
        before = dict(L.LAUNCHES)
        with pytest.raises(ValueError, match=frag):
            call()
        assert dict(L.LAUNCHES) == before, frag


def test_pos_gradient_through_composite():
    """A two-layer peel of 2 x 40 x 56 composited by raster.composite; d pos through coverage_image_loss equals d pos through the two
    torch lines within tests/test_gpu_composite.py's bound (rel-L2 1e-5; pos receives float atomics), d shaded bit for bit."""
    from nvdiffrecmc_b200.raster import composite
    from test_gpu_composite import _buffers, _scene
    rasts, pos, tri, topo = _scene(DEV, 2, (40, 56), 2)
    pos = pos.clone().requires_grad_(True)
    layers = [(b, r) for b, r in zip(_buffers(rasts, [("shaded", 4)], 11, nonfinite=False, strided=()), rasts)]
    _, r_np = _values(tuple(rasts[0].shape[:3]), 12)
    ref = _on_device(r_np, "sliced")
    grads = []
    for fn in (R.coverage_image_loss, _chain):
        shaded = composite(layers, pos, tri, topology=topo)["shaded"]
        out = fn(shaded, ref, "l1", "log_srgb")
        grads.append(torch.autograd.grad(out, [pos, shaded]))
    (gp, gs), (gp_want, gs_want) = grads
    _same(gs, gs_want, "d shaded")
    assert torch.isfinite(gp_want).all() and gp_want.abs().max() > 0
    e = float((gp - gp_want).double().norm() / gp_want.double().norm())
    assert e <= 1e-5, e
