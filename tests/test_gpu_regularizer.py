"""GPU: nvdiffrecmc_b200.regularizer (csrc/regularizer.cu) against the reference's own functions (the frozen fixture), per element
against the fp64 oracle, bit for bit against the fp32 oracle where the contract says so, and its launch properties: deterministic sums,
CUDA-graph capture, a device-resident upstream gradient without a host read, argument errors before any launch."""
import numpy as np
import pytest
import torch

import nvdiffrecmc_b200._lib as L
import nvdiffrecmc_b200.regularizer as R
from common import check_per_element, nan_bits
from oracle.regularizer import RegularizerOracle
from regularizer_cases import ARGS, CASES, assert_grad_close, assert_loss_close, fixture_case, grad_args

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _strided(x):
    """x [B,H,W,4] on the GPU as channels 2..5 of a [B,H,W,8] buffer: a non-dense view, as color_ref[..., :] slices are."""
    buf = torch.full(x.shape[:3] + (8,), float("nan"), device=DEV)
    buf[..., 2:6] = torch.as_tensor(x, device=DEV)
    return buf[..., 2:6]


def _product(fn, ins, lam, G, strided=("color_ref",)):
    """(loss, [gradient of each differentiable argument]) of the product, upstream gradient G (a device scalar)."""
    ts = []
    for a, x in zip(ARGS[fn], ins):
        t = _strided(x) if a in strided else torch.tensor(np.asarray(x), device=DEV)
        if a != "color_ref":
            t = t.detach().requires_grad_(True)
        ts.append(t)
    loss = getattr(R, fn)(*ts, *lam)
    loss.backward(torch.tensor(G, dtype=torch.float32, device=DEV))
    return loss.detach().cpu().numpy(), [t.grad.cpu().numpy() for a, t in zip(ARGS[fn], ts) if a != "color_ref"]


def _oracle(fn, ins, lam, f64=False, d_loss=None):
    o = RegularizerOracle.get(f64)
    f = getattr(o, fn)
    if d_loss is None:
        out = f(*ins, *lam)
        return float(out[0] if fn == "shading_loss" else out)
    g = f(*ins, *lam, d_loss=d_loss)
    return list(g) if isinstance(g, tuple) else [g]


@pytest.mark.parametrize("fn,case", CASES)
def test_reproduces_the_reference_fixture(fn, case):
    ins, lam, G, loss, grads = fixture_case(fn, case)
    got_loss, got = _product(fn, ins, lam, G)
    assert_loss_close(got_loss, loss, "%s/%s" % (fn, case))
    for a, g in zip(grad_args(fn), got):
        assert_grad_close(g, grads[a], fn, "%s/%s: d %s" % (fn, case, a))


# ---- per element against the fp64 oracle
SHAPES = [(8, 512, 512), (3, 37, 53)]       # the bench size; 5 883 pixels: the forward's last CTA and the backward's last block are ragged


def _inputs(fn, shape, seed):
    """Training-like operands of `shape` with the fixture's finite edge pixels in their first [2,24,40] block."""
    rng = np.random.default_rng(seed)
    B, H, W = shape
    a = np.where(rng.random((B, H, W, 1)) < 0.7, 1.0, np.where(rng.random((B, H, W, 1)) < 0.5, 0.0, rng.random((B, H, W, 1))))
    if fn == "shading_loss":
        ins = [np.concatenate([rng.uniform(-0.05, 2.0, (B, H, W, 3)), a], -1), np.concatenate([rng.uniform(-0.02, 0.8, (B, H, W, 3)), a], -1),
               np.concatenate([rng.random((B, H, W, 3)), a], -1)]
    elif fn == "material_smoothness_grad":
        ins = [np.concatenate([np.abs(rng.normal(0, s, (B, H, W, 3))), a], -1) for s in (0.1, 0.05, 0.2)]
    else:
        ins = [np.concatenate([rng.random((B, H, W, 3)), a], -1), np.concatenate([rng.random((B, H, W, 3)), a], -1)]
    ins = [x.astype(np.float32) for x in ins]
    edge = fixture_case(fn, "finite")[0]
    for x, e in zip(ins, edge):
        x[:2, :24, :40] = e
    return ins


# shading_loss: the step-tail bar, K = 16, plus a per-element floor R for the device's logf / powf, which are not glibc's (each within 2 ulp
# of the exact value, so img and tgt within 8 ulp): R = 8 * 2^-24 * (kappa * (|g_dl1| + |g_s2|) + |g_s1|) for the lights' luma gradient,
# with kappa = (|img| + |tgt|) / |img - tgt| the condition of the subtraction, g_dl1 and g_s2 the terms that carry |img - tgt| (through the
# error's numerator and its clamp(sum, eps) denominator) and g_s1 the term through the log-sRGB derivative (regularizer.cu's names).
# Perturbing the operands by one ulp does not move img by one ulp of img, so Delta alone cannot see a last-ulp difference of powf that
# the subtraction and the following sum of terms amplify (one pixel in 2^21 at 8x512^2, ratio 84 without the floor).
K_SHADING = 16


def _shading_floor(ins, lam, G):
    """The floor R above, per element of (d diffuse_light, d specular_light), in fp64 from the operands."""
    d, s, r = [np.asarray(x, np.float64) for x in ins]
    n3 = 3.0 * d[..., 0].size
    luma = lambda x: (x[..., 0] + x[..., 1] + x[..., 2]) / 3
    srgb = lambda f: np.where(f <= 0.0031308, f * 12.92, np.maximum(f, 0.0031308) ** (1 / 2.4) * 1.055 - 0.055)
    dl, sl, a = luma(d), luma(s), r[..., 3]
    tot = dl + sl
    x = tot * a
    u = np.clip(x, 0, 65535)
    L = np.log1p(u)
    img, tgt = srgb(L), srgb(np.log1p(np.clip(r[..., :3].max(-1) * a, 0, 65535)))
    ad, cs = np.abs(img - tgt), np.maximum(tot, 0.001)
    g_num = abs(G * lam[0] / n3) / cs
    g_dl1 = g_num * ad
    g_s2 = np.where(tot >= 0.001, g_num * ad * dl / cs, 0.0)
    dsrgb = np.where(L <= 0.0031308, 12.92, 1.055 / 2.4 * np.maximum(L, 1e-30) ** (1 / 2.4 - 1))
    g_s1 = np.where((x >= 0) & (x <= 65535), g_num * np.abs(dl) * dsrgb / (u + 1) * np.abs(a), 0.0)
    kappa = np.divide(np.abs(img) + np.abs(tgt), ad, out=np.zeros_like(ad), where=ad > 0)
    rd = 8 * 2.0 ** -24 * (kappa * (g_dl1 + g_s2) + g_s1)
    rs = 8 * 2.0 ** -24 * (kappa * g_s2 + g_s1)
    four = lambda v: np.concatenate([np.repeat(np.nan_to_num(v, nan=0.0)[..., None], 3, -1), np.zeros(v.shape + (1,))], -1)
    return [four(rd), four(rs)]


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("fn", list(ARGS))
def test_per_element_against_the_fp64_oracle(fn, shape):
    ins = _inputs(fn, shape, seed=list(ARGS).index(fn))
    lam = [float(x) for x in fixture_case(fn, "finite")[1]]
    G = 0.75
    strided = ("color_ref", "ks_grad")
    loss, got = _product(fn, ins, lam, G, strided)
    r64 = _oracle(fn, ins, lam, f64=True)
    assert abs(float(loss) - r64) <= 1e-6 * abs(r64), "%s loss %r, fp64 oracle %r" % (fn, float(loss), r64)
    names = ["d " + a for a in grad_args(fn)]
    if fn == "shading_loss":
        nd = len(names)
        f64 = lambda xs: _oracle(fn, list(xs) + ins[nd:], lam, True, G)
        f32 = lambda xs: _oracle(fn, list(xs) + ins[nd:], lam, False, G)
        check_per_element(fn, got, f64, f32, ins[:nd], K_SHADING, names, floor=_shading_floor(ins, lam, G), tag="regularizer")
    else:
        ref = _oracle(fn, ins, lam, False, G)
        for n, g, r in zip(names, got, ref):
            same = nan_bits(g) == nan_bits(r)
            assert same.all(), "%s %s: %d elements differ from the fp32 oracle, first %s (got %r, oracle %r)" % (
                fn, n, int((~same).sum()), tuple(np.argwhere(~same)[0]), g[~same][0], r[~same][0])


# ---- launch properties
def _tick(ts, lam):
    """The three calls as a geometry tick makes them, summed."""
    d, s, ref, kdg, ksg, nrg, kd = ts
    return (R.shading_loss(d, s, ref, *lam[0]) + R.material_smoothness_grad(kdg, ksg, nrg, *lam[1]) + R.chroma_loss(kd, ref, *lam[2]))


def _tick_inputs(shape, seed=3):
    sh = _inputs("shading_loss", shape, seed)
    ms = _inputs("material_smoothness_grad", shape, seed + 1)
    ch = _inputs("chroma_loss", shape, seed + 2)
    ts = [torch.tensor(x, device=DEV) for x in (sh[0], sh[1])] + [_strided(sh[2])] + [torch.tensor(x, device=DEV) for x in ms + [ch[0]]]
    for i in (0, 1, 3, 4, 5, 6):
        ts[i].requires_grad_(True)
    lam = [tuple(float(x) for x in fixture_case(fn, "finite")[1]) for fn in ARGS]
    return ts, lam


def _tick_run(ts, lam, G):
    loss = _tick(ts, lam)
    grads = torch.autograd.grad(loss, [ts[i] for i in (0, 1, 3, 4, 5, 6)], grad_outputs=G)
    return [loss.detach().clone()] + [g.clone() for g in grads]


def test_two_runs_are_bit_identical():
    ts, lam = _tick_inputs((8, 512, 512))
    G = torch.tensor(1.25, device=DEV)
    a = [x.cpu().numpy() for x in _tick_run(ts, lam, G)]
    b = [x.cpu().numpy() for x in _tick_run(ts, lam, G)]
    for x, y in zip(a, b):
        assert np.array_equal(nan_bits(x), nan_bits(y))


def test_cuda_graph_replay_matches_eager():
    ts, lam = _tick_inputs((3, 37, 53))
    G = torch.tensor(0.5, device=DEV)
    eager = [x.cpu().numpy() for x in _tick_run(ts, lam, G)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _tick_run(ts, lam, G)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = _tick_run(ts, lam, G)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(outs, eager):
        assert np.array_equal(nan_bits(x.cpu().numpy()), nan_bits(y))
    with torch.no_grad():                           # a new upstream gradient on the device is read by the replay
        G.fill_(2.0)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(outs[1:], eager[1:]):
        assert np.array_equal(nan_bits(x.cpu().numpy()), nan_bits(4.0 * y))


def test_device_upstream_gradient_without_a_host_read():
    ins = _inputs("material_smoothness_grad", (2, 40, 56), 4)
    lam = [0.1, 0.05, 0.025]
    ts = [torch.tensor(x, device=DEV, requires_grad=True) for x in ins]
    sh = [torch.tensor(x, device=DEV, requires_grad=i < 2) for i, x in enumerate(_inputs("shading_loss", (2, 40, 56), 5))]
    ch = [torch.tensor(x, device=DEV, requires_grad=i < 1) for i, x in enumerate(_inputs("chroma_loss", (2, 40, 56), 6))]
    G = torch.tensor(1.5, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")         # any synchronising call raises
    try:
        R.material_smoothness_grad(*ts, *lam).backward(G)
        R.shading_loss(*sh, 0.15, 0.0025).backward(G)
        R.chroma_loss(*ch, 0.025).backward(G)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    ref = _oracle("material_smoothness_grad", ins, lam, False, 1.5)
    for t, r in zip(ts, ref):
        assert np.array_equal(nan_bits(t.grad.cpu().numpy()), nan_bits(r))


def test_argument_errors_raise_before_any_launch():
    x = torch.rand(2, 8, 9, 4, device=DEV)
    cases = [
        ("diffuse_light", lambda: R.shading_loss(x[..., :3], x, x, 0.1, 0.1)),
        ("specular_light", lambda: R.shading_loss(x, torch.rand(2, 8, 10, 4, device=DEV), x, 0.1, 0.1)),
        ("color_ref", lambda: R.shading_loss(x, x, x.cpu(), 0.1, 0.1)),
        ("lambda_specular", lambda: R.shading_loss(x, x, x, 0.1, 1)),
        ("color_ref", lambda: R.shading_loss(x, x, x.clone().requires_grad_(True), 0.1, 0.1)),
        ("ks_grad", lambda: R.material_smoothness_grad(x, torch.rand(2, 8, 9, 3, device=DEV), x)),
        ("nrm_grad", lambda: R.material_smoothness_grad(x, x, torch.rand(1, 8, 9, 4, device=DEV))),
        ("kd_grad", lambda: R.material_smoothness_grad(x.cpu(), x, x)),
        ("lambda_nrm", lambda: R.material_smoothness_grad(x, x, x, lambda_nrm=torch.tensor(0.0))),
        ("kd", lambda: R.chroma_loss(x.double(), x, 0.1)),
        ("color_ref", lambda: R.chroma_loss(x, x[:1], 0.1)),
        ("lambda_chroma", lambda: R.chroma_loss(x, x, None)),
    ]
    for name, call in cases:
        before = dict(L.LAUNCHES)
        with pytest.raises(ValueError, match=name):
            call()
        assert dict(L.LAUNCHES) == before, name
