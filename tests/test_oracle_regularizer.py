"""CPU: the oracle's restatement of the image-space regularisers (render/regularizer.py:15-49) against the reference's own functions
(frozen in tests/golden/ref_regularizer.npz), against finite differences in fp64, and the public functions' signatures against the
reference's."""
import ast
import inspect
import os

import numpy as np
import pytest

from oracle.regularizer import RegularizerOracle
from regularizer_cases import ARGS, CASES, GOLDEN, assert_grad_close, assert_loss_close, fixture_case, grad_args

REF_REGULARIZER = "/root/reference/render/regularizer.py"
HAVE_REF = os.path.exists(REF_REGULARIZER)


def _run(o, fn, ins, lam, d_loss=None):
    f = getattr(o, fn)
    if d_loss is None:
        out = f(*ins, *lam)
        return out[0] if fn == "shading_loss" else out
    g = f(*ins, *lam, d_loss=d_loss)
    return g if isinstance(g, tuple) else (g,)


@pytest.mark.parametrize("fn,case", CASES)
def test_fp32_oracle_reproduces_the_reference(fn, case):
    ins, lam, G, loss, grads = fixture_case(fn, case)
    o = RegularizerOracle.get()
    assert_loss_close(_run(o, fn, ins, lam), loss, "%s/%s" % (fn, case))
    for a, g in zip(grad_args(fn), _run(o, fn, ins, lam, G)):
        assert_grad_close(g, grads[a], fn, "%s/%s: d %s" % (fn, case, a))


def test_fixture_covers_the_edge_classes():
    """The fixture holds every edge class the contract names."""
    ins, *_ = fixture_case("shading_loss", "finite")
    d, s, r = [np.asarray(x, np.float32) for x in ins]
    luma = lambda x: ((x[..., 0] + x[..., 1]) + x[..., 2]) / np.float32(3)
    eps = np.float32(0.001)
    ssum = luma(d) + luma(s)
    lit = ssum * r[..., 3]
    assert (ssum == eps).any() and (lit == 0).any() and (lit == 65535).any() and (lit > 65535).any()
    assert ((r[..., 3] == 0).any() and (r[..., 3] == 1).any() and ((r[..., 3] > 0) & (r[..., 3] < 1)).any())
    assert (d[..., :3] < 0).any() and (s[..., :3] < 0).any()
    L, t = np.log1p(np.float64(lit[(lit >= 0) & (lit < 1)])), float(np.float32(0.0031308))
    assert ((L > t) & (L < t + 1e-6)).any() and ((L < t) & (L > t - 1e-6)).any()
    kd, ref = [np.asarray(x, np.float32) for x in fixture_case("chroma_loss", "finite")[0]]
    for x in (kd, ref):
        v = x[..., :3].max(-1)
        assert (v == eps).any()
        assert ((x[..., 0] == x[..., 1]) & (x[..., 0] == x[..., 2])).any() and ((x[..., 0] == x[..., 1]) & (x[..., 2] < x[..., 0])).any()
    for fn in ARGS:
        ins = fixture_case(fn, "nonfinite")[0]
        assert any(np.isnan(x).any() for x in ins) and any(np.isinf(x).any() for x in ins)


# ---- fp64: finite differences and the adjoint identity, at points away from the kinks (ties, clamp boundaries, abs at 0, sRGB branch)
def _smooth_point(fn, rng, shape=(2, 5, 7)):
    """Inputs of fn with every kink at least a margin away: distinct channels, luma sums >> eps, lit values in (0, 65535) and away from
    the sRGB threshold, |img - tgt| > 0, values >> eps, coverage in (0, 1]."""
    B, H, W = shape
    a = rng.choice([1.0, 0.5, 0.25], size=(B, H, W, 1))
    rgb = lambda lo, hi: lo + (hi - lo) * (np.arange(3) / 2.0 * 0.3 + rng.random((B, H, W, 1)) * 0.7)      # strictly increasing channels
    if fn == "shading_loss":
        lit = np.where(rng.random((B, H, W, 1)) < 0.3, rng.uniform(2e-4, 1.5e-3, (B, H, W, 1)), rng.uniform(0.05, 3.0, (B, H, W, 1)))
        d = np.concatenate([lit * rgb(0.6, 1.2)[..., ::-1] / 0.9, a], -1)
        s = np.concatenate([lit * rgb(0.05, 0.4) / 0.9, a], -1)
        r = np.concatenate([rgb(0.1, 1.0) * rng.uniform(0.2, 3.0, (B, H, W, 1)), a], -1)
        return [d, s, r], [0.15, 0.0025]
    if fn == "material_smoothness_grad":
        return [np.concatenate([rng.uniform(0.01, 0.3, (B, H, W, 3)), rng.uniform(0.1, 1.0, (B, H, W, 1))], -1) for _ in range(3)], [0.1, 0.05, 0.025]
    kd = np.concatenate([rgb(0.05, 0.9), a], -1)
    ref = np.concatenate([rgb(0.1, 0.8)[..., ::-1], a], -1)
    return [kd, ref], [0.025]


def _fd_ok(fd, an, what):
    assert np.isfinite(an).all(), what
    assert abs(fd - an) <= 1e-6 * max(abs(an), 1e-3 * 1.0) + 1e-10, "%s: finite difference %r, analytic %r" % (what, fd, an)


@pytest.mark.parametrize("fn", list(ARGS))
def test_fp64_oracle_matches_finite_differences(fn):
    o = RegularizerOracle.get(True)
    rng = np.random.default_rng(5)
    ins, lam = _smooth_point(fn, rng)
    grads = _run(o, fn, ins, lam, 1.0)
    for k, a in enumerate(grad_args(fn)):
        g = grads[k]
        for _ in range(24):
            idx = tuple(rng.integers(0, n) for n in ins[k].shape)
            h = 1e-7 * max(1.0, abs(ins[k][idx]))
            up, dn = [x.copy() for x in ins], [x.copy() for x in ins]
            up[k][idx] += h
            dn[k][idx] -= h
            fd = (float(_run(o, fn, up, lam)) - float(_run(o, fn, dn, lam))) / (2 * h)
            _fd_ok(fd, g[idx], "%s: d %s%s" % (fn, a, idx))
        if fn == "chroma_loss":
            assert (g[..., 3] == 0).all()


@pytest.mark.parametrize("fn", list(ARGS))
def test_fp64_oracle_adjoint_identity(fn):
    """<grad(G), v> = G * d/dt loss(x + t v) for random directions v on every differentiable operand at once."""
    o = RegularizerOracle.get(True)
    rng = np.random.default_rng(9)
    ins, lam = _smooth_point(fn, rng)
    G = 0.75
    grads = _run(o, fn, ins, lam, G)
    nd = len(grad_args(fn))
    for _ in range(4):
        vs = [rng.standard_normal(x.shape) * np.abs(x) * 1e-1 for x in ins[:nd]]
        h = 1e-6
        f = lambda t: float(_run(o, fn, [x + t * v for x, v in zip(ins[:nd], vs)] + ins[nd:], lam))
        fd = G * (f(h) - f(-h)) / (2 * h)
        an = sum(float((g * v).sum()) for g, v in zip(grads, vs))
        assert abs(fd - an) <= 1e-6 * abs(an) + 1e-12, "%s: directional difference %r, adjoint %r" % (fn, fd, an)


# ---- signatures
@pytest.mark.skipif(not HAVE_REF, reason="needs the reference checkout")
def test_public_signatures_match_the_reference():
    import nvdiffrecmc_b200.regularizer as R
    tree = ast.parse(open(REF_REGULARIZER).read())
    ref = {f.name: f for f in tree.body if isinstance(f, ast.FunctionDef)}
    for name in ("shading_loss", "material_smoothness_grad", "chroma_loss"):
        args = ref[name].args
        names = [a.arg for a in args.args]
        defaults = [ast.literal_eval(d) for d in args.defaults]
        sig = inspect.signature(getattr(R, name))
        assert list(sig.parameters) == names, name
        got_defaults = [p.default for p in sig.parameters.values() if p.default is not inspect.Parameter.empty]
        assert got_defaults == defaults and all(type(a) is type(b) for a, b in zip(got_defaults, defaults)), name
        assert all(p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD for p in sig.parameters.values()), name


@pytest.mark.skipif(not HAVE_REF, reason="needs the reference checkout")
def test_generator_reproduces_the_fixture():
    import sys
    sys.path.insert(0, os.path.dirname(GOLDEN))
    import make_regularizer_golden
    new = make_regularizer_golden.generate()
    old = np.load(GOLDEN)
    assert sorted(new) == sorted(old.files)
    for k in old.files:
        a, b = np.asarray(new[k]), old[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        assert np.array_equal(a, b, equal_nan=True), k


def test_arguments_are_checked_before_any_launch():
    """The checks that need no GPU: a CPU tensor and another channel count raise ValueError naming the argument."""
    import torch
    import nvdiffrecmc_b200.regularizer as R
    x = torch.zeros(1, 2, 3, 4)
    with pytest.raises(ValueError, match="diffuse_light"):
        R.shading_loss(x, x, x, 0.1, 0.1)
    with pytest.raises(ValueError, match="kd_grad"):
        R.material_smoothness_grad(torch.zeros(1, 2, 3, 3), x, x)
    with pytest.raises(ValueError, match="kd"):
        R.chroma_loss(x, x, 0.1)
