"""Shared by the regulariser tests: the frozen reference fixture (tests/golden/ref_regularizer.npz) and the bar its reproductions are held
to."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_regularizer.npz")
ARGS = {"shading_loss": ("diffuse_light", "specular_light", "color_ref"), "material_smoothness_grad": ("kd_grad", "ks_grad", "nrm_grad"),
        "chroma_loss": ("kd", "color_ref")}
CASES = [(fn, case) for fn in ARGS for case in ("finite", "nonfinite")]


def grad_args(fn):
    return [a for a in ARGS[fn] if a != "color_ref"]


def fixture_case(fn, case):
    """-> (inputs in argument order, lambdas (floats), upstream gradient G, reference loss, {argument: reference gradient})."""
    d = np.load(GOLDEN)
    pre = "%s/%s/" % (fn, case)
    return ([d[pre + a] for a in ARGS[fn]], [float(x) for x in d[pre + "lambdas"]], float(d["G"]), d[pre + "loss"],
            {a: d[pre + "d_" + a] for a in grad_args(fn)})


def _ulp32(x):
    a = np.minimum(np.abs(np.asarray(x, np.float64)), np.finfo(np.float32).max).astype(np.float32)
    return np.nextafter(a, np.float32(np.inf)).astype(np.float64) - a.astype(np.float64)


def assert_loss_close(got, ref, what):
    got, ref = float(got), float(ref)
    if np.isnan(ref):
        assert np.isnan(got), "%s: loss %r, the reference has NaN" % (what, got)
    else:
        assert abs(got - ref) <= 1e-6 * abs(ref), "%s: loss %r, reference %r (rel %.3g)" % (what, got, ref, abs(got - ref) / abs(ref))


def assert_grad_close(got, ref, fn, what):
    """Element by element at the fixture's fp32 noise, with identical NaN, +-inf and exact-zero sets.  material_smoothness_grad and
    chroma_loss: 4 ulp32.  shading_loss: 1e-4 relative plus 1e-6 of the largest gradient -- torch's vectorised CPU log / pow, glibc's and
    the device's differ in the last ulp, and the log-sRGB chain and the |img - tgt| * luma / sum cancellations carry that to about 1e-5
    relative in a few elements."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    for pred, name in ((np.isnan, "NaN"), (np.isposinf, "+inf"), (np.isneginf, "-inf"), (lambda x: x == 0, "exact-zero")):
        bad = pred(got) != pred(ref)
        assert not bad.any(), "%s: %s set differs at %d elements, first %s (got %r, reference %r)" % (
            what, name, int(bad.sum()), tuple(np.argwhere(bad)[0]), got[bad][0], ref[bad][0])
    fin = np.isfinite(ref)
    if fn == "shading_loss":
        tol = 1e-4 * np.abs(ref) + 1e-6 * (np.abs(ref[fin]).max() if fin.any() else 0.0)
    else:
        tol = 4 * _ulp32(np.where(fin, ref, 0.0))
    err = np.abs(np.where(fin, got, 0.0) - np.where(fin, ref, 0.0))
    bad = err > tol
    assert not bad.any(), "%s: %d elements beyond the fixture's noise, first %s (got %r, reference %r)" % (
        what, int(bad.sum()), tuple(np.argwhere(bad)[0]), got[bad][0], ref[bad][0])
