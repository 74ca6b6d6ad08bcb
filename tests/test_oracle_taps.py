"""CPU: the oracle's restatement of shade()'s jittered regulariser taps (oracle/taps.c) against the reference's own shade(), frozen in
tests/golden/ref_jitter_taps.npz, against central finite differences in fp64, and the argument checks of `jitter_taps` that run before
any launch."""
import os

import numpy as np
import pytest
import torch

from oracle.taps import BUFFERS, taps_oracle
from taps_cases import ARGS, random_case
from nvdiffrecmc_b200 import _lib
from nvdiffrecmc_b200.regularizer import jitter_taps

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_jitter_taps.npz")
CASES = ["kd3", "kd4_nrm", "kd3_nrm", "mlp"]
# The golden's taps come from the reference's texture stub (grid_sample), whose texel coordinate ((2u - 1) + 1) W / 2 - 0.5 differs from
# the contract's u W - 0.5 by a few fp32 roundings: at most 4 ulp of W = 19, 4 * 2^-20 < 4e-6 texels.  A tap moves by that times the
# largest texel difference (below 2 for the fixture's unit normals and [0, 1) colours): < 8e-6; the buffers and gradients are a product
# of such a difference with weights and upstream gradients of order 1, plus fp32 roundings of the reference (< 1e-6).  Bar: 1e-5 absolute
# (the worst measured is 3.4e-6).
GOLDEN_BAR = 1e-5


def golden_case(case):
    z = np.load(GOLDEN)
    g = lambda k: z["%s/%s" % (case, k)] if "%s/%s" % (case, k) in z.files else None
    args = [g(k) for k in ARGS]
    G = {k: g("G_" + k) for k in BUFFERS if g("G_" + k) is not None}
    want_fwd = {k: g(k) for k in G}
    want_bwd = {k: g("d_" + k) for k in ARGS[2:] if g("d_" + k) is not None}
    return args, G, want_fwd, want_bwd


@pytest.mark.parametrize("f64", [True, False], ids=["fp64", "fp32"])
@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_reference_shade(case, f64):
    args, G, want_fwd, want_bwd = golden_case(case)
    o = taps_oracle(f64)
    got = o.forward(*args)
    assert sorted(got) == sorted(want_fwd)
    for k in want_fwd:
        err = np.abs(got[k].astype(np.float64) - want_fwd[k])
        assert err.max() <= GOLDEN_BAR, (case, k, err.max())
    d = o.backward(*args, G)
    assert sorted(d) == sorted(want_bwd)
    for k in want_bwd:
        err = np.abs(d[k].astype(np.float64) - want_bwd[k])
        assert err.max() <= GOLDEN_BAR, (case, k, err.max())
    print("[taps golden] %-8s %s forward %.2e, gradients %.2e" % (case, "fp64" if f64 else "fp32",
          max(np.abs(got[k] - want_fwd[k]).max() for k in want_fwd), max(np.abs(d[k] - want_bwd[k]).max() for k in want_bwd)))


@pytest.mark.parametrize("ckd,pn,mlp", [(3, False, False), (4, True, False), (3, True, True), (4, False, True)])
def test_fp64_adjoint_matches_finite_differences(ckd, pn, mlp):
    """Central differences (h = 1e-6) of sum_k <G_k, buffer_k> in every differentiable operand at random elements; random operands keep
    every |tap - value| and every squared length far from the abs kink and the 1e-20 clamp."""
    rng = np.random.default_rng(11 + ckd + 2 * pn + 4 * mlp)
    args = [None if a is None else a.astype(np.float64) for a in random_case(rng, 2, 7, 9, ckd, pn, mlp)]
    o = taps_oracle(True)
    fwd = o.forward(*args)
    G = {k: rng.normal(size=v.shape) for k, v in fwd.items()}
    d = o.backward(*args, G)
    loss = lambda a: sum(float((v * G[k]).sum()) for k, v in o.forward(*a).items())
    h, worst = 1e-6, 0.0
    for i, name in enumerate(ARGS):
        if name not in d:
            continue
        for _ in range(12):
            idx = tuple(int(rng.integers(0, s)) for s in args[i].shape)
            ap, am = list(args), list(args)
            ap[i], am[i] = args[i].copy(), args[i].copy()
            ap[i][idx] += h
            am[i][idx] -= h
            fd = (loss(ap) - loss(am)) / (2 * h)
            err = abs(fd - d[name][idx])
            worst = max(worst, err / (1 + abs(fd)))
            assert err <= 1e-6 * (1 + abs(fd)), (name, idx, fd, d[name][idx])
    print("[taps fd] ckd %d pn %d mlp %d: worst relative error %.2e" % (ckd, pn, mlp, worst))


def test_terms_modes():
    """abs >= |sum| and count = the number of non-zero terms: a pixel's direct term has one component per channel (kd's alpha up to five),
    plus four tap terms per pixel whose tap reads the element."""
    rng = np.random.default_rng(5)
    args = random_case(rng, 2, 5, 6, 4, True, False)
    o = taps_oracle()
    G = {k: rng.normal(size=v.shape).astype(np.float32) for k, v in o.forward(*args).items()}
    s, a, n = (o.backward(*args, G, terms=t) for t in ("sum", "abs", "count"))
    for k in s:
        assert np.all(a[k] >= np.abs(s[k]) * (1 - 1e-5)), k
        assert np.all(n[k] == np.round(n[k])) and n[k].max() >= 2, k
    assert n["kd"][..., 3].max() >= 5


def test_header_declares_both_entry_points():
    assert "mcs_jitter_taps_fwd" in _lib.EXPORTED_SYMBOLS and "mcs_jitter_taps_bwd" in _lib.EXPORTED_SYMBOLS
    assert _lib._ABI_VERSION == 2


def _cpu_args(ckd=3):
    B, H, W = 1, 4, 5
    t = lambda c: torch.zeros(B, H, W, c)
    return dict(rast=t(4), jitter=t(2), kd=t(ckd), ks=t(3), gb_normal=t(3))


@pytest.mark.parametrize("name,bad,what", [
    ("kd", torch.zeros(1, 4, 5, 5), "kd must be"), ("ks", torch.zeros(1, 4, 5, 4), "ks must be"),
    ("gb_normal", torch.zeros(1, 4, 5, 3, dtype=torch.float64), "gb_normal must be float32"), ("rast", torch.zeros(1, 4, 5, 3), "rast must be"),
    ("jitter", torch.zeros(4, 5, 2), "jitter must be"), ("perturbed_nrm", torch.zeros(1, 4, 5, 2), "perturbed_nrm must be"),
    ("kd", None, "kd must be a torch.Tensor"), ("rast", torch.zeros(1, 4, 5, 4), "rast must be a CUDA tensor")])
def test_argument_errors_name_the_argument(name, bad, what):
    before = sum(_lib.LAUNCHES.values())
    kw = _cpu_args()
    kw[name] = bad
    with pytest.raises(ValueError, match=what):
        jitter_taps(**kw)
    assert sum(_lib.LAUNCHES.values()) == before


@pytest.mark.parametrize("given", ["kd_jitter", "ks_jitter"])
def test_mlp_operands_go_together(given):
    kw = _cpu_args()
    kw[given] = torch.zeros(1, 4, 5, 3)
    with pytest.raises(ValueError, match="kd_jitter and ks_jitter go together.*got only %s" % given):
        jitter_taps(**kw)


def test_kd_jitter_takes_kd_channels():
    kw = _cpu_args(ckd=4)
    kw.update(kd_jitter=torch.zeros(1, 4, 5, 3), ks_jitter=torch.zeros(1, 4, 5, 3))
    with pytest.raises(ValueError, match=r"kd_jitter must be \[B,H,W,4\]"):
        jitter_taps(**kw)
