"""GPU: the bilateral denoiser's background skip is exact.

A warp whose outputs all have an exactly zero centre normal skips the tap loop when everything staged in its tile is finite (csrc/denoise.cu,
file header); its outputs come from the epilogue on zero accumulators.  The reference for such an output is the tap loop itself, run on the
same inputs with every other pixel of the image given a unit normal (a checkerboard), so that no warp is background and every warp runs
its loop: a zero-normal output does not depend on its taps' normals (each weight is FLT_EPS^128 = 0 times a factor in [0, 1], or NaN
from the depth term, whatever the tap normals), so the loop's result for it is the same with or without the checkerboard.  Two runs, one
per checkerboard parity, give every unchanged zero-normal output once.  They must agree bit for bit (NaN payloads aside) with the run
that skips: exactly (0, 0, 0, 1e-4) forward and (0, 0, 0) transposed where the tile is finite, and the loop's NaN wherever a NaN or
infinite depth, depth gradient, signal or upstream gradient reaches a zero-normal centre, so the skip must not fire there.

Every case runs through the single- and two-signal entry points, forward and transposed, on both staging kernels (contiguous signals: the
TMA-staged kernel where the radius allows it; strided views: the plain kernel), which must agree bit for bit.  sigma 2 (r = 11: both
directions TMA-staged), 3.2 (r = 19: the transposed filter falls back to the plain kernel) and 4.4 (r = 25: plain only, one signal; the
two-signal tile exceeds shared memory).  Shapes 2 x 45 x 72 (ragged 32 x 16 tiles both ways) and 1 x 37 x 70 (W % 4 != 0: plain only)."""
import ctypes as C

import numpy as np
import pytest
import torch

from common import _radius, nan_bits

pytestmark = pytest.mark.gpu

SIGMAS = [np.float32(2.0), np.float32(3.2), np.float32(4.4)]
SHAPES = [(2, 45, 72), (1, 37, 70)]
CASES = ["background", "mixed", "one_covered", "nonfinite"]
# the non-finite values, one per view of the "nonfinite" case, each at a background pixel: (array, channel, value)
POISON = [("zdz", 0, np.nan), ("zdz", 0, np.inf), ("zdz", 0, -np.inf), ("zdz", 1, np.nan), ("zdz", 1, "inf_next_to_inf_depth"),
          ("col", 0, np.nan), ("colB", 2, np.inf), ("gA", 1, np.nan), ("gB", 0, -np.inf)]


def _unit(shape, rng):
    n = rng.normal(size=shape + (3,)) + np.float64([0.2, 0.1, 1.5])
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


def _case(kind, shape, seed):
    """(col, colB, nrm, zdz, gA, gB) float32: background has a zero normal (both signs of zero) and depth 0, covered pixels a unit normal,
    a smooth depth with a step and dz = 0.01 (negative and zero in places)."""
    B, H, W = (len(POISON),) + shape[1:] if kind == "nonfinite" else shape
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    fg = np.zeros((B, H, W), bool)
    if kind in ("mixed", "nonfinite"):
        for b in range(B):                        # an ellipse per view: whole background tiles, mixed ones and whole covered ones
            cy, cx = rng.uniform(0.2, 0.8) * H, rng.uniform(0.2, 0.8) * W
            fg[b] = ((ys - cy) / (0.3 * H)) ** 2 + ((xs - cx) / (0.25 * W)) ** 2 < 1
    elif kind == "one_covered":
        fg[0, H // 2, W // 3] = True
    nrm = np.where(fg[..., None], _unit((B, H, W), rng), 0.0)
    nrm[~fg] *= np.where(rng.uniform(size=(~fg).sum()) < 0.5, -1.0, 1.0)[:, None]        # -0 and +0
    z = np.where(fg, 2.0 + 0.02 * xs + 0.01 * ys + 0.3 * (xs > W // 2), 0.0)
    dz = np.full((B, H, W), 0.01)
    dz[:, ::7, ::5] = -0.01
    dz[:, 3::11, 2::9] = 0.0
    zdz = np.stack([z, dz], -1).astype(np.float32)
    col, colB = [rng.uniform(0, 2, size=(B, H, W, 3)).astype(np.float32) for _ in range(2)]
    gA, gB = [rng.normal(size=(B, H, W, 4)).astype(np.float32) for _ in range(2)]
    a = dict(col=col, colB=colB, nrm=nrm.astype(np.float32), zdz=zdz, gA=gA, gB=gB)
    if kind == "nonfinite":
        for b, (name, c, v) in enumerate(POISON):
            bgy, bgx = np.nonzero(~fg[b])
            k = np.argmin((bgy - H // 2) ** 2 + (bgx - W // 2) ** 2)       # the background pixel nearest the centre
            y, x = bgy[k], bgx[k]
            if v == "inf_next_to_inf_depth":      # a guarded 1/dz of 0 next to an infinite depth difference
                a["zdz"][b, y, x, 1] = np.inf
                a["zdz"][b, y, x + 1 if x + 1 < W else x - 1, 0] = np.inf
            else:
                a[name][b, y, x, c] = v
    return a["col"], a["colB"], a["nrm"], a["zdz"], a["gA"], a["gB"]


def _filters(col, colB, nrm, zdz, gA, gB, sigma, dev):
    """Forward and transposed outputs [B,H,W,4] / [B,H,W,3] of every entry point (the two-signal ones only where their tile fits in shared memory), through every
    entry point on both staging kernels; all of them must agree bit for bit (NaN payloads aside)."""
    from nvdiffrecmc_b200 import _lib as L
    lib, sp = L.lib(), L.stream_ptr()
    r = _radius(sigma)
    two = 4 * 11 * (32 + 2 * r) * (16 + 2 * r) <= 227 * 1024
    t = lambda x: torch.tensor(x, device=dev)
    d = lambda x: C.byref(L.nhwc(x))
    wide = lambda x: torch.cat([x, torch.zeros_like(x[..., :1])], -1)[..., :x.shape[-1]]
    n, z = t(nrm), t(zdz)
    shape = tuple(col.shape[:3])
    runs = []
    for view in (lambda x: x, wide):
        a, b, ga, gb = view(t(col)), view(t(colB)), view(t(gA)), view(t(gB))
        f1, c1 = torch.empty(shape + (4,), device=dev), torch.empty(shape + (3,), device=dev)
        L.check(lib.mcs_bilateral_fwd(d(a), d(n), d(z), float(sigma), f1.data_ptr(), sp), "bilateral_fwd")
        L.check(lib.mcs_bilateral_bwd(d(n), d(z), float(sigma), d(ga), c1.data_ptr(), sp), "bilateral_bwd")
        run = {"fwd1": f1, "bwd1": c1}
        if two:
            fa, fb = torch.empty(shape + (4,), device=dev), torch.empty(shape + (4,), device=dev)
            ca, cb = torch.empty(shape + (3,), device=dev), torch.empty(shape + (3,), device=dev)
            L.check(lib.mcs_bilateral_fwd2(d(a), d(b), d(n), d(z), float(sigma), fa.data_ptr(), fb.data_ptr(), sp), "bilateral_fwd2")
            L.check(lib.mcs_bilateral_bwd2(d(n), d(z), float(sigma), d(ga), d(gb), ca.data_ptr(), cb.data_ptr(), sp), "bilateral_bwd2")
            run.update(fwd2A=fa, fwd2B=fb, bwd2A=ca, bwd2B=cb)
        runs.append({k: v.cpu().numpy() for k, v in run.items()})
    for k in runs[0]:
        assert np.array_equal(nan_bits(runs[0][k]), nan_bits(runs[1][k])), "%s: the two staging kernels disagree" % k
    if two:
        assert np.array_equal(nan_bits(runs[0]["fwd1"]), nan_bits(runs[0]["fwd2A"])), "forward: one and two signals disagree"
        assert np.array_equal(nan_bits(runs[0]["bwd1"]), nan_bits(runs[0]["bwd2A"])), "transposed: one and two signals disagree"
    return runs[0]


@pytest.mark.parametrize("kind", CASES)
@pytest.mark.parametrize("shape", SHAPES, ids=["2x45x72", "1x37x70"])
@pytest.mark.parametrize("sigma", SIGMAS, ids=["2", "3.2", "4.4"])
def test_background_skip_is_exact(dev, sigma, shape, kind):
    col, colB, nrm, zdz, gA, gB = _case(kind, shape, seed=shape[1] + shape[2])
    got = _filters(col, colB, nrm, zdz, gA, gB, sigma, dev)
    zero = (nrm == 0).all(-1)
    B, H, W = zero.shape
    checker = (np.arange(H)[:, None] + np.arange(W)[None, :]) % 2
    unit = _unit((B, H, W), np.random.default_rng(3)).astype(np.float32)
    for parity in (0, 1):
        lit = zero & (checker == parity)[None]
        forced = _filters(col, colB, np.where(lit[..., None], unit, nrm), zdz, gA, gB, sigma, dev)
        keep = zero & ~lit
        for k, v in got.items():
            assert np.array_equal(nan_bits(v[keep]), nan_bits(forced[k][keep])), "%s: %d of %d zero-normal outputs differ from the tap loop's" % (
                k, (nan_bits(v[keep]) != nan_bits(forced[k][keep])).any(-1).sum(), keep.sum())
    finite = all(np.isfinite(x).all() for x in (col, colB, zdz, gA, gB))
    if finite:
        for k, v in got.items():
            want = np.float32([0, 0, 0, 1e-4]) if v.shape[-1] == 4 else np.zeros(3, np.float32)
            assert np.array_equal(nan_bits(v[zero]), nan_bits(np.broadcast_to(want, v[zero].shape))), k
    else:
        # NaN reaches zero-normal centres: in the forward from a NaN or infinite depth and the inf-dz pair, in both directions from the signals
        nan_fwd = np.isnan(got["fwd1"][zero]).any(-1).sum()
        nan_bwd = np.isnan(got["bwd1"][zero]).any(-1).sum()
        assert nan_fwd > 0 and nan_bwd > 0, (nan_fwd, nan_bwd)
    if kind == "background":
        assert zero.all()
    if kind == "one_covered":
        assert (~zero).sum() == 1
