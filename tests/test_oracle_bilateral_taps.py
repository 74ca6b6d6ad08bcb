"""CPU: the denoiser oracle's single tap weight, Oracle.bilateral_tap_weight, is the weight its filters sum -- and the weight the compiled
reference kernels sum.  A filter run on an impulse lattice (common.impulse_lattice: exactly one non-zero tap in every window) returns that
one tap's weight times the impulse, which with power-of-two impulses is exact; the S^2 lattice offsets cover every in-image tap of every
pixel once.  So the export must equal these impulse responses bit for bit, forward (the centre's depth gradient) and transposed (the
tap's), on guides with a zero normal, zero and negative depth gradients at centres and at taps, and windows clipped by the image on
every side (the images are smaller than the r = 9 window)."""
import numpy as np
import pytest

from common import _degenerate_guides, _radius, impulse_lattice, oracle

VALS = np.float32([1.0, 2.0, 4.0])             # per channel: a channel swap shows
SIGMAS = [np.float32(1e-20), np.float32(0.6), np.float32(2 * 1050 / 1750)]      # r = 3, 5 and 9 (the ramp's first r = 9 iteration)
B, H, W = 2, 11, 13


def _same(a, b):
    """bit-for-bit equality in either precision (so +0 / -0 count)"""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _guides():
    nrm, zdz = _degenerate_guides(B, H, W, seed=5)
    assert (nrm[0, H // 2, W // 3] == 0).all() and zdz[0, H // 2, W // 3 + 1, 1] == 0 and (zdz[B - 1, H // 2, W // 2, 1] < 0)
    return nrm, zdz


def _impulse_responses(fwd, bwd, nrm, zdz, sigma):
    """(forward, transposed) impulse responses [S^2, B, H, W] per channel divided by VALS -- the three channels must agree bit for bit --
    and the lattice's (dy, dx)."""
    r = _radius(sigma)
    S2 = (2 * r + 1) ** 2
    sig, dy, dx = impulse_lattice(B, H, W, r, VALS)
    n, z = np.tile(nrm, (S2, 1, 1, 1)), np.tile(zdz, (S2, 1, 1, 1))
    g4 = np.concatenate([sig, np.full(sig.shape[:3] + (1,), 8.0, np.float32) * (sig[..., :1] != 0)], -1)    # weight channel unused
    out = []
    for resp in (fwd(sig, n, z, sigma)[..., :3], bwd(n, z, sigma, g4)):
        w = resp / VALS.astype(resp.dtype)
        assert np.array_equal(w[..., 0], w[..., 1]) and np.array_equal(w[..., 0], w[..., 2])
        out.append(np.ascontiguousarray(w[..., 0]).reshape(S2, B, H, W))
    return out, dy, dx


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("sigma", SIGMAS, ids=["1e-20", "0.6", "1.2"])
def test_tap_weight_is_the_impulse_response_of_the_filters(f64, sigma):
    o = oracle(f64)
    nrm, zdz = _guides()
    (wf, wb), dy, dx = _impulse_responses(o.bilateral_fwd, o.bilateral_bwd, nrm, zdz, sigma)
    pix = np.arange(B * H * W).reshape(1, B, H, W)
    ef = o.bilateral_tap_weight(nrm, zdz, sigma, pix, dy, dx)
    eb = o.bilateral_tap_weight(nrm, zdz, sigma, pix, dy, dx, transposed=True)
    assert _same(ef, wf) and _same(eb, wb)
    assert (ef > 0).any() and (ef == 0).any()                                    # taps in and out of the image
    assert np.array_equal(ef, eb) == (sigma < 1e-3)                              # the two depth gradients differ, except at the centre


def test_tap_weight_outside_the_window_or_the_image_is_zero():
    o = oracle()
    nrm, zdz = _guides()
    r = _radius(0.6)
    flat = np.ones((B, H, W, 3), np.float32) * np.float32([0, 0, 1])
    zflat = np.stack([np.ones((B, H, W)), np.full((B, H, W), 0.01)], -1).astype(np.float32)
    p = (1 * H + 5) * W + 6                                                       # view 1, (5, 6)
    w = o.bilateral_tap_weight(flat, zflat, 0.6, p, [0, 0, r, -r, r + 1, 0, -6, 0, H - 5], [0, r, r, -r, 0, -(r + 1), 0, -7, 0])
    assert (w[:4] > 0).all() and w[0] == 1 and (w[4:6] == 0).all()               # ring r in, ring r + 1 out
    assert (w[6:] == 0).all()                                                     # outside the image (rows / columns of no view)
    assert o.bilateral_tap_weight(nrm, zdz, 0.6, (H // 2) * W + W // 3, [0, 1], [1, 0])[0] == 0     # zero normal at the centre


@pytest.mark.parametrize("sigma", SIGMAS, ids=["1e-20", "0.6", "1.2"])
def test_tap_weight_is_the_impulse_response_of_the_compiled_reference(sigma):
    """bilateral_denoiser_fwd_kernel / _bwd_kernel of denoising.cu, unmodified, on the host (oracle/_ref)."""
    from oracle import Reference
    try:
        ref = Reference(oracle())
    except RuntimeError as e:
        pytest.skip(str(e))
    o = oracle()
    nrm, zdz = _guides()
    (wf, wb), dy, dx = _impulse_responses(ref.bilateral_fwd, ref.bilateral_bwd, nrm, zdz, sigma)
    pix = np.arange(B * H * W).reshape(1, B, H, W)
    assert _same(o.bilateral_tap_weight(nrm, zdz, sigma, pix, dy, dx), wf)
    assert _same(o.bilateral_tap_weight(nrm, zdz, sigma, pix, dy, dx, transposed=True), wb)
