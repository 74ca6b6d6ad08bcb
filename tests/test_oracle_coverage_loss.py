"""CPU: regularizer.coverage_image_loss's contract as the oracle helper states it (tests/coverage_loss_oracle.py) -- against the two lines
of the geometry passes evaluated by torch in fp64 with the package's image_loss(use_python=True), and against central finite differences
in fp64 -- and the argument checks of the C entries and of the Python function, without a device."""
import ctypes

import numpy as np
import pytest
import torch

import nvdiffrecmc_b200._lib as L
import nvdiffrecmc_b200.regularizer as R
import nvdiffrecmc_b200.renderutils as ru
from common import oracle
from coverage_loss_oracle import coverage_loss, coverage_loss_bwd, coverage_loss_px, cta_partials

LOSSES = ["l1", "mse", "relmse", "smape", "n2n"]
TONEMAPPERS = ["none", "log_srgb"]


def _operands(shape, seed):
    """shaded / ref [B,H,W,4] in the range where the kernels' clamps are inactive (rgb in (0, 65535)), ref alpha exactly 0, exactly 1
    and fractional."""
    rng = np.random.default_rng(seed)
    B, H, W = shape
    s = np.concatenate([rng.uniform(0.05, 3.0, (B, H, W, 3)), rng.uniform(0.0, 1.0, (B, H, W, 1))], -1)
    ra = rng.choice([0.0, 1.0, 0.5], (B, H, W, 1), p=[0.2, 0.5, 0.3]) * np.where(rng.random((B, H, W, 1)) < 0.3, rng.uniform(0.2, 1.0, (B, H, W, 1)), 1.0)
    ra[0, 0, 0] = 0.0; ra[0, 0, 1] = 1.0
    r = np.concatenate([rng.uniform(0.05, 3.0, (B, H, W, 3)), ra], -1)
    return s.astype(np.float32), r.astype(np.float32)


def _torch_chain(s, r, loss, tm):
    """The two lines of geometry/dmtet.py:229-230 in fp64 on the CPU: (loss, d shaded)."""
    st = torch.tensor(s, dtype=torch.float64, requires_grad=True)
    rt = torch.tensor(r, dtype=torch.float64)
    img_loss = torch.nn.functional.mse_loss(st[..., 3:], rt[..., 3:])
    img_loss = img_loss + ru.image_loss(st[..., 0:3] * rt[..., 3:], rt[..., 0:3] * rt[..., 3:], loss, tm, use_python=True)
    img_loss.backward()
    return float(img_loss.detach()), st.grad.numpy()


@pytest.mark.parametrize("tm", TONEMAPPERS)
@pytest.mark.parametrize("loss", LOSSES)
def test_fp64_oracle_equals_the_torch_chain(loss, tm):
    """Forward and d shaded.  The fp64 oracle keeps the reference kernel's fp32 constants -- eps = 0.01f, and in the log-sRGB 0.0031308f,
    1 / 2.4f, 1.055f and 0.439583f / 0.583333f for the derivative -- which the torch twin writes in fp64, so the two agree to 1e-8 (eps)
    and with the tonemap to 1e-6 (forward) and 1e-5 (gradient), rather than to rounding."""
    s, r = _operands((2, 7, 9), LOSSES.index(loss))
    o = oracle(f64=True)
    want, g_want = _torch_chain(s, r, loss, tm)
    got = coverage_loss(o, s, r, loss, tm)
    g = coverage_loss_bwd(o, s, r, loss, tm)
    rtol, gtol = (1e-8, 1e-8) if tm == "none" else (1e-6, 1e-5)
    assert abs(got - want) <= rtol * abs(want), (got, want)
    np.testing.assert_allclose(g, g_want, rtol=gtol, atol=gtol * np.abs(g_want).max())
    # the coverage term on its own is exact: alpha's gradient does not see the tonemap
    np.testing.assert_allclose(g[..., 3], g_want[..., 3], rtol=1e-13, atol=0)


@pytest.mark.parametrize("tm", TONEMAPPERS)
@pytest.mark.parametrize("loss", ["l1", "mse", "relmse", "smape"])
def test_fp64_gradient_matches_central_differences(loss, tm):
    """d shaded against central differences of the fp64 oracle's loss, on operands away from the clamps' kinks (premultiplied colours
    in (0, 65535), tone-mapped values above the sRGB threshold, |img - tgt| away from 0 for l1 / smape).  n2n is left out: its gradient
    treats the denominator as a constant (the reference's n2n backward, renderutils/loss.py's img.detach()), so it is not the derivative
    of its forward."""
    o = oracle(f64=True)
    rng = np.random.default_rng(7)
    B, H, W = 1, 3, 5
    s = np.concatenate([rng.uniform(0.2, 3.0, (B, H, W, 3)), rng.uniform(0.0, 1.0, (B, H, W, 1))], -1)
    r = np.concatenate([rng.uniform(0.2, 3.0, (B, H, W, 3)), rng.uniform(0.3, 1.0, (B, H, W, 1))], -1)
    keep = np.abs(s[..., :3] - r[..., :3]) > 0.05
    s[..., :3] = np.where(keep, s[..., :3], s[..., :3] + 0.3)
    g = coverage_loss_bwd(o, s, r, loss, tm)
    h = 1e-6
    fd = np.zeros_like(s)
    for idx in np.ndindex(s.shape):
        sp, sm = s.copy(), s.copy()
        sp[idx] += h; sm[idx] -= h
        fd[idx] = (coverage_loss(o, sp, r, loss, tm) - coverage_loss(o, sm, r, loss, tm)) / (2 * h)
    tol = 1e-7 if tm == "none" else 1e-5                     # the log-sRGB derivative's fp32 constants, as above
    np.testing.assert_allclose(g, fd, rtol=tol, atol=tol * np.abs(fd).max())


def test_cta_partials_restate_the_shuffle_order():
    """cta_partials sums each block of 256 in the kernel's order (restated here for the first block with scalar fp32 adds), within the
    bound of 255 fp32 additions of the fp64 sums; 33 x 31 pixels leave the last block one pixel short, which counts as 0."""
    rng = np.random.default_rng(3)
    v = rng.uniform(0, 1, 33 * 31).astype(np.float32)
    p = cta_partials(v)
    assert p.dtype == np.float32 and p.shape == (4,)
    pad = np.zeros(4 * 256, np.float64)
    pad[:v.size] = v
    ref = pad.reshape(4, 256).sum(1)
    assert (np.abs(p - ref) <= 255 * 2.0 ** -24 * ref * 1.01).all()
    x = v[:256].reshape(8, 32).astype(np.float32)
    for off in (16, 8, 4, 2, 1):
        x = x + x[:, np.arange(32) ^ off]
    s = np.float32(0)
    for w in range(8):
        s = np.float32(s + x[w, 0])
    assert p[0] == s
    cov, col = coverage_loss_px(oracle(), *_operands((1, 4, 5), 1))
    assert cov.dtype == np.float32 and col.dtype == np.float32 and cov.shape == (1, 4, 5)


# ---- argument checks without a device
def _desc(C=4, shape=(2, 4, 4), ptr=0x10000, strides=None):
    B, H, W = shape
    return L._desc(ptr, (B, H, W, C), strides or (H * W * C, W * C, C, 1))


def test_c_entries_refuse_bad_arguments_before_any_launch():
    """Each refusal returns non-zero with a message naming the problem; the descriptors point at fake addresses, so a check that went
    missing would end in a failed launch on this device-less machine, whose message names none of these."""
    if torch.cuda.is_available():
        pytest.skip("the calls would launch on the fake pointers")
    l = L.lib()
    g, P, O = _desc(), 0x30000, 0x40000
    by = ctypes.byref
    fwd = lambda a, b, li=0, ti=0, part=P, out=O: l.mcs_coverage_loss_fwd(a and by(a), b and by(b), li, ti, part, out, None)
    bwd = lambda a, b, li=0, ti=0, dl=P, di=O: l.mcs_coverage_loss_bwd(a and by(a), b and by(b), li, ti, dl, di, None)
    cases = [
        ("loss id", lambda f: f(g, g, li=5), b"unknown loss id 5"),
        ("negative loss id", lambda f: f(g, g, li=-1), b"unknown loss id -1"),
        ("tonemapper id", lambda f: f(g, g, ti=2), b"unknown tonemapper id 2"),
        ("null img", lambda f: f(None, g), b"img is null"),
        ("null ref pointer", lambda f: f(g, _desc(ptr=0)), b"ref is null"),
        ("img channels", lambda f: f(_desc(3), g), b"img must have 4 channels, got 3"),
        ("ref channels", lambda f: f(g, _desc(5)), b"ref must have 4 channels, got 5"),
        ("ref shape", lambda f: f(g, _desc(shape=(2, 4, 5))), b"ref must have the shape of img"),
        ("ref batch", lambda f: f(g, _desc(shape=(1, 4, 4))), b"ref must have the shape of img"),
        ("negative stride", lambda f: f(g, _desc(strides=(64, 16, -4, 1))), b"ref has a negative stride"),
        ("empty", lambda f: f(_desc(shape=(2, 0, 4)), _desc(shape=(2, 0, 4))), b"empty operands"),
        ("too many pixels", lambda f: f(_desc(shape=(2, 32768, 32768)), _desc(shape=(2, 32768, 32768))), b"at most 2^31 - 1"),
    ]
    for way, f in (("fwd", fwd), ("bwd", bwd)):
        for what, call, frag in cases:
            rc = call(f)
            msg = l.mcs_last_error() or b""
            assert rc != 0 and frag in msg and msg.startswith(b"coverage_loss_" + way.encode()), (way, what, msg)
    for what, rc in (("partials", fwd(g, g, part=None)), ("loss_out", fwd(g, g, out=None))):
        assert rc != 0 and l.mcs_last_error() == b"coverage_loss_fwd: null output pointer", what
    for what, rc in (("d_loss", bwd(g, g, dl=None)), ("d_img", bwd(g, g, di=None))):
        assert rc != 0 and l.mcs_last_error() == b"coverage_loss_bwd: null pointer argument", what
    assert bwd(g, g, di=O + 4) != 0 and b"16-byte aligned" in l.mcs_last_error()
    assert l.mcs_coverage_loss_num_partials(2, 4, 4) == 1 and l.mcs_coverage_loss_num_partials(1, 33, 31) == 4
    assert l.mcs_coverage_loss_num_partials(8, 512, 512) == l.mcs_image_loss_num_partials(8, 512, 512) == 8192


def test_python_errors_without_a_device():
    """Unknown names, and shaded's checks up to the device check, raise ValueError naming the problem, and nothing is launched (the
    checks of color_ref against shaded need shaded on a device: tests/test_gpu_coverage_loss.py)."""
    x = torch.rand(2, 4, 5, 4)
    cases = [
        ("unknown loss 'l2'", lambda: R.coverage_image_loss(x, x, "l2")),
        ("unknown tonemapper 'srgb'", lambda: R.coverage_image_loss(x, x, "l1", "srgb")),
        ("shaded must be \\[B,H,W,4\\]", lambda: R.coverage_image_loss(x[..., :3], x)),
        ("shaded must be float32", lambda: R.coverage_image_loss(x.double(), x)),
        ("shaded must be a torch.Tensor", lambda: R.coverage_image_loss(x.numpy(), x)),
        ("shaded must be a CUDA tensor", lambda: R.coverage_image_loss(x, x)),
    ]
    for frag, call in cases:
        before = dict(L.LAUNCHES)
        with pytest.raises(ValueError, match=frag):
            call()
        assert dict(L.LAUNCHES) == before, frag


def test_public_names():
    assert "coverage_image_loss" in R.__all__
    assert not hasattr(ru, "coverage_image_loss")
