"""CPU: the oracle's restatement of the training step's streaming tail.  orc_shade_combine (render.py:119-127: normalise the two denoiser
outputs, recombine the demodulated signals) in fp64 against central finite differences, against the same torch composition in float64
and through the adjoint identity; and the divisor rule of image_loss when img broadcasts against a batched target."""
import numpy as np
import pytest
import torch

from common import oracle


def _combine_inputs(shape=(2, 3, 5), seed=0):
    g = np.random.default_rng(seed)
    a4 = g.uniform(0.1, 2.0, shape + (4,)); b4 = g.uniform(0.1, 2.0, shape + (4,))
    a4[..., 3] = g.uniform(0.5, 3.0, shape); b4[..., 3] = g.uniform(0.5, 3.0, shape)
    kd = g.uniform(0.0, 1.0, shape + (3,)); ks = g.uniform(0.0, 1.0, shape + (3,))
    dout = g.normal(size=shape + (3,))
    return [a4, b4, kd, ks], dout


def _torch_combine(a4, b4, kd, ks, pbr):
    """render.py:119-127 as the reference writes it (denoiser.py's rgb / w normalisation first)."""
    da = a4[..., 0:3] / a4[..., 3:4]
    if not pbr:
        return da * kd
    db = b4[..., 0:3] / b4[..., 3:4]
    return da * (kd * (1.0 - ks[..., 2:3])) + db


@pytest.mark.parametrize("pbr", [True, False])
def test_shade_combine_fp64_matches_the_torch_composition(pbr):
    o = oracle(f64=True)
    ins, dout = _combine_inputs(seed=1)
    t = [torch.tensor(x, dtype=torch.float64, requires_grad=True) for x in ins]
    ref = _torch_combine(*t, pbr)
    ref.backward(torch.tensor(dout))
    out = o.shade_combine(*ins, pbr=pbr)
    np.testing.assert_allclose(out, ref.detach().numpy(), rtol=1e-12, atol=1e-12)
    grads = o.shade_combine_bwd(*ins, dout, pbr=pbr)
    for name, g, x in zip(("a4", "b4", "kd", "ks"), grads, t):
        want = x.grad.numpy() if x.grad is not None else np.zeros_like(g)
        np.testing.assert_allclose(g, want, rtol=1e-12, atol=1e-12, err_msg=name)


@pytest.mark.parametrize("pbr", [True, False])
def test_shade_combine_fp64_gradients_match_central_differences(pbr):
    o = oracle(f64=True)
    ins, dout = _combine_inputs(shape=(1, 2, 3), seed=2)
    grads = o.shade_combine_bwd(*ins, dout, pbr=pbr)
    f = lambda xs: float((o.shade_combine(*xs, pbr=pbr) * dout).sum())
    h = 1e-6
    for k, (x, g) in enumerate(zip(ins, grads)):
        fd = np.zeros_like(x)
        for idx in np.ndindex(x.shape):
            xp = [a.copy() for a in ins]; xm = [a.copy() for a in ins]
            xp[k][idx] += h; xm[k][idx] -= h
            fd[idx] = (f(xp) - f(xm)) / (2 * h)
        np.testing.assert_allclose(g, fd, rtol=1e-7, atol=1e-8, err_msg="operand %d" % k)


@pytest.mark.parametrize("pbr", [True, False])
def test_shade_combine_adjoint_identity(pbr):
    """<J v, w> = <v, J^T w> for random directions v (all four operands at once) and upstream gradients w; J v by forward-mode AD of
    the float64 torch composition."""
    o = oracle(f64=True)
    ins, w = _combine_inputs(shape=(2, 4, 3), seed=3)
    g = np.random.default_rng(4)
    for _ in range(3):
        v = [g.normal(size=x.shape) for x in ins]
        _, jv = torch.func.jvp(lambda *xs: _torch_combine(*xs, pbr), tuple(torch.tensor(x) for x in ins), tuple(torch.tensor(d) for d in v))
        lhs = float((jv.numpy() * w).sum())
        rhs = sum(float((d * gr).sum()) for d, gr in zip(v, o.shade_combine_bwd(*ins, w, pbr=pbr)))
        assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), 1.0), (lhs, rhs)


def test_shade_combine_fp32_and_fp64_agree():
    ins, dout = _combine_inputs(seed=5)
    a, b = oracle().shade_combine(*ins), oracle(f64=True).shade_combine(*ins)
    assert a.dtype == np.float32 and np.abs(a - b).max() <= 1e-6 * np.abs(b).max()
    for x, y in zip(oracle().shade_combine_bwd(*ins, dout), oracle(f64=True).shade_combine_bwd(*ins, dout)):
        assert np.abs(x - y).max() <= 1e-5 * max(np.abs(y).max(), 1e-30)


@pytest.mark.parametrize("f64", [False, True])
def test_image_loss_divides_by_the_pixels_of_img(f64):
    """renderutils/ops.py:494 divides the summed per-pixel loss by img.shape[0:3], not by the broadcast grid: with img [1,H,W,3] against
    a target [N,H,W,3] the loss is N times the mean per-pixel loss, and so is its gradient.  The oracle follows that rule."""
    o = oracle(f64=f64)
    g = np.random.default_rng(6)
    N, H, W = 3, 5, 7
    img = g.uniform(0.0, 2.0, (1, H, W, 3)).astype(np.float32); tgt = g.uniform(0.0, 2.0, (N, H, W, 3)).astype(np.float32)
    for loss in ("l1", "mse", "relmse", "smape", "n2n"):
        px = o.image_loss_px(img, tgt, loss, "log_srgb")
        assert px.shape == (N, H, W)
        v = o.image_loss(img, tgt, loss, "log_srgb")
        assert v == px.sum(dtype=np.float64) / (H * W)
        assert abs(v / (N * px.mean(dtype=np.float64)) - 1) < 1e-12
        # img batched, target broadcast: both counts agree, the plain mean
        assert abs(o.image_loss(tgt, img, loss, "log_srgb") - o.image_loss_px(tgt, img, loss, "log_srgb").mean(dtype=np.float64)) < 1e-12
        # the scalar upstream gradient is the per-pixel one with dout / (img's pixels) everywhere
        gi, gt = o.image_loss_bwd(img, tgt, loss, "log_srgb", dout=2.0)
        gi2, gt2 = o.image_loss_bwd(img, tgt, loss, "log_srgb", dout=np.full((N, H, W), 2.0 / (H * W)))
        assert np.array_equal(gi, gi2) and np.array_equal(gt, gt2) and gi.shape == (N, H, W, 3)


def test_image_loss_per_pixel_gradient_is_the_adjoint_of_the_per_pixel_loss():
    """image_loss_bwd with an [N,H,W] upstream gradient w: the gradient of sum(w * image_loss_px), checked by central differences in fp64.
    log_srgb to 1e-5 only: loss.cu:33-39 writes the derivative of x^(1/2.4) with the six-digit constants 0.439583 and 0.583333.  Not n2n:
    its gradient holds the denominator img^2 + eps constant (loss.cu:84-89, img.detach() in the PyTorch twin), so it is not the derivative."""
    o = oracle(f64=True)
    g = np.random.default_rng(7)
    img = g.uniform(0.2, 2.0, (2, 2, 3, 3)); tgt = g.uniform(0.2, 2.0, (2, 2, 3, 3))
    w = g.normal(size=(2, 2, 3))
    for loss, tm in [(l, t) for l in ("mse", "relmse", "smape", "l1") for t in ("none", "log_srgb")]:
        rtol = 1e-7 if tm == "none" else 1e-5
        gi, gt = o.image_loss_bwd(img, tgt, loss, tm, dout=w)
        f = lambda a, b: float((o.image_loss_px(a, b, loss, tm) * w).sum())
        h = 1e-6
        for x, gx, first in ((img, gi, True), (tgt, gt, False)):
            fd = np.zeros_like(x)
            for idx in np.ndindex(x.shape):
                xp, xm = x.copy(), x.copy()
                xp[idx] += h; xm[idx] -= h
                fd[idx] = ((f(xp, tgt) - f(xm, tgt)) if first else (f(img, xp) - f(img, xm))) / (2 * h)
            np.testing.assert_allclose(gx, fd, rtol=rtol, atol=1e-8, err_msg=loss + " " + tm)
