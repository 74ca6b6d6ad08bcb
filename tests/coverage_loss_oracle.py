"""regularizer.coverage_image_loss's contract stated on the CPU oracle of image_loss (orc_image_loss_fwd / _bwd) -- TEST INFRASTRUCTURE.

The geometry passes' image loss is mse(shaded.a, ref.a) + image_loss(shaded.rgb * ref.a, ref.rgb * ref.a): the colour term is the
oracle's image loss of the colours premultiplied in the oracle build's precision, the coverage term is restated here in numpy.  No C of its
own.  `cta_partials` restates the kernel's per-CTA summation order (csrc/lossmesh.cu) for fp32 terms."""
import numpy as np

LOSS_BLOCK = 256                                    # lossmesh.cu: one partial per 256 consecutive pixels


def _split(o, shaded, ref):
    s, r = np.asarray(shaded, o.dt), np.asarray(ref, o.dt)
    assert s.shape == r.shape and s.ndim == 4 and s.shape[3] == 4, (s.shape, r.shape)
    a = r[..., 3:]
    return s, r, s[..., :3] * a, r[..., :3] * a     # one multiply in the build's precision


def coverage_loss_px(o, shaded, ref, loss="l1", tonemapper="none"):
    """(coverage, colour), each [B,H,W] in o's precision: (shaded.a - ref.a)^2 and image_loss's per-pixel value of the premultiplied rgb."""
    s, r, img, tgt = _split(o, shaded, ref)
    d = s[..., 3] - r[..., 3]
    return d * d, o.image_loss_px(img, tgt, loss, tonemapper)


def coverage_loss(o, shaded, ref, loss="l1", tonemapper="none"):
    """The loss in double: both per-pixel terms summed in fp64 and divided by B*H*W."""
    cov, col = coverage_loss_px(o, shaded, ref, loss, tonemapper)
    n = cov.size
    return cov.sum(dtype=np.float64) / n + col.sum(dtype=np.float64) / n


def coverage_loss_bwd(o, shaded, ref, loss="l1", tonemapper="none", dout=1.0):
    """d shaded [B,H,W,4] for the upstream gradient dout: rgb = image_loss's d img (dout / (B*H*W) per pixel) * ref.a, alpha =
    2 / (B*H*W) * (shaded.a - ref.a) * dout."""
    s, r, img, tgt = _split(o, shaded, ref)
    n = s[..., 0].size
    gi, _ = o.image_loss_bwd(img, tgt, loss, tonemapper, dout=dout)
    ga = o.dt(2.0 / n) * (s[..., 3] - r[..., 3]) * o.dt(dout)
    return np.concatenate([gi * r[..., 3:], ga[..., None]], -1)


def cta_partials(px):
    """fp32 per-CTA sums of the per-pixel terms px in the kernel's order: 256 pixels per CTA, butterfly (xor 16, 8, 4, 2, 1) within each
    warp, then the eight warp sums added in warp order to 0."""
    v = np.asarray(px, np.float32).reshape(-1)
    P = (v.size + LOSS_BLOCK - 1) // LOSS_BLOCK
    x = np.zeros(P * LOSS_BLOCK, np.float32)
    x[:v.size] = v
    x = x.reshape(P, LOSS_BLOCK // 32, 32)
    lane = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        x = x + x[..., lane ^ off]
    s = np.zeros(P, np.float32)
    for w in range(LOSS_BLOCK // 32):
        s = s + x[:, w, 0]
    return s
