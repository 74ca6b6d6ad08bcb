"""GPU: the bilateral denoiser TAP BY TAP and PIXEL BY PIXEL against the fp64 oracle, at every radius of the training ramp.

Training sets sigma = 2 min(it / 1750, 1) (at least 1e-4); its first and last iteration at each radius are it = 0, 349 (r = 3), 350, 699
(r = 5), 700, 1049 (r = 7), 1050, 1399 (r = 9), 1400 and 1750 (r = 11), and each radius change falls on an fp32 sigma whose product with
2.5 rounds differently in double and in fp32.  Next to those, sigma 2.4 (r = 15: the transposed filter's last TMA-staged radius) and 3.0
(r = 17: the transposed filter falls back to the plain kernel).  Shapes: 2 x 45 x 72 (partial 32 x 16 tiles both ways, TMA-eligible),
1 x 37 x 70 (W % 4 != 0: the plain kernel only) and 1 x 9 x 16 (smaller than the window from r = 5 up).  Every case runs on both kernels
and through all four entry points (common._dn_both_paths), which must agree bit for bit.

The bar is check_per_element's: |got - r64| <= K max(Delta, |r32 - r64|) + R + 4 ulp32(r64), with Delta from +-1 ulp perturbations of
the inputs.  Tap weights get R = FLT_MIN + 8 x 2^-24 x w |ln w|: ex2.approx.ftz and the fp32 products flush a weight whose value is below
2^-126, and the exponent is rounded in fp32 (_exponent_rounding).  Filter outputs get R = (2r+1)^2 2^-24 A + (2r+1)^2 FLT_MIN max|signal|, A being the fp64 oracle on |signal| (the weights are >= 0, so A bounds the sum
of the terms' magnitudes): the first term bounds the fp32 summation in any order, the second the flushed weights."""
import numpy as np
import pytest
import torch

from common import _degenerate_guides, _dn_both_paths, _radius, check_per_element, impulse_lattice, oracle, same_bits

pytestmark = pytest.mark.gpu

K = 16
FLT_MIN = float(np.finfo(np.float32).tiny)
RAMP = [0, 349, 350, 699, 700, 1049, 1050, 1399, 1400, 1750]
SIGMAS = [np.float32(max(2.0 * min(it / 1750.0, 1.0), 1e-4)) for it in RAMP] + [np.float32(2.4), np.float32(3.0)]
SIGMA_IDS = ["it%d" % it for it in RAMP] + ["2.4", "3.0"]
SHAPES = [(2, 45, 72), (1, 37, 70), (1, 9, 16)]
GUIDES = ["degenerate", "silhouette"]
# power-of-two impulses, different per channel, signal and direction: products with a weight are exact, and a swap shows
V_FWD = (np.float32([1, 2, 4]), np.float32([8, 16, 32]))
V_BWD = (np.float32([64, 128, 256]), np.float32([512, 1024, 2048]))


def test_ramp_radii():
    assert [_radius(s) for s in SIGMAS] == [3, 3, 5, 5, 7, 7, 9, 9, 11, 11, 15, 17]


def _silhouette_guides(B, H, W, seed):
    """A bench-like G-buffer: background with depth 0 and a zero normal; foreground blobs with smooth depth, dz = 0.01 everywhere, and
    normals that are not unit length, |n|^2 in [0.9, 0.95], so that a centre's own weight (|n|^2)^128 (1.4e-6 .. 1.4e-3) straddles the
    weight floor 1e-4."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    nrm = np.zeros((B, H, W, 3)); z = np.zeros((B, H, W))
    for b in range(B):
        fg = np.zeros((H, W), bool)
        for _ in range(3):
            cy, cx = rng.uniform(0, H), rng.uniform(0, W)
            ry, rx = rng.uniform(0.2, 0.5) * H, rng.uniform(0.15, 0.4) * W
            fg |= ((ys - cy) / ry) ** 2 + ((xs - cx) / rx) ** 2 < 1
        n = np.stack([np.sin(xs * 0.21 + b), np.cos(ys * 0.17), 1.5 + 0.3 * np.sin((xs + ys) * 0.13)], -1)
        n /= np.linalg.norm(n, axis=-1, keepdims=True)
        n *= np.sqrt(rng.uniform(0.9, 0.95, size=(H, W, 1)))
        nrm[b][fg] = n[fg]
        z[b] = np.where(fg, 2.0 + 0.02 * xs + 0.01 * ys + 0.3 * (xs > W / 2), 0.0)
    zdz = np.stack([z, np.full((B, H, W), 0.01)], -1)
    return nrm.astype(np.float32), zdz.astype(np.float32)


def _guides(kind, shape):
    B, H, W = shape
    if kind == "silhouette":
        return _silhouette_guides(B, H, W, seed=H + W)
    return _degenerate_guides(B, H, W, seed=H + W)


def _floor(o64, filt, signal, r):
    """R of the module docstring for the filter `filt(|signal|)` (fp64 oracle)."""
    n = (2 * r + 1) ** 2
    a = np.asarray(filt(np.abs(np.asarray(signal, np.float64))), np.float64)
    m = float(np.abs(signal[..., :3]).max())
    if a.shape[-1] == 4:                                       # forward: the weight channel is the sum of the weights (signal 1)
        return n * 2.0 ** -24 * a + n * FLT_MIN * np.float64([m, m, m, 1.0])
    return n * 2.0 ** -24 * a + n * FLT_MIN * m


# ---------------------------------------------------------------------------------------------------------------------------------------
# a. tap by tap: impulse lattices
# ---------------------------------------------------------------------------------------------------------------------------------------
def _exponent_rounding(w64):
    """8 x 2^-24 x w |ln w|: the kernel forms a weight's exponent in fp32 -- k2 = -log2(e) / (2 sigma^2) rounded once on the host, then an
    FMA per tap -- so the exponent carries a rounding of a few units of 2^-24 relative to its size |ln w|.  Perturbing nrm and zdz does not
    reach it where the spatial term dominates (sigma is a scalar, not an input element), and the fp32 oracle's own exponent can land
    closer by chance.  Without this term, 19 of ~2e8 taps failed K = 16 on an H100 80GB HBM3 (700 W limit), all with the spatial term
    dominating, and their errors were at most 3.0 x 2^-24 x w |ln w|.  With it the worst ratio over all taps is 10.3."""
    w64 = np.asarray(w64, np.float64)
    return 8.0 * 2.0 ** -24 * w64 * np.abs(np.log(np.where(w64 > 0, w64, 1.0)))


def _quotients(out, vals, what):
    """out [..., >=3] / vals per channel: the three quotients must be one and the same weight, bit for bit."""
    q = [out[..., c] / vals[c] for c in range(3)]
    assert same_bits(q[0], q[1]) and same_bits(q[0], q[2]), "%s: the channels of one tap disagree" % what
    return q[0]


@pytest.mark.parametrize("guides", GUIDES)
@pytest.mark.parametrize("shape", SHAPES, ids=["2x45x72", "1x37x70", "1x9x16"])
@pytest.mark.parametrize("sigma", SIGMAS, ids=SIGMA_IDS)
def test_tap_by_tap(dev, sigma, shape, guides):
    """Every (pixel, tap) weight of the forward and the transposed filter, from the S^2 impulse lattices stacked along the batch (the guides
    repeat per lattice) plus one copy of the views without impulses.  Each weight within the bar (R as in the module docstring) of the oracle's
    bilateral_tap_weight on the same pairs; exactly +0 where the pixel's lattice point lies outside the image; nothing at all in the views
    without impulses (an impulse never shows in another view); the weight channel bit-identical across all lattices."""
    B, H, W = shape
    r = _radius(sigma)
    S2 = (2 * r + 1) ** 2
    nrm, zdz = _guides(guides, shape)
    lat = [impulse_lattice(B, H, W, r, v)[0] for v in V_FWD]
    glat = [impulse_lattice(B, H, W, r, np.append(v, np.float32(4096)))[0] for v in V_BWD]     # the weight channel of the gradient is unused
    _, dy, dx = impulse_lattice(B, H, W, r, V_FWD[0][:1])
    blank = lambda a: np.concatenate([a, np.zeros((B,) + a.shape[1:], np.float32)])
    n_rep, z_rep = np.tile(nrm, (S2 + 1, 1, 1, 1)), np.tile(zdz, (S2 + 1, 1, 1, 1))
    fA, fB, cA, cB = _dn_both_paths(blank(lat[0]), blank(lat[1]), n_rep, z_rep, blank(glat[0]), blank(glat[1]), sigma, dev)
    n = S2 * B
    for out in (fA, fB, cA, cB):
        assert same_bits(out[n:, ..., :3], np.zeros_like(out[n:, ..., :3])), "an impulse shows in a view without impulses"
    wsum = fA[..., 3].reshape(S2 + 1, B, H, W)
    assert same_bits(fB[..., 3], fA[..., 3]) and same_bits(wsum, np.broadcast_to(wsum[:1], wsum.shape)), "the weight channel depends on the signal"
    wf = _quotients(fA[:n], V_FWD[0], "forward A")
    assert same_bits(_quotients(fB[:n], V_FWD[1], "forward B"), wf), "the two forward signals weigh a tap differently"
    wb = _quotients(cA[:n], V_BWD[0], "transposed A")
    assert same_bits(_quotients(cB[:n], V_BWD[1], "transposed B"), wb), "the two transposed signals weigh a tap differently"
    wf, wb = wf.reshape(S2, B, H, W), wb.reshape(S2, B, H, W)
    ys, xs = np.arange(H)[None, None, :, None], np.arange(W)[None, None, None, :]
    out_img = (ys + dy < 0) | (ys + dy >= H) | (xs + dx < 0) | (xs + dx >= W)
    for w, what in ((wf, "forward"), (wb, "transposed")):
        assert same_bits(np.where(out_img, w, 0), np.zeros_like(w)), "%s: a tap outside the image has weight" % what
    pix = np.arange(B * H * W).reshape(1, B, H, W)
    o32, o64 = oracle(), oracle(f64=True)
    taps = lambda o: lambda ins: [o.bilateral_tap_weight(ins[0], ins[1], sigma, pix, dy, dx),
                                  o.bilateral_tap_weight(ins[0], ins[1], sigma, pix, dy, dx, transposed=True)]
    R = [FLT_MIN + _exponent_rounding(w) for w in taps(o64)([nrm, zdz])]
    check_per_element("bilateral r=%d %s %s taps" % (r, shape, guides), [wf, wb], taps(o64), taps(o32), [nrm, zdz], K,
                      ["forward weight", "transposed weight"], floor=R, tag="denoise")


# ---------------------------------------------------------------------------------------------------------------------------------------
# b. pixel by pixel: realistic signals
# ---------------------------------------------------------------------------------------------------------------------------------------
def _norm_floor(raw64, R):
    """R propagated through rgb / w (the weight channel R[..., 3])."""
    w = raw64[..., 3:]
    return R[..., :3] / w + np.abs(raw64[..., :3]) * R[..., 3:] / (w * w)


@pytest.mark.parametrize("guides", GUIDES)
@pytest.mark.parametrize("shape", SHAPES, ids=["2x45x72", "1x37x70", "1x9x16"])
@pytest.mark.parametrize("sigma", SIGMAS, ids=SIGMA_IDS)
def test_pixel_by_pixel(dev, sigma, shape, guides):
    """Random colours and signed upstream gradients: the raw forward [B,H,W,4] and the transposed filter (all four entry points, both
    kernels), ou.bilateral_denoiser's normalised output and its column gradient through the autograd of the division, and
    BilateralDenoiser.forward on the reference's 8-channel tensor (strided slices, _safe_normalize'd normals)."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.denoiser import BilateralDenoiser
    B, H, W = shape
    r = _radius(sigma)
    nrm, zdz = _guides(guides, shape)
    rng = np.random.default_rng(B * H * W + r)
    col, colB = [rng.uniform(0, 2, size=(B, H, W, 3)).astype(np.float32) for _ in range(2)]
    gA, gB = [rng.normal(size=(B, H, W, 4)).astype(np.float32) for _ in range(2)]
    g3 = rng.normal(size=(B, H, W, 3)).astype(np.float32)
    fA, fB, cA, cB = _dn_both_paths(col, colB, nrm, zdz, gA, gB, sigma, dev)
    o32, o64 = oracle(), oracle(f64=True)
    tag = "bilateral r=%d %s %s" % (r, shape, guides)
    fwd = lambda o: lambda ins: [o.bilateral_fwd(ins[0], ins[2], ins[3], sigma), o.bilateral_fwd(ins[1], ins[2], ins[3], sigma)]
    R = [_floor(o64, lambda s: o64.bilateral_fwd(s, nrm, zdz, sigma), c, r) for c in (col, colB)]
    worst = [check_per_element(tag + " forward", [fA, fB], fwd(o64), fwd(o32), [col, colB, nrm, zdz], K, ["A", "B"], floor=R, tag="denoise")]
    bwd = lambda o: lambda ins: [o.bilateral_bwd(ins[2], ins[3], sigma, ins[0]), o.bilateral_bwd(ins[2], ins[3], sigma, ins[1])]
    Rb = [_floor(o64, lambda s: o64.bilateral_bwd(nrm, zdz, sigma, s), g, r) for g in (gA, gB)]
    worst.append(check_per_element(tag + " transposed", [cA, cB], bwd(o64), bwd(o32), [gA, gB, nrm, zdz], K, ["A", "B"], floor=Rb, tag="denoise"))

    # ou.bilateral_denoiser and its column gradient (ops.py:139-141): the division's gradient g / w reaches the transposed filter
    t = lambda a: torch.tensor(a, device=dev)
    c = t(col).requires_grad_(True)
    out = ou.bilateral_denoiser(c, t(nrm), t(zdz), float(sigma))
    out.backward(t(g3))

    def norm_and_grad(o):
        def f(ins):
            raw = np.asarray(o.bilateral_fwd(ins[0], ins[1], ins[2], sigma))
            og = np.concatenate([ins[3] / raw[..., 3:], np.zeros_like(raw[..., 3:])], -1)
            return [raw[..., :3] / raw[..., 3:], o.bilateral_bwd(ins[1], ins[2], sigma, og)]
        return f
    raw64 = np.asarray(o64.bilateral_fwd(col, nrm, zdz, sigma), np.float64)
    og64 = np.concatenate([g3 / raw64[..., 3:], np.zeros_like(raw64[..., 3:])], -1)
    rel_w = R[0][..., 3:] / raw64[..., 3:]
    Rg = _floor(o64, lambda s: o64.bilateral_bwd(nrm, zdz, sigma, s), og64, r) + np.asarray(
        o64.bilateral_bwd(nrm, zdz, sigma, np.concatenate([np.abs(og64[..., :3]) * rel_w, np.zeros_like(rel_w)], -1)))
    worst.append(check_per_element(tag + " bilateral_denoiser", [out.detach().cpu().numpy(), c.grad.cpu().numpy()], norm_and_grad(o64),
                                   norm_and_grad(o32), [col, nrm, zdz, g3], K, ["normalised", "column gradient"],
                                   floor=[_norm_floor(raw64, R[0]), Rg], tag="denoise"))

    # BilateralDenoiser.forward: one [B,H,W,8] tensor, sliced; its normals are scaled, and _safe_normalize'd on the device
    den = BilateralDenoiser(influence=float(sigma) / 2)
    assert np.float32(den.sigma) == sigma
    x = t(np.concatenate([col, nrm * np.float32(0.7), zdz], -1))
    got = den.forward(x).cpu().numpy()
    from nvdiffrecmc_b200.denoiser import _safe_normalize
    n_used = _safe_normalize(x[..., 3:6]).cpu().numpy()
    nf = lambda o: lambda ins: [o.bilateral_denoiser(ins[0], ins[1], ins[2], sigma)]
    raw64m = np.asarray(o64.bilateral_fwd(col, n_used, zdz, sigma), np.float64)
    Rm = _floor(o64, lambda s: o64.bilateral_fwd(s, n_used, zdz, sigma), col, r)
    worst.append(check_per_element(tag + " BilateralDenoiser", [got], nf(o64), nf(o32), [col, n_used, zdz], K, ["forward"],
                                   floor=[_norm_floor(raw64m, Rm)], tag="denoise"))
    print("[denoise] %s: worst ratio %.3g" % (tag, max(worst)))


# ---------------------------------------------------------------------------------------------------------------------------------------
# c. the bench launch: 8 x 512^2 at sigma = 2, compared on crops
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_guides(dev):
    """The bench's denoiser guides: primary rays of its 8 views traced on the device, synth.assemble_gbuffer, the shading normal of
    prepare_shading_normal _safe_normalize'd, zdz = (depth, 0.01) -- as bench.py's shade() hands them to denoise_and_combine."""
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    from bench import WORKLOAD as wl, build_scene_numpy, view_pose
    from nvdiffrecmc_b200 import synth
    from nvdiffrecmc_b200.denoiser import _safe_normalize
    v, f, vn = build_scene_numpy(wl, 0)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=1)
    r, B = wl["res"], wl["views_per_gpu"]
    gbs = []
    for gi in range(B):
        ang, tilt = view_pose(gi)
        campos, ro, rd = synth.primary_rays(synth.orbit_view(ang, tilt=tilt), r)
        tid, tuv = ou.trace_closest(ctx, torch.tensor(ro.reshape(-1, 3), device=dev), torch.tensor(rd.reshape(-1, 3), device=dev))
        gbs.append(synth.assemble_gbuffer(v, f, vn, tid.cpu().numpy().reshape(r, r), tuv.cpu().numpy().reshape(r, r, 3), campos, seed=100 + gi))
    del ctx
    st = lambda k: torch.tensor(np.ascontiguousarray(np.stack([g[k] for g in gbs]), np.float32), device=dev)
    nrm = ru.prepare_shading_normal(st("pos"), st("view_pos").reshape(B, 1, 1, 3), None, st("smooth_nrm"), st("tangent"), st("geom_nrm"),
                                    two_sided_shading=True, opengl=True)
    depth = st("depth")
    zdz = torch.stack([depth, torch.full_like(depth, 0.01)], -1)
    return _safe_normalize(nrm).contiguous().cpu().numpy(), zdz.contiguous().cpu().numpy()


def _crops(nrm, r, rng):
    """(view, y0, x0) of 64 x 64 output blocks: the four corners of views 0 and 7, one across tile seams (x = 0 mod 32, y = 0 mod 16),
    the two blocks of most silhouette pixels (a zero normal next to a non-zero one) and two random ones."""
    B, H, W = nrm.shape[:3]
    out = [(b, y, x) for b in (0, B - 1) for y in (0, H - 64) for x in (0, W - 64)]
    out.append((3, 16 * 9 + 8, 32 * 5 + 16))
    bg = (nrm == 0).all(-1)
    edge = np.zeros_like(bg)
    edge[:, 1:] |= bg[:, 1:] != bg[:, :-1]
    edge[:, :, 1:] |= bg[:, :, 1:] != bg[:, :, :-1]
    counts = edge.reshape(B, H // 64, 64, W // 64, 64).sum((2, 4))
    for k in np.argsort(counts.reshape(-1))[::-1][:2]:
        b, by, bx = np.unravel_index(k, counts.shape)
        out.append((int(b), int(by) * 64, int(bx) * 64))
    for _ in range(2):
        out.append((int(rng.integers(B)), int(rng.integers(H - 64)), int(rng.integers(W - 64))))
    return out


def test_bench_launch_on_crops(dev, bench_guides):
    """denoise_and_combine's first launch (the two-signal forward) and its backward (the two-signal transposed filter) at the bench
    shape 8 x 512^2, sigma = 2 (r = 11), on both kernels.  Each crop of (64 + 2r)^2 pixels around a 64^2 block is filtered by the oracle as
    an image of its own; the pixels whose window the crop holds whole -- the block, and the crop's rim where it is the image's edge -- are
    compared per element."""
    nrm, zdz = bench_guides
    B, H, W = nrm.shape[:3]
    sigma = np.float32(2.0)
    r = _radius(sigma)
    rng = np.random.default_rng(17)
    diff, spec = [rng.uniform(0, 2, size=(B, H, W, 3)).astype(np.float32) for _ in range(2)]
    gA, gB = [rng.normal(size=(B, H, W, 4)).astype(np.float32) for _ in range(2)]
    outs = _dn_both_paths(diff, spec, nrm, zdz, gA, gB, sigma, dev)
    assert (nrm == 0).all(-1).mean() > 0.05 and (nrm != 0).any(-1).mean() > 0.05
    o32, o64 = oracle(), oracle(f64=True)
    filt = lambda o: lambda ins: [o.bilateral_fwd(ins[0], ins[4], ins[5], sigma), o.bilateral_fwd(ins[1], ins[4], ins[5], sigma),
                                  o.bilateral_bwd(ins[4], ins[5], sigma, ins[2]), o.bilateral_bwd(ins[4], ins[5], sigma, ins[3])]
    for b, y0, x0 in _crops(nrm, r, rng):
        ya, yb, xa, xb = max(y0 - r, 0), min(y0 + 64 + r, H), max(x0 - r, 0), min(x0 + 64 + r, W)
        ys, xs = np.arange(ya, yb)[:, None], np.arange(xa, xb)[None, :]
        whole = ((ys - r >= ya) | (ya == 0)) & ((ys + r < yb) | (yb == H)) & ((xs - r >= xa) | (xa == 0)) & ((xs + r < xb) | (xb == W))
        assert whole[y0 - ya:y0 - ya + 64, x0 - xa:x0 - xa + 64].all()
        cut = lambda a: np.ascontiguousarray(a[b:b + 1, ya:yb, xa:xb])
        ins = [cut(a) for a in (diff, spec, gA, gB, nrm, zdz)]
        got = [cut(a) for a in outs]
        R = [_floor(o64, lambda s: o64.bilateral_fwd(s, ins[4], ins[5], sigma), ins[k], r) for k in (0, 1)]
        R += [_floor(o64, lambda s: o64.bilateral_bwd(ins[4], ins[5], sigma, s), ins[k], r) for k in (2, 3)]
        ex = [np.broadcast_to(~whole[None, :, :, None], g.shape) for g in got]
        check_per_element("bilateral bench crop view %d (%d, %d)" % (b, y0, x0), got, filt(o64), filt(o32), ins, K,
                          ["forward diffuse", "forward specular", "transposed A", "transposed B"], exempt=ex, floor=R, tag="denoise")


# ---------------------------------------------------------------------------------------------------------------------------------------
# d. tiny sigma
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sigma", [np.float32(1e-20), np.float32(1e-22), np.float32(1e-24)], ids=["1e-20", "1e-22", "1e-24"])
def test_tiny_sigma(dev, sigma):
    """-log2(e) / (2 sigma^2) overflows fp32 below sigma ~ 4.6e-20.  The reference's centre tap is still -0 / (2 sigma^2) = -0, weight 1,
    so its output is finite -- close to the identity -- until 2 sigma^2 itself rounds to 0 (sigma ~ 2.6e-23); then its centre tap is NaN,
    and so is every colour it filters (the weight channel stays at the 1e-4 floor).  The product must follow: per element at 1e-20 and
    1e-22, NaN exactly where the fp32 oracle has it at 1e-24."""
    B, H, W = 2, 45, 72
    r = _radius(sigma)
    assert r == 3
    nrm, zdz = _degenerate_guides(B, H, W, seed=1)
    rng = np.random.default_rng(2)
    col, colB = [rng.uniform(0, 2, size=(B, H, W, 3)).astype(np.float32) for _ in range(2)]
    gA, gB = [rng.normal(size=(B, H, W, 4)).astype(np.float32) for _ in range(2)]
    outs = _dn_both_paths(col, colB, nrm, zdz, gA, gB, sigma, dev)
    o32, o64 = oracle(), oracle(f64=True)
    filt = lambda o: lambda ins: [o.bilateral_fwd(ins[0], ins[4], ins[5], sigma), o.bilateral_fwd(ins[1], ins[4], ins[5], sigma),
                                  o.bilateral_bwd(ins[4], ins[5], sigma, ins[2]), o.bilateral_bwd(ins[4], ins[5], sigma, ins[3])]
    ins = [col, colB, gA, gB, nrm, zdz]
    R = [_floor(o64, lambda s: o64.bilateral_fwd(s, nrm, zdz, sigma), ins[k], r) for k in (0, 1)]
    R += [_floor(o64, lambda s: o64.bilateral_bwd(nrm, zdz, sigma, s), ins[k], r) for k in (2, 3)]
    check_per_element("bilateral sigma %g" % sigma, outs, filt(o64), filt(o32), ins, K,
                      ["forward A", "forward B", "transposed A", "transposed B"], floor=R, tag="denoise")
    if sigma > 1e-23:
        assert all(np.isfinite(x).all() for x in outs)
        unit = (np.abs(np.sum(nrm.astype(np.float64) ** 2, -1) - 1) < 1e-6)[..., None]
        w = (nrm.astype(np.float64) ** 2).sum(-1, keepdims=True) ** 128
        assert np.allclose(np.where(unit, outs[0][..., :3], 0), np.where(unit, col * w, 0), rtol=1e-4, atol=0)   # the identity, weighed
    else:
        assert np.isnan(outs[0][..., :3]).all() and (outs[0][..., 3] == np.float32(1e-4)).all()
