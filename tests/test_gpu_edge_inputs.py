"""GPU parity on the inputs where kernels go wrong: the renderutils ops and env_shade on the edge inputs that tests/test_oracle_ref.py
runs through the oracle and the host-compiled reference (zero vectors, +-1, 1e-6, 1e4, back-facing and grazing geometry, a zero shading
normal, roughness 0 / 1, a probe with black texels), the denoiser on degenerate guides and at radii where an fp32 product 2.5 * sigma
would round differently from the reference's double one, and the image loss at the training shape.  The fast machinery of the kernels
(FMA contraction, the 4-pixel vector path and its scalar tail, ex2 / rsqrt approximations, env_shade's n.wi > 0 gate) is what separates
these inputs from the easy ones of the other GPU tests; the bars are the ones the oracle meets against the reference."""
import numpy as np
import pytest
import torch

from common import RU_OPS, _degenerate_guides, _dn_both_paths, _radius, env_shade_edge_case, oracle, rel_l2, ru_edge_inputs
from common import nan_bits as _bits

pytestmark = pytest.mark.gpu


def _close(got, want, want64, bar, what):
    """Same NaN / +-inf positions as the fp32 oracle; finite values within bar x (largest finite oracle magnitude).  On failure the
    message gives both fp32 sides' distance from the fp64 oracle, which tells which side is the noisy one."""
    got = np.asarray(got, np.float32); want = np.asarray(want, np.float32); want64 = np.asarray(want64, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "%s: NaN at %d product / %d oracle positions, %d differ" % (
        what, np.isnan(got).sum(), np.isnan(want).sum(), (np.isnan(got) != np.isnan(want)).sum())
    for inf in (np.isposinf, np.isneginf):
        assert np.array_equal(inf(got), inf(want)), "%s: infinities differ" % what
    ok = np.isfinite(want)
    if not ok.any():
        return
    scale = max(float(np.abs(want[ok]).max()), 1e-30)
    err = float(np.abs(got[ok].astype(np.float64) - want[ok]).max())
    if err > bar * scale:
        ok64 = ok & np.isfinite(want64)
        e_p = float(np.abs(got[ok64] - want64[ok64]).max()) if ok64.any() else float("nan")
        e_o = float(np.abs(want[ok64] - want64[ok64]).max()) if ok64.any() else float("nan")
        raise AssertionError("%s: max |product - oracle| %.3e > %.0e x %.3e; against fp64: product %.3e, fp32 oracle %.3e" % (
            what, err, bar, scale, e_p, e_o))


# ---------------------------------------------------------------------------------------------------------------------------------------
# renderutils ops
# ---------------------------------------------------------------------------------------------------------------------------------------
def _ru_fn(kernel, kw):
    import nvdiffrecmc_b200.renderutils as ru
    return {"lambert": ru.lambert, "frostbite": ru.frostbite_diffuse, "fresnel": ru._fresnel_shlick, "ndf": ru._ndf_ggx,
            "lambda": ru._lambda_ggx, "masking": ru._masking_smith,
            "specular": lambda *a: ru.pbr_specular(*a, **kw), "bsdf": lambda *a: ru.pbr_bsdf(*a, **kw),
            "psn": lambda *a: ru.prepare_shading_normal(*a, **kw)}[kernel]


def _ru_run(fn, ins, dout, dev, sliced):
    """Forward and every input gradient.  sliced=True passes each operand as the leading channels of a one-channel-wider tensor: a
    strided view, which the kernels load pixel by pixel (scalar path) instead of four pixels per 128-bit load."""
    xs = []
    for a in ins:
        c = a.shape[-1]
        w = torch.zeros(*a.shape[:-1], c + 1 if sliced else c, device=dev)
        w[..., :c] = torch.tensor(a, device=dev)
        w.requires_grad_(True)
        x = w[..., :c]
        assert x.is_contiguous() != sliced
        xs.append(x)
    out = fn(*xs)
    grads = torch.autograd.grad(out, xs, torch.tensor(dout, device=dev), allow_unused=True)
    return out.detach().cpu().numpy(), [np.zeros_like(a) if g is None else g.cpu().numpy() for g in grads]


def _ragged(a):
    """[1,6,8,c] -> [1,1,47,c]: pixel order reversed and the last original pixel dropped, so that pixels 0..2 (the zero, +1 and -1
    vectors) land in the ragged last group of 3 pixels, which a separate kernel instantiation handles."""
    return np.ascontiguousarray(a.reshape(1, 1, -1, a.shape[-1])[:, :, ::-1][:, :, 1:])


@pytest.mark.parametrize("kernel,fwd,bwd,chans,out_c,extras,kw", RU_OPS)
def test_renderutils_edge_inputs(dev, kernel, fwd, bwd, chans, out_c, extras, kw):
    """Every op of the table, forward and all input gradients, against the fp32 oracle on the edge inputs: identical NaN / inf
    positions, finite values within 2e-5 x scale forward and 1e-3 x scale backward.  Contiguous operands take the 4-pixel vector path,
    channel-slice views of the same values the scalar one: forward outputs must be bit-identical, and a pixel must get the same bits in
    a full 4-pixel group as in the ragged tail."""
    fn = _ru_fn(kernel, kw)
    o32, o64 = oracle(), oracle(f64=True)
    ins0, dout0 = ru_edge_inputs(chans, out_c)
    fwd_by_layout = {}
    for layout in ("grid", "ragged"):
        ins, dout = (ins0, dout0) if layout == "grid" else ([_ragged(a) for a in ins0], _ragged(dout0))
        want, want64 = getattr(o32, fwd)(*ins, **kw), getattr(o64, fwd)(*ins, **kw)
        g32, g64 = getattr(o32, bwd)(*ins, dout, **kw), getattr(o64, bwd)(*ins, dout, **kw)
        g32, g64 = (g32, g64) if isinstance(g32, tuple) else ((g32,), (g64,))
        outs = {}
        for sliced in (False, True):
            tag = "%s %s %s" % (kernel, layout, "slice" if sliced else "contiguous")
            out, grads = _ru_run(fn, ins, dout, dev, sliced)
            _close(out, want, want64, 2e-5, tag + " forward")
            assert len(grads) == len(g32)
            for i, (g, r32, r64) in enumerate(zip(grads, g32, g64)):
                _close(g, r32, r64, 1e-3, "%s gradient %d" % (tag, i))
            outs[sliced] = out
        assert np.array_equal(_bits(outs[False]), _bits(outs[True])), "%s %s: vector and scalar paths differ" % (kernel, layout)
        fwd_by_layout[layout] = outs[False].reshape(-1, out_c)
    assert np.array_equal(_bits(fwd_by_layout["ragged"][::-1]), _bits(fwd_by_layout["grid"][:-1])), \
        "%s: a pixel in the ragged tail differs from the same pixel in a full 4-pixel group" % kernel


# ---------------------------------------------------------------------------------------------------------------------------------------
# env_shade
# ---------------------------------------------------------------------------------------------------------------------------------------
def _es_tensors(c, dev):
    return [torch.tensor(c[k], device=dev) for k in ("mask", "ro", "pos", "nrm", "view", "kd", "ks", "light", "pdf", "rows", "cols")]


def _es_oracle_args(c):
    return (c["scene"], c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"],
            c["perms"])


@pytest.mark.parametrize("bsdf", ["pbr", "diffuse", "white"])
@pytest.mark.parametrize("shadow_scale", [1.0, 0.5])
def test_env_shade_edge_case(dev, bsdf, shadow_scale):
    """Zero and flipped shading normals, roughness 0 / 1, pure metal, black albedo, a probe with a black row and black texels.
    Texel records bit for bit on every pixel (the zero-normal pixel's BSDF samples included); visibility equal wherever the product
    traced.  The product never traces a ray with n.wi <= 0 -- all rays of the zero-normal pixel -- while the oracle does: its record
    there holds hits and misses, which radiance and gradients must not depend on.  Radiance within 1e-4 with the same NaN positions;
    gradients in all three backward modes within max(1e-4, 2 x the fp32 oracle's distance from the fp64 one)."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.optixutils import ops
    c = env_shade_edge_case()
    if bsdf == "white":
        c["kd"] = np.ones_like(c["kd"])        # render.py:107
    N, seed = c["N"], 21
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(c["verts"], device=dev), torch.tensor(c["tris"], device=dev), rebuild=1)
    perms = torch.tensor(c["perms"], device=dev)
    kw = dict(BSDF=bsdf, n_samples_x=N, rnd_seed=seed, shadow_scale=shadow_scale)
    diff, spec, rec_t, rec_v = ops.env_shade_records(ctx, *_es_tensors(c, dev), perms, **kw)
    o32, o64 = oracle(), oracle(f64=True)
    d_ref, s_ref, (rt, rv) = o32.env_shade(*_es_oracle_args(c), records=True, **kw)
    rec_t, rec_v = rec_t.cpu().numpy(), rec_v.cpu().numpy()
    assert np.array_equal(rec_t, rt), "env texel records differ on %d of %d rays" % ((rec_t != rt).sum(), rt.size)
    traced = rec_v != 2
    assert np.array_equal(rec_v[traced], rv[traced]), "visibility differs on %d traced rays" % (rec_v[traced] != rv[traced]).sum()
    zero = c["edge_px"][0]
    assert (rec_v[zero] == 2).all() and np.isin(rv[zero], (0, 1)).all()
    assert traced[c["mask"] > 0].mean() > 0.2
    for name, got, want in (("diffuse", diff, d_ref), ("specular", spec, s_ref)):
        got = got.cpu().numpy()
        assert np.array_equal(np.isnan(got), np.isnan(want)), name
        assert rel_l2(np.nan_to_num(got), np.nan_to_num(want)) < 1e-4, (name, rel_l2(np.nan_to_num(got), np.nan_to_num(want)))

    rng = np.random.default_rng(0)
    gd = rng.uniform(size=d_ref.shape).astype(np.float32); gs = rng.uniform(size=d_ref.shape).astype(np.float32)
    g32 = o32.env_shade(*_es_oracle_args(c), grads=(gd, gs), **kw)
    g64 = o64.env_shade(o64.scene(c["verts"], c["tris"]), *_es_oracle_args(c)[1:], grads=(gd, gs),
                        sampling_gbuffer=(c["pos"], c["nrm"], c["kd"], c["ks"]), **kw)
    default_mode = ops.HIT_RECORD_REPLAY
    for replay in ("rays", "bits", None):
        ops.HIT_RECORD_REPLAY = replay
        try:
            mask, ro, pos, nrm, view, kd, ks, light, pdf, rows, cols = _es_tensors(c, dev)
            for x in (pos, nrm, kd, ks, light):
                x.requires_grad_(True)
            d, s = ou.optix_env_shade(ctx, mask, ro, pos, nrm, view, kd, ks, light, pdf, rows, cols, perms=perms, **kw)
            torch.autograd.backward([d, s], [torch.tensor(gd, device=dev), torch.tensor(gs, device=dev)])
        finally:
            ops.HIT_RECORD_REPLAY = default_mode
        for name, x, r32, r64 in zip(("pos", "nrm", "kd", "ks", "light"), (pos, nrm, kd, ks, light), g32, g64):
            got = x.grad.cpu().numpy() if x.grad is not None else np.zeros_like(r32)
            assert np.array_equal(np.isnan(got), np.isnan(r32)), (replay, name)
            got, r32, r64 = np.nan_to_num(got), np.nan_to_num(r32), np.nan_to_num(r64)
            if np.abs(r64).max() == 0:
                assert np.abs(got).max() == 0, (replay, name)
                continue
            floor = rel_l2(r32, r64)
            assert rel_l2(got, r64) < max(1e-4, 2.0 * floor), (replay, name, rel_l2(got, r64), floor)


# ---------------------------------------------------------------------------------------------------------------------------------------
# bilateral denoiser
# ---------------------------------------------------------------------------------------------------------------------------------------
def _dn_check_oracle(col, colB, nrm, zdz, gA, gB, sigma, outs):
    o = oracle()
    for k, (got, want) in enumerate(zip(outs, (o.bilateral_fwd(col, nrm, zdz, sigma), o.bilateral_fwd(colB, nrm, zdz, sigma),
                                               o.bilateral_bwd(nrm, zdz, sigma, gA), o.bilateral_bwd(nrm, zdz, sigma, gB)))):
        assert np.isfinite(got).all(), k
        assert rel_l2(got, want) < 1e-4, (k, rel_l2(got, want))


@pytest.mark.parametrize("sigma", [0.6, 2.0, 3.0])
def test_denoiser_degenerate_guides(dev, sigma):
    """sigma 3.0 gives r = 17: the forward still fits the TMA kernel's tensor-map box, the backward (four-channel upstream gradients,
    72 x 4 > 256 elements) falls back to the plain kernel even for contiguous operands."""
    assert _radius(3.0) == 17
    B, H, W = 2, 45, 72
    nrm, zdz = _degenerate_guides(B, H, W, seed=int(sigma * 10))
    rng = np.random.default_rng(3)
    col, colB = [rng.uniform(0, 2, size=(B, H, W, 3)).astype(np.float32) for _ in range(2)]
    gA, gB = [rng.uniform(0, 1, size=(B, H, W, 4)).astype(np.float32) for _ in range(2)]
    outs = _dn_both_paths(col, colB, nrm, zdz, gA, gB, sigma, dev)
    _dn_check_oracle(col, colB, nrm, zdz, gA, gB, sigma, outs)
    assert (outs[0][0, H // 2, W // 3, :3] == 0).all() and outs[0][0, H // 2, W // 3, 3] == np.float32(1e-4)    # zero normal: no tap has weight


@pytest.mark.parametrize("sigma,r", [(2.4, 15), (3.2, 19)])
def test_denoiser_radius_is_computed_in_double(dev, sigma, r):
    """fl32(2.4) * 2.5 = 6.0000002 and fl32(3.2) * 2.5 = 8.0000001 in double: the reference filters over 2 ceil(.) + 1 = 15 and 19 pixels
    in each direction, one ring more than the fp32 products 6 and 8 would give.  With flat guides and a signal that is zero except at one
    pixel, the centre output is > 0 when that pixel lies on ring r and exactly 0 when it lies on ring r + 1, forward and transposed, on
    both kernels."""
    assert _radius(sigma) == r
    B, H, W = 1, 48, 48
    cy, cx = 24, 24
    nrm = np.zeros((B, H, W, 3), np.float32); nrm[..., 2] = 1.0
    zdz = np.stack([np.ones((B, H, W)), np.full((B, H, W), 0.01)], -1).astype(np.float32)
    for (dy, dx), inside in (((0, r), True), ((-r, -r), True), ((r, 3), True), ((0, r + 1), False), ((-(r + 1), -(r + 1)), False),
                             ((5, -(r + 1)), False)):
        col = np.zeros((B, H, W, 3), np.float32); col[0, cy + dy, cx + dx] = 1.0
        g4 = np.zeros((B, H, W, 4), np.float32); g4[0, cy + dy, cx + dx] = 1.0
        fa, _, ga, _ = _dn_both_paths(col, col, nrm, zdz, g4, g4, sigma, dev)
        for what, v in (("forward", fa[0, cy, cx, :3]), ("transposed", ga[0, cy, cx])):
            if inside:
                assert (v > 0).all(), (what, dy, dx, v)
            else:
                assert (v == 0).all(), (what, dy, dx, v)


def test_denoiser_large_sigma(dev):
    """sigma 4.5 (r = 25): the two-signal plain kernel needs (5 + 6) x 82 x 66 floats = 238 128 bytes of shared memory and the TMA box
    would be 88 x 3 > 256 elements wide, so bilateral_denoiser2 raises; the single-signal filter (173 KB) runs and matches the oracle."""
    import nvdiffrecmc_b200.optixutils as ou
    assert _radius(4.5) == 25
    B, H, W = 1, 40, 64
    nrm, zdz = _degenerate_guides(B, H, W, seed=45)
    col = np.random.default_rng(4).uniform(0, 2, size=(B, H, W, 3)).astype(np.float32)
    t = lambda a: torch.tensor(a, device=dev)
    c = t(col).requires_grad_(True)
    out = ou.bilateral_denoiser(c, t(nrm), t(zdz), 4.5)
    o = oracle()
    raw = o.bilateral_fwd(col, nrm, zdz, 4.5)
    assert rel_l2(out.detach().cpu().numpy(), raw[..., :3] / raw[..., 3:]) < 1e-4
    g = np.random.default_rng(5).uniform(size=out.shape).astype(np.float32)
    out.backward(t(g))
    og = np.concatenate([g / raw[..., 3:], np.zeros_like(raw[..., 3:])], -1)
    assert rel_l2(c.grad.cpu().numpy(), o.bilateral_bwd(nrm, zdz, 4.5, og)) < 1e-4
    with pytest.raises(RuntimeError, match=r"bilateral: sigma 4\.500 needs a 238128-byte tile \(> 227 KB shared memory\)"):
        ou.bilateral_denoiser2(t(col), t(col), t(nrm), t(zdz), 4.5)


# ---------------------------------------------------------------------------------------------------------------------------------------
# image loss at the training shape
# ---------------------------------------------------------------------------------------------------------------------------------------
def _tonemap64(x):
    """loss.cu:28-46 log-sRGB in double, on the fp32 values the kernels read."""
    s = np.log(np.asarray(x, np.float64) + 1.0)
    return np.where(s > 0.0031308, np.power(np.maximum(s, 0.0031308), 1.0 / 2.4) * 1.055 - 0.055, 12.92 * np.maximum(s, 0.0))


def _l1_grad_close(got, want, ties, what):
    """The L1 gradient is sign(tm(img) - tm(target)) x tm'(.): where the two tone-mapped values are within a few fp32 ulps of each other
    (ties), the sign is not determined by fp32 arithmetic -- CUDA's and the host libm's powf / logf differ in the last bit, and the fp32
    oracle itself is then 6e-5 from the fp64 one on this image.  Everywhere else the 1e-5 bar; at the ties the magnitude."""
    got = np.asarray(got, np.float64); want = np.asarray(want, np.float64)
    assert ties.mean() < 1e-5, (what, int(ties.sum()))
    assert rel_l2(np.where(ties, 0.0, got), np.where(ties, 0.0, want)) < 1e-5, (what, rel_l2(np.where(ties, 0.0, got), np.where(ties, 0.0, want)))
    g, w = got[ties], want[ties]
    assert ((g == 0) | (w == 0) | (np.abs(np.abs(g) - np.abs(w)) <= 1e-5 * np.abs(w))).all(), (what, g, w)


@pytest.mark.parametrize("target_batch", [8, 1])
def test_image_loss_at_the_training_shape(dev, target_batch):
    """8 x 512^2 with the bench's loss ('l1' after 'log_srgb'): thousands of per-block partials instead of the handful of the small
    tests, and a target broadcast over the batch ([1,H,W,3], its gradient summed over the views).  Forward within 1e-5 of the oracle
    and bit-deterministic across calls; gradients within 1e-5 wherever fp32 determines the sign of the L1 term (_l1_grad_close)."""
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.renderutils.ops import _image_loss_func
    B, H, W = 8, 512, 512
    g = torch.Generator().manual_seed(8)
    img = (torch.rand(B, H, W, 3, generator=g) * 4).to(dev); tgt = (torch.rand(target_batch, H, W, 3, generator=g) * 4).to(dev)
    img[0, 0, 0] = -0.5; img[3, 100, 7] = 70000.0; tgt[0, 1, 0] = 0.0
    img.requires_grad_(True); tgt.requires_grad_(True)
    v = ru.image_loss(img, tgt, loss="l1", tonemapper="log_srgb")
    v.backward()
    ni, nt = img.detach().cpu().numpy(), tgt.detach().cpu().numpy()
    o = oracle()
    ref = o.image_loss(ni, nt, "l1", "log_srgb")
    assert abs(float(v.detach()) / ref - 1) < 1e-5, (float(v.detach()), ref)
    gi, gt = o.image_loss_bwd(ni, nt, "l1", "log_srgb")
    a, b = _tonemap64(ni), _tonemap64(nt)
    ties = np.abs(a - b) <= 4 * 2.0 ** -23 * np.maximum(np.abs(a), np.abs(b))        # [8,H,W,3]
    _l1_grad_close(img.grad.cpu().numpy(), gi, ties, "image gradient")
    if target_batch == 1:
        gt = gt.sum(axis=0, keepdims=True, dtype=np.float64)
        tt = ties.any(axis=0, keepdims=True)                                            # summed over the views: leave out every tie
        assert rel_l2(np.where(tt, 0.0, tgt.grad.cpu().numpy()), np.where(tt, 0.0, gt)) < 1e-5
    else:
        _l1_grad_close(tgt.grad.cpu().numpy(), gt, ties, "target gradient")
    with torch.no_grad():
        parts = [_image_loss_func.apply(img, tgt, "l1", "log_srgb") for _ in range(2)]
        assert parts[0].numel() >= 1024 and torch.equal(parts[0], parts[1])
        assert float(ru.image_loss(img, tgt, loss="l1", tonemapper="log_srgb")) == float(v.detach())
