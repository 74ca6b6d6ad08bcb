"""GPU: env_shade PER PIXEL -- diffuse and specular radiance and the pos / nrm / kd / ks gradients -- and its light gradient PER TEXEL
against the fp64 oracle, at the sample counts, shadow ramp and launch shapes that training runs.

The bar is check_per_element's (tests/common.py) with a reduction floor R:
    |got - r64| <= K * max(Delta, |r32 - r64|) + R + 4 * ulp32(r64),    R = n * 2^-24 * A
r64 / r32 are the fp64 / fp32 oracle.  A is the fp64 oracle's sum of the absolute values of the element's per-ray terms (abs_terms), so R
bounds what summing the same n terms in another order can change: the kernel adds a pixel's rays lane by lane and then across the warp,
and scatters the light gradient with atomics.  n is the number of terms: the pixel's rays with V != 0, or the rays with V != 0 that read
the texel, counted from the fp32 oracle's records.  Delta is the largest change of r64 when the EVALUATED operands (pos, nrm, kd, ks,
light and the upstream gradients) move by +-1 ulp while the sampling decisions keep the unperturbed G-buffer (sampling_gbuffer); view and
ro, which steer sampling and visibility, stay put.  With the sample set fixed Delta is continuous.

Records: the env texel of every ray bit for bit against the fp32 oracle, visibility wherever the product traced.  NaN and +-inf must sit
where the fp32 oracle has them.  Exempt pixels: where the fp64 oracle's records differ from the fp32 ones (its direction arithmetic
flips a texel or a visibility bit) the fp64 values belong to another sample set.  Those pixels, and the texels their differing rays read,
are held to the fp32 oracle within 1e-4 * A instead; they must be at most 1 % of the covered pixels.

Every case runs the backward in all three modes (HIT_RECORD_REPLAY "rays", "bits" and None: ray-record replay, visibility-bit replay,
re-tracing) and checks the forward of each of those launches and of the records launch.  Cases larger than a few hundred pixels are
compared on a pixel selection: the product runs the whole launch with upstream gradients zero outside the selection, the oracle runs
view by view with the mask restricted to it (every pixel depends only on its own global index), as tests/parity_check.py does."""
import numpy as np
import pytest
import torch

from common import _sample_px, _ulp32, check_per_element, env_shade_edge_case, make_case, oracle

pytestmark = pytest.mark.gpu
K = 16
U32 = 2.0 ** -24
EXEMPT_MAX = 0.01                   # exempt pixels: at most this fraction of the covered pixels of the selection
EXEMPT_REL = 1e-4                   # ... held to the fp32 oracle within EXEMPT_REL * A
TAG = "env_shade"
MODES = ("rays", "bits", None)
GRADS = ("pos", "nrm", "kd", "ks")
SHADOW_RAMP = [0.0, float(np.float32(1.0 / 1750.0)), 0.5, 1.0]     # min(iteration / 1750, 1): the first two iterations of DMTet's pass


def _np(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------------------------
# the product: one records launch and one forward + backward per backward mode, outputs at the selection
# ---------------------------------------------------------------------------------------------------------------------------------------
def _product(c, sel, dev, kw, dg, sg):
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.optixutils import ops
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(c["verts"], device=dev), torch.tensor(c["tris"], device=dev), rebuild=1)
    t = lambda k: torch.tensor(c[k], device=dev)
    a = [t(k) for k in ("mask", "ro", "pos", "nrm", "view", "kd", "ks", "light", "pdf", "rows", "cols")]
    perms = t("perms")
    sel_t = torch.tensor(sel, device=dev)
    d, s, rt, rv = ops.env_shade_records(ctx, *a, perms, **kw)
    out = dict(fwd=[_np(d[sel_t]), _np(s[sel_t])], rt=_np(rt[sel_t]), rv=_np(rv[sel_t]), grads=[])
    del rt, rv
    default = ops.HIT_RECORD_REPLAY
    for mode in MODES:
        ops.HIT_RECORD_REPLAY = mode
        try:
            leaf = [x.clone().requires_grad_(True) for x in (a[2], a[3], a[5], a[6], a[7])]        # pos, nrm, kd, ks, light
            d, s = ou.optix_env_shade(ctx, a[0], a[1], leaf[0], leaf[1], a[4], leaf[2], leaf[3], leaf[4], a[8], a[9], a[10], perms=perms, **kw)
            torch.autograd.backward([d, s], [torch.tensor(dg, device=dev), torch.tensor(sg, device=dev)])
            torch.cuda.synchronize()
        finally:
            ops.HIT_RECORD_REPLAY = default
        out["fwd"] += [_np(d[sel_t]), _np(s[sel_t])]
        out["grads"] += [_np(x.grad[sel_t]) for x in leaf[:4]] + [_np(leaf[4].grad)]
        outside = ~sel_t
        if bool(outside.any()):
            assert all(float(x.grad[outside].abs().max()) == 0 for x in leaf[:4]), "%s: gradient outside the selection" % mode
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# the oracle on the selection, with the evaluated operands given separately from the sampling ones
# ---------------------------------------------------------------------------------------------------------------------------------------
def _oracle(o, scene, c, sel, kw, ev, grads=False, records=False, abs_terms=False):
    """o.env_shade on the pixels of sel (bool [B,H,W]) of the case c.  ev: the evaluated operands -- pos, nrm, kd, ks [n_sel,3] at sel,
    light [Hl,Wl,3] and, for the backward, dg / sg [n_sel,3]; the sampling decisions use c's own pos / nrm / kd / ks.  View by view, mask
    restricted to sel, batch_offset = the view's global index.  Returns [diff, spec] or [pos, nrm, kd, ks, light] gradients (per-pixel
    outputs at sel, [n_sel,3]; the light gradient summed over the views) and, with records, (texel, vis) at sel [n_sel, 2 N^2]."""
    B = c["mask"].shape[0]
    full = {k: c[k].copy() for k in GRADS}
    for k in GRADS:
        full[k][sel] = ev[k]
    if grads:
        up = [np.zeros_like(c["pos"]) for _ in range(2)]
        up[0][sel], up[1][sel] = ev["dg"], ev["sg"]
    per_px, light_g, rec = [], None, []
    for b in range(B):
        if not sel[b].any():
            continue
        s = slice(b, b + 1)
        m = (c["mask"][s] * sel[s]).astype(np.float32)
        view = c["view"][s] if c["view"].shape[0] == B else c["view"]
        args = (scene, m, c["ro"][s], full["pos"][s], full["nrm"][s], view, full["kd"][s], full["ks"][s], ev["light"], c["pdf"], c["rows"],
                c["cols"], c["perms"])
        r = o.env_shade(*args, sampling_gbuffer=(c["pos"][s], c["nrm"][s], c["kd"][s], c["ks"][s]), batch_offset=kw["batch_offset"] + b,
                        grads=(up[0][s], up[1][s]) if grads else None, records=records, abs_terms=abs_terms, parallel_bwd=True,
                        **{k: v for k, v in kw.items() if k != "batch_offset"})
        if records:
            rec.append((r[2][0][0][sel[b]], r[2][1][0][sel[b]]))
        per_px.append([x[0][sel[b]] for x in r[:(4 if grads else 2)]])
        if grads:
            light_g = r[4] if light_g is None else light_g + r[4]
    out = [np.concatenate([p[k] for p in per_px]) for k in range(len(per_px[0]))]
    if grads:
        out.append(light_g)
    if records:
        return out, (np.concatenate([x[0] for x in rec]), np.concatenate([x[1] for x in rec]))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# one case
# ---------------------------------------------------------------------------------------------------------------------------------------
def _run(what, dev, c, sel=None, bsdf="pbr", shadow_scale=1.0, seed=11, batch_offset=0, vis_mode="brute", upstream_seed=1):
    """Product against oracle on the case c (pixels sel, default all).  Returns the worst ratio over every output."""
    B, H, W = c["mask"].shape
    if sel is None:
        sel = np.ones((B, H, W), bool)
    N = c["N"]
    S2 = 2 * N * N
    kw = dict(BSDF=bsdf, n_samples_x=N, rnd_seed=seed, shadow_scale=shadow_scale, batch_offset=batch_offset)
    okw = dict(kw, vis_mode=vis_mode)
    g = np.random.default_rng(upstream_seed)
    dg = (g.uniform(-1, 1, (B, H, W, 3)) * sel[..., None]).astype(np.float32)
    sg = (g.uniform(-1, 1, (B, H, W, 3)) * sel[..., None]).astype(np.float32)
    prod = _product(c, sel, dev, kw, dg, sg)

    o32, o64 = oracle(), oracle(f64=True)
    sc32, sc64 = c["scene"], o64.scene(c["verts"], c["tris"])
    cov = c["mask"][sel] > 0
    ncov = int(cov.sum())
    assert ncov > 0
    ev = dict(pos=c["pos"][sel], nrm=c["nrm"][sel], kd=c["kd"][sel], ks=c["ks"][sel], light=c["light"], dg=dg[sel], sg=sg[sel])
    f_keys, b_keys = ["pos", "nrm", "kd", "ks", "light"], ["pos", "nrm", "kd", "ks", "light", "dg", "sg"]

    # ---- records: product vs fp32 oracle; fp64 vs fp32 decides the exempt pixels -----------------------------------------------------
    fwd32, (rt32, rv32) = _oracle(o32, sc32, c, sel, okw, ev, records=True)
    fwd64, (rt64, rv64) = _oracle(o64, sc64, c, sel, okw, ev, records=True)
    bad = prod["rt"] != rt32
    assert not bad.any(), "%s: env texel records differ from the fp32 oracle on %d of %d rays" % (what, bad.sum(), bad.size)
    traced = (prod["rv"] != 2) & cov[:, None]
    bad = traced & (prod["rv"] != rv32)
    assert not bad.any(), "%s: visibility differs from the fp32 oracle on %d traced rays" % (what, bad.sum())
    if shadow_scale == 0.0:
        assert not traced.any(), "%s: shadow_scale = 0 traced %d rays" % (what, traced.sum())
    else:
        assert traced[cov].mean() > 0.2
    flip = (rt32 != rt64) | ((rv32 != rv64) & traced)
    ex_px = flip.any(-1) & cov
    where = np.argwhere(sel)[ex_px]
    print("[%s] %s: %d covered pixels, %d exempt %s" % (TAG, what, ncov, ex_px.sum(), [tuple(int(v) for v in p) for p in where]))
    assert ex_px.sum() <= EXEMPT_MAX * ncov, "%s: %d of %d covered pixels have fp64 records that differ from fp32 ones: %s" % (
        what, ex_px.sum(), ncov, [tuple(int(v) for v in p) for p in where])
    Hl, Wl = c["light"].shape[:2]
    texel = lambda rt: (rt >> 16) * Wl + (rt & 0xFFFF)
    ex_tex = np.zeros(Hl * Wl, bool)
    ex_tex[texel(rt32[flip & cov[:, None]])] = True
    ex_tex[texel(rt64[flip & cov[:, None]])] = True
    ex_tex = np.broadcast_to(ex_tex.reshape(Hl, Wl, 1), (Hl, Wl, 3))
    ex_pxc = np.broadcast_to(ex_px[:, None], (ex_px.size, 3))

    # ---- term counts and reduction floors ------------------------------------------------------------------------------------------
    live = (rt32 >= 0) & cov[:, None] & ((rv32 == 1) | (shadow_scale != 1.0))          # rays with V != 0
    n_px = live.sum(-1).astype(np.float64)[:, None]
    n_tex = np.bincount(texel(rt32[live]), minlength=Hl * Wl).astype(np.float64).reshape(Hl, Wl, 1)
    a_fwd = _oracle(o64, sc64, c, sel, okw, ev, abs_terms=True)
    a_bwd = _oracle(o64, sc64, c, sel, okw, ev, grads=True, abs_terms=True)

    def exempt_check(name, got, r32, a, ex):
        got, r32, a = [np.asarray(x, np.float64)[ex] for x in (got, r32, a)]
        ok = np.isfinite(r32)
        err = np.abs(got - r32)[ok]
        lim = (EXEMPT_REL * a + 4 * _ulp32(r32))[ok]
        assert (err <= lim).all(), "%s: %s: exempt elements beyond %g x A of the fp32 oracle (worst %.3g x A)" % (
            what, name, EXEMPT_REL, (err / np.maximum(a[ok], 1e-30)).max())

    # ---- forward: the records launch and the forward launch of every backward mode ---------------------------------------------------
    nf = len(prod["fwd"]) // 2
    ins = [ev[k] for k in f_keys]
    f64 = lambda x: fwd64 * nf if x is ins else _oracle(o64, sc64, c, sel, okw, dict(ev, **dict(zip(f_keys, x)))) * nf
    names = ["%s (%s)" % (n, l) for l in ("records launch",) + tuple("mode %s" % m for m in MODES) for n in ("diff", "spec")]
    w = check_per_element(what + " forward", prod["fwd"], f64, lambda x: fwd32 * nf, ins, K, names, exempt=[ex_pxc] * (2 * nf),
                          floor=[n_px * U32 * a for a in a_fwd] * nf, tag=TAG)
    for k in range(2 * nf):
        exempt_check(names[k], prod["fwd"][k], fwd32[k % 2], a_fwd[k % 2], ex_pxc)

    # ---- backward in all three modes --------------------------------------------------------------------------------------------------
    ins = [ev[k] for k in b_keys]
    bwd32 = _oracle(o32, sc32, c, sel, okw, ev, grads=True)
    f64 = lambda x: _oracle(o64, sc64, c, sel, okw, dict(ev, **dict(zip(b_keys, x))), grads=True) * len(MODES)
    names = ["d_%s (mode %s)" % (n, m) for m in MODES for n in f_keys]
    floors = [n_px * U32 * a for a in a_bwd[:4]] + [n_tex * U32 * a_bwd[4]]
    exempt = [ex_pxc] * 4 + [ex_tex]
    w2 = check_per_element(what + " backward", prod["grads"], f64, lambda x: bwd32 * len(MODES), ins, K, names,
                           exempt=exempt * len(MODES), floor=floors * len(MODES), tag=TAG)
    for k, got in enumerate(prod["grads"]):
        exempt_check(names[k], got, bwd32[k % 5], a_bwd[k % 5], exempt[k % 5])
    return max(w, w2)


# ---------------------------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shadow_scale", SHADOW_RAMP, ids=["ss0", "ss1over1750", "ss0.5", "ss1"])
@pytest.mark.parametrize("bsdf", ["pbr", "diffuse", "white"])
def test_bsdfs_along_the_shadow_ramp(dev, bsdf, shadow_scale):
    """24^2 x 2 views, N = 4, every pixel.  shadow_scale 0 is DMTet's first iteration: nothing is traced, every ray has V = 1 and
    records 2; fp32(1/1750) its second, where an occluded ray keeps V = 1 - 1/1750.  K = 16; worst ratio on an H100 80GB HBM3 (700 W
    limit): radiance 1.0, per-pixel gradients 1.04, light gradient 1.81."""
    c = make_case(res=24, B=2, N=4, seed=4)
    if bsdf == "white":
        c["kd"] = np.ones_like(c["kd"])        # render.py:107
    _run("%s ss=%g" % (bsdf, shadow_scale), dev, c, bsdf=bsdf, shadow_scale=shadow_scale)


def _window(B, H, W, y0, x0, h, w, b=0):
    sel = np.zeros((B, H, W), bool)
    sel[b, y0:y0 + h, x0:x0 + w] = True
    return sel


@pytest.mark.parametrize("N", [1, 5, 8, 9, 12, 32])
def test_sample_counts(dev, N):
    """2 N^2 sample slots per pixel: N = 1 one sample pair; 5 (50 slots) crosses a 32-bit hit word; 8 fills the 128-slot queue once;
    9, 12 and 32 take 2, 3 and 16 fills (the last one partial for 9 and 12), and at 32 the replay kernel walks records of up to 2 048
    rays 32 at a time.  24^2 x 2, every pixel for N <= 8; a covered 10 x 10 crop of view 0 for 9, 12 and 32 (BVH visibility at 32).
    K = 16; worst ratio on an H100: radiance 1.1, per-pixel gradients 3.5 (N = 1), light gradient 1.91."""
    c = make_case(res=24, B=2, N=N, seed=5)
    sel = None
    if N >= 9:
        sel = _window(2, 24, 24, 8, 8, 10, 10)
        assert (c["mask"][sel] > 0).mean() > 0.8
    _run("N=%d" % N, dev, c, sel=sel, seed=13, vis_mode="bvh" if N == 32 else "brute")


@pytest.mark.parametrize("shadow_scale", [1.0, 0.0])
@pytest.mark.parametrize("bsdf", ["pbr", "diffuse", "white"])
def test_edge_inputs(dev, bsdf, shadow_scale):
    """env_shade_edge_case(): zero and flipped shading normals, roughness 0 / 1, pure metal, black albedo, a probe with a black row and
    black texels.  Every pixel.  K = 16; worst ratio on an H100: radiance 1.0, per-pixel gradients
    1.03, light gradient 1.5."""
    c = env_shade_edge_case()
    if bsdf == "white":
        c["kd"] = np.ones_like(c["kd"])
    _run("edge %s ss=%g" % (bsdf, shadow_scale), dev, c, bsdf=bsdf, shadow_scale=shadow_scale, seed=21)


def test_persistent_grid_tails(dev):
    """3 views of 97 x 131 (38 121 pixels: the last 32-pixel chunk holds 9), so chunks straddle rows and views; N = 8, batch_offset = 2.
    Selection: the last two chunks, the chunks across both view boundaries, row 0 and the last row of every view, and 1 500 random
    pixels.  K = 16; worst ratio on an H100: radiance 0.93, per-pixel gradients 0.99, light gradient 1.41."""
    c = make_case(res=131, B=3, N=8, seed=6)
    for k in ("mask", "ro", "pos", "nrm", "kd", "ks"):
        c[k] = np.ascontiguousarray(c[k][:, 17:17 + 97])
    B, H, W = c["mask"].shape
    n = B * H * W
    assert n % 32 == 9
    idx = [np.arange(n - 9 - 32, n)]
    for b in (1, 2):
        idx.append(np.arange(b * H * W - 40, b * H * W + 40))
    for b in range(B):
        idx += [(b * H) * W + np.arange(W), (b * H + H - 1) * W + np.arange(W)]
    idx.append(np.random.default_rng(3).integers(0, n, 1500))
    sel = np.zeros(n, bool)
    sel[np.concatenate(idx)] = True
    _run("tails 3x97x131", dev, c, sel=sel.reshape(B, H, W), seed=17, batch_offset=2, vis_mode="bvh")


def test_bench_launch(dev):
    """The bench's launch: 8 views x 512^2 of its mesh (G-buffer as bench.py builds it), N = 8, its probe resolution.  The product runs
    the whole launch; the oracle the selection: the first and last pixel, the last 32-pixel chunk, rows 0, 1 and H - 1 of the first and
    last view and 2 000 random pixels.  K = 16; worst ratio on an H100: radiance 0.99, per-pixel gradients
    1.0, light gradient 2.1."""
    import nvdiffrecmc_b200.optixutils as ou
    from bench import WORKLOAD as wl, build_scene_numpy, view_pose
    from nvdiffrecmc_b200 import synth
    o = oracle()
    v, f, vn = build_scene_numpy(wl, 0)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=1)
    r, B, N = wl["res"], wl["views_per_gpu"], wl["n_samples_x"]
    gbs = []
    for gi in range(B):
        ang, tilt = view_pose(gi)
        campos, ro, rd = synth.primary_rays(synth.orbit_view(ang, tilt=tilt), r)
        tid, tuv = ou.trace_closest(ctx, torch.tensor(ro.reshape(-1, 3), device=dev), torch.tensor(rd.reshape(-1, 3), device=dev))
        gbs.append(synth.assemble_gbuffer(v, f, vn, _np(tid).reshape(r, r), _np(tuv).reshape(r, r, 3), campos, seed=100 + gi))
    del ctx
    st = lambda k: np.ascontiguousarray(np.stack([g[k] for g in gbs]), np.float32)
    view = st("view_pos").reshape(B, 1, 1, 3)
    pos, mask = st("pos"), st("mask")
    nrm = o.prepare_shading_normal(pos, view, None, st("smooth_nrm"), st("tangent"), st("geom_nrm"), two_sided_shading=True, opengl=True)
    nrm = (nrm * (mask[..., None] > 0)).astype(np.float32)
    light = synth.random_light(wl["light_res"], seed=2)
    pdf, rows, cols = o.update_pdf(light)
    c = dict(verts=v, tris=f, scene=o.scene(v, f), mask=mask, ro=(pos + nrm * np.float32(0.001)).astype(np.float32), pos=pos, nrm=nrm,
             view=view, kd=st("kd"), ks=st("ks"), light=light, pdf=pdf, rows=rows, cols=cols, perms=synth.make_perms(N, seed=3), N=N)
    sel = np.zeros(B * r * r, bool)
    sel[_sample_px(B, r, r, n_rand=2000, seed=5, group=32)] = True
    sel[[0, B * r * r - 1]] = True
    _run("bench 8x512^2", dev, c, sel=sel.reshape(B, r, r), seed=12345, vis_mode="bvh")
