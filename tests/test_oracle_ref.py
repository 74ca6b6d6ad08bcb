"""CPU: the oracle against the REFERENCE ITSELF -- the unmodified raygen program of render/optixutils/c_src/envsampling/kernel.cu
(with bsdf.h, math_utils.h, common.h, accessor.h, params.h) compiled for the host by oracle/ref_shim and run here (oracle/_ref).
The shadow-ray hit/miss decision is the one thing that source delegates to the closed OptiX runtime; it is supplied by the oracle's
visibility predicate, everything else (RNG, strata, CDF sampling, lat-long mapping, MIS, BSDF forward and hand-derived adjoints,
gradient scatter) is the reference's own code.  Skipped where neither /root/reference nor a prebuilt oracle/_ref library exists."""
import numpy as np
import pytest

from common import RU_OPS as _RU_OPS, env_shade_edge_case, make_case, oracle, rel_l2, ru_edge_inputs


@pytest.fixture(scope="module")
def ref():
    from oracle import Reference
    try:
        return Reference(oracle())
    except RuntimeError as e:
        pytest.skip(str(e))


def _args(c, kd=None):
    return (c["scene"], c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"] if kd is None else kd, c["ks"], c["light"], c["pdf"], c["rows"],
            c["cols"], c["perms"])


@pytest.mark.parametrize("bsdf", ["pbr", "diffuse", "white"])
@pytest.mark.parametrize("N,light,lhw,shadow", [(4, "random", (32, 64), 1.0), (3, "hdr", (64, 128), 0.5), (8, "random", (16, 16), 1.0)])
def test_forward_matches_the_compiled_reference(ref, bsdf, N, light, lhw, shadow):
    c = make_case(res=20, B=2, N=N, light=light, light_hw=lhw, seed=N)
    kd = np.ones_like(c["kd"]) if bsdf == "white" else None
    kw = dict(BSDF=bsdf, n_samples_x=N, rnd_seed=11, shadow_scale=shadow)
    d_r, s_r = ref.env_shade(*_args(c, kd), **kw)
    d_o, s_o = oracle().env_shade(*_args(c, kd), **kw)
    # host libm vs the oracle's fixed transcendental kernels may move a few rays per million to a neighbouring texel: 1e-4 bar, typically 1e-7
    assert rel_l2(d_o, d_r) < 1e-4 and np.abs(d_o - d_r).max() < 1e-3 * max(np.abs(d_r).max(), 1e-6)
    if bsdf == "pbr":
        assert rel_l2(s_o, s_r) < 1e-4
    else:
        assert np.abs(s_r).max() == 0 and np.abs(s_o).max() == 0
    m = c["mask"] <= 0
    assert (d_r[m] == 0).all() and (d_o[m] == 0).all()


@pytest.mark.parametrize("bsdf", ["pbr", "diffuse"])
def test_backward_matches_the_compiled_reference_within_fp32_noise(ref, bsdf):
    """The hand-derived GGX adjoints are ill-conditioned in fp32 (DESIGN.md section 2): reference and oracle are both ~2-4e-4 away from the
    fp64 evaluation of the same samples, so they are compared with each other relative to that noise floor."""
    N = 4
    c = make_case(res=20, B=2, N=N, seed=2)
    g = np.random.default_rng(0)
    gd = g.uniform(size=c["pos"].shape).astype(np.float32); gs = g.uniform(size=c["pos"].shape).astype(np.float32)
    kw = dict(BSDF=bsdf, n_samples_x=N, rnd_seed=11)
    g_r = ref.env_shade(*_args(c), grads=(gd, gs), **kw)
    g_o = oracle().env_shade(*_args(c), grads=(gd, gs), **kw)
    o64 = oracle(f64=True)
    g64 = o64.env_shade(o64.scene(c["verts"], c["tris"]), *_args(c)[1:], grads=(gd, gs), sampling_gbuffer=(c["pos"], c["nrm"], c["kd"], c["ks"]), **kw)
    for name, a, b, r in zip(("pos", "nrm", "kd", "ks", "light"), g_o, g_r, g64):
        if np.abs(b).max() == 0:
            assert np.abs(a).max() == 0, name                    # 'diffuse': no kd / ks / pos gradient in either
            continue
        floor = max(rel_l2(b, r), rel_l2(a, r))                  # fp32 noise of this quantity on this input
        assert rel_l2(a, b) < 2.0 * floor + 1e-5, (name, rel_l2(a, b), floor)
        assert rel_l2(a, r) < 1e-3 and rel_l2(b, r) < 1e-3, name


def test_visibility_modes_and_determinism(ref):
    c = make_case(res=16, B=1, N=4, seed=1)
    a = ref.env_shade(*_args(c), n_samples_x=4, rnd_seed=3, vis_mode="brute")
    b = ref.env_shade(*_args(c), n_samples_x=4, rnd_seed=3, vis_mode="bvh")
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])           # canonical LBVH == brute force, also through the reference
    d = ref.env_shade(*_args(c), n_samples_x=4, rnd_seed=4)
    assert not np.array_equal(a[0], d[0])


@pytest.mark.parametrize("sigma", [1e-4, 0.7, 2.0, 2.4, 3.2, 4.4])
def test_denoiser_matches_the_compiled_reference_kernels(ref, sigma):
    """bilateral_denoiser_fwd_kernel / _bwd_kernel of denoising.cu, unmodified, on the host: the oracle restatement is bit-identical.
    At sigma 2.4, 3.2 and 4.4 the radius 2 ceil(2.5 sigma) + 1, whose product denoising.cu rounds in double, is one ring wider than an
    fp32 product gives (fl32(2.4) * 2.5 = 6.0000002): with flat guides the taps of that ring carry weight, and the outputs move."""
    g = np.random.default_rng(1)
    if sigma <= 2.0:
        B, H, W = 2, 21, 17
        col = g.uniform(size=(B, H, W, 3)).astype(np.float32)
        nrm = g.normal(size=(B, H, W, 3)).astype(np.float32); nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
        nrm[0, 3, 4] = 0                                               # degenerate guide normal
        zdz = np.stack([g.uniform(1, 2, size=(B, H, W)), g.uniform(0.0, 0.02, size=(B, H, W))], -1).astype(np.float32)
        zdz[1, 5, 5, 1] = 0                                            # zero depth gradient: the FLT_EPS guard (denoising.cu:59,118)
    else:
        B, H, W = 1, 48, 48
        col = g.uniform(size=(B, H, W, 3)).astype(np.float32)
        nrm = np.zeros((B, H, W, 3), np.float32); nrm[..., 2] = 1.0
        zdz = np.stack([np.ones((B, H, W)), np.full((B, H, W), 0.01)], -1).astype(np.float32)
    o = oracle()
    assert np.array_equal(o.bilateral_fwd(col, nrm, zdz, sigma), ref.bilateral_fwd(col, nrm, zdz, sigma))
    og = g.uniform(size=(B, H, W, 4)).astype(np.float32)
    assert np.array_equal(o.bilateral_bwd(nrm, zdz, sigma, og), ref.bilateral_bwd(nrm, zdz, sigma, og))


@pytest.mark.parametrize("kernel,fwd,bwd,chans,out_c,extras,kw", _RU_OPS)
def test_renderutils_kernels_match_the_compiled_reference(ref, kernel, fwd, bwd, chans, out_c, extras, kw):
    """The CUDA kernels of render/renderutils/c_src/bsdf.cu and normal.cu themselves (unmodified, host build) on the reference tests'
    input distribution (torch.rand, tests/test_bsdf.py): where the CUDA code and the PyTorch twin differ (safe-normalize, division by
    the raw cosine), this is the flavour the oracle -- and the product -- must follow."""
    g = np.random.default_rng(len(chans) * 7 + out_c)
    ins = [g.uniform(size=(2, 9, 11, c)).astype(np.float32) for c in chans]
    o = oracle()
    a = getattr(o, fwd)(*ins, **kw)
    b = ref.renderutils(kernel + "_fwd", ins, out_c, f0=extras[0], i0=extras[1], i1=extras[2])
    assert rel_l2(a, b) < 2e-6, (kernel, rel_l2(a, b))
    dout = g.uniform(size=b.shape).astype(np.float32)
    ga = getattr(o, bwd)(*ins, dout, **kw)
    gb = ref.renderutils(kernel + "_bwd", ins, dout=dout, f0=extras[0], i0=extras[1], i1=extras[2])
    ga = ga if isinstance(ga, (list, tuple)) else [ga]
    assert len(ga) == len(gb)
    # the GGX adjoints (arm / alpha gradients of pbr_specular, pbr_bsdf) carry fp32 noise of a few 1e-4 on this input distribution
    # (tests/test_gpu_elementwise.py measures it against the fp64 oracle); everything else agrees to ~1e-6
    tol = 2e-4 if kernel in ("bsdf", "specular") else 2e-5
    for i, (x, y) in enumerate(zip(ga, gb)):
        assert rel_l2(x, y) < tol, (kernel, i, rel_l2(x, y))


def test_renderutils_broadcast_view_position(ref):
    """view_pos / light_pos arrive as [1,1,1,3] (render.py passes the camera position broadcast): tensor.h:32 nhwcIndex semantics."""
    g = np.random.default_rng(3)
    full = lambda: g.uniform(size=(2, 5, 6, 3)).astype(np.float32)
    kd, arm, pos, nrm = full(), full(), full(), full()
    view = g.uniform(size=(1, 1, 1, 3)).astype(np.float32); light = g.uniform(size=(2, 1, 1, 3)).astype(np.float32)
    a = oracle().pbr_bsdf(kd, arm, pos, nrm, view, light)
    b = ref.renderutils("bsdf_fwd", [kd, arm, pos, nrm, view, light], 3, f0=0.08, i0=0)
    assert rel_l2(a, b) < 2e-6


@pytest.mark.parametrize("loss", ["l1", "mse", "relmse", "smape", "n2n"])
@pytest.mark.parametrize("tm", ["none", "log_srgb"])
def test_image_loss_matches_the_compiled_reference(ref, loss, tm):
    """imgLossFwdKernel / imgLossBwdKernel of loss.cu, unmodified ('n2n' selected by its enum: the reference's string mapping never
    reaches it, torch_bindings.cpp:727-737).  Bit-identical per-pixel losses and gradients, clamp / zero-gradient edges included."""
    g = np.random.default_rng(5)
    img = (g.uniform(size=(2, 9, 7, 3)) * 4).astype(np.float32); tgt = (g.uniform(size=(2, 9, 7, 3)) * 4).astype(np.float32)
    img[0, 0, 0] = -0.5; img[0, 0, 1] = 70000.0; tgt[0, 1, 0] = 0.0
    o = oracle()
    assert abs(o.image_loss(img, tgt, loss, tm) / ref.image_loss(img, tgt, loss, tm) - 1) < 1e-7
    ga, gb = o.image_loss_bwd(img, tgt, loss, tm), ref.image_loss(img, tgt, loss, tm, dout=1.0)
    assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])


@pytest.mark.parametrize("is_points", [True, False])
@pytest.mark.parametrize("bp", [1, 3])
def test_xfm_matches_the_compiled_reference(ref, is_points, bp):
    g = np.random.default_rng(6)
    pts = g.uniform(size=(bp, 37, 3)).astype(np.float32); mtx = g.uniform(size=(3, 4, 4)).astype(np.float32)
    o = oracle()
    a, b = o.xfm(pts, mtx, is_points), ref.xfm(pts, mtx, is_points)
    assert np.array_equal(a, b)
    d = g.uniform(size=b.shape).astype(np.float32)
    assert np.array_equal(o.xfm_bwd(mtx, d, is_points), ref.xfm(pts, mtx, is_points, dout=d))


@pytest.mark.parametrize("kernel,fwd,bwd,chans,out_c,extras,kw", _RU_OPS)
def test_renderutils_edge_inputs_match_the_compiled_reference(ref, kernel, fwd, bwd, chans, out_c, extras, kw):
    """Inputs the reference tests never draw: zero vectors (safe-normalise guard), back-facing / grazing configurations (the cosine
    gates of bsdf.cu:146-160, 236), roughness at both ends of its clamp range, negative and > 1 values.  Forward values and gradients of
    the oracle must follow the compiled CUDA source through every branch; NaNs must appear in the same places."""
    ins, dout = ru_edge_inputs(chans, out_c)
    o = oracle()
    a = getattr(o, fwd)(*ins, **kw)
    b = ref.renderutils(kernel + "_fwd", ins, out_c, f0=extras[0], i0=extras[1], i1=extras[2])
    assert np.array_equal(np.isnan(a), np.isnan(b)), kernel
    ok = ~np.isnan(b)
    scale = max(float(np.abs(b[ok]).max()), 1e-30) if ok.any() else 1.0
    assert np.abs(a[ok] - b[ok]).max() <= 2e-5 * scale, (kernel, np.abs(a[ok] - b[ok]).max(), scale)
    assert dout.shape == b.shape
    ga =getattr(o, bwd)(*ins, dout, **kw)
    gb = ref.renderutils(kernel + "_bwd", ins, dout=dout, f0=extras[0], i0=extras[1], i1=extras[2])
    ga = ga if isinstance(ga, (list, tuple)) else [ga]
    for i, (x, y) in enumerate(zip(ga, gb)):
        assert np.array_equal(np.isnan(x), np.isnan(y)), (kernel, i)
        ok = ~np.isnan(y) & np.isfinite(y)
        if ok.any():
            scale = max(float(np.abs(y[ok]).max()), 1e-30)
            assert np.abs(x[ok] - y[ok]).max() <= 1e-3 * scale, (kernel, i, np.abs(x[ok] - y[ok]).max(), scale)


def test_env_shade_edge_materials_and_geometry_match_the_compiled_reference(ref):
    """Pixels the synthetic scenes never contain: zero shading normal, camera behind the surface (NdotV < 0: bsdf_pdf's early-out,
    kernel.cu:376-378), roughness 0 and 1 (min-roughness clamp), pure metal, black albedo, and a probe with black rows / texels."""
    c = env_shade_edge_case()
    args = _args(c)
    kw = dict(BSDF="pbr", n_samples_x=c["N"], rnd_seed=21)
    d_r, s_r = ref.env_shade(*args, **kw)
    d_o, s_o = oracle().env_shade(*args, **kw)
    assert np.array_equal(np.isnan(d_r), np.isnan(d_o)) and np.array_equal(np.isnan(s_r), np.isnan(s_o))
    f = lambda a: np.nan_to_num(a)
    assert rel_l2(f(d_o), f(d_r)) < 1e-4 and rel_l2(f(s_o), f(s_r)) < 1e-4
    g = np.random.default_rng(0)
    gd = g.uniform(size=d_r.shape).astype(np.float32); gs = g.uniform(size=d_r.shape).astype(np.float32)
    g_r = ref.env_shade(*args, grads=(gd, gs), **kw)
    g_o = oracle().env_shade(*args, grads=(gd, gs), **kw)
    for name, a, b in zip(("pos", "nrm", "kd", "ks", "light"), g_o, g_r):
        assert np.array_equal(np.isnan(a), np.isnan(b)), name
        assert rel_l2(f(a), f(b)) < 2e-3, (name, rel_l2(f(a), f(b)))        # fp32 noise of the GGX adjoints, larger at the roughness clamp


@pytest.mark.parametrize("seed,N,light,lhw", [(2, 4, "random", (32, 64)), (3, 8, "hdr", (64, 128)), (5, 3, "random", (256, 256))])
def test_traced_rays_of_the_reference_hit_the_texels_the_oracle_records(ref, seed, N, light, lhw):
    """Per-RAY agreement, not only per-pixel sums: the OptiX stand-in logs the direction of every shadow ray the reference's raygen
    program traces (sample-slot order: light i, BSDF i, ...); mapped to env texels they must equal the oracle's per-ray texel record --
    the record the CUDA product reproduces bit-exactly (tests/test_gpu_envshade.py).  Host libm vs the oracle's fixed transcendental
    kernels could move a ray across a texel border in the last ulp: tolerated at 1e-4 of the rays, observed 0 of 208 512."""
    c = make_case(res=28, B=2, N=N, seed=seed, light=light, light_hw=lhw)
    args = (c["scene"], c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"], c["perms"])
    o = oracle()
    d_r, s_r, dirs = ref.env_shade(*args, n_samples_x=N, rnd_seed=11, ray_log=True)
    d_o, s_o, (rt, rv) = o.env_shade(*args, n_samples_x=N, rnd_seed=11, records=True)
    m = c["mask"] > 0
    assert np.isfinite(dirs[m]).all() and np.isnan(dirs[~m]).all()          # exactly 2 n^2 rays per covered pixel, none elsewhere
    assert np.abs(np.linalg.norm(dirs[m], axis=-1) - 1).max() < 1e-3
    tex = o.dirs_to_texels(dirs[m], lhw[0], lhw[1])
    want = rt.reshape(dirs.shape[:-1])[m]
    assert (tex != want).mean() <= 1e-4, int((tex != want).sum())
