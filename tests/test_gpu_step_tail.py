"""GPU: the per-pixel ops around env_shade in every training step -- prepare_shading_normal, pbr_bsdf / pbr_specular, shade_combine (the
second launch of denoise_and_combine), image_loss -- and xfm_points / xfm_vectors, PER ELEMENT against the fp64 oracle, at the bench's
shapes and operand layouts (vector loads next to strided and broadcast scalar loads in one launch, ragged 4-pixel groups that straddle a
view, channel slices, transposed matrices, stride-0 upstream gradients).

The bar (check_per_element): with r64 the fp64 oracle, r32 the fp32 oracle and Delta the largest change of r64 over N_PERT seeded
perturbations of every input element by +-1 fp32 ulp (a per-element sensitivity estimate), every finite element must satisfy
    |got - r64| <= K * max(Delta, |r32 - r64|) + 4 * ulp32(r64)
and NaN / +-inf must sit where the fp32 oracle has them.  These ops use contracted fast math and device powf / logf, so they are not
bit-exact; K is calibrated per op on an H100 and each test's docstring gives the worst ratio (|got - r64| - 4 ulp) / max(Delta, |r32 - r64|)
observed there.  8 x 512^2 cases are compared on a sample (_sample_px): every pixel of rows 0, 1 and H-1 of the first and last view,
20 000 random pixels and the last 4-pixel group, gathered into [1,1,K,C] for the oracle."""
import types

import numpy as np
import pytest
import torch

from common import _sample_px, _take, check_per_element, oracle, same_bits
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------------------------
# prepare_shading_normal at the bench's layout
# ---------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_gbuffer(dev):
    """The bench's G-buffer: 8 views x 512^2 of its mesh, primary rays traced on the device as bench.py does, synth.assemble_gbuffer."""
    import nvdiffrecmc_b200.optixutils as ou
    from bench import WORKLOAD as wl, build_scene_numpy, view_pose
    v, f, vn = build_scene_numpy(wl, 0)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=1)
    r, B = wl["res"], wl["views_per_gpu"]
    gbs = []
    for gi in range(B):
        ang, tilt = view_pose(gi)
        campos, ro, rd = synth.primary_rays(synth.orbit_view(ang, tilt=tilt), r)
        tid, tuv = ou.trace_closest(ctx, torch.tensor(ro.reshape(-1, 3), device=dev), torch.tensor(rd.reshape(-1, 3), device=dev))
        gbs.append(synth.assemble_gbuffer(v, f, vn, _np(tid).reshape(r, r), _np(tuv).reshape(r, r, 3), campos, seed=100 + gi))
    del ctx
    st = lambda k: np.ascontiguousarray(np.stack([g[k] for g in gbs]), np.float32)
    return dict(pos=st("pos"), view=st("view_pos").reshape(B, 1, 1, 3), smooth_nrm=st("smooth_nrm"), tangent=st("tangent"),
                geom_nrm=st("geom_nrm"))


PSN_NAMES = ["pos", "view_pos", "perturbed_nrm", "smooth_nrm", "smooth_tng", "geom_nrm"]


def _psn_device(ins_t, dout_t, two_sided, opengl):
    """Forward through the public op (perturbed_nrm=None: the [1,1,1,3] default) and the six full-grid gradients of its backward launch
    (before a broadcast operand's gradient is summed)."""
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.renderutils.ops import _call, _default_perturbed_nrm
    pos, view, sn, st, gn = ins_t
    out = ru.prepare_shading_normal(pos, view, None, sn, st, gn, two_sided_shading=two_sided, opengl=opengl)
    grads = _call("prepare_shading_normal_bwd", [pos, view, _default_perturbed_nrm(pos.device), sn, st, gn], (int(two_sided), int(opengl)),
                  (3,) * 6, dout=dout_t)
    torch.cuda.synchronize()
    return out, grads


def _psn_check(what, ins_np, dout_np, out, grads, two_sided, opengl, idx, K):
    pn = np.array([0.0, 0.0, 1.0], np.float32).reshape(1, 1, 1, 3)
    grid = out.shape[:3]
    ins = [_take(x, grid, idx) for x in (ins_np[0], ins_np[1], pn, ins_np[2], ins_np[3], ins_np[4])]
    d = _take(dout_np, grid, idx)
    kw = dict(two_sided_shading=two_sided, opengl=opengl)
    o32, o64 = oracle(), oracle(f64=True)
    got = [_take(_np(out), grid, idx)]
    w = check_per_element(what + " forward", got, lambda a: [o64.prepare_shading_normal(*a, **kw)], lambda a: [o32.prepare_shading_normal(*a, **kw)],
                          ins, K, ["out"])
    got = [_take(_np(g), grid, idx) for g in grads]
    # d_perturbed_nrm.z: with perturbed_nrm = (0, 0, 1) the shading normal's pre-normalisation vector is the unit smooth normal itself, and
    # this component of the gradient is that vector's radial part, which the normalisation's adjoint removes -- exactly 0 in exact
    # arithmetic, an fp32 cancellation residue in the kernel (up to ~1e-7 |d_out|) that neither Delta nor the fp32 oracle (which happens
    # to cancel exactly) measures.  It is held to 2K ulps of the pixel's |d_out| instead.
    radial = np.zeros(got[2].shape, bool)
    radial[..., 2] = True
    w2 = check_per_element(what + " backward", got, lambda a: list(o64.prepare_shading_normal_bwd(*a[:6], a[6], **kw)),
                           lambda a: list(o32.prepare_shading_normal_bwd(*a[:6], a[6], **kw)), ins + [d], K, ["d_" + n for n in PSN_NAMES],
                           exempt=[None, None, radial, None, None, None])
    r64 = o64.prepare_shading_normal_bwd(*ins, d, **kw)[2][..., 2]
    bound = 2 * K * 2.0 ** -23 * np.linalg.norm(d.astype(np.float64), axis=-1)
    excess = np.abs(got[2][..., 2] - r64) / np.maximum(bound, 1e-30)
    assert (excess <= 1.0).all(), "%s: d_perturbed_nrm.z beyond %d ulps of |d_out| (worst %.3g x)" % (what, 2 * K, excess.max())
    print("[step-tail] %-60s worst ratio %.3g (of %d ulps of |d_out|)" % (what + " backward: d_perturbed_nrm.z", excess.max() * 2 * K, 2 * K))
    return max(w, w2)


K_PSN = 16


@pytest.mark.parametrize("two_sided", [True, False])
@pytest.mark.parametrize("opengl", [True, False])
def test_prepare_shading_normal_at_the_bench_layout(dev, bench_gbuffer, two_sided, opengl):
    """8 x 512^2, view_pos [8,1,1,3] and the default perturbed normal [1,1,1,3] (strided scalar loads) next to contiguous G-buffer operands
    (vector loads) in one launch, as every bench step calls it; forward and all six gradients.  With two_sided and opengl, an operand whose
    data pointer is 4 bytes past 16-byte alignment (so it takes the scalar path) gives bit-identical results.
    K = 16; worst ratio on an H100 80GB HBM3 (700 W limit): forward 1.1, gradients 5.2; d_perturbed_nrm.z (see _psn_check) 11 ulps of
    |d_out| against its bound of 32."""
    gb = bench_gbuffer
    ins_np = [gb["pos"], gb["view"], gb["smooth_nrm"], gb["tangent"], gb["geom_nrm"]]
    B, H, W = gb["pos"].shape[:3]
    dout_np = np.random.default_rng(21).normal(size=(B, H, W, 3)).astype(np.float32)
    ins_t = [torch.tensor(x, device=dev) for x in ins_np]
    dout_t = torch.tensor(dout_np, device=dev)
    out, grads = _psn_device(ins_t, dout_t, two_sided, opengl)
    _psn_check("prepare_shading_normal %s/%s" % (two_sided, opengl), ins_np, dout_np, out, grads, two_sided, opengl, _sample_px(B, H, W), K_PSN)
    if two_sided and opengl:
        buf = torch.empty(ins_t[0].numel() + 1, device=dev)
        mis = buf[1:].view(ins_t[0].shape)
        mis.copy_(ins_t[0])
        assert mis.is_contiguous() and mis.data_ptr() % 16 == 4
        out2, grads2 = _psn_device([mis] + ins_t[1:], dout_t, two_sided, opengl)
        assert same_bits(_np(out2), _np(out)), "a 4-byte-offset pos changes the forward"
        for n, a, b in zip(PSN_NAMES, grads2, grads):
            assert same_bits(_np(a), _np(b)), "a 4-byte-offset pos changes d_%s" % n


@pytest.mark.parametrize("shape", [(3, 7, 5), (2, 9, 13), (3, 9, 13)], ids=["npx%4=1", "npx%4=2", "npx%4=3"])
@pytest.mark.parametrize("two_sided,opengl", [(True, True), (False, False)])
def test_prepare_shading_normal_ragged_tail_straddles_the_last_view(dev, shape, two_sided, opengl):
    """B*H*W = 1, 2, 3 (mod 4) with H*W odd, so 4-pixel groups cross view boundaries and the last group is partial; view_pos [B,1,1,3]
    changes at every view.  Every pixel.  K = 16 (the worst ratios are within those of the bench-layout test)."""
    B, H, W = shape
    g = np.random.default_rng(sum(shape) + 7 * two_sided)
    pos = g.normal(size=shape + (3,)).astype(np.float32)
    view = (g.normal(size=(B, 1, 1, 3)) * 4).astype(np.float32)
    sn, st, gn = [g.normal(size=shape + (3,)).astype(np.float32) for _ in range(3)]
    dout = g.normal(size=shape + (3,)).astype(np.float32)
    ins_np = [pos, view, sn, st, gn]
    out, grads = _psn_device([torch.tensor(x, device=dev) for x in ins_np], torch.tensor(dout, device=dev), two_sided, opengl)
    _psn_check("prepare_shading_normal %s" % (shape,), ins_np, dout, out, grads, two_sided, opengl, np.arange(B * H * W), K_PSN)


# ---------------------------------------------------------------------------------------------------------------------------------------
# pbr_bsdf / pbr_specular
# ---------------------------------------------------------------------------------------------------------------------------------------
K_BSDF = 16
BSDF_NAMES = ["kd", "arm", "pos", "nrm", "view_pos", "light_pos"]
SPEC_NAMES = ["col", "nrm", "wo", "wi", "alpha"]


def _ew_device(op, ins_t, scalars, fwd, bwd_ch, dout_t):
    from nvdiffrecmc_b200.renderutils.ops import _call
    out = fwd(*ins_t)
    grads = _call(op + "_bwd", list(ins_t), scalars, bwd_ch, dout=dout_t)
    torch.cuda.synchronize()
    return _np(out), [_np(x) for x in grads]


def _bsdf_case(dev, what, ins_np, bsdf, K):
    import nvdiffrecmc_b200.renderutils as ru
    ins_t = [x if isinstance(x, torch.Tensor) else torch.tensor(x, device=dev) for x in ins_np]
    ins_np = [_np(x) for x in ins_t]
    grid = np.broadcast_shapes(*[x.shape[:3] for x in ins_np])
    dout = np.random.default_rng(31).uniform(size=grid + (3,)).astype(np.float32)
    out, grads = _ew_device("pbr_bsdf", ins_t, (0.08, 1 if bsdf == "frostbite" else 0), lambda *a: ru.pbr_bsdf(*a, bsdf=bsdf), (3,) * 6,
                            torch.tensor(dout, device=dev))
    o32, o64 = oracle(), oracle(f64=True)
    kw = dict(min_roughness=0.08, bsdf=bsdf)
    w = check_per_element(what + " pbr_bsdf(%s) forward" % bsdf, [out], lambda a: [o64.pbr_bsdf(*a, **kw)], lambda a: [o32.pbr_bsdf(*a, **kw)],
                          ins_np, K, ["out"])
    w2 = check_per_element(what + " pbr_bsdf(%s) backward" % bsdf, grads, lambda a: list(o64.pbr_bsdf_bwd(*a[:6], a[6], **kw)),
                           lambda a: list(o32.pbr_bsdf_bwd(*a[:6], a[6], **kw)), ins_np + [dout], K, ["d_" + n for n in BSDF_NAMES])
    return max(w, w2)


def _spec_case(dev, what, ins_t, K):
    import nvdiffrecmc_b200.renderutils as ru
    ins_np = [_np(x) for x in ins_t]
    grid = np.broadcast_shapes(*[x.shape[:3] for x in ins_np])
    dout = np.random.default_rng(32).uniform(size=grid + (3,)).astype(np.float32)
    out, grads = _ew_device("pbr_specular", ins_t, (0.08,), lambda *a: ru.pbr_specular(*a), (3, 3, 3, 3, 1), torch.tensor(dout, device=dev))
    o32, o64 = oracle(), oracle(f64=True)
    w = check_per_element(what + " pbr_specular forward", [out], lambda a: [o64.pbr_specular(*a)], lambda a: [o32.pbr_specular(*a)], ins_np, K, ["out"])
    w2 = check_per_element(what + " pbr_specular backward", grads, lambda a: list(o64.pbr_specular_bwd(*a[:5], a[5])),
                           lambda a: list(o32.pbr_specular_bwd(*a[:5], a[5])), ins_np + [dout], K, ["d_" + n for n in SPEC_NAMES])
    return max(w, w2)


def _rand(shape, seed):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed)).numpy()


R = (2, 37, 29)


@pytest.mark.parametrize("bsdf", ["lambert", "frostbite"])
def test_pbr_bsdf_per_element_on_the_reference_distribution(dev, bsdf):
    """The rel-L2 test's inputs (torch.rand, un-normalised normals, random view / light positions; test_gpu_elementwise.py) held per
    element.  K = 16; worst ratio on an H100: forward 1.0, gradients 5.6."""
    _bsdf_case(dev, "R", [_rand(R + (3,), i) for i in range(6)], bsdf, K_BSDF)


def test_pbr_specular_per_element_on_the_reference_distribution(dev):
    """As above for pbr_specular.  K = 16; worst ratio on an H100: forward 1.0, gradients 6.3."""
    _spec_case(dev, "R", [torch.tensor(_rand(R + (c,), i), device=dev) for i, c in enumerate([3, 3, 3, 3, 1])], K_BSDF)


def _mixed_inputs(dev, seed):
    """4 x 128 x 96 operands of every layout the kernel distinguishes: contiguous (vector loads), channel slices of an 8-channel tensor
    (strided scalar loads), [B,1,1,3] and [1,1,1,3] (broadcast)."""
    g = np.random.default_rng(seed)
    B, H, W = 4, 128, 96
    t8 = torch.tensor(g.uniform(size=(B, H, W, 8)).astype(np.float32), device=dev)
    pos = g.uniform(size=(B, H, W, 3)).astype(np.float32)
    n = g.normal(size=(B, H, W, 3)) * 0.4 + [0.0, 0.0, 1.0]
    nrm = (n / np.linalg.norm(n, axis=-1, keepdims=True)).astype(np.float32)
    view = (np.array([0.5, 0.5, 3.0]) + g.normal(size=(B, 1, 1, 3)) * 0.5).astype(np.float32)
    light = np.array([[[[0.3, 0.2, 4.0]]]], np.float32)
    return t8, pos, nrm, view, light


@pytest.mark.parametrize("bsdf", ["lambert", "frostbite"])
def test_pbr_bsdf_per_element_with_mixed_operand_layouts(dev, bsdf):
    """kd contiguous, arm a channel slice, pos / nrm contiguous, view_pos [4,1,1,3], light_pos [1,1,1,3], in one launch.  K = 16; worst ratio on an H100:
    forward 1.0, gradients 6.2."""
    t8, pos, nrm, view, light = _mixed_inputs(dev, 41)
    kd = torch.tensor(_rand((4, 128, 96, 3), 42), device=dev)
    arm = t8[..., 2:5]
    assert not arm.is_contiguous()
    _bsdf_case(dev, "mixed", [kd, arm, torch.tensor(pos, device=dev), torch.tensor(nrm, device=dev), torch.tensor(view, device=dev),
                              torch.tensor(light, device=dev)], bsdf, K_BSDF)


def test_pbr_specular_per_element_with_mixed_operand_layouts(dev):
    """col contiguous, nrm a channel slice, wo [4,1,1,3], wi contiguous, alpha a one-channel slice.  K = 16; worst ratio on an H100: forward 1.0,
    gradients 6.2."""
    t8, pos, nrm, view, light = _mixed_inputs(dev, 43)
    t8[..., 0:3] = torch.tensor(nrm, device=dev)
    wo = view / np.linalg.norm(view, axis=-1, keepdims=True)
    wi = np.broadcast_to(light / np.linalg.norm(light), pos.shape) + (pos - 0.5) * 0.2
    col = torch.tensor(_rand((4, 128, 96, 3), 44), device=dev)
    _spec_case(dev, "mixed", [col, t8[..., 0:3], torch.tensor(wo.astype(np.float32), device=dev), torch.tensor(wi.astype(np.float32), device=dev),
                              t8[..., 7:8]], K_BSDF)


# ---------------------------------------------------------------------------------------------------------------------------------------
# shade_combine (denoise_and_combine's second launch)
# ---------------------------------------------------------------------------------------------------------------------------------------
K_COMBINE = 16


def _combine_inputs(shape, seed):
    """a4 / b4: rgb weighted sums with weights log-uniform from the denoiser's 1e-4 floor to 1e4 (every 97th exactly at the floor);
    kd / ks: channel slices 0:3 and 4:7 of one 8-channel tensor, ks.z exactly 0 or 1 on about half the pixels."""
    g = np.random.default_rng(seed)

    def raw():
        w = np.exp(g.uniform(np.log(1e-4), np.log(1e4), shape)).astype(np.float32)
        w.reshape(-1)[::97] = np.float32(1e-4)
        a = np.empty(shape + (4,), np.float32)
        a[..., 3] = w
        a[..., :3] = g.uniform(0.0, 2.0, shape + (3,)) * w[..., None]
        return a
    a4, b4 = raw(), raw()
    t8 = g.uniform(0.0, 1.0, shape + (8,)).astype(np.float32)
    sel = g.random(shape)
    t8[..., 6][sel < 0.25] = 0.0
    t8[..., 6][sel > 0.75] = 1.0
    dout = g.normal(size=shape + (3,)).astype(np.float32)
    return a4, b4, t8, dout


@pytest.mark.parametrize("bsdf", ["pbr", "diffuse"])
def test_shade_combine_per_element_at_the_bench_shape(dev, bsdf):
    """8 x 512^2: forward and every gradient of shade_combine against orc_shade_combine (render.py:119-127 in the reference's order); the
    kernel computes A * (1/w) * kd * (1 - ks.z) + B * (1/w_B) with contraction.  kd / ks are strided channel slices.  K = 16; worst ratio on an H100:
    forward 0 (within 4 ulps everywhere), gradients 1.7."""
    from nvdiffrecmc_b200.optixutils.ops import shade_combine
    B, H, W = 8, 512, 512
    pbr = bsdf == "pbr"
    a4, b4, t8, dout = _combine_inputs((B, H, W), 51)
    a4t, b4t, t8t = [torch.tensor(x, device=dev).requires_grad_(True) for x in (a4, b4, t8)]
    kd, ks = t8t[..., 0:3], t8t[..., 4:7]
    out = shade_combine(a4t, b4t, kd, ks, BSDF=bsdf)
    out.backward(torch.tensor(dout, device=dev))
    torch.cuda.synchronize()
    idx = _sample_px(B, H, W)
    grid = (B, H, W)
    ins = [_take(x, grid, idx) for x in (a4, b4, t8[..., 0:3], t8[..., 4:7])]
    d = _take(dout, grid, idx)
    o32, o64 = oracle(), oracle(f64=True)
    check_per_element("shade_combine(%s) forward" % bsdf, [_take(_np(out), grid, idx)], lambda a: [o64.shade_combine(*a, pbr=pbr)],
                      lambda a: [o32.shade_combine(*a, pbr=pbr)], ins, K_COMBINE, ["out"])
    tg = _np(t8t.grad)
    got = [_take(_np(a4t.grad), grid, idx), _take(tg[..., 0:3], grid, idx)]
    names = ["d_a4", "d_kd"]
    pick = lambda r: [r[0], r[2]]
    if pbr:
        got += [_take(_np(b4t.grad), grid, idx), _take(tg[..., 4:7], grid, idx)]
        names += ["d_b4", "d_ks"]
        pick = lambda r: [r[0], r[2], r[1], r[3]]
    else:
        assert b4t.grad is None and not tg[..., 3:].any()
    check_per_element("shade_combine(%s) backward" % bsdf, got, lambda a: pick(o64.shade_combine_bwd(*a[:4], a[4], pbr=pbr)),
                      lambda a: pick(o32.shade_combine_bwd(*a[:4], a[4], pbr=pbr)), ins + [d], K_COMBINE, names)


def test_shade_combine_rejects_a4_or_b4_smaller_than_the_grid(dev):
    """Every output takes a4's [B,H,W]: an a4 (or, for 'pbr', a b4) that spans less than the broadcast grid of the operands is refused
    with a RuntimeError naming it, by the Python op and by the C entry points, before any launch."""
    import ctypes as C
    from nvdiffrecmc_b200 import _lib as L
    from nvdiffrecmc_b200.optixutils.ops import shade_combine
    full4 = torch.rand(2, 4, 5, 4, device=dev) + 0.5
    small4 = torch.rand(1, 4, 5, 4, device=dev) + 0.5
    kd, ks = torch.rand(2, 4, 5, 3, device=dev), torch.rand(2, 4, 5, 3, device=dev)
    with pytest.raises(RuntimeError, match="a4"):
        shade_combine(small4, full4, kd, ks, 'pbr')
    with pytest.raises(RuntimeError, match="b4"):
        shade_combine(full4, small4, kd, ks, 'pbr')
    with pytest.raises(RuntimeError, match="a4"):
        shade_combine(small4, None, kd, None, 'diffuse')
    # the C entries on their own; every output buffer is sized for the full grid and must come back untouched
    d = lambda t: C.byref(L.nhwc(t))
    outs = [torch.full((2, 4, 5, c), 7.0, device=dev) for c in (3, 4, 4, 3, 3)]
    for a, b, name in ((small4, full4, "a4"), (full4, small4, "b4")):
        rc = L.lib().mcs_shade_combine_fwd(d(a), d(b), d(kd), d(ks), 1, outs[0].data_ptr(), L.stream_ptr())
        assert rc != 0 and name in L.lib().mcs_last_error().decode()
        rc = L.lib().mcs_shade_combine_bwd(d(a), d(b), d(kd), d(ks), 1, d(kd), outs[1].data_ptr(), outs[2].data_ptr(), outs[3].data_ptr(),
                                           outs[4].data_ptr(), L.stream_ptr())
        assert rc != 0 and name in L.lib().mcs_last_error().decode()
    rc = L.lib().mcs_shade_combine_bwd(d(full4), d(full4), d(kd[:1]), d(ks[:1]), 1, d(torch.rand(3, 4, 5, 3, device=dev)), outs[1].data_ptr(),
                                       outs[2].data_ptr(), outs[3].data_ptr(), outs[4].data_ptr(), L.stream_ptr())
    assert rc != 0 and "a4" in L.lib().mcs_last_error().decode()       # a larger upstream gradient counts too
    torch.cuda.synchronize()
    assert all(bool((o == 7.0).all()) for o in outs)
    # broadcast kd / ks stay allowed, and their gradients come back summed to their shapes
    a = full4.clone().requires_grad_(True); k1 = kd[:1].clone().requires_grad_(True)
    shade_combine(a, full4, k1, ks[:1], 'pbr').sum().backward()
    assert k1.grad.shape == k1.shape


# ---------------------------------------------------------------------------------------------------------------------------------------
# image_loss: per-CTA partials and the partial -> pixel mapping of the backward
# ---------------------------------------------------------------------------------------------------------------------------------------
K_LOSS = 16
# The log_srgb backward of mse / relmse / n2n is proportional to d = tm(img) - tm(target).  Device logf / powf differ from glibc by a few ulps
# of tm(x), and where img and target are close the subtraction turns that into a relative error of d many times larger; perturbing the
# inputs by one ulp moves tm(x) by less than one of its own ulps (the tone map compresses), so Delta does not see it.
K_LOSS_CANCEL = 256
LOSS_BLOCK = 256                                    # lossmesh.cu: one partial per 256 consecutive grid pixels
IL_SHAPE = (3, 97, 131)                             # 38 121 pixels: 149 partials, the last one ragged


def _tonemap64(x, tm):
    x = np.clip(np.asarray(x, np.float64), 0.0, 65535.0)
    if tm == "none":
        return x
    s = np.log(x + 1.0)
    return np.where(s > 0.0031308, np.power(np.maximum(s, 0.0031308), 1.0 / 2.4) * 1.055 - 0.055, 12.92 * np.maximum(s, 0.0))


def _partials(px, dtype):
    n = px.size
    P = (n + LOSS_BLOCK - 1) // LOSS_BLOCK
    p = np.zeros(P * LOSS_BLOCK, dtype)
    p[:n] = px.reshape(-1)
    return p.reshape(P, LOSS_BLOCK).sum(1, dtype=dtype)


def _loss_layout(dev, layout, seed):
    """('rgba', 'img_broadcast') -> (img, target) device tensors with requires_grad leaves (leaf_img, leaf_tgt) and the numpy values.
    rgba: img = shaded[..., :3] of an RGBA tensor, target [1,H,W,3]; img_broadcast: img [1,H,W,3], target [N,H,W,3]."""
    N, H, W = IL_SHAPE
    g = np.random.default_rng(seed)
    if layout == "rgba":
        li = g.uniform(0.0, 4.0, (N, H, W, 4)).astype(np.float32); lt = g.uniform(0.0, 4.0, (1, H, W, 3)).astype(np.float32)
        li[0, 0, 0, :3] = -0.5; li[1, 50, 7, :3] = 70000.0; lt[0, 1, 0] = 0.0            # clamped / zero-gradient pixels
    else:
        li = g.uniform(0.0, 4.0, (1, H, W, 3)).astype(np.float32); lt = g.uniform(0.0, 4.0, (N, H, W, 3)).astype(np.float32)
        li[0, 0, 0] = -0.5; li[0, 50, 7] = 70000.0; lt[2, 1, 0] = 0.0
    leaf_i = torch.tensor(li, device=dev).requires_grad_(True); leaf_t = torch.tensor(lt, device=dev).requires_grad_(True)
    img = leaf_i[..., :3] if layout == "rgba" else leaf_i
    return img, leaf_t, leaf_i, leaf_t


def _reduce_to(g, shape, dtype):
    ax = tuple(k for k in range(g.ndim) if shape[k] == 1 and g.shape[k] != 1)
    return g.sum(axis=ax, keepdims=True, dtype=dtype) if ax else g.astype(dtype)


@pytest.mark.parametrize("layout", ["rgba", "img_broadcast"])
@pytest.mark.parametrize("tm", ["none", "log_srgb"])
@pytest.mark.parametrize("loss", ["l1", "mse", "relmse", "smape", "n2n"])
def test_image_loss_partials_and_weighted_backward(dev, loss, tm, layout):
    """3 x 97 x 131 (149 partials, the last one ragged).  Every per-CTA partial against the fp64 sum of the oracle's per-pixel losses over
    the same 256 grid pixels; the scalar loss divided by img's pixel count (so N times the mean for a broadcast img, as the reference);
    the backward driven by a distinct seeded weight per partial, so every pixel's gradient carries the weight of its own partial.
    For l1 and smape the gradient's sign at a tie between the tone-mapped values is not determined by fp32 (test_gpu_edge_inputs's
    _l1_grad_close): ties are left out of the bar and must agree in magnitude (or be zero on one side).  K = 16 (worst ratio on an H100:
    partials 1.0, gradients 6.2), except K_LOSS_CANCEL = 256 for the log_srgb gradients of mse / relmse / n2n (worst 142, see there)."""
    from nvdiffrecmc_b200.renderutils.ops import _image_loss_func
    import nvdiffrecmc_b200.renderutils as ru
    img, tgt, leaf_i, leaf_t = _loss_layout(dev, layout, 61)
    ni, nt = _np(img), _np(tgt)
    o32, o64 = oracle(), oracle(f64=True)
    parts = _image_loss_func.apply(img, tgt, loss, tm)
    P = parts.numel()
    assert P == (np.prod(IL_SHAPE) + LOSS_BLOCK - 1) // LOSS_BLOCK
    check_per_element("image_loss(%s,%s,%s) partials" % (loss, tm, layout), [_np(parts)],
                      lambda a: [_partials(o64.image_loss_px(a[0], a[1], loss, tm), np.float64)],
                      lambda a: [_partials(o32.image_loss_px(a[0], a[1], loss, tm), np.float32)], [ni, nt], K_LOSS, ["partial"])
    v = float(ru.image_loss(img, tgt, loss=loss, tonemapper=tm))
    ref = o64.image_loss(ni, nt, loss, tm)
    assert abs(v / ref - 1) < 1e-5, (v, ref)
    assert ref == o64.image_loss_px(ni, nt, loss, tm).sum() / (ni.shape[0] * ni.shape[1] * ni.shape[2])
    # backward: one distinct weight per partial
    w = np.random.default_rng(62).uniform(0.5, 1.5, P).astype(np.float32)
    ((parts * torch.tensor(w, device=dev)).sum()).backward()
    torch.cuda.synchronize()
    gi = _np(leaf_i.grad)
    if layout == "rgba":
        assert not gi[..., 3].any()
        gi = gi[..., :3]
    got = [gi, _np(leaf_t.grad)]
    dpx = np.repeat(w, LOSS_BLOCK)[:int(np.prod(IL_SHAPE))].reshape(IL_SHAPE)
    shapes = [ni.shape, nt.shape]

    def bwd(o, dt):
        return lambda a: [_reduce_to(x, s, dt) for x, s in zip(o.image_loss_bwd(a[0], a[1], loss, tm, dout=a[2]), shapes)]
    exempt = None
    if loss in ("l1", "smape"):
        ta, tb = _tonemap64(ni, tm), _tonemap64(nt, tm)
        ties = np.abs(ta - tb) <= 4 * 2.0 ** -23 * np.maximum(np.abs(ta), np.abs(tb))             # full grid [N,H,W,3]
        exempt = [_reduce_to(ties, s, np.int64) > 0 for s in shapes]
        g64 = [_reduce_to(x, s, np.float64) for x, s in zip(o64.image_loss_bwd(ni, nt, loss, tm, dout=dpx), shapes)]
        for gg, ww, e, s in zip(got, g64, exempt, shapes):
            assert e.mean() < 1e-3, ("ties", int(e.sum()))
            if s[0] == 1 and IL_SHAPE[0] != 1:
                continue                                    # summed over the views: a tie in one view leaves the sum undetermined
            a, b = gg[e].astype(np.float64), ww[e]
            assert ((a == 0) | (b == 0) | (np.abs(np.abs(a) - np.abs(b)) <= 1e-5 * np.abs(b))).all(), ("tie magnitudes", a, b)
    K = K_LOSS_CANCEL if tm == "log_srgb" and loss in ("mse", "relmse", "n2n") else K_LOSS
    check_per_element("image_loss(%s,%s,%s) backward" % (loss, tm, layout), got, bwd(o64, np.float64), bwd(o32, np.float32), [ni, nt, dpx],
                      K, ["d_img", "d_target"], exempt=exempt)


# ---------------------------------------------------------------------------------------------------------------------------------------
# xfm_points / xfm_vectors
# ---------------------------------------------------------------------------------------------------------------------------------------
K_XFM = 16


def _xfm_points(dev, layout, bp, V, g):
    """[bp,V,3] points as 'aos': a [..., :3] view of a [bp,V,4] tensor (strides 4V, 4, 1), or 'soa': a [bp,3,V] tensor transposed
    (strides 3V, 1, V)."""
    if layout == "aos":
        return torch.tensor((g.normal(size=(bp, V, 4)) * 3).astype(np.float32), device=dev)[..., :3]
    return torch.tensor((g.normal(size=(bp, 3, V)) * 3).astype(np.float32), device=dev).transpose(1, 2)


@pytest.mark.parametrize("layout", ["aos", "soa"])
@pytest.mark.parametrize("B,bp", [(1, 1), (8, 1), (8, 8)])
@pytest.mark.parametrize("V", [1, 255, 256, 257, 100003])
def test_xfm_strided_operands_per_element(dev, V, B, bp, layout):
    """Points as a strided view, the matrix as m.transpose(1, 2) of a contiguous tensor, and upstream gradients expanded with stride 0
    over the batch and over the vertices, handed to the backward as they are.  Forward and points gradient per element.  'soa' points
    have a channel stride of V.  K = 16; worst ratio on an H100: forward 3.3, gradient 5.2."""
    from nvdiffrecmc_b200.renderutils.ops import _xfm_func
    import nvdiffrecmc_b200.renderutils as ru
    g = np.random.default_rng(V + 10 * B + bp)
    pts = _xfm_points(dev, layout, bp, V, g)
    m0 = torch.tensor(g.normal(size=(B, 4, 4)).astype(np.float32), device=dev)
    mtx = m0.transpose(1, 2)
    assert mtx.stride()[1:] == (1, 4) and pts.stride(2) == (1 if layout == "aos" else V)
    o32, o64 = oracle(), oracle(f64=True)
    np_p, np_m = _np(pts), _np(mtx)
    for is_points, fn in ((True, ru.xfm_points), (False, ru.xfm_vectors)):
        C4 = 4 if is_points else 3
        what = "xfm_%s V=%d B=%d bp=%d %s" % ("points" if is_points else "vectors", V, B, bp, layout)
        out = fn(pts, mtx)
        check_per_element(what + " forward", [_np(out)], lambda a: [o64.xfm(a[0], a[1], is_points)], lambda a: [o32.xfm(a[0], a[1], is_points)],
                          [np_p, np_m], K_XFM, ["out"])
        ctx = types.SimpleNamespace(saved_tensors=(pts, mtx), isPoints=is_points)
        for k, dshape in enumerate([(1, V, C4), (B, 1, C4)]):
            dout = torch.tensor(g.uniform(-1, 1, dshape).astype(np.float32), device=dev).expand(B, V, C4)
            gp = _xfm_func.backward(ctx, dout)[0]
            torch.cuda.synchronize()
            dnp = np.ascontiguousarray(_np(dout))

            def bwd(o, dt):
                return lambda a: [_reduce_to(o.xfm_bwd(a[0], a[1], is_points), (bp, V, 3), dt)]
            check_per_element(what + " backward (stride-0 %s)" % ("batch" if k == 0 else "vertex"), [_np(gp)], bwd(o64, np.float64),
                              bwd(o32, np.float32), [np_m, dnp], K_XFM, ["d_points"])
