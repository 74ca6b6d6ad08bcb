"""The image-space regularisers of both geometry passes on the GPU: drop-ins for the reference's `shading_loss`,
`material_smoothness_grad` and `chroma_loss` (render/regularizer.py:15-49), run by the kernels of csrc/regularizer.cu (contract stated
there: torch's conventions for ties of max, clamp boundaries, abs at 0, the sRGB branch and the means' denominators), and
`jitter_taps`, the producer of their inputs in shade() (render/render.py:50-97), run by the kernels of csrc/taps.cu, and
`coverage_image_loss`, the image loss the geometry passes put in front of them (geometry/dmtet.py:229-230, geometry/dlmesh.py:75-76): the
coverage MSE plus `image_loss` of the colour premultiplied by the target's alpha, run by the kernels of csrc/lossmesh.cu.

Each function returns a 0-dim fp32 device tensor, as `torch.mean(...) * lambda` does.  Forward and backward are one streaming launch
each (plus a one-CTA finish in the forward), make no host synchronisation and can be captured in a CUDA graph; the backward reads its
upstream gradient from the device.  Gradients flow to every rendered operand, all four channels (alpha comes from the composite and
depends on the geometry); `kd`'s alpha gets exactly 0 and `color_ref` is the constant target.

Operands are fp32 CUDA [B,H,W,4] tensors of one B, H, W, with any strides (`color_ref` is often a slice); `material_smoothness_grad`'s
kd_grad may also be [B,H,W,5], the transparency configuration's 4-channel kd with alpha appended.  A wrong channel count, a shape
mismatch, a CPU tensor, a non-float lambda or a `color_ref` that requires grad raises ValueError before anything is launched, as does
an unknown loss or tonemapper name for `coverage_image_loss`.
"""
import torch

from . import _lib as L
from .renderutils.ops import _loss_ids

__all__ = ["shading_loss", "material_smoothness_grad", "chroma_loss", "jitter_taps", "coverage_image_loss"]


def _check(fn, named, lambdas, chans=None):
    """ValueError naming the argument unless every (name, tensor) of `named` is an fp32 CUDA [B,H,W,C] tensor of the first one's B, H, W on
    its device, with C = 4 or one of chans[name], every (name, value) of `lambdas` is a Python float, and color_ref (if given) does not
    require grad."""
    first_name, first = named[0]
    for name, t in named:
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: %s must be a torch.Tensor, got %s" % (fn, name, type(t).__name__))
        if t.dtype != torch.float32:
            raise ValueError("%s: %s must be float32, got %s" % (fn, name, t.dtype))
        want = (chans or {}).get(name, (4,))
        if t.dim() != 4 or t.shape[3] not in want:
            raise ValueError("%s: %s must be [B,H,W,%s], got %s" % (fn, name, "|".join(map(str, want)), tuple(t.shape)))
        if not t.is_cuda:
            raise ValueError("%s: %s must be a CUDA tensor, got %s" % (fn, name, t.device))
        if t.shape[:3] != first.shape[:3]:
            raise ValueError("%s: %s has shape %s, %s has %s" % (fn, name, tuple(t.shape), first_name, tuple(first.shape)))
        if t.device != first.device:
            raise ValueError("%s: %s is on %s, %s on %s" % (fn, name, t.device, first_name, first.device))
        if t.numel() == 0:
            raise ValueError("%s: %s is empty" % (fn, name))
        if any(s >= 2 ** 31 for s in t.stride()):
            raise ValueError("%s: %s has a stride beyond int32" % (fn, name))
        if name == "color_ref" and t.requires_grad:
            raise ValueError("%s: color_ref is the constant target and must not require grad" % fn)
    if first.shape[0] * first.shape[1] * first.shape[2] >= 2 ** 31:
        raise ValueError("%s: at most 2^31 - 1 pixels" % fn)
    for name, v in lambdas:
        if not isinstance(v, float):
            raise ValueError("%s: %s must be a float, got %s" % (fn, name, type(v).__name__))


def _partials(fn, t, k):
    B, H, W = t.shape[:3]
    return torch.empty(k * getattr(L.lib(), "mcs_%s_num_partials" % fn)(B, H, W), dtype=torch.float64, device=t.device)


def _grad(t):
    return torch.empty(t.shape, dtype=torch.float32, device=t.device)


def _upstream(d_loss):
    return d_loss.to(torch.float32).contiguous()


# ---- shading_loss ----
def _shading_fwd(d, s, r, ld, ls):
    loss = torch.empty((), dtype=torch.float32, device=d.device)
    means = torch.empty(2, dtype=torch.float32, device=d.device)
    L.check(L.lib().mcs_shading_loss_fwd(L.nhwc(d), L.nhwc(s), L.nhwc(r), ld, ls, _partials("shading_loss", d, 3).data_ptr(), loss.data_ptr(),
                                         means.data_ptr(), L.stream_ptr()), "shading_loss_fwd")
    return loss, means


class _ShadingLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, d, s, r, ld, ls):
        loss, means = _shading_fwd(d, s, r, ld, ls)
        ctx.save_for_backward(d, s, r, means)
        ctx.lambdas = (ld, ls)
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        d, s, r, means = ctx.saved_tensors
        gd, gs = _grad(d), _grad(s)
        L.check(L.lib().mcs_shading_loss_bwd(L.nhwc(d), L.nhwc(s), L.nhwc(r), *ctx.lambdas, means.data_ptr(), _upstream(d_loss).data_ptr(),
                                             gd.data_ptr(), gs.data_ptr(), L.stream_ptr()), "shading_loss_bwd")
        return (gd if ctx.needs_input_grad[0] else None), (gs if ctx.needs_input_grad[1] else None), None, None, None


def shading_loss(diffuse_light, specular_light, color_ref, lambda_diffuse, lambda_specular):
    """The reference's monochrome shading regulariser: the log-sRGB error of the lights' luma against color_ref's value, weighted by the
    diffuse share, plus mean specular luma over mean diffuse luma.  -> 0-dim fp32 tensor, differentiable in both lights."""
    _check("shading_loss", [("diffuse_light", diffuse_light), ("specular_light", specular_light), ("color_ref", color_ref)],
           [("lambda_diffuse", lambda_diffuse), ("lambda_specular", lambda_specular)])
    if torch.is_grad_enabled() and (diffuse_light.requires_grad or specular_light.requires_grad):
        return _ShadingLoss.apply(diffuse_light, specular_light, color_ref, lambda_diffuse, lambda_specular)
    return _shading_fwd(diffuse_light.detach(), specular_light.detach(), color_ref, lambda_diffuse, lambda_specular)[0]


# ---- material_smoothness_grad ----
def _smooth_fwd(k, s, n, lam):
    loss = torch.empty((), dtype=torch.float32, device=k.device)
    L.check(L.lib().mcs_material_smoothness_grad_fwd(L.nhwc(k), L.nhwc(s), L.nhwc(n), *lam, _partials("material_smoothness_grad", k, 3).data_ptr(),
                                                     loss.data_ptr(), L.stream_ptr()), "material_smoothness_grad_fwd")
    return loss


class _MaterialSmoothness(torch.autograd.Function):
    @staticmethod
    def forward(ctx, k, s, n, lkd, lks, lnrm):
        ctx.save_for_backward(k, s, n)
        ctx.lambdas = (lkd, lks, lnrm)
        return _smooth_fwd(k, s, n, ctx.lambdas)

    @staticmethod
    def backward(ctx, d_loss):
        k, s, n = ctx.saved_tensors
        gk, gs, gn = _grad(k), _grad(s), _grad(n)
        L.check(L.lib().mcs_material_smoothness_grad_bwd(L.nhwc(k), L.nhwc(s), L.nhwc(n), *ctx.lambdas, _upstream(d_loss).data_ptr(),
                                                         gk.data_ptr(), gs.data_ptr(), gn.data_ptr(), L.stream_ptr()),
                "material_smoothness_grad_bwd")
        return tuple(g if need else None for g, need in zip((gk, gs, gn), ctx.needs_input_grad[:3])) + (None, None, None)


def material_smoothness_grad(kd_grad, ks_grad, nrm_grad, lambda_kd=0.25, lambda_ks=0.1, lambda_nrm=0.0):
    """The reference's material smoothness regulariser over the jittered-tap differences kd_grad, ks_grad, nrm_grad (rgb, coverage
    alpha).  kd_grad may have 5 channels (`jitter_taps` of a 4-channel kd): luma from channels 0..2, alpha from the last, and channel 3
    gets a gradient of exactly 0.  -> 0-dim fp32 tensor, differentiable in every channel of each."""
    _check("material_smoothness_grad", [("kd_grad", kd_grad), ("ks_grad", ks_grad), ("nrm_grad", nrm_grad)],
           [("lambda_kd", lambda_kd), ("lambda_ks", lambda_ks), ("lambda_nrm", lambda_nrm)], chans={"kd_grad": (4, 5)})
    if torch.is_grad_enabled() and (kd_grad.requires_grad or ks_grad.requires_grad or nrm_grad.requires_grad):
        return _MaterialSmoothness.apply(kd_grad, ks_grad, nrm_grad, lambda_kd, lambda_ks, lambda_nrm)
    return _smooth_fwd(kd_grad.detach(), ks_grad.detach(), nrm_grad.detach(), (lambda_kd, lambda_ks, lambda_nrm))


# ---- chroma_loss ----
def _chroma_fwd(k, r, lc):
    loss = torch.empty((), dtype=torch.float32, device=k.device)
    L.check(L.lib().mcs_chroma_loss_fwd(L.nhwc(k), L.nhwc(r), lc, _partials("chroma_loss", k, 1).data_ptr(), loss.data_ptr(), L.stream_ptr()),
            "chroma_loss_fwd")
    return loss


class _ChromaLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, k, r, lc):
        ctx.save_for_backward(k, r)
        ctx.lc = lc
        return _chroma_fwd(k, r, lc)

    @staticmethod
    def backward(ctx, d_loss):
        k, r = ctx.saved_tensors
        gk = _grad(k)
        L.check(L.lib().mcs_chroma_loss_bwd(L.nhwc(k), L.nhwc(r), ctx.lc, _upstream(d_loss).data_ptr(), gk.data_ptr(), L.stream_ptr()),
                "chroma_loss_bwd")
        return gk, None, None


def chroma_loss(kd, color_ref, lambda_chroma):
    """The reference's chroma regulariser: |kd / value(kd) - color_ref / value(color_ref)| where color_ref covers, over rgb.  -> 0-dim
    fp32 tensor, differentiable in kd's rgb (kd's alpha gets 0)."""
    _check("chroma_loss", [("kd", kd), ("color_ref", color_ref)], [("lambda_chroma", lambda_chroma)])
    if torch.is_grad_enabled() and kd.requires_grad:
        return _ChromaLoss.apply(kd, color_ref, lambda_chroma)
    return _chroma_fwd(kd.detach(), color_ref, lambda_chroma)


# ---- jitter_taps ----
_TAP_OPERANDS = ("rast", "jitter", "kd", "ks", "gb_normal", "perturbed_nrm", "kd_jitter", "ks_jitter")


def _check_taps(named):
    """ValueError naming the argument unless every given operand is an fp32 CUDA [B,H,W,C] tensor of rast's B, H, W and device with its
    channel count, kd_jitter / ks_jitter come together and jitter does not require grad.  rast may require grad (rasterize's output is
    differentiable in the vertices); only its coverage test is read, which has no gradient, as in the reference."""
    fn = "jitter_taps"
    rast = named["rast"]
    if (named["kd_jitter"] is None) != (named["ks_jitter"] is None):
        raise ValueError("%s: kd_jitter and ks_jitter go together (the MLP path), got only %s" % (
            fn, "kd_jitter" if named["ks_jitter"] is None else "ks_jitter"))
    chans = {"rast": (4,), "jitter": (2,), "kd": (3, 4), "ks": (3,), "gb_normal": (3,), "perturbed_nrm": (3,), "ks_jitter": (3,)}
    given = [(name, named[name]) for name in _TAP_OPERANDS if named[name] is not None or name in ("rast", "jitter", "kd", "ks", "gb_normal")]
    for name, t in given:
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: %s must be a torch.Tensor, got %s" % (fn, name, type(t).__name__))
        if t.dtype != torch.float32:
            raise ValueError("%s: %s must be float32, got %s" % (fn, name, t.dtype))
        want = chans[name] if name in chans else (named["kd"].shape[3],)      # kd_jitter: kd's channels (kd is checked before it)
        if t.dim() != 4 or t.shape[3] not in want:
            raise ValueError("%s: %s must be [B,H,W,%s], got %s" % (fn, name, "|".join(map(str, want)), tuple(t.shape)))
    for name, t in given:
        if not t.is_cuda:
            raise ValueError("%s: %s must be a CUDA tensor, got %s" % (fn, name, t.device))
        if t.shape[:3] != rast.shape[:3]:
            raise ValueError("%s: %s has B,H,W %s, rast has %s" % (fn, name, tuple(t.shape[:3]), tuple(rast.shape[:3])))
        if t.device != rast.device:
            raise ValueError("%s: %s is on %s, rast on %s" % (fn, name, t.device, rast.device))
        if any(s >= 2 ** 31 or s < 0 for s in t.stride()):
            raise ValueError("%s: %s has a stride outside int32" % (fn, name))
    if named["jitter"].requires_grad:
        raise ValueError("%s: jitter is a constant and must not require grad (its gradient would be dropped)" % fn)
    if rast.shape[0] * rast.shape[1] * rast.shape[2] >= 2 ** 31:
        raise ValueError("%s: at most 2^31 - 1 pixels" % fn)


def _desc(t):
    return None if t is None else L.nhwc(t)


def _taps_fwd(ops):
    rast, kd, pn = ops[0], ops[2], ops[5]
    B, H, W = rast.shape[:3]
    dev = rast.device
    outs = [torch.empty(B, H, W, kd.shape[3] + 1, dtype=torch.float32, device=dev)]
    outs += [torch.empty(B, H, W, 4, dtype=torch.float32, device=dev) for _ in range(2 if pn is None else 3)]
    if B * H * W:
        descs = [_desc(t) for t in ops]
        L.check(L.lib().mcs_jitter_taps_fwd(*descs, *[o.data_ptr() for o in outs], *([None] if pn is None else []), L.stream_ptr()),
                "jitter_taps_fwd")
    return outs


class _JitterTaps(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *ops):
        ctx.has_pn, ctx.mlp = ops[5] is not None, ops[6] is not None
        ctx.save_for_backward(*ops)
        return tuple(_taps_fwd(ops))

    @staticmethod
    def backward(ctx, *d_outs):
        ops = ctx.saved_tensors
        rast, kd = ops[0], ops[2]
        B, H, W = rast.shape[:3]
        dev = rast.device
        ckd = kd.shape[3]
        grads4 = [torch.zeros(B, H, W, 4, dtype=torch.float32, device=dev) for _ in range(4 if ctx.has_pn else 3)]
        gj = [torch.empty(B, H, W, ckd, dtype=torch.float32, device=dev), torch.empty(B, H, W, 3, dtype=torch.float32, device=dev)] \
            if ctx.mlp else [None, None]
        ups = [g.to(torch.float32).contiguous() for g in d_outs]
        if B * H * W:
            ptr = lambda t: None if t is None else t.data_ptr()
            L.check(L.lib().mcs_jitter_taps_bwd(*[_desc(t) for t in ops], *[u.data_ptr() for u in ups], *([None] if not ctx.has_pn else []),
                                                *[g.data_ptr() for g in grads4], *([None] if not ctx.has_pn else []), ptr(gj[0]), ptr(gj[1]),
                                                L.stream_ptr()), "jitter_taps_bwd")
        d_kd = grads4[0] if ckd == 4 else grads4[0][..., :3]
        d = [None, None, d_kd, grads4[1][..., :3], grads4[2][..., :3], grads4[3][..., :3] if ctx.has_pn else None, gj[0], gj[1]]
        return tuple(g if need else None for g, need in zip(d, ctx.needs_input_grad))


def jitter_taps(rast, jitter, kd, ks, gb_normal, perturbed_nrm=None, kd_jitter=None, ks_jitter=None):
    """The jittered regulariser differences of the reference's shade() (render/render.py:50-97), one launch each way: -> {"kd_grad":
    [B,H,W,Ckd+1], "ks_grad", "normal_grad" and, when perturbed_nrm is given, "perturbed_nrm_grad": [B,H,W,4]}, each with shade()'s
    alpha appended, ready for its `buffers` dict.

    rast [B,H,W,4] and jitter [B,H,W,2] (pixel_grid + the caller's offset draw) are constants; kd [B,H,W,3|4], ks, gb_normal and
    perturbed_nrm [B,H,W,3], any strides.  With kd_jitter and ks_jitter (the MLP texture's jittered sample, all_tex_jitter[...,0:3] /
    [...,3:6]) the differences are the MLP path's (no tap, no grad weight); else kd and ks are tapped at jitter.  Differentiable in kd,
    ks, gb_normal, perturbed_nrm, kd_jitter and ks_jitter."""
    ops = (rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter)
    _check_taps(dict(zip(_TAP_OPERANDS, ops)))
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ops):
        outs = _JitterTaps.apply(*ops)
    else:
        outs = _taps_fwd(tuple(None if t is None else t.detach() for t in ops))
    names = ["kd_grad", "ks_grad", "normal_grad", "perturbed_nrm_grad"]
    return dict(zip(names, outs))


# ---- coverage_image_loss ----
def _coverage_fwd(s, r, ids):
    B, H, W = s.shape[:3]
    loss = torch.empty((), dtype=torch.float32, device=s.device)
    partials = torch.empty(2 * L.lib().mcs_coverage_loss_num_partials(B, H, W), dtype=torch.float32, device=s.device)
    L.check(L.lib().mcs_coverage_loss_fwd(L.nhwc(s), L.nhwc(r), *ids, partials.data_ptr(), loss.data_ptr(), L.stream_ptr()), "coverage_loss_fwd")
    return loss


class _CoverageImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s, r, ids):
        ctx.save_for_backward(s, r)
        ctx.ids = ids
        return _coverage_fwd(s, r, ids)

    @staticmethod
    def backward(ctx, d_loss):
        if not ctx.needs_input_grad[0]:
            return None, None, None
        s, r = ctx.saved_tensors
        gs = _grad(s)
        L.check(L.lib().mcs_coverage_loss_bwd(L.nhwc(s), L.nhwc(r), *ctx.ids, _upstream(d_loss).data_ptr(), gs.data_ptr(), L.stream_ptr()),
                "coverage_loss_bwd")
        return gs, None, None


def coverage_image_loss(shaded, color_ref, loss='l1', tonemapper='none'):
    """The geometry passes' image loss (geometry/dmtet.py:229-230, geometry/dlmesh.py:75-76):
        mse_loss(shaded[..., 3:], color_ref[..., 3:]) + image_loss(shaded[..., 0:3] * color_ref[..., 3:], color_ref[..., 0:3] * color_ref[..., 3:],
                                                                   loss, tonemapper)
    with `image_loss` the package's renderutils op (so 'n2n' is honoured) and loss / tonemapper one of train.py's createLoss pairs.  The
    first term is the silhouette loss: shaded's alpha is the composited coverage.  -> 0-dim fp32 tensor, differentiable in all four
    channels of shaded; color_ref is the constant target."""
    ids = _loss_ids(loss, tonemapper)
    _check("coverage_image_loss", [("shaded", shaded), ("color_ref", color_ref)], [])
    if torch.is_grad_enabled() and shaded.requires_grad:
        return _CoverageImageLoss.apply(shaded, color_ref, ids)
    return _coverage_fwd(shaded.detach(), color_ref, ids)
