"""Drop-in replacement for the BSDF / shading-normal part of render/renderutils/ops.py.

Every op keeps the reference signature including the `use_python=` validation switch
(renderutils/ops.py:101,124,146,168,194,244,278,315,355); the CUDA path calls libmcshade through the
C ABI.  Gradients of broadcast inputs come back full-size from the kernel and are reduced by
`_reduce_like` (the reference leaves that to autograd's sum_to_size, tensor.h:61,75).
"""
import ctypes as C

import torch

from .. import _lib as L
from . import bsdf as _tb


def _prep(*ts):
    L.require_cuda(*ts)
    out = []
    for t in ts:
        if t.dim() != 4:
            raise RuntimeError("expected [minibatch, height, width, channels] tensors, got shape %s" % (tuple(t.shape),))
        out.append(t if t.dtype == torch.float32 else t.float())
    return out


def _grid(*ts):
    return tuple(max(t.shape[d] for t in ts) for d in range(3))


def _reduce_like(g, ref):
    """Sum a full-grid gradient down to the (broadcast) shape of its input."""
    if tuple(g.shape) == tuple(ref.shape):
        return g
    return g.sum_to_size(ref.shape)


def _call(name, ins, extra, n_out_ch, dout=None):
    """Run mcs_<name>: ins (+ dout) as mcs_tensor views, outputs freshly allocated contiguous fp32."""
    ins = _prep(*ins)
    allt = ins + (_prep(dout) if dout is not None else [])
    N, H, W = _grid(*allt)
    outs = [torch.empty(N, H, W, c, dtype=torch.float32, device=ins[0].device) for c in n_out_ch]
    descs = [L.nhwc(t) for t in ins]
    args = [C.byref(d) for d in descs] + list(extra)
    if dout is not None:
        dd = L.nhwc(allt[-1])
        args.append(C.byref(dd))
    args += [o.data_ptr() for o in outs] + [L.stream_ptr()]
    L.check(getattr(L.lib(), "mcs_" + name)(*args), name)
    return outs


def _finite(out, name):
    if torch.is_anomaly_enabled():
        assert torch.all(torch.isfinite(out)), "Output of %s contains inf or NaN" % name
    return out


# ---------------------------------------------------------------------------------------------
class _ew_func(torch.autograd.Function):
    """mcs_<name>_fwd / mcs_<name>_bwd on the operands `ins`, with `scalars` after the operands in both calls: one output of fwd_ch
    channels forward, one gradient per operand backward (bwd_ch[i] channels, reduced to the operand's shape)."""
    @staticmethod
    def forward(ctx, name, scalars, fwd_ch, bwd_ch, *ins):
        ctx.name, ctx.scalars, ctx.bwd_ch = name, scalars, bwd_ch
        ctx.save_for_backward(*ins)
        return _call(name + "_fwd", ins, scalars, [fwd_ch])[0]

    @staticmethod
    def backward(ctx, dout):
        ins = ctx.saved_tensors
        g = _call(ctx.name + "_bwd", ins, ctx.scalars, ctx.bwd_ch, dout=dout)
        return (None,) * 4 + tuple(_reduce_like(a, b) for a, b in zip(g, ins))


def _fresnel_shlick(f0, f90, cosTheta, use_python=False):
    """renderutils/ops.py:89-109"""
    out = _tb.fresnel_schlick(f0, f90, cosTheta) if use_python else _ew_func.apply("fresnel_shlick", (), 3, (3, 3, 1), f0, f90, cosTheta)
    return _finite(out, "_fresnel_shlick")


def _ndf_ggx(alphaSqr, cosTheta, use_python=False):
    """renderutils/ops.py:112-132"""
    out = _tb.ndf_ggx(alphaSqr, cosTheta) if use_python else _ew_func.apply("ndf_ggx", (), 1, (1, 1), alphaSqr, cosTheta)
    return _finite(out, "_ndf_ggx")


def _lambda_ggx(alphaSqr, cosTheta, use_python=False):
    """renderutils/ops.py:134-154"""
    out = _tb.lambda_ggx(alphaSqr, cosTheta) if use_python else _ew_func.apply("lambda_ggx", (), 1, (1, 1), alphaSqr, cosTheta)
    return _finite(out, "_lambda_ggx")


def _masking_smith(alphaSqr, cosThetaI, cosThetaO, use_python=False):
    """renderutils/ops.py:156-176"""
    if use_python:
        out = _tb.masking_smith(alphaSqr, cosThetaI, cosThetaO)
    else:
        out = _ew_func.apply("masking_smith", (), 1, (1, 1, 1), alphaSqr, cosThetaI, cosThetaO)
    return _finite(out, "_masking_smith")


# ---------------------------------------------------------------------------------------------
_DEFAULT_PNRM = {}


def _default_perturbed_nrm(device):
    """[1,1,1,3] = (0, 0, 1), created once per device (the reference builds it from a Python list on every call, ops.py:217-218 -- a
    pageable host-to-device copy that would also break CUDA-graph capture of the step)."""
    key = str(device)
    if key not in _DEFAULT_PNRM:
        t = torch.zeros(1, 1, 1, 3, dtype=torch.float32, device=device)
        t[..., 2] = 1.0
        _DEFAULT_PNRM[key] = t
    return _DEFAULT_PNRM[key]


def prepare_shading_normal(pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm, two_sided_shading=True, opengl=True, use_python=False):
    """renderutils/ops.py:181-227.  Builds the tangent frame, perturbs by the normal map, flips for
    two-sided shading and bends back-facing normals towards the camera.  All tensors are
    [minibatch, height, width, 3] or broadcastable."""
    if perturbed_nrm is None:
        perturbed_nrm = _default_perturbed_nrm(pos.device)
    if use_python:
        out = _tb.prepare_shading_normal(pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm, two_sided_shading, opengl)
    else:
        out = _ew_func.apply("prepare_shading_normal", (int(two_sided_shading), int(opengl)), 3, (3,) * 6,
                             pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm)
    return _finite(out, "prepare_shading_normal")


# ---------------------------------------------------------------------------------------------
def lambert(nrm, wi, use_python=False):
    """renderutils/ops.py:244-264 -> [minibatch, height, width, 1]"""
    out = _tb.lambert(nrm, wi) if use_python else _ew_func.apply("lambert", (), 1, (3, 3), nrm, wi)
    return _finite(out, "lambert")


def frostbite_diffuse(nrm, wi, wo, linearRoughness, use_python=False):
    """renderutils/ops.py:278-300"""
    if use_python:
        out = _tb.frostbite_diffuse(nrm, wi, wo, linearRoughness)
    else:
        out = _ew_func.apply("frostbite", (), 1, (3, 3, 3, 1), nrm, wi, wo, linearRoughness)
    return _finite(out, "frostbite_diffuse")


def pbr_specular(col, nrm, wo, wi, alpha, min_roughness=0.08, use_python=False):
    """renderutils/ops.py:315-339; alpha is [minibatch, height, width, 1]"""
    if use_python:
        out = _tb.pbr_specular(col, nrm, wo, wi, alpha, min_roughness)
    else:
        out = _ew_func.apply("pbr_specular", (min_roughness,), 3, (3, 3, 3, 3, 1), col, nrm, wo, wi, alpha)
    return _finite(out, "pbr_specular")


def pbr_bsdf(kd, arm, pos, nrm, view_pos, light_pos, min_roughness=0.08, bsdf="lambert", use_python=False):
    """renderutils/ops.py:355-386.  Diffuse (Lambert or Frostbite) + GGX specular for a point light.
    kd: albedo, arm: (occlusion/spec attenuation, linear roughness, metalness)."""
    BSDF = 1 if bsdf == 'frostbite' else 0
    if use_python:
        out = _tb.pbr_bsdf(kd, arm, pos, nrm, view_pos, light_pos, min_roughness, BSDF)
    else:
        out = _ew_func.apply("pbr_bsdf", (min_roughness, BSDF), 3, (3,) * 6, kd, arm, pos, nrm, view_pos, light_pos)
    return _finite(out, "pbr_bsdf")


# ---------------------------------------------------------------------------------------------
# Row f3 of SURVEY section 8: image loss and mesh transforms
_LOSS_IDS = {"l1": 0, "mse": 1, "relmse": 2, "smape": 3, "n2n": 4}
_TONEMAPPERS = {"none": 0, "log_srgb": 1}


def _loss_ids(loss, tonemapper):
    """The reference's CUDA path maps every unknown loss name to L1 (strToLoss, torch_bindings.cpp:727-737) -- which is how 'n2n'
    silently became L1 there.  Unknown names raise here."""
    if loss not in _LOSS_IDS:
        raise ValueError("image_loss: unknown loss %r (expected one of %s)" % (loss, sorted(_LOSS_IDS)))
    if tonemapper not in _TONEMAPPERS:
        raise ValueError("image_loss: unknown tonemapper %r (expected one of %s)" % (tonemapper, sorted(_TONEMAPPERS)))
    return _LOSS_IDS[loss], _TONEMAPPERS[tonemapper]


class _image_loss_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, target, loss, tonemapper):
        img, target = _prep(img, target)
        ctx.loss, ctx.tonemapper = loss, tonemapper
        ctx.save_for_backward(img, target)
        N, H, W = _grid(img, target)
        nparts = L.lib().mcs_image_loss_num_partials(N, H, W)
        out = torch.empty(nparts, dtype=torch.float32, device=img.device)
        a, b = L.nhwc(img), L.nhwc(target)
        li, ti = _loss_ids(loss, tonemapper)
        L.check(L.lib().mcs_image_loss_fwd(C.byref(a), C.byref(b), li, ti, out.data_ptr(),
                                           L.stream_ptr()), "image_loss (forward)")
        return out

    @staticmethod
    def backward(ctx, dout):
        img, target = ctx.saved_tensors
        N, H, W = _grid(img, target)
        gi = torch.empty(N, H, W, 3, dtype=torch.float32, device=img.device)
        gt = torch.empty(N, H, W, 3, dtype=torch.float32, device=img.device)
        d = dout.float()
        dd = L._desc(d.data_ptr(), [d.shape[0], 1, 1, 1], [d.stride(0), 0, 0, 0])
        a, b = L.nhwc(img), L.nhwc(target)
        li, ti = _loss_ids(ctx.loss, ctx.tonemapper)
        L.check(L.lib().mcs_image_loss_bwd(C.byref(a), C.byref(b), li, ti, C.byref(dd),
                                           gi.data_ptr(), gt.data_ptr(), L.stream_ptr()), "image_loss (backward)")
        return _reduce_like(gi, img), _reduce_like(gt, target), None, None


def image_loss(img, target, loss='l1', tonemapper='none', use_python=False):
    """renderutils/ops.py:476-498.  HDR image loss, tonemapping + loss fused in one kernel.  loss in ['l1', 'mse', 'smape', 'relmse', 'n2n']
    (FIX: the reference's CUDA path silently computes l1 for 'n2n'), tonemapper in ['none', 'log_srgb'].  Returns a scalar."""
    _loss_ids(loss, tonemapper)
    if use_python:
        from .loss import image_loss_fn
        out = image_loss_fn(img, target, loss, tonemapper)
    else:
        out = _image_loss_func.apply(img, target, loss, tonemapper)
        out = torch.sum(out) / (img.shape[0] * img.shape[1] * img.shape[2])
    return _finite(out, "image_loss")


class _xfm_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, matrix, isPoints):
        L.require_cuda(points, matrix)
        points = points if points.dtype == torch.float32 else points.float()
        matrix = matrix if matrix.dtype == torch.float32 else matrix.float()
        if points.dim() != 3 or points.shape[2] != 3 or matrix.dim() != 3:
            raise RuntimeError("xfm: points must be [1|B, V, 3] and matrix [B, 4, 4]")
        ctx.save_for_backward(points, matrix)
        ctx.isPoints = isPoints
        B, V = matrix.shape[0], points.shape[1]
        out = torch.empty(B, V, 4 if isPoints else 3, dtype=torch.float32, device=points.device)
        p = L._desc(points.data_ptr(), list(points.shape) + [1], list(points.stride()) + [0])
        m = L._desc(matrix.data_ptr(), list(matrix.shape) + [1], list(matrix.stride()) + [0])
        L.check(L.lib().mcs_xfm_fwd(C.byref(p), C.byref(m), int(isPoints), out.data_ptr(), L.stream_ptr()), "xfm (forward)")
        return out

    @staticmethod
    def backward(ctx, dout):
        points, matrix = ctx.saved_tensors
        B, V = matrix.shape[0], points.shape[1]
        d = dout.float()
        g = torch.empty(B, V, 3, dtype=torch.float32, device=points.device)
        p = L._desc(points.data_ptr(), list(points.shape) + [1], list(points.stride()) + [0])
        m = L._desc(matrix.data_ptr(), list(matrix.shape) + [1], list(matrix.stride()) + [0])
        dd = L._desc(d.data_ptr(), list(d.shape) + [1], list(d.stride()) + [0])
        L.check(L.lib().mcs_xfm_bwd(C.byref(p), C.byref(m), C.byref(dd), int(ctx.isPoints), g.data_ptr(), L.stream_ptr()), "xfm (backward)")
        return (g.sum_to_size(points.shape) if tuple(g.shape) != tuple(points.shape) else g), None, None


def xfm_points(points, matrix, use_python=False):
    """renderutils/ops.py:501-519: [1|B,V,3] x [B,4,4] -> homogeneous [B,V,4]."""
    if use_python:
        out = torch.matmul(torch.nn.functional.pad(points, pad=(0, 1), mode='constant', value=1.0), torch.transpose(matrix, 1, 2))
    else:
        out = _xfm_func.apply(points, matrix, True)
    return _finite(out, "xfm_points")


def xfm_vectors(vectors, matrix, use_python=False):
    """renderutils/ops.py:521-540: [1|B,V,3] x [B,4,4] -> [B,V,3] (w = 0)."""
    if use_python:
        out = torch.matmul(torch.nn.functional.pad(vectors, pad=(0, 1), mode='constant', value=0.0), torch.transpose(matrix, 1, 2))[..., 0:3].contiguous()
    else:
        out = _xfm_func.apply(vectors, matrix, False)
    return _finite(out, "xfm_vectors")
