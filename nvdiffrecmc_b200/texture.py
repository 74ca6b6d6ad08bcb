"""Trainable 2-D textures on the GPU: a drop-in `Texture2D` for the reference's (render/texture.py:33-100) whose automatic mip chain is
built and differentiated by the kernels of csrc/texture.cu (contract stated there), and whose `clamp_` / `normalize_` are one launch each
over every level.

`mip_chain(tex)` returns levels 1..L of the reference's automatic chain: each level halves both sides, rounding down, by the 2 x 2 average
(avg_pool2d's float order, bit for bit), until either side is 1.  Its backward is the reference's `texture2d_mip.backward` folded over the
whole chain in one launch: the gradient of a coarser level reaches the finer one as the clamped bilinear look-up of a quarter of it at the
finer texels' centres, added to the finer level's own gradient.  Levels with no incoming gradient cost nothing.  For power-of-two sides
this is the reference's arithmetic bit for bit; for others the reference's `torch.linspace` grid differs from the exact texel centres by
an ulp.  Like the reference, the backward fails for a chain with a level pooled from an odd side (it raises RuntimeError naming the level).

Swapping the class in is one assignment, made before any mesh or material is loaded; `create_trainable`, `load_texture2D`,
`srgb_to_rgb` / `rgb_to_srgb` and render/material.py look `Texture2D` up at call time:

    import render.texture, nvdiffrecmc_b200.texture
    render.texture.Texture2D = nvdiffrecmc_b200.texture.Texture2D
"""
import ctypes

import numpy as np
import torch

from . import _lib as L
from .raster import texture

__all__ = ["Texture2D", "mip_chain"]
_MAX_LEVELS = 16


def chain_shapes(H, W):
    """(H_k, W_k) of the automatic chain of an H x W texture: halve both sides until either is 1."""
    shapes = [(H, W)]
    while shapes[-1][0] > 1 and shapes[-1][1] > 1:
        shapes.append((shapes[-1][0] // 2, shapes[-1][1] // 2))
    return shapes


def _table(shapes, ptrs, Bt, C):
    """mcs_texture_levels of dense [Bt, h, w, C] levels; a None pointer is an absent level."""
    lv = L.mcs_texture_levels()
    lv.n_levels, lv.C = len(shapes), C
    for k, ((h, w), p) in enumerate(zip(shapes, ptrs)):
        lv.ptr[k], lv.h[k], lv.w[k], lv.batch_stride[k] = p, h, w, h * w * C
    return lv


class _mip_chain_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tex):
        ctx.set_materialize_grads(False)
        Bt, H, W, C = tex.shape
        shapes = chain_shapes(H, W)
        levels = [torch.empty(Bt, h, w, C, dtype=torch.float32, device=tex.device) for h, w in shapes[1:]]
        lv = _table(shapes, [tex.data_ptr()] + [t.data_ptr() for t in levels], Bt, C)
        L.check(L.lib().mcs_mip_chain_fwd(ctypes.byref(lv), Bt, L.stream_ptr()), "mip_chain_fwd", L.lib().mcs_mip_chain_fwd_launches(len(shapes)))
        ctx.shape = tuple(tex.shape)
        return tuple(levels)

    @staticmethod
    def backward(ctx, *grads):
        Bt, H, W, C = ctx.shape
        shapes = chain_shapes(H, W)
        live = [k + 1 for k, g in enumerate(grads) if g is not None]
        if not live:
            return None
        odd = next((k for k, (h, w) in enumerate(shapes[:-1]) if h % 2 or w % 2), None)
        if odd is not None and live[-1] > odd:
            raise RuntimeError("mip_chain: level %d (%d x %d) has an odd side, and the 2 x 2 average that pools it into level %d has no "
                               "backward (the reference's texture2d_mip.backward returns %d x %d there); only chains whose pooled levels "
                               "are even in both sides are differentiable" % (odd, *shapes[odd], odd + 1, 2 * shapes[odd + 1][0], 2 * shapes[odd + 1][1]))
        gs = [None] + [None if g is None else g.to(torch.float32).contiguous() for g in grads]
        n = live[-1] + 1
        d_base = torch.empty(ctx.shape, dtype=torch.float32, device=next(g for g in gs if g is not None).device)
        lv = _table(shapes[:n], [None if g is None else g.data_ptr() for g in gs[:n]], Bt, C)
        L.check(L.lib().mcs_mip_chain_bwd(ctypes.byref(lv), Bt, d_base.data_ptr(), L.stream_ptr()), "mip_chain_bwd")
        return d_base


def mip_chain(tex):
    """Levels 1..L ([Bt, H >> k, W >> k, C] fp32) of the automatic mip chain of tex [Bt, H, W, C] (fp32 CUDA, any C >= 1): the 2 x 2
    average of the previous level until either side is 1; an empty list when tex already has a side of 1.  Differentiable in tex."""
    if not isinstance(tex, torch.Tensor) or tex.dim() != 4 or tex.dtype != torch.float32:
        raise ValueError("mip_chain: tex must be an fp32 [Bt,H,W,C] tensor, got %s" % (
            "%s %s" % (tuple(tex.shape), tex.dtype) if isinstance(tex, torch.Tensor) else type(tex).__name__))
    if min(tex.shape) < 1:
        raise ValueError("mip_chain: tex has an empty dimension %s" % (tuple(tex.shape),))
    L.require_cuda(tex)
    if len(chain_shapes(tex.shape[1], tex.shape[2])) > _MAX_LEVELS:
        raise ValueError("mip_chain: a %d x %d texture has more than %d levels" % (tex.shape[1], tex.shape[2], _MAX_LEVELS))
    if tex.shape[1] == 1 or tex.shape[2] == 1:
        return []
    return list(_mip_chain_func.apply(tex.contiguous()))


def _in_place_table(fn, mips):
    """Level table of a texture's levels for an in-place update: fp32 CUDA, contiguous, one minibatch and channel count."""
    for k, m in enumerate(mips):
        if not isinstance(m, torch.Tensor) or m.dim() != 4 or m.dtype != torch.float32 or not m.is_cuda:
            raise ValueError("%s: level %d must be an fp32 CUDA [Bt,H,W,C] tensor" % (fn, k))
        if not m.is_contiguous():
            raise ValueError("%s: level %d is not contiguous" % (fn, k))
        if m.shape[0] != mips[0].shape[0] or m.shape[3] != mips[0].shape[3]:
            raise ValueError("%s: level %d is %s; its minibatch and channels must be those of level 0 %s" % (fn, k, tuple(m.shape), tuple(mips[0].shape)))
    if len(mips) > _MAX_LEVELS:
        raise ValueError("%s: %d levels; at most %d are supported" % (fn, len(mips), _MAX_LEVELS))
    Bt, C = mips[0].shape[0], mips[0].shape[3]
    return _table([tuple(m.shape[1:3]) for m in mips], [m.data_ptr() for m in mips], Bt, C), Bt


def _written(mips):
    for m in mips:                     # what an in-place torch op does: saved copies of these levels are now stale
        torch.autograd.graph.increment_version(m)


class Texture2D:
    """The reference's Texture2D: `init` is a numpy array, a constant (1-D), an [H,W,C] or [Bt,H,W,C] tensor, or a custom chain (a list of
    [Bt,H_k,W_k,C] levels; a one-element list is its tensor).  `.data` holds the [Bt,H,W,C] tensor or the list, `.min_max` the clamp
    bounds."""

    def __init__(self, init, min_max=None):
        if isinstance(init, np.ndarray):
            init = torch.tensor(init, dtype=torch.float32, device='cuda')
        elif isinstance(init, list) and len(init) == 1:
            init = init[0]
        if isinstance(init, list) or len(init.shape) == 4:
            self.data = init
        elif len(init.shape) == 3:
            self.data = init[None, ...]
        else:
            self.data = init[None, None, None, :]
        self.min_max = min_max

    def sample(self, texc, texc_deriv, filter_mode='linear-mipmap-linear'):
        """Filtered look-up (raster.texture) of the custom chain, or of the texture and its automatic chain.  'linear' reads level 0 only,
        so the chain is not built."""
        if isinstance(self.data, list):
            return texture(self.data[0], texc, texc_deriv, mip=self.data[1:], filter_mode=filter_mode)
        mipmap = filter_mode == 'linear-mipmap-linear' or (filter_mode == 'auto' and texc_deriv is not None)
        if mipmap and self.data.shape[1] > 1 and self.data.shape[2] > 1:
            return texture(self.data, texc, texc_deriv, mip=mip_chain(self.data), filter_mode=filter_mode)
        return texture(self.data, texc, texc_deriv, filter_mode=filter_mode)

    def getRes(self):
        return self.getMips()[0].shape[1:3]

    def getChannels(self):
        return self.getMips()[0].shape[3]

    def getMips(self):
        return self.data if isinstance(self.data, list) else [self.data]

    def parameters(self):
        return self.getMips()

    def clamp_(self):
        """Clamp every level in place, channel c to [min_max[0][c], min_max[1][c]] (NaN texels stay NaN), in one launch; a no-op without
        min_max.  The bounds stay on the device: min_max must be two fp32 CUDA tensors of at least C entries."""
        if self.min_max is None:
            return
        mips = self.getMips()
        lv, Bt = _in_place_table("clamp_", mips)
        C = lv.C
        mm = self.min_max
        if not (isinstance(mm, (list, tuple)) and len(mm) == 2 and all(isinstance(b, torch.Tensor) and b.dtype == torch.float32 and b.is_cuda
                                                                       and b.dim() == 1 and b.shape[0] >= C for b in mm)):
            raise ValueError("clamp_: min_max must be two fp32 CUDA 1-D tensors of at least %d entries" % C)
        lo, hi = (b.contiguous() for b in mm)
        L.check(L.lib().mcs_mip_clamp(ctypes.byref(lv), Bt, lo.data_ptr(), hi.data_ptr(), L.stream_ptr()), "mip_clamp")
        _written(mips)

    def normalize_(self):
        """Normalise every texel of every level in place (util.safe_normalize: x / sqrt(max(dot(x, x), 1e-20))), in one launch; C = 3."""
        mips = self.getMips()
        lv, Bt = _in_place_table("normalize_", mips)
        if lv.C != 3:
            raise ValueError("normalize_: the texture must have 3 channels, got %d" % lv.C)
        L.check(L.lib().mcs_mip_normalize(ctypes.byref(lv), Bt, L.stream_ptr()), "mip_normalize")
        _written(mips)
