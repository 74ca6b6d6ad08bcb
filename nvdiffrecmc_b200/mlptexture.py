"""`MLPTexture3D`: the reference's neural material texture (render/mlptexture.py:47-103) with its `sample` fused into one forward and one
backward CUDA kernel (csrc/mlptexture.cu, semantics stated there): AABB normalisation, clamp, the hash-grid encoding of
`nvdiffrecmc_b200.tinycudann`, the bias-free ReLU MLP and the sigmoid scaled into min_max.

The module holds the reference's parameters under the reference's names (`encoder.params`, `net.net.<i>.weight`), built and initialised
in the reference's order, so the same torch seed gives the same weights and `state_dict()`s are interchangeable.  The gradients are the
ones the reference's two backward hooks produce, without hooks: d params is 128 x the true gradient (train.py:443 divides it by 8), d texc
and d W are unscaled.  With `render.mlptexture.MLPTexture3D = nvdiffrecmc_b200.mlptexture.MLPTexture3D` (after the `tinycudann` swap)
train.py and material.py pick it up unmodified.
"""
import ctypes

import numpy as np
import torch

from . import _lib as L
from . import tinycudann as tcnn

__all__ = ["MLPTexture3D"]

_SUPPORTED = "supported: internal_dims 32, hidden 1..4, channels 1..8"
GRADIENT_SCALING = 128.0        # render/mlptexture.py:71: the encoder's params see 128 x their gradient


def _check_config(channels, internal_dims, hidden):
    if internal_dims != 32:
        raise ValueError("MLPTexture3D: internal_dims %r is not provided; %s" % (internal_dims, _SUPPORTED))
    if not (isinstance(hidden, int) and 1 <= hidden <= 4):
        raise ValueError("MLPTexture3D: hidden %r is not provided; %s" % (hidden, _SUPPORTED))
    if not (isinstance(channels, int) and 1 <= channels <= 8):
        raise ValueError("MLPTexture3D: channels %r is not provided; %s" % (channels, _SUPPORTED))


class _MLP(torch.nn.Module):
    """The reference's `_MLP` parameters: `net` is a Sequential of bias-free Linear + ReLU, moved to the GPU, then kaiming-uniform
    initialised (render/mlptexture.py:18-41).  No backward hook: the fused kernel produces the hooks' gradients."""

    def __init__(self, cfg):
        super().__init__()
        net = (torch.nn.Linear(cfg["n_input_dims"], cfg["n_neurons"], bias=False), torch.nn.ReLU())
        for _ in range(cfg["n_hidden_layers"] - 1):
            net = net + (torch.nn.Linear(cfg["n_neurons"], cfg["n_neurons"], bias=False), torch.nn.ReLU())
        net = net + (torch.nn.Linear(cfg["n_neurons"], cfg["n_output_dims"], bias=False),)
        self.net = torch.nn.Sequential(*net).cuda()
        self.net.apply(self._init_weights)

    @staticmethod
    def _init_weights(m):
        if type(m) == torch.nn.Linear:
            torch.nn.init.kaiming_uniform_(m.weight, nonlinearity="relu")

    def weights(self):
        return [m.weight for m in self.net if isinstance(m, torch.nn.Linear)]


def _ptrs(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() if t is not None else None for t in tensors])


class _mlptex_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, params, aabb, min_max, lv, hidden, C, *weights):
        n = x.shape[0]
        out = torch.empty(n, C, dtype=torch.float32, device=x.device)
        enc = torch.empty(n, 32, dtype=torch.float32, device=x.device)
        _launch_fwd(x, params, aabb, min_max, lv, hidden, C, weights, out, enc)
        ctx.save_for_backward(x, params, aabb, min_max, enc, *weights)
        ctx.lv, ctx.hidden, ctx.C = lv, hidden, C
        return out

    @staticmethod
    def backward(ctx, d_out):
        x, params, aabb, min_max, enc, *weights = ctx.saved_tensors
        need_x, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_w = list(ctx.needs_input_grad[7:])
        n, hidden, C = x.shape[0], ctx.hidden, ctx.C
        d_x = torch.empty_like(x) if need_x else None
        d_p = torch.zeros_like(params) if need_p else None
        d_w = [torch.zeros_like(w) if nw else None for w, nw in zip(weights, need_w)]
        if n > 0 and (need_x or need_p or any(need_w)):
            ws = None
            if any(need_w):
                ws = torch.empty(max(1, L.lib().mcs_mlptex_workspace_bytes(n, hidden, C) // 4), dtype=torch.float32, device=x.device)
            g = d_out.to(torch.float32).contiguous()
            L.check(L.lib().mcs_mlptex_bwd(x.data_ptr(), n, aabb.data_ptr(), min_max.data_ptr(), params.data_ptr(), ctypes.byref(ctx.lv),
                                           hidden, C, _ptrs(weights), enc.data_ptr(), g.data_ptr(), d_p.data_ptr() if need_p else None,
                                           d_x.data_ptr() if need_x else None, _ptrs(d_w), ws.data_ptr() if ws is not None else None,
                                           L.stream_ptr()), "mlptex_bwd_dw" if any(need_w) else "mlptex_bwd")
            if need_p:
                d_p.mul_(GRADIENT_SCALING)
        return (d_x, d_p, None, None, None, None, None, *d_w)


class _mlptex_pair_func(torch.autograd.Function):
    """(x, x + off) through the MLP texture in one launch each way; d x = d_plain + d_jit, d off = d_jit, d W = d W plain + d W jit."""

    @staticmethod
    def forward(ctx, x, off, params, aabb, min_max, lv, hidden, C, *weights):
        n = x.shape[0]
        out, out_jit = [torch.empty(n, C, dtype=torch.float32, device=x.device) for _ in range(2)]
        enc, enc_jit = [torch.empty(n, 32, dtype=torch.float32, device=x.device) for _ in range(2)]
        _launch_pair_fwd(x, off, params, aabb, min_max, lv, hidden, C, weights, out, out_jit, enc, enc_jit)
        ctx.save_for_backward(x, off, params, aabb, min_max, enc, enc_jit, *weights)
        ctx.lv, ctx.hidden, ctx.C = lv, hidden, C
        ctx.set_materialize_grads(False)          # an unused output's gradient is passed to the kernel as null (zero)
        return out, out_jit

    @staticmethod
    def backward(ctx, d_out, d_out_jit):
        x, off, params, aabb, min_max, enc, enc_jit, *weights = ctx.saved_tensors
        need_x, need_o, need_p = ctx.needs_input_grad[:3]
        need_w = list(ctx.needs_input_grad[8:])
        n, hidden, C = x.shape[0], ctx.hidden, ctx.C
        d_x = torch.empty_like(x) if need_x else None
        d_o = torch.empty_like(off) if need_o else None
        d_p = torch.zeros_like(params) if need_p else None
        d_w = [torch.zeros_like(w) if nw else None for w, nw in zip(weights, need_w)]
        if n > 0 and (need_x or need_o or need_p or any(need_w)):
            ws = None
            if any(need_w):
                ws = torch.empty(max(1, 2 * L.lib().mcs_mlptex_workspace_bytes(n, hidden, C) // 4), dtype=torch.float32, device=x.device)
            g, gj = [d.to(torch.float32).contiguous() if d is not None else None for d in (d_out, d_out_jit)]
            ptr = lambda v: v.data_ptr() if v is not None else None
            L.check(L.lib().mcs_mlptex_pair_bwd(x.data_ptr(), off.data_ptr(), n, aabb.data_ptr(), min_max.data_ptr(), params.data_ptr(),
                                                ctypes.byref(ctx.lv), hidden, C, _ptrs(weights), enc.data_ptr(), enc_jit.data_ptr(), ptr(g),
                                                ptr(gj), ptr(d_p), ptr(d_x), ptr(d_o), _ptrs(d_w), ptr(ws), L.stream_ptr()),
                    "mlptex_pair_bwd_dw" if any(need_w) else "mlptex_pair_bwd")
            if need_p:
                d_p.mul_(GRADIENT_SCALING)
        return (d_x, d_o, d_p, None, None, None, None, None, *d_w)


def _launch_fwd(x, params, aabb, min_max, lv, hidden, C, weights, out, enc):
    if x.shape[0] == 0:                 # an empty tensor has no storage to point at
        return
    L.check(L.lib().mcs_mlptex_fwd(x.data_ptr(), x.shape[0], aabb.data_ptr(), min_max.data_ptr(), params.data_ptr(), ctypes.byref(lv), hidden, C,
                                   _ptrs(weights), out.data_ptr(), enc.data_ptr() if enc is not None else None, L.stream_ptr()), "mlptex_fwd")


def _launch_pair_fwd(x, off, params, aabb, min_max, lv, hidden, C, weights, out, out_jit, enc, enc_jit):
    if x.shape[0] == 0:
        return
    ptr = lambda v: v.data_ptr() if v is not None else None
    L.check(L.lib().mcs_mlptex_pair_fwd(x.data_ptr(), off.data_ptr(), x.shape[0], aabb.data_ptr(), min_max.data_ptr(), params.data_ptr(),
                                        ctypes.byref(lv), hidden, C, _ptrs(weights), out.data_ptr(), out_jit.data_ptr(), ptr(enc), ptr(enc_jit),
                                        L.stream_ptr()), "mlptex_pair_fwd")


class MLPTexture3D(torch.nn.Module):
    """The reference's `MLPTexture3D(AABB, channels=3, internal_dims=32, hidden=2, min_max=None)` on the current CUDA device.
    `sample(texc [..., 3])` -> [..., channels] fp32, differentiable in texc, `encoder.params` and every `net.net` weight.
    `sample_pair(texc, offset)` -> (sample(texc), sample(texc + offset)) in one launch each way, bit for bit."""

    def __init__(self, AABB, channels=3, internal_dims=32, hidden=2, min_max=None):
        super().__init__()
        _check_config(channels, internal_dims, hidden)
        self.channels = channels
        self.internal_dims = internal_dims
        self.AABB = AABB
        self.min_max = min_max

        desired_resolution, base_grid_resolution, num_levels = 4096, 16, 16
        per_level_scale = np.exp(np.log(desired_resolution / base_grid_resolution) / (num_levels - 1))
        enc_cfg = {"otype": "HashGrid", "n_levels": num_levels, "n_features_per_level": 2, "log2_hashmap_size": 19,
                   "base_resolution": base_grid_resolution, "per_level_scale": per_level_scale}
        self.encoder = tcnn.Encoding(3, enc_cfg)
        mlp_cfg = {"n_input_dims": self.encoder.n_output_dims, "n_output_dims": self.channels, "n_hidden_layers": hidden,
                   "n_neurons": self.internal_dims}
        self.net = _MLP(mlp_cfg)
        self.hidden = hidden

    def _operands(self, texc):
        if not isinstance(texc, torch.Tensor) or not texc.is_floating_point():
            raise TypeError("MLPTexture3D.sample: texc must be a floating-point tensor")
        if texc.dim() < 1 or texc.shape[-1] != 3:
            raise ValueError("MLPTexture3D.sample: texc must be [..., 3], got %s" % (tuple(texc.shape),))
        if self.min_max is None:
            raise ValueError("MLPTexture3D.sample: min_max is not set")
        dev = self.encoder.params.device
        aabb = torch.stack([torch.as_tensor(self.AABB[0]), torch.as_tensor(self.AABB[1])]).to(dev, torch.float32).contiguous()
        mm = torch.stack([torch.as_tensor(self.min_max[0]), torch.as_tensor(self.min_max[1])]).to(dev, torch.float32).contiguous()
        if aabb.shape != (2, 3) or mm.shape != (2, self.channels):
            raise ValueError("MLPTexture3D.sample: AABB must be [2,3] and min_max [2,%d]" % self.channels)
        weights = self.net.weights()
        for w in weights + [self.encoder.params]:
            if w.dtype != torch.float32 or not w.is_contiguous() or w.device != dev:
                raise ValueError("MLPTexture3D: parameters must stay contiguous fp32 tensors on %s" % dev)
        L.require_cuda(texc, self.encoder.params)
        return aabb, mm, weights

    def sample(self, texc):
        aabb, mm, weights = self._operands(texc)
        x = texc.reshape(-1, 3).to(torch.float32).contiguous()
        params, lv, C = self.encoder.params, self.encoder._lv, self.channels
        if torch.is_grad_enabled() and (x.requires_grad or params.requires_grad or any(w.requires_grad for w in weights)):
            out = _mlptex_func.apply(x, params, aabb, mm, lv, self.hidden, C, *weights)
        else:
            out = torch.empty(x.shape[0], C, dtype=torch.float32, device=x.device)
            _launch_fwd(x, params, aabb, mm, lv, self.hidden, C, weights, out, None)
        return out.view(*texc.shape[:-1], C)

    def sample_pair(self, texc, offset):
        """(sample(texc), sample(texc + offset)) -- render.py:63-64's plain and jittered samples of every pixel -- evaluated together:
        one forward and one backward launch (plus the d W sum), bit for bit the two calls' outputs and their gradients summed by
        autograd (d texc = d_plain + d_jit, d offset = d_jit, d W = d W plain + d W jit; d params as float atomics, like sample's).
        texc and offset: [..., 3] of the same shape, floating point, on one device; the jittered point is fp32(texc) + fp32(offset)."""
        for name, v in (("texc", texc), ("offset", offset)):
            if not isinstance(v, torch.Tensor) or not v.is_floating_point():
                raise ValueError("MLPTexture3D.sample_pair: %s must be a floating-point tensor" % name)
        if texc.shape != offset.shape:
            raise ValueError("MLPTexture3D.sample_pair: texc %s and offset %s differ in shape" % (tuple(texc.shape), tuple(offset.shape)))
        if texc.dim() < 1 or texc.shape[-1] != 3:
            raise ValueError("MLPTexture3D.sample_pair: texc and offset must be [..., 3], got %s" % (tuple(texc.shape),))
        if offset.device != texc.device:
            raise ValueError("MLPTexture3D.sample_pair: offset is on %s, texc on %s" % (offset.device, texc.device))
        aabb, mm, weights = self._operands(texc)
        x = texc.reshape(-1, 3).to(torch.float32).contiguous()
        off = offset.reshape(-1, 3).to(torch.float32).contiguous()
        params, lv, C = self.encoder.params, self.encoder._lv, self.channels
        if torch.is_grad_enabled() and (x.requires_grad or off.requires_grad or params.requires_grad or any(w.requires_grad for w in weights)):
            out, out_jit = _mlptex_pair_func.apply(x, off, params, aabb, mm, lv, self.hidden, C, *weights)
        else:
            out, out_jit = [torch.empty(x.shape[0], C, dtype=torch.float32, device=x.device) for _ in range(2)]
            _launch_pair_fwd(x, off, params, aabb, mm, lv, self.hidden, C, weights, out, out_jit, None, None)
        shape = (*texc.shape[:-1], C)
        return out.view(shape), out_jit.view(shape)

    def clamp_(self):
        pass

    def cleanup(self):
        tcnn.free_temporary_memory()
