"""Multiresolution hash-grid encoding: a stand-in for the part of tiny-cuda-nn the reference's `MLPTexture3D` uses
(render/mlptexture.py:11,57-73,103; train.py:443 reads `encoder.params.grad`).

`Encoding(3, {"otype": "HashGrid", ...})` is an `nn.Module` with a flat fp32 `params` parameter and a forward that maps points
`x [N,3]` (normally in [0,1]^3) to `[N, 2 * n_levels]` fp32 features, differentiable in `x` and `params`, through the CUDA kernels of
csrc/hashgrid.cu (semantics stated there).  With `sys.modules["tinycudann"] = nvdiffrecmc_b200.tinycudann` the reference's
`render/mlptexture.py` runs unmodified.  Only the configuration the reference uses is supported: 3 input dimensions, 2 features per
level, linear interpolation.  Everything is fp32 (tiny-cuda-nn computes in fp16); the parameters are initialised uniformly in
[-1e-4, 1e-4] from a CPU generator, so they are the same on every machine, but they are not tiny-cuda-nn's values.
"""
import ctypes
import math

import torch

from .. import _lib as L

__all__ = ["Encoding", "free_temporary_memory", "level_table"]

_SUPPORTED = ("supported: otype 'HashGrid' with n_input_dims 3, n_features_per_level 2, interpolation 'Linear', n_levels 1..16")


def level_table(n_levels, log2_hashmap_size, base_resolution, per_level_scale):
    """The level geometry as a dict of Python lists (offset has n_levels + 1 entries), computed in double precision:
    scale_l = fl32(base * per_level_scale^l - 1), res_l = ceil(scale_l) + 1, size_l = min(next_multiple_of_8(res_l^3), 2^log2) (2^log2
    if res_l^3 >= 2^31), dense iff res_l^3 <= size_l."""
    import numpy as np
    cap = 1 << int(log2_hashmap_size)
    offset, res, scale, dense_mask = [0], [], [], 0
    for l in range(n_levels):
        s = float(np.float32(float(base_resolution) * math.pow(float(per_level_scale), l) - 1.0))
        r = int(math.ceil(s)) + 1
        r3 = r ** 3
        size = cap if r3 >= 1 << 31 else min((r3 + 7) // 8 * 8, cap)
        if r3 <= size:
            dense_mask |= 1 << l
        offset.append(offset[-1] + size)
        res.append(r)
        scale.append(s)
    return {"n_levels": n_levels, "offset": offset, "res": res, "scale": scale, "dense_mask": dense_mask}


def _c_levels(t):
    lv = L.mcs_hashgrid_levels()
    lv.n_levels = t["n_levels"]
    for l in range(t["n_levels"]):
        lv.res[l] = t["res"][l] & 0xFFFFFFFF
        lv.scale[l] = t["scale"][l]
    for l, o in enumerate(t["offset"]):
        lv.offset[l] = o
    lv.dense_mask = t["dense_mask"]
    return lv


def _parse(n_input_dims, cfg):
    cfg = dict(cfg)
    if cfg.get("otype") != "HashGrid":
        raise ValueError("tinycudann.Encoding: otype %r is not provided; %s" % (cfg.get("otype"), _SUPPORTED))
    if n_input_dims != 3:
        raise ValueError("tinycudann.Encoding: n_input_dims %r is not provided; %s" % (n_input_dims, _SUPPORTED))
    if cfg.get("n_features_per_level", 2) != 2:
        raise ValueError("tinycudann.Encoding: n_features_per_level %r is not provided; %s" % (cfg["n_features_per_level"], _SUPPORTED))
    if cfg.get("interpolation", "Linear") != "Linear":
        raise ValueError("tinycudann.Encoding: interpolation %r is not provided; %s" % (cfg["interpolation"], _SUPPORTED))
    n_levels, log2 = int(cfg.get("n_levels", 16)), int(cfg.get("log2_hashmap_size", 19))
    base, pls = float(cfg.get("base_resolution", 16)), float(cfg.get("per_level_scale", 2.0))
    if not 1 <= n_levels <= 16:
        raise ValueError("tinycudann.Encoding: n_levels %d is not provided; %s" % (n_levels, _SUPPORTED))
    if not 3 <= log2 <= 27:
        raise ValueError("tinycudann.Encoding: log2_hashmap_size must be in 3..27 (got %d)" % log2)
    if not (math.isfinite(base) and math.isfinite(pls) and base > 0 and pls > 0):
        raise ValueError("tinycudann.Encoding: base_resolution and per_level_scale must be finite and positive")
    t = level_table(n_levels, log2, base, pls)
    if t["offset"][-1] * 2 >= 1 << 32:
        raise ValueError("tinycudann.Encoding: the table has %d entries, more than the 2^31 the kernels index" % t["offset"][-1])
    return t


def init_params(n_params, seed=1337):
    """Uniform in [-1e-4, 1e-4] from a CPU generator (identical on every machine)."""
    g = torch.Generator().manual_seed(int(seed))
    return (torch.rand(n_params, generator=g, dtype=torch.float32) * 2.0 - 1.0) * 1e-4


class _hashgrid_func(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, params, lv):
        n = x.shape[0]
        out = torch.empty(n, 2 * lv.n_levels, dtype=torch.float32, device=x.device)
        if n > 0:                  # an empty tensor has no storage to point at
            L.check(L.lib().mcs_hashgrid_fwd(x.data_ptr(), n, params.data_ptr(), ctypes.byref(lv), out.data_ptr(), L.stream_ptr()), "hashgrid_fwd")
        ctx.save_for_backward(x, params)
        ctx.lv = lv
        return out

    @staticmethod
    def backward(ctx, d_out):
        x, params = ctx.saved_tensors
        need_x, need_p = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_x or need_p):
            return None, None, None
        if x.shape[0] == 0:
            return torch.zeros_like(x) if need_x else None, torch.zeros_like(params) if need_p else None, None
        g = d_out.to(torch.float32).contiguous()
        d_x = torch.empty_like(x) if need_x else None
        d_p = torch.zeros_like(params) if need_p else None
        L.check(L.lib().mcs_hashgrid_bwd(x.data_ptr(), x.shape[0], params.data_ptr(), ctypes.byref(ctx.lv), g.data_ptr(),
                                         d_p.data_ptr() if need_p else None, d_x.data_ptr() if need_x else None, L.stream_ptr()),
                "hashgrid_bwd_both" if need_x and need_p else "hashgrid_bwd")
        return d_x, d_p, None


class Encoding(torch.nn.Module):
    """tiny-cuda-nn's `Encoding(n_input_dims, encoding_config, seed=1337, dtype=None)` for `otype: "HashGrid"` on the current CUDA
    device.  `params` is the flat fp32 table (2 features per entry, tiny-cuda-nn's layout); `forward(x [N,3])` returns [N, n_output_dims]
    fp32."""

    def __init__(self, n_input_dims, encoding_config, seed=1337, dtype=None):
        super().__init__()
        if dtype not in (None, torch.float32):
            raise ValueError("tinycudann.Encoding: dtype %r is not provided; params and outputs are fp32" % (dtype,))
        self.n_input_dims = n_input_dims
        self.encoding_config = dict(encoding_config)
        self.levels = _parse(n_input_dims, encoding_config)
        self._lv = _c_levels(self.levels)
        self.n_output_dims = 2 * self.levels["n_levels"]
        self.seed = seed
        dev = torch.device("cuda", torch.cuda.current_device())
        self.params = torch.nn.Parameter(init_params(2 * self.levels["offset"][-1], seed).to(dev))

    def forward(self, x):
        if not isinstance(x, torch.Tensor):
            raise TypeError("tinycudann.Encoding: x must be a tensor")
        L.require_cuda(x, self.params)
        if not x.is_floating_point():
            raise TypeError("tinycudann.Encoding: x must be floating point, got %s" % x.dtype)
        if x.dim() != 2 or x.shape[1] != self.n_input_dims:
            raise ValueError("tinycudann.Encoding: x must be [N,%d], got %s" % (self.n_input_dims, tuple(x.shape)))
        if self.params.dtype != torch.float32 or self.params.dim() != 1 or not self.params.is_contiguous():
            raise ValueError("tinycudann.Encoding: params must stay a contiguous flat fp32 tensor")
        if self.params.numel() != 2 * self.levels["offset"][-1]:
            raise ValueError("tinycudann.Encoding: params has %d values, the table needs %d" % (self.params.numel(), 2 * self.levels["offset"][-1]))
        if x.device != self.params.device:
            raise ValueError("tinycudann.Encoding: x is on %s, params on %s" % (x.device, self.params.device))
        return _hashgrid_func.apply(x.to(torch.float32).contiguous(), self.params, self._lv)

    def extra_repr(self):
        return "n_input_dims=%d, n_output_dims=%d, params=%d" % (self.n_input_dims, self.n_output_dims, self.params.numel())


def free_temporary_memory():
    """tiny-cuda-nn releases its scratch arenas here; these kernels allocate nothing beyond the caller's tensors."""
