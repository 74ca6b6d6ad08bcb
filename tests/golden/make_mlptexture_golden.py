"""Generates tests/golden/ref_mlptexture.npz by running the UNMODIFIED reference `render/mlptexture.py` (MLPTexture3D) on the CPU.

  * `tinycudann` is a stand-in backed by the fp32 CPU oracle of the hash-grid encoding (oracle/hashgrid.c), with the contract's
    parameter initialisation (seed 1337);
  * `.cuda()` on modules is redirected to the CPU for the duration of the run (the reference moves its MLP to 'cuda', mlptexture.py:27);
  * the texture has the reference's hard-coded configuration (16 levels, 2^19, base 16, 6 channels as train.py:162-166 builds it),
    256 points partly outside the AABB (so the clamp of `sample()` is exercised) and a seeded upstream gradient.

Stored: the MLP weights, AABB, min_max, points, `sample()` output, upstream gradient, `d points`, `d` of every MLP weight and
`encoder.params.grad` after the reference's backward hooks (x128 through the MLP's input hook, /128 on the encoder's input), the last
as its nonzero (index, value) pairs.  Nothing from the reference is copied into this repository.
    python tests/golden/make_mlptexture_golden.py
"""
import contextlib
import importlib
import os
import sys
import types

import numpy as np
import torch

REF = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_mlptexture.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def oracle_tinycudann():
    """A `tinycudann` module with the surface mlptexture.py uses, computing on CPU tensors through the fp32 oracle."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle.hashgrid import hashgrid_oracle, init_params
    orc = hashgrid_oracle()
    m = types.ModuleType("oracle_tinycudann")

    class _F(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, params, lv):
            ctx.save_for_backward(x, params)
            ctx.lv = lv
            return torch.from_numpy(orc.forward(x.detach().numpy(), params.detach().numpy(), lv))

        @staticmethod
        def backward(ctx, dy):
            x, params = ctx.saved_tensors
            dp, dx = orc.backward(x.numpy(), params.detach().numpy(), ctx.lv, dy.contiguous().numpy())
            return torch.from_numpy(dx), torch.from_numpy(dp), None

    class Encoding(torch.nn.Module):
        def __init__(self, n_input_dims, encoding_config, seed=1337, dtype=None):
            super().__init__()
            assert n_input_dims == 3 and encoding_config["otype"] == "HashGrid" and encoding_config["n_features_per_level"] == 2
            self.lv = orc.levels(encoding_config)
            self.n_input_dims, self.n_output_dims = 3, 2 * self.lv["n_levels"]
            self.params = torch.nn.Parameter(torch.from_numpy(init_params(2 * int(self.lv["offset"][-1]), seed)))

        def forward(self, x):
            return _F.apply(x.to(torch.float32).contiguous(), self.params, self.lv)

    m.Encoding = Encoding
    m.free_temporary_memory = lambda: None
    return m


@contextlib.contextmanager
def reference_mlptexture(tcnn):
    """Yields the reference's render/mlptexture.py imported with `tcnn` as `tinycudann`; module `.cuda()` is a no-op without a GPU."""
    saved = {k: sys.modules.get(k) for k in ("tinycudann", "render", "render.mlptexture")}
    for k in saved:
        sys.modules.pop(k, None)
    sys.modules["tinycudann"] = tcnn
    sys.path.insert(0, REF)
    cuda = torch.nn.Module.cuda
    if not torch.cuda.is_available():
        torch.nn.Module.cuda = lambda self, device=None: self
    try:
        yield importlib.import_module("render.mlptexture")
    finally:
        torch.nn.Module.cuda = cuda
        sys.path.remove(REF)
        for k in ("tinycudann", "render", "render.mlptexture"):
            sys.modules.pop(k, None)
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v


def generate():
    with reference_mlptexture(oracle_tinycudann()) as mt:
        torch.manual_seed(0)                                    # kaiming_uniform_ of the MLP weights (mlptexture.py:29,38)
        aabb = torch.tensor([[-1.0, -0.5, -0.8], [1.1, 0.9, 0.7]])
        min_max = [torch.tensor([0.0, 0.0, 0.0, 0.0, 0.08, 0.0]), torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, 1.0])]
        tex = mt.MLPTexture3D(aabb, channels=6, min_max=min_max)
        g = torch.Generator().manual_seed(7)
        pts = (torch.rand(256, 3, generator=g) * 1.2 - 0.1) * (aabb[1] - aabb[0]) + aabb[0]
        pts = pts.reshape(1, 16, 16, 3).requires_grad_(True)
        out = tex.sample(pts)
        dout = torch.randn(out.shape, generator=g)
        out.backward(dout)
        pg = tex.encoder.params.grad
        nz = torch.nonzero(pg).reshape(-1)
        d = {"aabb": aabb.numpy(), "min_max": torch.stack(min_max).numpy(), "points": pts.detach().numpy(), "out": out.detach().numpy(),
             "dout": dout.numpy(), "d_points": pts.grad.numpy(), "params_grad_idx": nz.numpy().astype(np.int32),
             "params_grad_val": pg[nz].numpy(), "params_head": tex.encoder.params.detach()[:8].numpy()}
        lin = [m for m in tex.net.net if isinstance(m, torch.nn.Linear)]
        for k, m in enumerate(lin):
            d["w%d" % k] = m.weight.detach().numpy()
            d["d_w%d" % k] = m.weight.grad.numpy()
    return d


if __name__ == "__main__":
    d = generate()
    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(d["params_grad_idx"]), "nonzero params.grad entries")
