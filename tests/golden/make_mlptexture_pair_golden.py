"""Generates tests/golden/ref_mlptexture_pair.npz by running the UNMODIFIED reference `render/mlptexture.py` (MLPTexture3D) on the CPU,
with render.py:63-64's two lines -- the jittered sample and the plain sample of every pixel -- executed as the reference writes them.

  * `tinycudann` and `.cuda()` as in make_mlptexture_golden.py (the fp32 hash-grid oracle, the contract's initialisation, seed 1337);
  * gb_pos is a 2 x 13 x 19 G-buffer: covered pixels on a sphere cap partly outside the AABB (so the clamp is exercised), uncovered ones
    at the origin, as interpolate leaves them; it requires grad;
  * the noise is one frozen draw of N(0, 0.01) (render.py draws it with torch.normal on the GPU);
  * both samples get a seeded upstream gradient, zero at uncovered pixels (composite_buffer blends them with alpha 0), which also keeps
    the nonzero d params few enough for a small fixture.

Stored: the MLP weights, AABB, min_max, gb_pos, the noise, both upstream gradients, both samples, gb_pos.grad, `d` of every MLP weight
and `encoder.params.grad` after the reference's hooks, the last as its nonzero (index, value) pairs.  Nothing from the reference is
copied into this repository.
    python tests/golden/make_mlptexture_pair_golden.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_mlptexture_golden import oracle_tinycudann, reference_mlptexture  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_mlptexture_pair.npz")
B, H, W = 2, 13, 19


def gbuffer(g, aabb):
    """gb_pos [B,H,W,3] and coverage [B,H,W]: a sphere cap seen from two views, 0 where uncovered."""
    v, u = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    pos = torch.zeros(B, H, W, 3)
    cov = torch.zeros(B, H, W, dtype=torch.bool)
    for b in range(B):
        cx, cy, r = (-0.3, 0.1, 0.42) if b == 0 else (0.35, -0.2, 0.38)
        du, dv = (u - cx) / r, (v - cy) / r
        inside = du * du + dv * dv < 1
        dz = torch.sqrt(torch.clamp(1 - du * du - dv * dv, min=0))
        p = torch.stack([du, dv, dz], -1) * (0.6 + 0.1 * b) + torch.tensor([0.1, 0.2, -0.3 + 0.2 * b])
        p = p + 0.002 * torch.randn(p.shape, generator=g)
        pos[b][inside] = p[inside]
        cov[b] = inside
    return pos, cov


def generate():
    with reference_mlptexture(oracle_tinycudann()) as mt:
        torch.manual_seed(0)                                    # kaiming_uniform_ of the MLP weights
        aabb = torch.tensor([[-1.0, -0.5, -0.8], [1.1, 0.9, 0.7]])
        min_max = [torch.tensor([0.0, 0.0, 0.0, 0.0, 0.08, 0.0]), torch.tensor([1.0, 1.0, 1.0, 1.0, 1.0, 1.0])]
        tex = mt.MLPTexture3D(aabb, channels=6, min_max=min_max)
        g = torch.Generator().manual_seed(11)
        pos, cov = gbuffer(g, aabb)
        gb_pos = pos.clone().requires_grad_(True)
        noise = torch.normal(mean=0, std=0.01, size=gb_pos.shape, generator=g)
        material = {"kd_ks": tex}
        # render.py:63-64, the noise draw frozen
        all_tex_jitter = material['kd_ks'].sample(gb_pos + noise)
        all_tex = material['kd_ks'].sample(gb_pos)
        dout = torch.randn(all_tex.shape, generator=g) * cov[..., None]
        dout_jit = torch.randn(all_tex.shape, generator=g) * cov[..., None]
        torch.autograd.backward([all_tex_jitter, all_tex], [dout_jit, dout])
        pg = tex.encoder.params.grad
        nz = torch.nonzero(pg).reshape(-1)
        d = {"aabb": aabb.numpy(), "min_max": torch.stack(min_max).numpy(), "gb_pos": pos.numpy(), "noise": noise.numpy(),
             "dout": dout.numpy(), "dout_jit": dout_jit.numpy(), "out": all_tex.detach().numpy(), "out_jit": all_tex_jitter.detach().numpy(),
             "d_gb_pos": gb_pos.grad.numpy(), "params_grad_idx": nz.numpy().astype(np.int32), "params_grad_val": pg[nz].numpy(),
             "params_head": tex.encoder.params.detach()[:8].numpy()}
        lin = [m for m in tex.net.net if isinstance(m, torch.nn.Linear)]
        for k, m in enumerate(lin):
            d["w%d" % k] = m.weight.detach().numpy()
            d["d_w%d" % k] = m.weight.grad.numpy()
    return d


if __name__ == "__main__":
    d = generate()
    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(d["params_grad_idx"]), "nonzero params.grad entries;",
          int((d["dout"] != 0).any(-1).sum()), "covered pixels")
