"""Freeze the reference's jittered regulariser taps into tests/golden/ref_jitter_taps.npz: the reference's own shade() (render/render.py:30-164,
imported UNMODIFIED through tests/refshade.reference_render and run on the CPU with autograd on) produces kd_grad, ks_grad, normal_grad
and perturbed_nrm_grad; this script records the torch.normal draws shade() makes (the uv offset, and the MLP path's position noise), the
jitter its first texture tap reads, the four buffers, and the autograd gradients of sum_k <G_k, buffer_k> over those four buffers only,
for fixed upstream gradients G_k.

shade() runs with bsdf='kd', which shades with kd alone, so neither env_shade nor the denoiser is called; the taps do not depend on the
BSDF.  nvdiffrast's texture is refshade's grid_sample stub (bilinear, clamped borders); its texel coordinate is ((2u - 1) + 1) W / 2 - 0.5
rather than u W - 0.5, so the taps match the contract's to a few ulp of the coordinate, not bit for bit.

Cases, each [2, 13, 19] (non-square, odd, B = 2), coverage about 70 % with the borders partly covered:
  * "kd3":      texture path, kd of 3 channels, no normal map;
  * "kd4_nrm":  texture path, kd of 4 channels (alpha), with a normal map;
  * "kd3_nrm":  texture path, kd of 3 channels, with a normal map;
  * "mlp":      the MLP path, material['kd_ks'] a smooth deterministic function of the position (6 channels).
ks is always the [..., 0:3] slice of a 4-channel sample, as shade() takes it.
Run: python tests/golden/make_taps_golden.py   (only where the reference checkout exists)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refshade  # noqa: E402

OUT = os.path.join(HERE, "ref_jitter_taps.npz")
B, H, W = 2, 13, 19
CASES = {"kd3": (3, False, False), "kd4_nrm": (4, True, False), "kd3_nrm": (3, True, False), "mlp": (3, False, True)}
BUFFERS = ["kd_grad", "ks_grad", "normal_grad", "perturbed_nrm_grad"]


def _unit(rng, shape, z=0.0):
    v = rng.normal(size=shape).astype(np.float32)
    v[..., 2] += z
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)


class _Tex:
    def __init__(self, img):
        self.img = img

    def sample(self, texc, texc_deriv, filter_mode='linear-mipmap-linear'):
        return self.img


class _KdKs:
    """A smooth deterministic 6-channel field of the position; every sample is returned as a fresh leaf, so its gradient is recorded."""
    M = torch.tensor(np.random.default_rng(7).normal(size=(3, 6)).astype(np.float32) * 3.0)

    def __init__(self):
        self.calls = []

    def sample(self, x):
        out = (0.5 + 0.4 * torch.sin(x.detach() @ self.M + 0.3)).requires_grad_(True)
        self.calls.append(out)
        return out


def make_case(name, seed):
    ckd, nrm_map, mlp = CASES[name]
    rng = np.random.default_rng(seed)
    cov = rng.random((B, H, W)) < 0.7
    rast = np.zeros((B, H, W, 4), np.float32)
    rast[..., 0:2] = rng.random((B, H, W, 2))
    rast[..., 2] = rng.random((B, H, W))
    rast[..., 3] = np.where(cov, rng.integers(1, 50, (B, H, W)), 0).astype(np.float32)
    inp = dict(rast=rast, gb_depth=np.stack([rng.random((B, H, W)), np.full((B, H, W), 0.01)], -1).astype(np.float32),
               gb_pos=rng.normal(size=(B, H, W, 3)).astype(np.float32), gb_geometric_normal=_unit(rng, (B, H, W, 3)),
               gb_normal=_unit(rng, (B, H, W, 3)), gb_tangent=_unit(rng, (B, H, W, 3)),
               view_pos=rng.normal(size=(B, 1, 1, 3)).astype(np.float32) * 3,
               kd=rng.random((B, H, W, ckd)).astype(np.float32), ks4=rng.random((B, H, W, 4)).astype(np.float32))
    if nrm_map:
        inp["perturbed_nrm"] = _unit(rng, (B, H, W, 3), z=1.5)
    G = {k: rng.normal(size=(B, H, W, ckd + 1 if k == "kd_grad" else 4)).astype(np.float32) for k in BUFFERS}
    return inp, G


def run_case(name, seed):
    ckd, nrm_map, mlp = CASES[name]
    inp, G = make_case(name, seed)
    torch.manual_seed(seed)
    ou, ru = refshade.oracle_backends(None, None)
    leaf = lambda k: torch.tensor(inp[k]).requires_grad_(True)
    kd, ks4, nrm = leaf("kd"), leaf("ks4"), leaf("gb_normal")
    pn = leaf("perturbed_nrm") if nrm_map else None
    kdks = _KdKs()
    if mlp:
        material = {"bsdf": "kd", "kd_ks": kdks}
    else:
        material = {"bsdf": "kd", "kd": _Tex(kd), "ks": _Tex(ks4)}
        if nrm_map:
            material["normal"] = _Tex(pn)
    draws, uvs = [], []
    with refshade.reference_render(ou, ru) as (render, light, den):
        normal, dr = torch.normal, sys.modules["nvdiffrast.torch"]
        texture = dr.texture

        def rec_normal(*a, **k):
            out = normal(*a, **k)
            draws.append(out.detach().clone())
            return out

        def rec_texture(tex, uv, *a, **k):
            uvs.append(uv.detach().clone())
            return texture(tex, uv, *a, **k)
        torch.normal, dr.texture = rec_normal, rec_texture
        try:
            t = lambda k: torch.tensor(inp[k])
            texc = torch.zeros(B, H, W, 2)
            buffers = render.shade(refshade._Flags(), t("rast"), t("gb_depth"), t("gb_pos"), t("gb_geometric_normal"), nrm, t("gb_tangent"),
                                   texc, texc, t("view_pos"), None, material, None, None, None, None, 1.0)
        finally:
            torch.normal = normal
    names = BUFFERS if nrm_map else BUFFERS[:3]
    loss = sum((buffers[k] * torch.tensor(G[k])).sum() for k in names)
    loss.backward()
    out = {"rast": inp["rast"], "jitter": uvs[0].numpy(), "offset": draws[0].numpy(), "gb_normal": inp["gb_normal"],
           "d_gb_normal": nrm.grad.numpy()}
    if mlp:
        J, T = kdks.calls
        out.update(pos_noise=draws[1].numpy(), kd=T.detach()[..., 0:3].numpy(), ks=T.detach()[..., 3:6].numpy(),
                   kd_jitter=J.detach()[..., 0:3].numpy(), ks_jitter=J.detach()[..., 3:6].numpy(), d_kd=T.grad[..., 0:3].numpy(),
                   d_ks=T.grad[..., 3:6].numpy(), d_kd_jitter=J.grad[..., 0:3].numpy(), d_ks_jitter=J.grad[..., 3:6].numpy())
    else:
        out.update(kd=inp["kd"], ks=inp["ks4"][..., 0:3], d_kd=kd.grad.numpy(), d_ks=ks4.grad[..., 0:3].numpy())
        if nrm_map:
            out.update(perturbed_nrm=inp["perturbed_nrm"], d_perturbed_nrm=pn.grad.numpy())
    for k in names:
        out[k] = buffers[k].detach().numpy()
        out["G_" + k] = G[k]
    return {"%s/%s" % (name, k): np.ascontiguousarray(v, np.float32) for k, v in out.items()}


def main():
    data = {}
    for seed, name in enumerate(CASES):
        data.update(run_case(name, 100 + seed))
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, len(data), "arrays")


if __name__ == "__main__":
    main()
