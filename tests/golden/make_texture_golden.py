"""Generates tests/golden/ref_texture2d.npz by running the UNMODIFIED reference `render/texture.py` and `render/light.py` on the CPU.

  * the reference modules are imported through tests/refshade.py's `reference_render` (stub nvdiffrast, CPU redirection), unedited;
  * the stub's `dr.texture` is replaced by an autograd function with nvdiffrast's signature computing on the fp32 oracle
    (oracle/texture.c: forward, d tex per level, d uv, d uv_da);
  * `texture2d_mip.backward` builds its look-up grid with `torch.linspace(..., device="cuda")`; that factory is redirected to the CPU
    for the duration of the run;
  * `texc` / `texc_deriv` are render_layer's `gb_texc` / `gb_texc_deriv` from ref_render_layer_db.npz, the derivatives scaled per pixel by
    2^s, s uniform in [-2, 8], so that every level of the chains and both clamps of the level of detail are used.

Cases (outputs, and for the Texture2D cases the gradients to every level, texc and texc_deriv for a seeded upstream gradient):
  auto   Texture2D(32 x 96 x 4).sample: the automatic chain of texture2d_mip (avg_pool, 32 x 96 down to 1 x 3), whose backward reaches the
         base texture through the reference's own `dr.texture(dout * 0.25, uv, filter_mode='linear', boundary_mode='clamp')`.  That
         backward returns twice the pooled size, so it only differentiates chains whose pooled levels are even in both sides (48 x 80
         pools 3 x 5 into 1 x 2 and fails inside the reference);
  custom create_trainable(48 x 80 x 4, auto_mipmaps=False).sample: a custom chain, gradients to every level;
  const  Texture2D(constant of 3).sample: a 1x1 texture (mip=None);
  env    EnvironmentLight(base 16 x 32 x 3).generate_image((12, 20)): 'linear', 'wrap'; forward only (the reference decorates it, as
         its probe loader, with @torch.no_grad()).
    python tests/golden/make_texture_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_texture2d.npz")
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

AUTO_HW = (32, 96)
TEX_HW = (48, 80)
ENV_RES = (12, 20)


def inputs():
    """texc [2,24,32,2], texc_deriv [2,24,32,4] (fp32), the base textures and upstream gradients, all seeded."""
    d = np.load(os.path.join(HERE, "ref_render_layer_db.npz"))
    rng = np.random.default_rng(2024)
    texc = d["gb_texc"].astype(np.float32)
    s = rng.uniform(-2.0, 8.0, texc.shape[:3] + (1,))
    deriv = (d["gb_texc_deriv"] * 2.0 ** s).astype(np.float32)
    base = rng.uniform(0, 1, TEX_HW + (4,)).astype(np.float32)
    auto = rng.uniform(0, 1, AUTO_HW + (4,)).astype(np.float32)
    const = np.array([0.25, 0.5, 0.75], np.float32)
    env = rng.uniform(0, 2, (16, 32, 3)).astype(np.float32)
    g = {k: rng.normal(size=texc.shape[:3] + (c,)).astype(np.float32) for k, c in (("auto", 4), ("custom", 4), ("const", 3))}
    return texc, deriv, auto, base, const, env, g


def oracle_texture():
    """nvdiffrast's `texture` signature on the fp32 oracle (CPU tensors), differentiable in tex, every mip level, uv and uv_da."""
    from oracle.texture import texture_oracle
    o = texture_oracle()

    class Fn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, filter_mode, boundary_mode, uv, uv_da, *levels):
            ctx.save_for_backward(uv, uv_da, *levels)
            ctx.modes = (filter_mode, boundary_mode)
            n = [t.detach().numpy() for t in levels]
            return torch.from_numpy(o.forward(n, uv.detach().numpy(), None if uv_da is None else uv_da.detach().numpy(), filter_mode, boundary_mode))

        @staticmethod
        def backward(ctx, dout):
            uv, uv_da, *levels = ctx.saved_tensors
            f, b = ctx.modes
            dt, duv, dda = o.backward([t.detach().numpy() for t in levels], uv.detach().numpy(), None if uv_da is None else uv_da.detach().numpy(),
                                      dout.contiguous().numpy(), f, b)
            if f == "linear":
                dt = dt + [None] * (len(levels) - 1)
            return (None, None, torch.from_numpy(duv), None if dda is None else torch.from_numpy(dda), *[None if t is None else torch.from_numpy(t) for t in dt])

    def texture(tex, uv, uv_da=None, mip_level_bias=None, mip=None, filter_mode='auto', boundary_mode='wrap', max_mip_level=None):
        assert mip_level_bias is None and max_mip_level is None
        if filter_mode == 'auto':
            filter_mode = 'linear-mipmap-linear' if uv_da is not None else 'linear'
        levels = [tex] + (list(mip) if mip is not None and filter_mode != 'linear' else [])
        return Fn.apply(filter_mode, boundary_mode, uv, uv_da if filter_mode != 'linear' else None, *levels)
    return texture


def generate():
    from refshade import reference_render
    import importlib
    texc, deriv, auto, base, const, env, g = inputs()
    out = {"texc": texc, "texc_deriv": deriv, "auto_base": auto, "base": base, "const": const, "env_base": env}
    for k, v in g.items():
        out["dout_" + k] = v
    linspace = torch.linspace

    def cpu_linspace(*a, **k):
        if str(k.get("device", "")).startswith("cuda"):
            k["device"] = "cpu"
        return linspace(*a, **k)

    empty = type(sys)("unused_backend")
    with reference_render(empty, empty) as (render, light, _den):
        tex_mod = importlib.import_module("render.texture")
        tex_mod.dr.texture = oracle_texture()
        torch.linspace = cpu_linspace
        try:
            for case in ("auto", "custom", "const"):
                uv = torch.from_numpy(texc).requires_grad_(True)
                da = torch.from_numpy(deriv).requires_grad_(True)
                if case == "auto":
                    leaf = torch.from_numpy(auto).requires_grad_(True)
                    t = tex_mod.Texture2D(leaf)                      # holds leaf[None]: the gradient lands on the leaf
                elif case == "custom":
                    t = tex_mod.create_trainable(torch.from_numpy(base), auto_mipmaps=False)
                else:
                    t = tex_mod.Texture2D(const.copy())
                    t.data.requires_grad_(True)
                y = t.sample(uv, da)
                y.backward(torch.from_numpy(g[case]))
                out["out_" + case] = y.detach().numpy()
                out["d_texc_" + case] = uv.grad.numpy()
                out["d_texc_deriv_" + case] = da.grad.numpy()
                for k, m in enumerate(t.getMips()):
                    out["d_level%d_%s" % (k, case)] = (leaf.grad[None] if case == "auto" else m.grad).numpy()
                    if case == "custom":
                        out["level%d_custom" % k] = m.detach().numpy()
            out["out_env"] = light.EnvironmentLight(torch.from_numpy(env)).generate_image(list(ENV_RES)).numpy()
        finally:
            torch.linspace = linspace
    return out


if __name__ == "__main__":
    d = generate()
    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", ", ".join("%s %s" % (k, v.shape) for k, v in sorted(d.items())))
