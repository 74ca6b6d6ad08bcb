"""Times render_mesh's layer compositing: nvdiffrecmc_b200.raster.composite (csrc/composite.cu, one launch per layer each way) against
the reference's composite_buffer (render/render.py:284-291) run per key with torch.lerp and raster.antialias, on the bench mesh with rast at
8 x 512^2.

Four workloads: "pass1", render_layer's pass-1 buffer set (eleven 4-channel buffers) and one layer; "pass2", the pass-2 set (twelve
4-channel buffers and a 5-channel kd_grad) and 8 depth-peeled layers, as with transparency; and both again with spp = 2 ("pass1_spp2",
"pass2_spp2"): output 8 x 256^2, the buffers MSAA-shaded at 256^2 and the chain that of render_mesh with --spp 2 (render.py:247-250,
313-330), which upscales every buffer and the background nearest, composites at 512^2 and box-filters with avg_pool_nhwc.  Buffers are
random with fractional alphas and 'shaded' starts from a background.  Per workload: the forward under no_grad (the dataset's reference
render) and forward + backward of sum_k <G_k, out_k> into every buffer, the background and the clip-space positions.  Every timing is the
median of --reps CUDA-event timings of --inner calls each, the fused op and the chain alternating, in two runs; torch.cuda's peak
allocation of one call of each arm is reported beside them.  Before any time is quoted the two are checked to agree on the same inputs
(forward bit for bit, gradients to 1e-5 relative L2).  Prints one JSON document with the card's name and power limit, read in the same run.

    python tools/compbench.py [--reps 15] [--inner 3] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nvdiffrecmc_b200 import raster, synth  # noqa: E402
from tapbench import alternate, card  # noqa: E402

PASS1 = [(k, 4) for k in ("shaded", "z_grad", "normal", "geometric_normal", "kd", "ks", "kd_grad", "ks_grad", "normal_grad", "diffuse_light",
                          "specular_light")]
PASS2 = [(k, 5 if k == "kd_grad" else c) for k, c in PASS1] + [("perturbed_nrm", 4), ("perturbed_nrm_grad", 4)]


def up(x, H, W):
    """scale_img_nhwc(x, (H, W), mag='nearest') (render.py:247-250, 313-319); full-resolution tensors pass through"""
    if tuple(x.shape[1:3]) == (H, W):
        return x
    return torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), (H, W), mode="nearest").permute(0, 2, 3, 1).contiguous()


def chain(layers, pos, tri, background, topology, spp):
    """composite_buffer(key, layers, bg, True) for every key (render.py:321-330), raster.antialias for dr.antialias; with spp > 1 the
    buffers and background upscaled first and every key box-filtered by avg_pool_nhwc after"""
    H, W = layers[0][1].shape[1:3]
    out = {}
    for key in layers[0][0]:
        accum = up(background[key], H, W) if key in background else torch.zeros(*layers[0][1].shape[:3], layers[0][0][key].shape[3],
                                                                                  device=pos.device)
        for buffers, rast in reversed(layers):
            b = up(buffers[key], H, W)
            alpha = (rast[..., -1:] > 0).float() * b[..., -1:]
            accum = torch.lerp(accum, torch.cat((b[..., :-1], torch.ones_like(b[..., -1:])), dim=-1), alpha)
            accum = raster.antialias(accum.contiguous(), rast, pos, tri, topology)
        out[key] = torch.nn.functional.avg_pool2d(accum.permute(0, 3, 1, 2), spp).permute(0, 2, 3, 1).contiguous() if spp > 1 else accum
    return out


def fused(layers, pos, tri, background, topology, spp):
    return raster.composite(layers, pos, tri, background=background, topology=topology, spp=spp)


def inputs(spec, n_layers, spp, B=8, res=(512, 512), seed=0):
    """(layers, pos, tri, background, topology, spp, leaves, upstream gradients) on the bench mesh; rast at res, buffers, background and
    gradients at res / spp"""
    import bench
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    vt, ft = torch.tensor(v, device="cuda"), torch.tensor(f, device="cuda")
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32),
                       device="cuda")
    with raster.DepthPeeler(ctx, mtx, res) as p:
        rasts = [p.rasterize_next_layer()[0] for _ in range(n_layers)]
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device="cuda")
    out = (res[0] // spp, res[1] // spp)
    layers = [({k: rnd(B, *out, c).requires_grad_(True) for k, c in spec}, r) for r in rasts]
    bg = {"shaded": rnd(B, *out, 4).requires_grad_(True)}
    pos = ru.xfm_points(vt[None], mtx).detach().requires_grad_(True)
    leaves = [b[k] for b, _ in layers for k, _ in spec] + [bg["shaded"], pos]
    G = [torch.randn(B, *out, c, generator=g, device="cuda") for _, c in spec]
    return layers, pos, ft, bg, raster.antialias_topology(ft), spp, leaves, G


def fwd_bwd(impl, args, leaves, G):
    def run():
        out = impl(*args)
        return torch.autograd.grad(list(out.values()), leaves, G)
    return run


def agree(args, leaves, G):
    """(forward bit-identical with NaNs in the same places, worst gradient relative L2)"""
    a, b = fused(*args), chain(*args)
    same = all(torch.equal(torch.nan_to_num(a[k], 7.0).view(torch.int32), torch.nan_to_num(b[k], 7.0).view(torch.int32))
               and torch.equal(a[k].isnan(), b[k].isnan()) for k in a)
    ga, gb = fwd_bwd(fused, args, leaves, G)(), fwd_bwd(chain, args, leaves, G)()
    return same, max(float((x - y).double().norm() / max(float(y.double().norm()), 1e-30)) for x, y in zip(ga, gb))


def peak_mib(fn):
    """torch.cuda.max_memory_allocated over one call of fn, and what was allocated before it, in MiB"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    del r
    return {"peak": peak / 2 ** 20, "before": base / 2 ** 20}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--inner", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "compbench needs a GPU"
    res = {"card": card(), "reps": a.reps, "inner": a.inner, "workloads": {}}
    for name, spec, n_layers, spp in (("pass1", PASS1, 1, 1), ("pass2", PASS2, 8, 1), ("pass1_spp2", PASS1, 1, 2), ("pass2_spp2", PASS2, 8, 2)):
        layers, pos, tri, bg, topo, spp, leaves, G = inputs(spec, n_layers, spp)
        args = (layers, pos, tri, bg, topo, spp)
        same, gl2 = agree(args, leaves, G)
        assert same and gl2 < 1e-5, "%s: fused op and chain disagree (%s, %.3g)" % (name, same, gl2)
        mem = {}
        for arm, impl in (("fused", fused), ("chain", chain)):
            with torch.no_grad():
                mem[arm] = {"fwd_mib": peak_mib(lambda: impl(*args))}
            mem[arm]["fwd_bwd_mib"] = peak_mib(fwd_bwd(impl, args, leaves, G))
        runs = []
        for _ in range(2):
            with torch.no_grad():
                fwd = alternate({"fused": lambda: fused(*args), "chain": lambda: chain(*args)}, a.reps, a.inner, a.warmup)
            fb = alternate({"fused": fwd_bwd(fused, args, leaves, G), "chain": fwd_bwd(chain, args, leaves, G)}, a.reps, a.inner, a.warmup)
            runs.append({"fwd_ms": fwd, "fwd_bwd_ms": fb})
        res["workloads"][name] = {"B": 8, "rast_res": 512, "spp": spp, "out_res": 512 // spp, "layers": n_layers, "buffers": len(spec),
                                  "channels": sum(c for _, c in spec), "agree_grad_rel_l2": gl2, "max_memory_allocated": mem, "runs": runs}
        del layers, pos, bg, leaves, G, args
        torch.cuda.empty_cache()
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
