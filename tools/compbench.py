"""Times render_mesh's layer compositing: nvdiffrecmc_b200.raster.composite (csrc/composite.cu, one launch per layer each way) against
the reference's composite_buffer (render/render.py:284-291) run per key with torch.lerp and raster.antialias, on the bench mesh at 8 x 512^2.

Two workloads: "pass1", render_layer's pass-1 buffer set (eleven 4-channel buffers) and one layer; "pass2", the pass-2 set (twelve
4-channel buffers and a 5-channel kd_grad) and 8 depth-peeled layers, as with transparency.  Buffers are random with fractional alphas
and 'shaded' starts from a background.  Per workload: the forward under no_grad (the dataset's reference render) and forward + backward
of sum_k <G_k, out_k> into every buffer, the background and the clip-space positions.  Every timing is the median of --reps CUDA-event
timings of --inner calls each, the fused op and the chain alternating, in two runs.  Before any time is quoted the two are checked to
agree on the same inputs (forward bit for bit, gradients to 1e-5 relative L2).  Prints one JSON document with the card's name and power
limit, read in the same run.

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


def chain(layers, pos, tri, background, topology):
    """composite_buffer(key, layers, bg, True) for every key (render.py:321-330), raster.antialias for dr.antialias"""
    out = {}
    for key in layers[0][0]:
        accum = background[key] if key in background else torch.zeros_like(layers[0][0][key])
        for buffers, rast in reversed(layers):
            b = buffers[key]
            alpha = (rast[..., -1:] > 0).float() * b[..., -1:]
            accum = torch.lerp(accum, torch.cat((b[..., :-1], torch.ones_like(b[..., -1:])), dim=-1), alpha)
            accum = raster.antialias(accum.contiguous(), rast, pos, tri, topology)
        out[key] = accum
    return out


def fused(layers, pos, tri, background, topology):
    return raster.composite(layers, pos, tri, background=background, topology=topology)


def inputs(spec, n_layers, B=8, res=(512, 512), seed=0):
    """(layers, pos, tri, background, topology, leaves, upstream gradients) on the bench mesh"""
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
    layers = [({k: rnd(B, *res, c).requires_grad_(True) for k, c in spec}, r) for r in rasts]
    bg = {"shaded": rnd(B, *res, 4).requires_grad_(True)}
    pos = ru.xfm_points(vt[None], mtx).detach().requires_grad_(True)
    leaves = [b[k] for b, _ in layers for k, _ in spec] + [bg["shaded"], pos]
    G = [torch.randn(B, *res, c, generator=g, device="cuda") for _, c in spec]
    return layers, pos, ft, bg, raster.antialias_topology(ft), leaves, G


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--inner", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "compbench needs a GPU"
    res = {"card": card(), "reps": a.reps, "inner": a.inner, "workloads": {}}
    for name, spec, n_layers in (("pass1", PASS1, 1), ("pass2", PASS2, 8)):
        layers, pos, tri, bg, topo, leaves, G = inputs(spec, n_layers)
        args = (layers, pos, tri, bg, topo)
        same, gl2 = agree(args, leaves, G)
        assert same and gl2 < 1e-5, "%s: fused op and chain disagree (%s, %.3g)" % (name, same, gl2)
        runs = []
        for _ in range(2):
            with torch.no_grad():
                fwd = alternate({"fused": lambda: fused(*args), "chain": lambda: chain(*args)}, a.reps, a.inner, a.warmup)
            fb = alternate({"fused": fwd_bwd(fused, args, leaves, G), "chain": fwd_bwd(chain, args, leaves, G)}, a.reps, a.inner, a.warmup)
            runs.append({"fwd_ms": fwd, "fwd_bwd_ms": fb})
        res["workloads"][name] = {"B": 8, "res": 512, "layers": n_layers, "buffers": len(spec), "channels": sum(c for _, c in spec),
                                  "agree_grad_rel_l2": gl2, "runs": runs}
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
