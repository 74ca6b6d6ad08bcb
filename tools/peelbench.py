"""Developer tool: CUDA-event timings of depth peeling through the raw C ABI (no Python wrappers inside the timed region).

  1. mcs_rasterize and mcs_rasterize_peel layer 0 at 8 x 512^2 on the bench mesh, alternated in one process (the peel state's
     load / store is the only difference between the two launches);
  2. each of 8 peeled layers at 8 x 512^2 on the bench mesh and on the 1.08 M-triangle grid, with the covered pixels of the layer.

Each timed launch starts from a copy of the state the previous layer left (restored outside the timed region).  Prints the card
name and power limit with the numbers, and one JSON line.
usage: python tools/peelbench.py [out.json]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import bench
import nvdiffrecmc_b200.optixutils as ou
from nvdiffrecmc_b200 import _lib as L, synth

dev = torch.device("cuda:0")
B, H, W, LAYERS, REPS = 8, 512, 512, 8, 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(dev)


def event_ms(fn, before=None, reps=REPS):
    ts = []
    for _ in range(reps + 2):
        if before is not None:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts[2:]))


def scene(kind):
    if kind == "bench":
        v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    else:
        v, f = synth.scene_mesh("grid1m")
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=1)
    torch.cuda.synchronize()
    return ctx, int(f.shape[0])


mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32), device=dev)
lib, st = L.lib(), L.stream_ptr()
rast = torch.empty(B, H, W, 4, device=dev)
state = torch.zeros(B, H, W, device=dev)
out = {"card": card(), "shape": [B, H, W], "reps": REPS}
print("card (name, power limit):", out["card"], flush=True)

ctx, T = scene("bench")
h = ctx.cpp_wrapper


def plain():
    lib.mcs_rasterize(h, mtx.data_ptr(), B, H, W, rast.data_ptr(), st)


def peel():
    lib.mcs_rasterize_peel(h, mtx.data_ptr(), B, H, W, state.data_ptr(), rast.data_ptr(), st)


alt = {"rasterize_ms": [], "peel_layer0_ms": []}
for _ in range(5):
    alt["rasterize_ms"].append(round(event_ms(plain), 4))
    alt["peel_layer0_ms"].append(round(event_ms(peel, before=state.zero_), 4))
out["layer0_alternated"] = alt
print("layer 0, alternated:", alt, flush=True)

for kind in ("bench", "grid1m"):
    if kind == "grid1m":
        del ctx
        ctx, T = scene(kind)
        h = ctx.cpp_wrapper
    rows = []
    state.zero_()
    for k in range(LAYERS):
        start = state.clone()
        ms = event_ms(peel, before=lambda: state.copy_(start))
        cov = int((rast[..., 3] > 0).sum())
        rows.append({"layer": k, "ms": round(ms, 4), "covered_px": cov})
        print(kind, rows[-1], flush=True)
    out[kind] = {"triangles": T, "layers": rows}

print(json.dumps(out))
if len(sys.argv) > 1:
    json.dump(out, open(sys.argv[1], "w"), indent=1)
