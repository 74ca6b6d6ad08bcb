"""Developer tool: CUDA-event timings of the screen-space derivatives through the raw C ABI (no Python wrappers inside the timed region),
on the bench mesh at 8 x 512^2:

  1. the rast_db launch alone (mcs_rast_db);
  2. rasterize without and with it (mcs_rasterize, then mcs_rasterize + mcs_rast_db), alternated in one process;
  3. interpolate of v_pos_clip [V,4] and v_tex [V,2] with diff_attrs='all', forward (mcs_interpolate_fwd + mcs_interpolate_da_fwd) and
     backward (mcs_interpolate_bwd + mcs_interpolate_da_bwd into d attr and d rast_db), each against the same call without derivatives;
  4. the derivative block that render_layer adds per layer (render.py:225-234: rast_db, and out_da of v_tex and v_pos_clip).

Prints the card name and power limit with the numbers, and one JSON line.
usage: python tools/dbbench.py [out.json]"""
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
import nvdiffrecmc_b200.renderutils as ru
from nvdiffrecmc_b200 import _lib as L, synth

dev = torch.device("cuda:0")
B, H, W, REPS = 8, 512, 512, 30


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


v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
ctx = ou.OptiXContext()
vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
V, T = v.shape[0], f.shape[0]
mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32), device=dev)
pos = ru.xfm_points(vt[None], mtx).contiguous()             # [B,V,4]
pos1 = pos[0].contiguous()                                  # [V,4], the unbatched attribute layout
tex = torch.rand(V, 2, device=dev)
lib, st, h = L.lib(), L.stream_ptr(), ctx.cpp_wrapper
rast = torch.empty(B, H, W, 4, device=dev)
db = torch.empty(B, H, W, 4, device=dev)
torch.cuda.synchronize()
out = {"card": card(), "shape": [B, H, W], "triangles": T, "vertices": V}
print("card (name, power limit):", out["card"], flush=True)


def plain():
    lib.mcs_rasterize(h, mtx.data_ptr(), B, H, W, rast.data_ptr(), st)


def rast_db():
    lib.mcs_rast_db(pos.data_ptr(), V * 4, V, ft.data_ptr(), T, rast.data_ptr(), B, H, W, db.data_ptr(), st)


def with_db():
    plain(); rast_db()


L.check(lib.mcs_rasterize(h, mtx.data_ptr(), B, H, W, rast.data_ptr(), st), "rasterize")
L.check(lib.mcs_rast_db(pos.data_ptr(), V * 4, V, ft.data_ptr(), T, rast.data_ptr(), B, H, W, db.data_ptr(), st), "rast_db")
torch.cuda.synchronize()
cov = int((rast[..., 3] > 0).sum())
out["covered_px"] = cov
alt = {"rasterize_ms": [], "rasterize_plus_rast_db_ms": [], "rast_db_ms": []}
for _ in range(5):
    alt["rasterize_ms"].append(round(event_ms(plain), 4))
    alt["rasterize_plus_rast_db_ms"].append(round(event_ms(with_db), 4))
    alt["rast_db_ms"].append(round(event_ms(rast_db), 4))
out["rasterize"] = {k: float(np.median(x)) for k, x in alt.items()}
out["rasterize"]["alternated"] = alt
print("rasterize:", out["rasterize"], flush=True)

ops = {}
for name, a in (("v_pos_clip", pos1), ("v_tex", tex)):
    C = a.shape[1]
    o = torch.empty(B, H, W, C, device=dev); da = torch.empty(B, H, W, 2 * C, device=dev)
    g, gda = torch.randn_like(o), torch.randn_like(da)
    d_a = torch.zeros_like(a); d_db = torch.empty_like(db)
    common = (a.data_ptr(), 0, V, C, ft.data_ptr(), T, rast.data_ptr())
    fwd = lambda: lib.mcs_interpolate_fwd(*common, B, H, W, o.data_ptr(), st)
    da_fwd = lambda: lib.mcs_interpolate_da_fwd(*common, db.data_ptr(), B, H, W, C, None, da.data_ptr(), st)
    bwd = lambda: lib.mcs_interpolate_bwd(*common, B, H, W, g.data_ptr(), d_a.data_ptr(), st)
    da_bwd = lambda: lib.mcs_interpolate_da_bwd(*common, db.data_ptr(), B, H, W, C, None, gda.data_ptr(), d_a.data_ptr(), d_db.data_ptr(), st)
    ops[name] = {"fwd_ms": event_ms(fwd), "fwd_with_da_ms": event_ms(lambda: (fwd(), da_fwd())), "da_fwd_ms": event_ms(da_fwd),
                 "bwd_ms": event_ms(bwd, before=d_a.zero_), "bwd_with_da_ms": event_ms(lambda: (bwd(), da_bwd()), before=d_a.zero_),
                 "da_bwd_ms": event_ms(da_bwd, before=d_a.zero_)}
    print(name, {k: round(x, 4) for k, x in ops[name].items()}, flush=True)
out["interpolate"] = ops

# render_layer's derivative block per layer: rast_db + out_da of v_tex + out_da of v_pos_clip (the forward interpolations of v_tex and
# v_pos_clip exist without derivatives too)
da_t = torch.empty(B, H, W, 4, device=dev); da_p = torch.empty(B, H, W, 8, device=dev)


def block():
    rast_db()
    lib.mcs_interpolate_da_fwd(tex.data_ptr(), 0, V, 2, ft.data_ptr(), T, rast.data_ptr(), db.data_ptr(), B, H, W, 2, None, da_t.data_ptr(), st)
    lib.mcs_interpolate_da_fwd(pos.data_ptr(), V * 4, V, 4, ft.data_ptr(), T, rast.data_ptr(), db.data_ptr(), B, H, W, 4, None, da_p.data_ptr(), st)


out["derivative_block_ms"] = event_ms(block)
print("render_layer derivative block (rast_db + 2 x out_da): %.4f ms" % out["derivative_block_ms"], flush=True)
print(json.dumps(out))
if len(sys.argv) > 1:
    json.dump(out, open(sys.argv[1], "w"), indent=1)
