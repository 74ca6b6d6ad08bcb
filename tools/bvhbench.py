"""Developer tool: rebuild / refit timing (CUDA events, L2 flushed) at the bench mesh (7 k triangles) and the 1.08 M-triangle grid --
the whole mcs_bvh_build, so up to 16 384 triangles it includes the shadow view's clustering (k_ploc, k_emit_shadow);
run under `ncu --metrics gpu__time_duration.sum` for the per-kernel split.  usage: python tools/bvhbench.py [reps]"""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import nvdiffrecmc_b200.optixutils as ou
from nvdiffrecmc_b200 import synth
dev = torch.device("cuda:0")
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
flush = torch.empty(1 << 29, dtype=torch.uint8, device=dev)
meshes = (("blob+torus", 4), ("bob-like", 4), ("blob+torus", 5), ("grid1m", 0))
if os.environ.get("BB_ONLY"):
    meshes = tuple(m for m in meshes if m[0] == os.environ["BB_ONLY"])
for kind, level in meshes:
    v, f = synth.scene_mesh(kind, level=level)
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ctx = ou.OptiXContext()
    for _ in range(3):
        ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    ts, tr = [], []
    for mode, acc in ((1, ts), (0, tr)):
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); ou.optix_build_bvh(ctx, vt, ft, rebuild=mode); e1.record(); torch.cuda.synchronize()
            acc.append(e0.elapsed_time(e1))
    T = int(ft.shape[0])
    ms = float(np.median(ts))
    print(json.dumps({"mesh": kind, "level": level, "triangles": T, "rebuild_us": round(ms * 1e3, 1), "refit_us": round(float(np.median(tr)) * 1e3, 1),
                      "rebuild_gbs_at_248B_per_tri": round(T * 248 / ms / 1e6, 1), "frac_of_hbm_6485": round(T * 248 / ms / 1e6 / 6485.5, 3)}), flush=True)
