"""Developer tool: shadow-ray rays, 4-wide node visits and leaf-triangle tests of the fused env_shade forward kernel at the bench
configuration (bench.py WORKLOAD, 5 forward launches with new seeds).  Needs the counting variant, never the shipped build:
    tools/build_variant.sh count_sah -DMCS_COUNT_TRAVERSAL=1                         # shadow view with its SAH topology
    tools/build_variant.sh count_lbvh -DMCS_COUNT_TRAVERSAL=1 -DMCS_SAH_MAX_TRIS=0   # shadow view = LBVH grandchild collapse
    MCS_LIB=nvdiffrecmc_b200/lib/variants/count_sah.so python tools/tracecount.py"""
import ctypes as C
import json
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import bench
from nvdiffrecmc_b200 import _lib as L

dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
wl = dict(bench.WORKLOAD)
w = bench.GpuWorkload(wl, 0, 1, dev, views=wl["views_per_gpu"])
torch.cuda.synchronize()
fn = L.lib().mcs_trace_counts          # AttributeError: MCS_LIB does not point at a counting variant
fn.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
fn.restype = C.c_int
out = (C.c_ulonglong * 3)()
assert fn(out, 1) == 0
launches = 5
bench.time_env_kernels(w, reps=launches, warm=0)
assert fn(out, 1) == 0
rays, visits, tests = (int(x) for x in out)
print(json.dumps({"lib": os.path.basename(L.LIB_PATH), "mesh": wl["mesh"], "triangles": int(w.tris.shape[0]), "forward_launches": launches,
                  "rays": rays, "visits_per_ray": round(visits / max(rays, 1), 3), "tri_tests_per_ray": round(tests / max(rays, 1), 3)}), flush=True)
