"""Developer tool: bilateral denoiser forward (one / two signals) and backward at 8 x 512^2, sigma = 2, on both staging kernels in one run.
Contiguous signals take the TMA-staged kernel; the same values passed as strided views (the leading channels of a one-channel-wider
tensor) take the plain kernel.  Prints the card name and power limit with the numbers.  usage: python tools/dnbench.py"""
import os, sys, json, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import nvdiffrecmc_b200.optixutils as ou
from nvdiffrecmc_b200.optixutils.ops import _bilateral_denoiser2_func
dev = torch.device("cuda:0")
flush = torch.empty(1 << 29, dtype=torch.uint8, device=dev)
def timed(fn, reps=20):
    fn(); fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(dev)
g = torch.Generator().manual_seed(0)
B, H, W = 8, 512, 512
col = torch.rand(B, H, W, 3, generator=g).to(dev); colB = torch.rand(B, H, W, 3, generator=g).to(dev)
nrm = torch.nn.functional.normalize(torch.rand(B, H, W, 3, generator=g).to(dev) - 0.5, dim=-1)
zdz = torch.stack([torch.rand(B, H, W, generator=g).to(dev) + 1, torch.full((B, H, W), 0.01, device=dev)], -1)
wide = lambda x: torch.cat([x, torch.zeros_like(x[..., :1])], -1)[..., :x.shape[-1]]      # same values, strided: not TMA-able
out = {"card": card}
for path, view in (("tma", lambda x: x), ("plain", wide)):
    a, b = view(col), view(colB)
    assert a.is_contiguous() == (path == "tma")
    with torch.no_grad():
        f1 = timed(lambda: ou.bilateral_denoiser(a, nrm, zdz, 2.0))
        f2 = timed(lambda: ou.bilateral_denoiser2(a, b, nrm, zdz, 2.0))
    cg = col.clone().requires_grad_(True); cgb = colB.clone().requires_grad_(True)
    ya, yb = _bilateral_denoiser2_func.apply(cg, cgb, nrm, zdz, 2.0)
    ga, gb = view(torch.rand_like(ya)), view(torch.rand_like(yb))          # autograd hands the views to the backward as they are
    b2 = timed(lambda: torch.autograd.grad([ya, yb], [cg, cgb], [ga, gb], retain_graph=True))
    out[path] = {"bwd2_ms": round(b2, 4), "fwd1_ms": round(f1, 4), "fwd2_ms": round(f2, 4), "gtaps_per_s_fwd2": round(B * H * W * 529 / f2 / 1e6, 1)}
print(json.dumps(out))
