"""Developer tool: CUDA-event timings of the filtered texture look-up on bench.py's shape, 8 x 512^2 pixels, with uv / uv_da from
rasterizing the bench mesh with a spherical texture coordinate (rasterize(grad_db=True) -> interpolate(diff_attrs='all')):

  1. Texture2D.sample x 3 as render.py:70-73 calls it: kd 1024^2 x 4, ks 1024^2 x 3, normal 1024^2 x 3, each with its full chain (11 levels),
     'linear-mipmap-linear', 'wrap'; forward, and backward into every level, uv and uv_da;
  2. the five jittered regulariser taps of render.py:54,75-95 ('linear', 'clamp'; C = 1, 4, 3, 3, 3), forward and backward;
  3. the same contract in plain PyTorch (grid_sample per level plus the level-of-detail blend, autograd), timed in the same process and
     checked against the kernels' outputs.

Bytes per call are counted from shapes: per pixel uv (8 B), uv_da (16 B), out or d out (4 C B), d uv / d uv_da in the backward, plus each
chain read once (forward) or read and its gradient written once (backward).  The achieved rate is those bytes over the time, against the
3.35 TB/s data-sheet HBM3 figure.  Prints the card name and power limit with the numbers, and one JSON line.  MCS_LIB= selects a library
variant (tools/build_variant.sh); TB_QUICK=1 skips the PyTorch comparison.
usage: python tools/texbench.py [out.json]"""
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
from nvdiffrecmc_b200 import synth
from nvdiffrecmc_b200.raster import interpolate, rasterize, texture

dev = torch.device("cuda:0")
B, H, W, REPS = 8, 512, 512, 25
PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(dev)


def event_ms(fn, reps=REPS):
    ts = []
    for _ in range(reps + 3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts[3:]))


def chain(C, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    lv = [torch.rand(1, 1024, 1024, C, device=dev, generator=g)]
    while lv[-1].shape[1] > 1:
        lv.append(torch.nn.functional.avg_pool2d(lv[-1].permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1).contiguous())
    return [x.requires_grad_(True) for x in lv]


def torch_texture(levels, uv, uv_da):
    """The contract in plain PyTorch: bilinear 'wrap' per level by grid_sample on a circularly padded level, major-axis LOD, blend."""
    H0, W0 = levels[0].shape[1], levels[0].shape[2]
    a, b, c, d = uv_da[..., 0] * W0, uv_da[..., 1] * W0, uv_da[..., 2] * H0, uv_da[..., 3] * H0
    A, Bq, Cq = a * a + c * c, b * b + d * d, a * b + c * d
    M = (A + Bq) * 0.5 + torch.sqrt(((A - Bq) * 0.5) ** 2 + Cq * Cq)
    lam = (0.5 * torch.log2(M)).nan_to_num(0.0).clamp(0, len(levels) - 1)
    l0 = lam.floor()
    f = (lam - l0)[..., None]
    out = 0
    uvw = uv - uv.floor()
    for k, t in enumerate(levels):
        w0 = torch.where(l0 == k, 1 - f[..., 0], torch.zeros_like(lam)) + torch.where((l0 + 1 == k), f[..., 0], torch.zeros_like(lam))
        if not bool((w0 > 0).any()):
            continue
        h, w = t.shape[1], t.shape[2]
        p = torch.cat([t[:, :, -1:], t, t[:, :, :1]], 2)
        p = torch.cat([p[:, -1:], p, p[:, :1]], 1).permute(0, 3, 1, 2).expand(uv.shape[0], -1, -1, -1)
        g = torch.stack([(uvw[..., 0] * w + 1) / (w + 2), (uvw[..., 1] * h + 1) / (h + 2)], -1) * 2 - 1
        s = torch.nn.functional.grid_sample(p, g, mode="bilinear", padding_mode="border", align_corners=False).permute(0, 2, 3, 1)
        out = out + w0[..., None] * s
    return out


v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
ctx = ou.OptiXContext()
vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
cdir = vt - vt.mean(0)
cdir = cdir / cdir.norm(dim=-1, keepdim=True)
v_tex = torch.stack([0.5 + torch.atan2(cdir[:, 2], cdir[:, 0]) / (2 * np.pi), torch.acos(cdir[:, 1].clamp(-1, 1)) / np.pi], -1).contiguous()
mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32), device=dev)
pos = ru.xfm_points(vt[None], mtx).contiguous()
with torch.no_grad():
    rast, db = rasterize(ctx, mtx, (H, W), pos=pos, tri=ft, grad_db=True)
    uv, uv_da = interpolate(v_tex, rast, ft, rast_db=db, diff_attrs="all")
mask = (rast[..., 3:] > 0).float()
uv, uv_da = uv.contiguous(), uv_da.contiguous()
out = {"card": card(), "shape": [B, H, W], "covered_px": int(mask.sum()), "lib": os.environ.get("MCS_LIB", "default")}
print("card (name, power limit):", out["card"], "| library:", out["lib"], flush=True)
texs = {"kd": chain(4, 1), "ks": chain(3, 2), "normal": chain(3, 3)}
px = B * H * W
res = {}
for name, lv in texs.items():
    C = lv[0].shape[3]
    chain_bytes = sum(x.numel() for x in lv) * 4
    uvg, dag = uv.clone().requires_grad_(True), uv_da.clone().requires_grad_(True)
    with torch.no_grad():
        fwd = lambda: texture(lv[0], uv, uv_da, mip=lv[1:])
        y = fwd()
    dy = (torch.randn_like(y) * mask).contiguous()                 # the reference's masked loss: background pixels carry no gradient
    y_ag = texture(lv[0], uvg, dag, mip=lv[1:])

    def bwd():
        torch.autograd.grad(y_ag, [uvg, dag] + lv, dy, retain_graph=True)

    fb = px * (8 + 16 + 4 * C) + chain_bytes
    bb = px * (8 + 16 + 4 * C + 8 + 16) + 2 * chain_bytes
    r = {"fwd_ms": event_ms(fwd), "bwd_ms": event_ms(bwd), "fwd_bytes": fb, "bwd_bytes": bb}
    r["fwd_TBps"], r["bwd_TBps"] = fb / r["fwd_ms"] / 1e9, bb / r["bwd_ms"] / 1e9
    r["fwd_frac_hbm"], r["bwd_frac_hbm"] = r["fwd_TBps"] * 1e12 / PEAK, r["bwd_TBps"] * 1e12 / PEAK
    if not os.environ.get("TB_QUICK"):
        with torch.no_grad():
            ref = torch_texture(lv, uv, uv_da)
        r["torch_max_abs_diff"] = float((ref - y).abs().max())
        r["torch_rel_l2"] = float((ref - y).norm() / y.norm())
        r["torch_fwd_ms"] = event_ms(lambda: torch_texture([x.detach() for x in lv], uv, uv_da), reps=5)
        yt = torch_texture(lv, uvg, dag)
        r["torch_bwd_ms"] = event_ms(lambda: torch.autograd.grad(yt, lv, dy, retain_graph=True), reps=5)
    res[name] = r
    print(name, {k: round(x, 4) if isinstance(x, float) else x for k, x in r.items()}, flush=True)
out["sample"] = res
out["sample_x3_fwd_ms"] = sum(r["fwd_ms"] for r in res.values())
out["sample_x3_bwd_ms"] = sum(r["bwd_ms"] for r in res.values())

g = torch.Generator(device=dev).manual_seed(0)
ys, xs = torch.meshgrid((torch.arange(H, device=dev) + 0.5) / H, (torch.arange(W, device=dev) + 0.5) / W, indexing="ij")
jitter = (torch.stack((xs, ys), -1)[None] + torch.randn(B, H, W, 2, device=dev, generator=g) * 0.005).contiguous()
imgs = [torch.rand(B, H, W, C, device=dev, generator=g).requires_grad_(True) for C in (1, 4, 3, 3, 3)]
with torch.no_grad():
    taps_fwd = lambda: [texture(im, jitter, filter_mode="linear", boundary_mode="clamp") for im in imgs]
    ys_ = taps_fwd()
ys_ag = [texture(im, jitter, filter_mode="linear", boundary_mode="clamp") for im in imgs]
dys = [torch.randn_like(y) for y in ys_]
out["taps"] = {"fwd_ms": event_ms(taps_fwd),
               "bwd_ms": event_ms(lambda: torch.autograd.grad(ys_ag, imgs, dys, retain_graph=True)),
               "fwd_bytes": sum(px * (8 + 8 * im.shape[3]) for im in imgs), "bwd_bytes": sum(px * (8 + 8 * im.shape[3]) for im in imgs)}
gs = lambda: [torch.nn.functional.grid_sample(im.permute(0, 3, 1, 2), jitter * 2 - 1, mode="bilinear", padding_mode="border", align_corners=False)
              for im in imgs]
with torch.no_grad():
    out["taps"]["grid_sample_fwd_ms"] = event_ms(gs)
for k in ("fwd", "bwd"):
    out["taps"][k + "_TBps"] = out["taps"][k + "_bytes"] / out["taps"][k + "_ms"] / 1e9
print("five taps:", {k: round(x, 4) for k, x in out["taps"].items()}, flush=True)
print("Texture2D.sample x3: fwd %.3f ms, bwd %.3f ms" % (out["sample_x3_fwd_ms"], out["sample_x3_bwd_ms"]), flush=True)
print(json.dumps(out))
if len(sys.argv) > 1:
    json.dump(out, open(sys.argv[1], "w"), indent=1)
