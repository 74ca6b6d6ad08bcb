"""Developer tool: CUDA-event timings of Texture2D's automatic mip chain on pass 2's three trainable 1024^2 textures (kd x 4, ks x 3,
normal x 3 channels, 11 levels each), against the reference's per-level torch composition (render/texture.py:20-30: avg_pool2d per level,
and a backward that builds a linspace grid and samples a quarter of the coarser gradient with raster.texture), timed in the same process
after checking that the two agree:

  1. chain forward of the three textures;
  2. fold (the chain's backward) of the three, every level with an incoming gradient;
  3. clamp_ on the three and normalize_ on the normal map, as train.py:467-476 calls them after each optimizer step;
  4. Texture2D.sample x 3 forward and backward, 'linear-mipmap-linear', 'wrap', at 8 x 512^2 pixels whose uv is uniform and whose footprint
     spans every level of the chain.

Bytes per call are counted from shapes (each level read or written once as the step needs it), and the achieved rate is against the
3.35 TB/s data-sheet HBM3 figure.  Prints the card name and power limit with the numbers, and one JSON line.
usage: python tools/mipbench.py [out.json]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from nvdiffrecmc_b200.raster import texture
from nvdiffrecmc_b200.texture import Texture2D, mip_chain

dev = torch.device("cuda:0")
B, H, W, RES, REPS = 8, 512, 512, 1024, 25
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


class Pool(torch.autograd.Function):
    """The reference's texture2d_mip on raster.texture."""
    @staticmethod
    def forward(ctx, x):
        return torch.nn.functional.avg_pool2d(x.permute(0, 3, 1, 2), (2, 2)).permute(0, 2, 3, 1).contiguous()

    @staticmethod
    def backward(ctx, dout):
        h, w = dout.shape[1], dout.shape[2]
        gy, gx = torch.meshgrid(torch.linspace(0.25 / h, 1 - 0.25 / h, 2 * h, device=dev), torch.linspace(0.25 / w, 1 - 0.25 / w, 2 * w, device=dev),
                                indexing="ij")
        return texture(dout * 0.25, torch.stack((gx, gy), -1)[None].contiguous(), filter_mode="linear", boundary_mode="clamp")


def pool_chain(x):
    lv = [x]
    while lv[-1].shape[1] > 1 and lv[-1].shape[2] > 1:
        lv.append(Pool.apply(lv[-1]))
    return lv[1:]


class RefTexture2D(Texture2D):
    """The reference's sample, clamp_ and normalize_ (render/texture.py:57-100) on raster.texture."""
    def sample(self, texc, texc_deriv, filter_mode="linear-mipmap-linear"):
        return texture(self.data, texc, texc_deriv, mip=pool_chain(self.data), filter_mode=filter_mode)

    def clamp_(self):
        for mip in self.getMips():
            for i in range(mip.shape[-1]):
                mip[..., i].clamp_(min=self.min_max[0][i], max=self.min_max[1][i])

    def normalize_(self):
        with torch.no_grad():
            for mip in self.getMips():
                mip.copy_(mip / torch.sqrt(torch.clamp(torch.sum(mip * mip, -1, keepdim=True), min=1e-20)))


def rel_l2(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


g = torch.Generator(device=dev).manual_seed(0)
mm = lambda lo, hi: [torch.tensor(lo, dtype=torch.float32, device=dev), torch.tensor(hi, dtype=torch.float32, device=dev)]
spec = {"kd": (4, mm([0.0] * 4, [1.0] * 4)), "ks": (3, mm([0.0, 0.08, 0.0], [0.0, 1.0, 1.0])), "normal": (3, mm([-1, -1, 0], [1, 1, 1]))}
init = {k: torch.rand(1, RES, RES, C, device=dev, generator=g) * 1.2 - 0.1 for k, (C, _) in spec.items()}
ours = {k: Texture2D(init[k].clone().requires_grad_(True), min_max=spec[k][1]) for k in spec}
ref = {k: RefTexture2D(init[k].clone().requires_grad_(True), min_max=spec[k][1]) for k in spec}
uv = torch.rand(B, H, W, 2, device=dev, generator=g)
uv_da = (torch.randn(B, H, W, 4, device=dev, generator=g) * 2.0 ** (torch.rand(B, H, W, 1, device=dev, generator=g) * 12 - 1) / RES).contiguous()
dys = {k: torch.randn(B, H, W, spec[k][0], device=dev, generator=g) for k in spec}

out = {"card": card(), "textures": {k: [RES, RES, C] for k, (C, _) in spec.items()}, "pixels": [B, H, W]}
print("card (name, power limit):", out["card"], flush=True)
level_elems = {k: sum(x.numel() for x in [init[k]] + pool_chain(init[k])) for k in spec}
base_elems = {k: init[k].numel() for k in spec}
res, check = {}, {}

# 1. chain forward
with torch.no_grad():
    fwd_ours = lambda: [mip_chain(t.data) for t in ours.values()]
    fwd_ref = lambda: [pool_chain(t.data) for t in ref.values()]
    a, b = fwd_ours(), fwd_ref()
check["chain_fwd_bit_equal"] = all(torch.equal(x, y) for la, lb in zip(a, b) for x, y in zip(la, lb))
by = sum(4 * (level_elems[k] + level_elems[k] - base_elems[k]) for k in spec)
res["chain_fwd"] = {"ms": event_ms(fwd_ours), "torch_ms": event_ms(fwd_ref), "bytes": by}

# 2. fold
grads = {k: [torch.randn_like(x) for x in pool_chain(init[k])] for k in spec}


def fold(chain, texs):
    lv = {k: chain(t.data) for k, t in texs.items()}
    return lambda: [torch.autograd.grad(lv[k], t.data, grads[k], retain_graph=True)[0] for k, t in texs.items()]


fold_ours, fold_ref = fold(mip_chain, ours), fold(pool_chain, ref)
check["fold_bit_equal"] = all(torch.equal(x, y) for x, y in zip(fold_ours(), fold_ref()))
by = sum(4 * level_elems[k] for k in spec)                # G_1..G_L read, d level 0 written
res["fold"] = {"ms": event_ms(fold_ours), "torch_ms": event_ms(fold_ref), "bytes": by}


# 3. clamp_ + normalize_ (each timed call starts from the same texels)
def update(texs):
    def run():
        with torch.no_grad():
            for k, t in texs.items():
                t.data.copy_(init[k])
            for t in texs.values():
                t.clamp_()
            texs["normal"].normalize_()
    return run


@torch.no_grad()
def copy_only():
    for k, t in ours.items():
        t.data.copy_(init[k])


with torch.no_grad():
    update(ours)(); update(ref)()
check["clamp_normalize_max_abs_diff"] = max(float((ours[k].data - ref[k].data).detach().abs().max()) for k in spec)
by = sum(2 * 4 * base_elems[k] for k in spec) + 2 * 4 * base_elems["normal"]
copy_ms = event_ms(copy_only)
res["clamp_normalize"] = {"ms": event_ms(update(ours)) - copy_ms, "torch_ms": event_ms(update(ref)) - copy_ms, "bytes": by,
                          "note": "minus %.4f ms of restoring the texels" % copy_ms}
with torch.no_grad():
    for k in spec:
        ours[k].data.copy_(init[k]); ref[k].data.copy_(init[k])


# 4. Texture2D.sample x 3, forward + backward
def sample_step(texs):
    def run():
        ys = [t.sample(uv, uv_da) for t in texs.values()]
        return torch.autograd.grad(ys, [t.data for t in texs.values()], [dys[k] for k in texs]), ys
    return run


(ga, ya), (gb, yb) = sample_step(ours)(), sample_step(ref)()
check["sample_out_bit_equal"] = all(torch.equal(x, y) for x, y in zip(ya, yb))
check["sample_grad_rel_l2"] = max(rel_l2(x, y) for x, y in zip(ga, gb))
res["sample_x3_fwd_bwd"] = {"ms": event_ms(sample_step(ours)), "torch_ms": event_ms(sample_step(ref))}

for k, r in res.items():
    if "bytes" in r:
        r["TBps"] = r["bytes"] / r["ms"] / 1e9
        r["frac_hbm"] = r["TBps"] * 1e12 / PEAK
    print(k, {a: round(v, 4) if isinstance(v, float) else v for a, v in r.items()}, flush=True)
print("agreement with the torch composition:", check, flush=True)
out.update(res)
out["check"] = check
print(json.dumps(out))
if len(sys.argv) > 1:
    json.dump(out, open(sys.argv[1], "w"), indent=1)
