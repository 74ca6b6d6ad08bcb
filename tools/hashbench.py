"""Developer tool: CUDA-event timings of the hash-grid encoding (csrc/hashgrid.cu) on the positions MLPTexture3D samples in training.

Workload: a G-buffer of the bench mesh (rasterize + interpolate of the positions, 8 views) at 8 x 512^2 and 8 x 800^2.  As in
render.py:61-64 each pixel is sampled twice, at gb_pos and at gb_pos + N(0, 0.01); uncovered pixels interpolate to gb_pos = 0, so
after the AABB normalisation they all land on one spot (the jittered ones within 0.01 of it), and their upstream gradient is zero
(composite_buffer blends them with alpha 0).  The raw kernels run on both samples as one call of 2 x B x H x W points.

Timed (median of REPS after warm-up):
  fwd            mcs_hashgrid_fwd
  bwd_params     mcs_hashgrid_bwd, d params only (into a zeroed buffer, zeroing outside the timed region)
  bwd_params_dx  mcs_hashgrid_bwd, d params and d x
  sample         MLPTexture3D.sample twice (normalise, clamp, encode, 3 bias-free Linear + ReLU, sigmoid), forward + backward, as the
                 torch composition (encoding kernels + torch MLP) and as the fused drop-in nvdiffrecmc_b200.mlptexture.MLPTexture3D
                 (csrc/mlptexture.cu), the two arms alternated twice; the encode-only composition for scale
  sample_pair    MLPTexture3D.sample_pair(gb_pos, noise), forward + backward, alternated twice with the fused two-call arm after checking
                 that the two arms' outputs agree bit for bit; with both arms' launches of our kernels per step (counted by the binding)
  sample_no_grad the fused forward alone under torch.no_grad() at 2048^2 points (render_uv's bake at texture_res)
  torch_*        the same encoding written in plain PyTorch (gather + weighted sum, autograd), the comparison arm; its backward (an
                 accumulating index_put of 128 values per point) takes seconds per call, so it is the median of 3
Prints the card name and power limit, the table bytes touched per point (16 levels x 8 corners x 8 B) and the achieved rate.
  HB_RAW=1   only the raw kernels (for A/B runs of library variants selected with MCS_LIB=...)
usage: python tools/hashbench.py [out.json]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ctypes
import numpy as np
import torch
import bench
import nvdiffrecmc_b200.optixutils as ou
from nvdiffrecmc_b200 import _lib as L, synth
from nvdiffrecmc_b200.raster import rasterize, interpolate
from nvdiffrecmc_b200.tinycudann import Encoding
from nvdiffrecmc_b200.mlptexture import MLPTexture3D

dev = torch.device("cuda:0")
REPS = 25
B = 8
CFG = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16,
       "per_level_scale": float(np.exp(np.log(4096 / 16) / 15))}
BYTES_PER_POINT = 16 * 8 * 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(dev)


def event_ms(fn, before=None, reps=REPS, warm=3, label=None):
    ts = []
    for k in range(reps + warm):
        if before is not None:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        if k >= warm:
            ts.append(e0.elapsed_time(e1))
    if label:
        print("  %s: %.3f ms" % (label, float(np.median(ts))), flush=True)
    return float(np.median(ts))


def gbuffer(res):
    """gb_pos [B,H,W,3] of the bench mesh (0 where uncovered), the mesh AABB and the coverage mask."""
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    ctx = ou.OptiXContext()
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32), device=dev)
    rast = rasterize(ctx, mtx, (res, res))
    pos, _ = interpolate(vt, rast, ft)
    aabb = torch.stack([vt.min(0).values, vt.max(0).values])
    return pos.detach(), aabb, rast[..., 3] > 0


def torch_encoding(x, params, lv):
    """The contract in plain PyTorch: per level, gather the 8 corners and sum their weighted features (autograd through both)."""
    P = params.view(-1, 2)
    outs = []
    M = 0xFFFFFFFF
    for l in range(lv["n_levels"]):
        s, res, off = lv["scale"][l], lv["res"][l], lv["offset"][l]
        size = lv["offset"][l + 1] - off
        p = x * s + 0.5
        g = torch.floor(p)
        t = p - g
        gi = g.to(torch.int64)
        y = 0
        for c in range(8):
            b = [(c >> d) & 1 for d in range(3)]
            cx, cy, cz = [gi[:, d] + b[d] for d in range(3)]
            if (lv["dense_mask"] >> l) & 1:
                idx = ((cx + cy * res + cz * (res * res)) & M) % size
            else:
                idx = ((cx & M) ^ ((cy * 2654435761) & M) ^ ((cz * 805459861) & M)) % size
            w = torch.ones_like(t[:, 0])
            for d in range(3):
                w = w * (t[:, d] if b[d] else 1 - t[:, d])
            y = y + w[:, None] * P[off + idx]
        outs.append(y)
    return torch.cat(outs, -1)


def run_size(res, raw_only):
    pos, aabb, cov = gbuffer(res)
    gen = torch.Generator(device=dev).manual_seed(0)
    noise = torch.randn(pos.shape, device=dev, generator=gen) * 0.01
    jit = pos + noise
    norm = lambda q: torch.clamp((q.view(-1, 3) - aabb[0][None]) / (aabb[1] - aabb[0])[None], 0, 1).contiguous()
    x = torch.cat([norm(jit), norm(pos)])
    n = x.shape[0]
    keep = torch.cat([cov.reshape(-1), cov.reshape(-1)]).float()[:, None]
    dy = torch.randn(n, 32, device=dev, generator=gen) * keep
    enc = Encoding(3, CFG)
    with torch.no_grad():
        enc.params.uniform_(-1, 1, generator=gen)
    lib, st, lv = L.lib(), L.stream_ptr(), ctypes.byref(enc._lv)
    out = torch.empty(n, 32, device=dev)
    dp = torch.zeros_like(enc.params)
    dx = torch.empty_like(x)
    ptr = enc.params.data_ptr()
    r = {"points": n, "covered": float(cov.float().mean())}
    r["fwd_ms"] = event_ms(lambda: lib.mcs_hashgrid_fwd(x.data_ptr(), n, ptr, lv, out.data_ptr(), st))
    r["bwd_params_ms"] = event_ms(lambda: lib.mcs_hashgrid_bwd(x.data_ptr(), n, ptr, lv, dy.data_ptr(), dp.data_ptr(), None, st), before=dp.zero_)
    r["bwd_params_dx_ms"] = event_ms(lambda: lib.mcs_hashgrid_bwd(x.data_ptr(), n, ptr, lv, dy.data_ptr(), dp.data_ptr(), dx.data_ptr(), st),
                                     before=dp.zero_)
    r["bwd_dx_ms"] = event_ms(lambda: lib.mcs_hashgrid_bwd(x.data_ptr(), n, ptr, lv, dy.data_ptr(), None, dx.data_ptr(), st))
    for k in ("fwd", "bwd_params", "bwd_params_dx"):
        r[k + "_GBps"] = round(n * BYTES_PER_POINT / (r[k + "_ms"] * 1e-3) / 1e9, 1)
    print(res, json.dumps(r), flush=True)
    if raw_only:
        return r
    # MLPTexture3D.sample, twice (jittered + plain), forward + backward
    net = torch.nn.Sequential(torch.nn.Linear(32, 32, bias=False), torch.nn.ReLU(), torch.nn.Linear(32, 32, bias=False), torch.nn.ReLU(),
                              torch.nn.Linear(32, 6, bias=False)).to(dev)
    lo, hi = torch.zeros(6, device=dev), torch.ones(6, device=dev)
    g6 = torch.randn(2, B, res, res, 6, device=dev, generator=gen) * cov[None, ..., None]
    pj, pp = jit.clone().requires_grad_(True), pos.clone().requires_grad_(True)

    def sample(q, mlp=True):
        e = enc(norm(q))
        if not mlp:
            return e
        return (torch.sigmoid(net(e)) * (hi - lo)[None] + lo[None]).view(*q.shape[:-1], 6)

    def step(mlp=True):
        a, b = sample(pj, mlp), sample(pp, mlp)
        if mlp:
            (a * g6[0]).sum().backward()
            (b * g6[1]).sum().backward()
        else:
            a.backward(dy[:n // 2]); b.backward(dy[n // 2:])

    tex = MLPTexture3D(aabb, channels=6, min_max=[lo, hi])
    with torch.no_grad():
        tex.encoder.params.copy_(enc.params)
        for w, m in zip(tex.net.weights(), [m for m in net if isinstance(m, torch.nn.Linear)]):
            w.copy_(m.weight)

    def fused_step():
        (tex.sample(pj) * g6[0]).sum().backward()
        (tex.sample(pp) * g6[1]).sum().backward()

    for rnd in range(2):                 # the two arms alternated, twice
        r["sample_fwd_bwd_ms_%d" % rnd] = event_ms(step, reps=20, label="sample fwd+bwd, torch MLP (round %d)" % rnd)
        r["fused_sample_fwd_bwd_ms_%d" % rnd] = event_ms(fused_step, reps=20, label="sample fwd+bwd, fused (round %d)" % rnd)
    r["sample_fwd_bwd_ms"] = min(r["sample_fwd_bwd_ms_0"], r["sample_fwd_bwd_ms_1"])
    r["fused_sample_fwd_bwd_ms"] = min(r["fused_sample_fwd_bwd_ms_0"], r["fused_sample_fwd_bwd_ms_1"])
    # the pair: both samples of every pixel in one launch each way, the jittered point formed in the kernel from the same noise
    pq = pos.clone().requires_grad_(True)

    def pair_step():
        a, b = tex.sample_pair(pq, noise)
        ((b * g6[0]).sum() + (a * g6[1]).sum()).backward()

    with torch.no_grad():
        a_p, b_p = tex.sample_pair(pos, noise)
        if not (torch.equal(a_p, tex.sample(pos)) and torch.equal(b_p, tex.sample(jit))):
            raise RuntimeError("sample_pair and the two sample calls disagree")
    for arm, fn in (("fused", fused_step), ("pair", pair_step)):
        L.LAUNCHES.clear()
        fn()
        r["%s_launches_per_step" % arm] = dict(L.LAUNCHES)
    for rnd in range(2):
        r["fused_sample_fwd_bwd_ms_pair_round_%d" % rnd] = event_ms(fused_step, reps=20, label="sample fwd+bwd, fused two calls (round %d)" % rnd)
        r["pair_sample_fwd_bwd_ms_%d" % rnd] = event_ms(pair_step, reps=20, label="sample_pair fwd+bwd (round %d)" % rnd)
    r["pair_sample_fwd_bwd_ms"] = min(r["pair_sample_fwd_bwd_ms_0"], r["pair_sample_fwd_bwd_ms_1"])
    r["encode_only_fwd_bwd_ms"] = event_ms(lambda: step(False), reps=20, label="encode only fwd+bwd")
    r["mlp_share"] = round(1 - r["encode_only_fwd_bwd_ms"] / r["sample_fwd_bwd_ms"], 3)
    with torch.no_grad():
        a_f, a_t = tex.sample(pp), sample(pp)
    r["fused_vs_torch_out_max_abs"] = float((a_f - a_t).abs().max())
    del tex
    # plain PyTorch comparison arm: forward, and forward + backward of d params and d x
    lvd = {"n_levels": 16, "dense_mask": enc.levels["dense_mask"], "scale": enc.levels["scale"], "res": enc.levels["res"], "offset": enc.levels["offset"]}
    try:
        pt = enc.params.detach().clone().requires_grad_(True)
        with torch.no_grad():
            r["torch_fwd_ms"] = event_ms(lambda: torch_encoding(x, pt, lvd), reps=20, warm=1, label="torch fwd")
        xt = x.clone().requires_grad_(True)
        if n <= 1 << 23:
            r["torch_fwd_bwd_ms"] = event_ms(lambda: torch_encoding(xt, pt, lvd).backward(dy), reps=3, warm=1, label="torch fwd+bwd")
        else:
            r["torch_fwd_bwd_ms"] = "not measured: one call took 39 s at 2 x 8 x 512^2 (H100 80GB HBM3, 400 W)"
        with torch.no_grad():
            ref = torch_encoding(x, pt, lvd)
        enc_out = torch.empty_like(out)
        lib.mcs_hashgrid_fwd(x.data_ptr(), n, ptr, lv, enc_out.data_ptr(), st)
        r["torch_vs_kernel_max_abs"] = float((ref - enc_out).abs().max())
    except torch.cuda.OutOfMemoryError:
        r["torch_fwd_bwd_ms"] = "out of memory"
    torch.cuda.empty_cache()
    return r


if __name__ == "__main__":
    raw = bool(os.environ.get("HB_RAW"))
    res_list = [int(s) for s in os.environ.get("HB_RES", "512,800").split(",")]
    out = {"card": card(), "lib": L.LIB_PATH, "bytes_per_point": BYTES_PER_POINT, "reps": REPS}
    print("card (name, power limit):", out["card"], flush=True)
    for res in res_list:
        out["2x%dx%d^2" % (B, res)] = run_size(res, raw)
        print(res, json.dumps(out["2x%dx%d^2" % (B, res)]), flush=True)
    if not raw:
        # render_uv bakes the texture once at texture_res (2048^2 points), forward only
        tex = MLPTexture3D(torch.tensor([[0.0] * 3, [1.0] * 3], device=dev), channels=6, min_max=[torch.zeros(6, device=dev), torch.ones(6, device=dev)])
        q = torch.rand(2048 * 2048, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
        with torch.no_grad():
            out["sample_no_grad_2048^2_ms"] = event_ms(lambda: tex.sample(q), reps=20, label="fused sample, no_grad, 2048^2")
    print(json.dumps(out))
    if len(sys.argv) > 1:
        json.dump(out, open(sys.argv[1], "w"), indent=1)
