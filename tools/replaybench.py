"""Developer tool: CUDA-event time of the env_shade replay backward (mcs_env_shade_bwd_replay) alone on the bench workload, for
several builds of libmcshade loaded into one process and alternated on the SAME ray record, with their outputs compared.

usage: python tools/replaybench.py [--reps 20] [--warm 5] [--rounds 2] [--profile-steps K] [--out FILE] [label=path/to/libmcshade.so ...]

The in-tree library (or MCS_LIB) is loaded as `tree`; it runs the forward pass that writes the record.  Every other build only runs
the replay, which takes no context, on the same preallocated buffers.  Per round and build: `warm` untimed launches, then the median
of `reps` launches, each bracketed by CUDA events on the launching stream (as bench.time_env_kernels).  The per-pixel gradients
(pos, normal, kd, ks) of each build are compared bit for bit with the first build's; the light gradient, summed with float atomics
in a run-dependent order, by relative L2.  --profile-steps K > 0 adds a torch.profiler run of K eager training steps (a run of its
own, after the timing) and lists the step's kernels by device time.  The card, its power limit and the SM clock sampled during the
timed launches are printed with the numbers."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import bench
from nvdiffrecmc_b200 import _lib as L


def bind(path):
    lib = C.CDLL(path)
    for name in ("mcs_env_shade_bwd_replay", "mcs_last_error"):
        args, res = L._SIGNATURES[name]
        getattr(lib, name).argtypes = args
        getattr(lib, name).restype = res
    return lib


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def profile_step(w, steps):
    """Kernel list of `steps` eager training steps, by device time, from torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        w.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            w.step()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t > 0:
            rows.append((e.key, t / 1e3 / steps, e.count // steps))
    rows.sort(key=lambda r: -r[1])
    total = sum(r[1] for r in rows)
    return {"steps": steps, "device_ms_per_step": round(total, 3),
            "kernels": [{"name": k[:110], "ms_per_step": round(t, 3), "share_pct": round(100 * t / total, 1), "calls_per_step": n}
                        for k, t, n in rows[:25]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=0)
    ap.add_argument("--out", default=None)
    ap.add_argument("libs", nargs="*", help="label=path of further builds to alternate with the in-tree one")
    a = ap.parse_args()

    dev = torch.device("cuda:0")
    wl = dict(bench.WORKLOAD)
    w = bench.GpuWorkload(wl, 0, 1, dev)
    tree = L.lib()
    libs = [("tree", tree)] + [(s.split("=", 1)[0], bind(s.split("=", 1)[1])) for s in a.libs]

    # inputs and buffers as bench.time_env_kernels sets them up; upstream gradients seeded, not constant
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.optixutils import ops
    gb, N = w.gb, wl["n_samples_x"]
    with torch.no_grad():
        nrm = ru.prepare_shading_normal(gb["pos"], gb["view"], None, gb["smooth_nrm"], gb["tangent"], gb["geom_nrm"])
        ro = gb["pos"] + nrm * 0.001
        kd = w.kd_tex.detach()[gb["texel"]].contiguous(); ks = w.ks_tex.detach()[gb["texel"]].contiguous()
        light = w.lgt.base.detach().contiguous()
    B, H, W_ = ro.shape[:3]
    slots = 2 * N * N
    d = ops._env_descs(gb["mask"], ro, gb["pos"], nrm, gb["view"], kd, ks, light, w.lgt._pdf, w.lgt.rows[:, 0], w.lgt.cols, w.perms)
    diff = torch.empty(B, H, W_, 3, device=dev); spec = torch.empty_like(diff)
    rec_cnt = torch.empty(B, H, W_, dtype=torch.int32, device=dev)
    rec_rays = torch.empty(B, H, W_, 5, slots, device=dev)
    g = [torch.empty(B, H, W_, 3, device=dev) for _ in range(4)]
    lg = torch.empty(light.shape[0], light.shape[1], 3, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    gd = torch.rand(B, H, W_, 3, device=dev, generator=gen); gs = torch.rand(B, H, W_, 3, device=dev, generator=gen)
    dsc = [L.nhwc(gb["pos"]), L.nhwc(nrm), L.nhwc(gb["view"]), L.nhwc(kd), L.nhwc(ks), L.view_hwc(light)]
    dg, sg = L.nhwc(gd), L.nhwc(gs)
    sp = L.stream_ptr()
    L.check(tree.mcs_env_shade_fwd(w.ctx.cpp_wrapper, *[C.byref(x) for x in d], 0, N, 1000, None, 1.0, int(w.offset), diff.data_ptr(), spec.data_ptr(),
                                   None, rec_cnt.data_ptr(), rec_rays.data_ptr(), slots, sp), "optix_env_shade (forward)")
    torch.cuda.synchronize()
    rays = int(rec_cnt.sum())

    def replay(lib):
        st = lib.mcs_env_shade_bwd_replay(*[C.byref(x) for x in dsc], 0, N, 1.0, C.byref(dg), C.byref(sg), rec_cnt.data_ptr(), rec_rays.data_ptr(),
                                          slots, g[0].data_ptr(), g[1].data_ptr(), g[2].data_ptr(), g[3].data_ptr(), lg.data_ptr(), sp)
        if st != 0:
            raise RuntimeError("mcs_env_shade_bwd_replay failed: %s" % lib.mcs_last_error())

    clk = bench.ClockSampler(0).start()
    times = {k: [] for k, _ in libs}
    outs = {}
    clk.begin()
    for _ in range(a.rounds):
        for label, lib in libs:
            ms = []
            for r in range(a.warm + a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); replay(lib); e1.record()
                torch.cuda.synchronize()
                if r >= a.warm:
                    ms.append(e0.elapsed_time(e1))
            times[label].append(float(np.median(ms)))
            if label not in outs:
                outs[label] = [t.clone() for t in g + [lg]]
    clk.end(); clk.close()

    first = libs[0][0]
    ref = outs[first]
    cmp = {}
    for label, o in outs.items():
        cmp[label] = {"pixel_grads_bit_equal_to_" + first: all(torch.equal(x, y) for x, y in zip(o[:4], ref[:4])),
                      "pixel_grads_max_abs_diff": max(float((x - y).abs().max()) for x, y in zip(o[:4], ref[:4])),
                      "light_grad_rel_l2": float((o[4] - ref[4]).double().norm() / ref[4].double().norm().clamp_min(1e-30))}
    res = {"card": card(), "clock": clk.summary(), "workload": {"views": B, "res": [H, W_], "n_samples_x": N, "recorded_rays": rays},
           "replay_ms_median_per_round": {k: [round(t, 3) for t in v] for k, v in times.items()},
           "replay_ms": {k: round(float(np.median(v)), 3) for k, v in times.items()},
           "grad_rays_per_us": {k: round(rays / float(np.median(v)) / 1e3, 1) for k, v in times.items()}, "outputs": cmp}
    if a.profile_steps > 0:
        res["profile"] = profile_step(w, a.profile_steps)
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
