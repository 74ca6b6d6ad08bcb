"""Developer tool: the bilateral denoiser's raw C-ABI launches -- forward with one and two signals, transposed filter with one and two
signals -- on both staging kernels, on the bench's own G-buffer (8 x 512^2, its 8 views, guide normals and depth built as shade() builds
them: about half of the pixels are background), for several builds of libmcshade loaded into one process and alternated.

usage: python tools/dnbench.py [--reps 20] [--warm 3] [--rounds 2] [--out FILE] [label=path/to/libmcshade.so ...]

The in-tree library (or MCS_LIB) is `tree`.  Contiguous signals take the TMA-staged kernel; the same values passed as strided views
(the leading channels of a one-channel-wider tensor) take the plain kernel.  Signals and upstream gradients are seeded uniform values.
Per round, launch and build: `warm` untimed launches, then the median of `reps` launches, each bracketed by CUDA events after a 512 MB
L2 flush.  Every build's outputs are compared bit for bit with the first build's before any time is printed.  Prints the card, its
power limit and the SM clock sampled during the timed launches, and the share of background output strips and tiles."""
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

OPS = ("mcs_bilateral_fwd", "mcs_bilateral_fwd2", "mcs_bilateral_bwd", "mcs_bilateral_bwd2")


def bind(path):
    lib = C.CDLL(path)
    for name in OPS + ("mcs_last_error",):
        args, res = L._SIGNATURES[name]
        getattr(lib, name).argtypes = args
        getattr(lib, name).restype = res
    return lib


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warm", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("libs", nargs="*", help="label=path of further builds to alternate with the in-tree one")
    a = ap.parse_args()

    dev = torch.device("cuda:0")
    wl = dict(bench.WORKLOAD)
    w = bench.GpuWorkload(wl, 0, 1, dev)
    libs = [("tree", L.lib())] + [(s.split("=", 1)[0], bind(s.split("=", 1)[1])) for s in a.libs]

    # the guides as GpuWorkload.shade() hands them to denoise_and_combine
    import nvdiffrecmc_b200.renderutils as ru
    from nvdiffrecmc_b200.denoiser import _safe_normalize
    gb = w.gb
    with torch.no_grad():
        nrm = _safe_normalize(ru.prepare_shading_normal(gb["pos"], gb["view"], None, gb["smooth_nrm"], gb["tangent"], gb["geom_nrm"],
                                                        two_sided_shading=True, opengl=True)).contiguous()
        zdz = torch.stack([gb["depth"], torch.full_like(gb["depth"], 0.01)], -1)
    sigma = float(w.denoiser.sigma)
    B, H, W = nrm.shape[:3]
    bg = (nrm == 0).all(-1)
    strips = bg.reshape(B, H // 2, 2, W // 32, 32).all(4).all(2)
    tiles = bg.reshape(B, H // 16, 16, W // 32, 32).all(4).all(2)
    gen = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda c: torch.rand(B, H, W, c, device=dev, generator=gen)
    col, colB, gA, gB = rnd(3), rnd(3), rnd(4) - 0.5, rnd(4) - 0.5
    wide = lambda x: torch.cat([x, torch.zeros_like(x[..., :1])], -1)[..., :x.shape[-1]]      # same values, strided: not TMA-able
    outs = {c: [torch.empty(B, H, W, c, device=dev) for _ in range(2)] for c in (3, 4)}      # transposed / forward outputs, A and B
    flush = torch.empty(1 << 29, dtype=torch.uint8, device=dev)
    sp = L.stream_ptr()

    def launch(lib, op, view):
        d = lambda t: C.byref(L.nhwc(t))
        oa, ob = [o.data_ptr() for o in outs[4 if "fwd" in op else 3]]
        n, z = d(nrm), d(zdz)
        if op == "mcs_bilateral_fwd":
            st = lib.mcs_bilateral_fwd(d(view(col)), n, z, sigma, oa, sp)
        elif op == "mcs_bilateral_fwd2":
            st = lib.mcs_bilateral_fwd2(d(view(col)), d(view(colB)), n, z, sigma, oa, ob, sp)
        elif op == "mcs_bilateral_bwd":
            st = lib.mcs_bilateral_bwd(n, z, sigma, d(view(gA)), oa, sp)
        else:
            st = lib.mcs_bilateral_bwd2(n, z, sigma, d(view(gA)), d(view(gB)), oa, ob, sp)
        if st != 0:
            raise RuntimeError("%s failed: %s" % (op, lib.mcs_last_error()))

    paths = (("tma", lambda x: x), ("plain", wide))
    times = {(p, op, lb): [] for p, _ in paths for op in OPS for lb, _ in libs}
    ref, equal = {}, {}
    clk = bench.ClockSampler(0).start()
    clk.begin()
    for _ in range(a.rounds):
        for p, view in paths:
            for op in OPS:
                for lb, lib in libs:
                    o = outs[4 if "fwd" in op else 3]
                    for t in o:
                        t.fill_(float("nan"))
                    ms = []
                    for i in range(a.warm + a.reps):
                        flush.zero_()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(); launch(lib, op, view); e1.record()
                        torch.cuda.synchronize()
                        if i >= a.warm:
                            ms.append(e0.elapsed_time(e1))
                    times[(p, op, lb)].append(float(np.median(ms)))
                    got = [t.view(torch.int32).clone() for t in o[:2 if op.endswith("2") else 1]]
                    key = (p, op)
                    if key not in ref:
                        ref[key] = got
                    eq = all(torch.equal(x, y) for x, y in zip(got, ref[key]))
                    equal[(p, op, lb)] = equal.get((p, op, lb), True) and eq
    clk.end(); clk.close()

    first = libs[0][0]
    bad = [k for k, v in equal.items() if not v]
    if bad:
        raise SystemExit("outputs differ from %s's bit for bit: %s" % (first, bad))
    res = {"card": card(), "clock": clk.summary(),
           "workload": {"views": B, "res": [H, W], "sigma": sigma, "radius": 2 * int(np.ceil(sigma * 2.5)) + 1,
                        "background_px": round(float(bg.float().mean()), 4), "background_32x2_strips": round(float(strips.float().mean()), 4),
                        "background_32x16_tiles": round(float(tiles.float().mean()), 4)},
           "outputs_bit_equal_to_" + first: True,
           "ms_median_per_round": {"%s %s %s" % k: [round(t, 4) for t in v] for k, v in times.items()},
           "ms": {"%s %s %s" % k: round(float(np.median(v)), 4) for k, v in times.items()}}
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
