"""Times the image-space regularisers (nvdiffrecmc_b200.regularizer, csrc/regularizer.cu) against a plain-PyTorch composition of the same
contract, at the training sizes 8x512^2 and 8x800^2 with training-like operands.

Per size: each function's forward and forward + backward through the public API, the three together as a geometry tick calls them
(forward + backward), and the raw C-ABI launches (forward, backward) with preallocated buffers.  Every timing is the median of --reps
CUDA-event timings of --inner calls each, after --warmup calls; the product and the composition alternate within one run.  Before any
time is quoted, the two are checked to agree on the same inputs (loss to 1e-5 relative, gradients to 1e-4 relative L2).  Prints one
JSON document with the card's name and power limit, read in the same run.

    python tools/regbench.py [--reps 25] [--inner 10] [--warmup 5] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import nvdiffrecmc_b200._lib as L  # noqa: E402
import nvdiffrecmc_b200.regularizer as R  # noqa: E402

EPS, SRGB_T = 0.001, 0.0031308
LAMBDAS = {"shading_loss": (0.15, 0.0025), "material_smoothness_grad": (0.1, 0.05, 0.025), "chroma_loss": (0.025,)}


# ---- the baseline: the contract of csrc/regularizer.cu written as a torch composition (per pixel; a mean over three identical channel
#      copies is the mean over one)
def _luma(x):
    return ((x[..., 0] + x[..., 1]) + x[..., 2]) / 3


def _value(x):
    return torch.max(x[..., 0:3], dim=-1).values            # the first maximal channel gets the gradient


def _srgb(f):
    return torch.where(f <= SRGB_T, f * 12.92, torch.clamp(f, min=SRGB_T) ** (1.0 / 2.4) * 1.055 - 0.055)


def t_shading(d, s, r, ld, ls):
    dl, sl, a = _luma(d), _luma(s), r[..., 3]
    tot = dl + sl
    img = _srgb(torch.log(torch.clamp(tot * a, 0, 65535) + 1))
    tgt = _srgb(torch.log(torch.clamp(_value(r) * a, 0, 65535) + 1))
    err = torch.abs(img - tgt) * dl / torch.clamp(tot, min=EPS)
    return err.mean() * ld + sl.mean() / torch.clamp(dl.mean(), min=EPS) * ls


def t_smooth(k, s, n, lk, ls, ln):
    return (_luma(k) * k[..., 3]).mean() * lk + (s[..., 0:3] * s[..., 3:4]).mean() * ls + (n[..., 0:3] * n[..., 3:4]).mean() * ln


def t_chroma(k, r, lc):
    ck = torch.clamp(_value(k), min=EPS)[..., None]
    cr = torch.clamp(_value(r), min=EPS)[..., None]
    return torch.abs((k[..., 0:3] / ck - r[..., 0:3] / cr) * r[..., 3:4]).mean() * lc


BASE = {"shading_loss": t_shading, "material_smoothness_grad": t_smooth, "chroma_loss": t_chroma}
NDIFF = {"shading_loss": 2, "material_smoothness_grad": 3, "chroma_loss": 1}


def inputs(B, H, W, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device="cuda")
    alpha = (rnd(B, H, W, 1) < 0.7).float()
    ref_buf = torch.cat([rnd(B, H, W, 3), alpha, rnd(B, H, W, 4)], -1)          # color_ref is a slice, as in the tick
    ref = ref_buf[..., 0:4]
    lit = lambda lo, hi: torch.cat([lo + (hi - lo) * rnd(B, H, W, 3), alpha], -1)
    return {"shading_loss": [lit(-0.05, 2.0), lit(-0.02, 0.8), ref], "material_smoothness_grad": [lit(0, 0.2), lit(0, 0.1), lit(0, 0.4)],
            "chroma_loss": [lit(0, 1), ref]}


def timed(fn, reps, inner, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(inner):
            fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / inner)
    ts.sort()
    return ts[len(ts) // 2]


def alternate(arms, reps, inner, warmup):
    """{name: median ms} of each zero-argument callable of `arms`, their timings interleaved."""
    for f in arms.values():
        timed(f, 1, 1, warmup)
    samples = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            samples[k].append(timed(f, 1, inner, 0))
    return {k: sorted(v)[len(v) // 2] for k, v in samples.items()}


def fwd_bwd(fn, ops, lam, impl):
    ops = [o.detach().requires_grad_(i < NDIFF[fn]) for i, o in enumerate(ops)]
    G = torch.ones((), device="cuda")

    def run():
        loss = impl(*ops, *lam)
        return torch.autograd.grad(loss, ops[:NDIFF[fn]], grad_outputs=G)
    return run


def agree(fn, ops, lam):
    """(loss rel. difference, worst gradient rel. L2) between the product and the composition."""
    ops = [o.detach().requires_grad_(i < NDIFF[fn]) for i, o in enumerate(ops)]
    lp, lb = getattr(R, fn)(*ops, *lam), BASE[fn](*ops, *lam)
    gp = torch.autograd.grad(lp, ops[:NDIFF[fn]])
    gb = torch.autograd.grad(lb, ops[:NDIFF[fn]])
    rel = abs(float(lp) - float(lb)) / abs(float(lb))
    gl2 = max(float((a - b).norm() / b.norm()) for a, b in zip(gp, gb))
    return rel, gl2


def raw_launches(fn, ops, lam):
    """(forward, backward) zero-argument callables of the bare C-ABI entries with preallocated buffers."""
    lib, st = L.lib(), L.stream_ptr()
    B, H, W = ops[0].shape[:3]
    views = [L.nhwc(o) for o in ops]
    k = 1 if fn == "chroma_loss" else 3
    part = torch.empty(k * getattr(lib, "mcs_%s_num_partials" % fn)(B, H, W), dtype=torch.float64, device="cuda")
    loss, means, dl = torch.empty((), device="cuda"), torch.empty(2, device="cuda"), torch.ones((), device="cuda")
    grads = [torch.empty_like(o, memory_format=torch.contiguous_format) for o in ops[:NDIFF[fn]]]
    f_fwd, f_bwd = getattr(lib, "mcs_%s_fwd" % fn), getattr(lib, "mcs_%s_bwd" % fn)
    fwd_args = [*views, *lam, part.data_ptr(), loss.data_ptr()] + ([means.data_ptr()] if fn == "shading_loss" else []) + [st]
    bwd_args = [*views, *lam] + ([means.data_ptr()] if fn == "shading_loss" else []) + [dl.data_ptr()] + [g.data_ptr() for g in grads] + [st]
    f_fwd(*fwd_args)
    return (lambda: f_fwd(*fwd_args)), (lambda: f_bwd(*bwd_args))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--inner", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "regbench needs a GPU"
    res = {"card": card(), "reps": a.reps, "inner": a.inner, "sizes": {}}
    for B, H, W in ((8, 512, 512), (8, 800, 800)):
        ins = inputs(B, H, W)
        row = {}
        for fn in LAMBDAS:
            ops, lam = ins[fn], LAMBDAS[fn]
            rel, gl2 = agree(fn, ops, lam)
            assert rel < 1e-5 and gl2 < 1e-4, "%s: product and composition disagree (loss %.3g, gradient %.3g)" % (fn, rel, gl2)
            with torch.no_grad():
                det = [o.detach() for o in ops]
                fwd = alternate({"fused": lambda: getattr(R, fn)(*det, *lam), "torch": lambda: BASE[fn](*det, *lam)}, a.reps, a.inner, a.warmup)
            fb = alternate({"fused": fwd_bwd(fn, ops, lam, getattr(R, fn)), "torch": fwd_bwd(fn, ops, lam, BASE[fn])}, a.reps, a.inner, a.warmup)
            rf, rb = raw_launches(fn, ops, lam)
            raw = alternate({"fwd": rf, "bwd": rb}, a.reps, a.inner, a.warmup)
            row[fn] = {"agree_loss_rel": rel, "agree_grad_rel_l2": gl2, "fwd_ms": fwd, "fwd_bwd_ms": fb, "raw_abi_ms": raw}
        sh, ms, ch = ins["shading_loss"], ins["material_smoothness_grad"], ins["chroma_loss"]
        dif = [sh[0], sh[1], ms[0], ms[1], ms[2], ch[0]]

        def tick(impl):
            ops = [o.detach().requires_grad_(True) for o in dif]
            G = torch.ones((), device="cuda")

            def run():
                loss = (impl["shading_loss"](ops[0], ops[1], sh[2], *LAMBDAS["shading_loss"])
                        + impl["material_smoothness_grad"](ops[2], ops[3], ops[4], *LAMBDAS["material_smoothness_grad"])
                        + impl["chroma_loss"](ops[5], ch[1], *LAMBDAS["chroma_loss"]))
                return torch.autograd.grad(loss, ops, grad_outputs=G)
            return run
        prod = {fn: getattr(R, fn) for fn in LAMBDAS}
        row["tick_fwd_bwd_ms"] = alternate({"fused": tick(prod), "torch": tick(BASE)}, a.reps, a.inner, a.warmup)
        res["sizes"]["%dx%dx%d" % (B, H, W)] = row
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
