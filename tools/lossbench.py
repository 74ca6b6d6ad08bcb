"""Times the geometry passes' image loss (geometry/dmtet.py:229-230, geometry/dlmesh.py:75-76): the two torch lines with the package's
renderutils.image_loss against nvdiffrecmc_b200.regularizer.coverage_image_loss (csrc/lossmesh.cu), forward + backward, at 8 x 512^2 with
training-like operands (a composited shaded buffer, color_ref a slice of a wider buffer as prepare_batch leaves it).

Before any time is quoted, the two are checked on the same inputs: d shaded bit for bit and the loss to 1e-6 relative.  Each timing is
the median of --reps CUDA-event timings of --inner calls, after --warmup calls, the two arms alternated.  Then one torch.profiler run
of each arm lists its kernels (name, launch count and device time) for one forward + backward.  Prints one JSON document with the card's name and
power limit, read in the same run.

    python tools/lossbench.py [--loss l1] [--tonemapper log_srgb] [--reps 25] [--inner 20] [--warmup 10] [--out FILE]
"""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import nvdiffrecmc_b200.regularizer as R  # noqa: E402
import nvdiffrecmc_b200.renderutils as ru  # noqa: E402


def chain(shaded, color_ref, loss, tonemapper):
    img_loss = torch.nn.functional.mse_loss(shaded[..., 3:], color_ref[..., 3:])
    img_loss += ru.image_loss(shaded[..., 0:3] * color_ref[..., 3:], color_ref[..., 0:3] * color_ref[..., 3:], loss, tonemapper)
    return img_loss


def inputs(B, H, W, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device="cuda")
    cov = (rnd(B, H, W, 1) < 0.6).float()
    edge = (rnd(B, H, W, 1) < 0.05).float()
    alpha = torch.clamp(cov + edge * rnd(B, H, W, 1), 0, 1)                     # mostly 0 / 1, fractional at silhouette edges
    shaded = torch.cat([rnd(B, H, W, 3) * 2.0 * alpha, alpha], -1)
    ref_buf = torch.cat([rnd(B, H, W, 3) * 2.0, (rnd(B, H, W, 1) < 0.6).float(), rnd(B, H, W, 4)], -1)
    return shaded, ref_buf[..., 0:4]


def step(fn, shaded, ref, loss, tonemapper):
    s = shaded.detach().requires_grad_(True)
    G = torch.ones((), device="cuda")

    def run():
        out = fn(s, ref, loss, tonemapper)
        return out, torch.autograd.grad(out, s, grad_outputs=G)[0]
    return run


def timed(fn, inner):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(inner):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / inner


def alternate(arms, reps, inner, warmup):
    """{name: {median, min, max} ms} of each zero-argument callable, their timings interleaved."""
    for f in arms.values():
        for _ in range(warmup):
            f()
    torch.cuda.synchronize()
    samples = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            samples[k].append(timed(f, inner))
    return {k: {"median": sorted(v)[len(v) // 2], "min": min(v), "max": max(v)} for k, v in samples.items()}


def kernels(fn):
    """[(kernel or memset name, launches, device microseconds)] of one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    n, us = collections.Counter(), collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            n[e.name] += 1
            us[e.name] += e.device_time_total
    return [[k[:120], v, round(us[k], 2)] for k, v in sorted(n.items())]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loss", default="l1")
    ap.add_argument("--tonemapper", default="log_srgb")
    ap.add_argument("--shape", default="8,512,512")
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--inner", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "lossbench needs a GPU"
    B, H, W = (int(x) for x in a.shape.split(","))
    shaded, ref = inputs(B, H, W)
    arms = {"chain": step(chain, shaded, ref, a.loss, a.tonemapper), "coverage_image_loss": step(R.coverage_image_loss, shaded, ref, a.loss,
                                                                                                   a.tonemapper)}
    (lc, gc), (lp, gp) = arms["chain"](), arms["coverage_image_loss"]()
    same = bool(torch.equal(gc.view(torch.int32), gp.view(torch.int32)))
    rel = abs(float(lp) - float(lc)) / abs(float(lc))
    assert same and rel <= 1e-6, "coverage_image_loss and the chain disagree (d shaded bit for bit: %s, loss rel %.3g)" % (same, rel)
    res = {"card": card(), "shape": [B, H, W], "loss": a.loss, "tonemapper": a.tonemapper, "reps": a.reps, "inner": a.inner,
           "agree": {"d_shaded_bit_for_bit": same, "loss_rel": rel}}
    res["fwd_bwd_ms"] = alternate(arms, a.reps, a.inner, a.warmup)
    with torch.no_grad():
        det = shaded.detach()
        fwd = {"chain": lambda: chain(det, ref, a.loss, a.tonemapper), "coverage_image_loss": lambda: R.coverage_image_loss(det, ref, a.loss,
                                                                                                                        a.tonemapper)}
        res["fwd_no_grad_ms"] = alternate(fwd, a.reps, a.inner, a.warmup)
    res["fwd_bwd_ms_second_run"] = alternate(dict(reversed(list(arms.items()))), a.reps, a.inner, a.warmup)
    res["kernels_fwd_bwd"] = {k: kernels(f) for k, f in arms.items()}
    res["launches_fwd_bwd"] = {k: sum(x[1] for x in v) for k, v in res["kernels_fwd_bwd"].items()}
    res["device_us_fwd_bwd"] = {k: round(sum(x[2] for x in v), 2) for k, v in res["kernels_fwd_bwd"].items()}
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
