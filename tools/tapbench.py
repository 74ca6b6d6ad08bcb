"""Times the jittered regulariser taps (nvdiffrecmc_b200.regularizer.jitter_taps, csrc/taps.cu) against the reference's lines of shade()
(render/render.py:50-97) composed from raster.texture and torch ops, at the training sizes 8 x 512^2 and 8 x 800^2.

Two configurations, with training-like operands (70 % coverage, jitter = pixel grid + N(0, 0.005)): "texture" (kd [..,3], ks the
[..., 0:3] slice of a 4-channel sample, gb_normal and a normal map: five taps) and "mlp" (kd / ks and their jittered samples as slices of
6-channel MLP outputs, gb_normal tapped).  Per size and configuration: the forward under no_grad (the dataset's reference render) and
forward + backward of sum_k <G_k, buffer_k>.  Every timing is the median of --reps CUDA-event timings of --inner calls each, the fused op
and the composition alternating, in two runs.  Before any time is quoted the two are checked to agree on the same inputs (kd_grad,
ks_grad, normal_grad bit for bit; perturbed_nrm_grad to 1e-5, as torch's own order of the three-element sums meets pixels where
sn(tap(p)) nearly cancels sn(p); gradients to 1e-5 relative L2).  Prints one JSON document with the card's
name and power limit, read in the same run.

    python tools/tapbench.py [--reps 25] [--inner 10] [--warmup 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from nvdiffrecmc_b200 import raster  # noqa: E402
from nvdiffrecmc_b200.regularizer import jitter_taps  # noqa: E402


def _sn(x):
    return x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=1e-20))


def composition(rast, jitter, kd, ks, gb_normal, perturbed_nrm=None, kd_jitter=None, ks_jitter=None):
    """render.py:50-97 with raster.texture as dr.texture, and the buffers' alpha as at :151-153,161-163"""
    tex = lambda t: raster.texture(t.contiguous(), jitter, filter_mode='linear', boundary_mode='clamp')
    mask = (rast[..., -1:] > 0).float()
    grad_weight = mask * tex(mask)
    m011 = torch.tensor([0, 1, 1], dtype=torch.float32, device="cuda")[None, None, None, :]
    if kd_jitter is not None:
        kd_grad = torch.abs(kd_jitter - kd)
        ks_grad = torch.abs(ks_jitter - ks) * m011
    else:
        kd_grad = torch.abs(tex(kd) - kd) * grad_weight
        ks_grad = torch.abs(tex(ks) - ks) * m011 * grad_weight
    alpha = kd[..., 3:4] if kd.shape[-1] == 4 else torch.ones_like(kd[..., 0:1])
    nrm_grad = torch.abs(tex(gb_normal) - gb_normal) * grad_weight
    out = {"kd_grad": torch.cat((kd_grad, alpha), -1), "ks_grad": torch.cat((ks_grad, alpha), -1), "normal_grad": torch.cat((nrm_grad, alpha), -1)}
    if perturbed_nrm is not None:
        pg = 1.0 - _sn(_sn(tex(perturbed_nrm)) + _sn(perturbed_nrm))[..., 2:3]
        out["perturbed_nrm_grad"] = torch.cat((pg.repeat(1, 1, 1, 3) * grad_weight, alpha), -1)
    return out


def inputs(cfg, B, H, W, seed=0):
    """(operands with the differentiable ones as leaves or slices of leaves, the leaves, upstream gradients)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g, device="cuda")
    nrm = lambda: torch.nn.functional.normalize(torch.randn(B, H, W, 3, generator=g, device="cuda") + torch.tensor([0, 0, 1.5], device="cuda"), dim=-1)
    rast = torch.zeros(B, H, W, 4, device="cuda")
    rast[..., 3] = (rnd(B, H, W) < 0.7).float() * 7
    y, x = torch.meshgrid((torch.arange(H, device="cuda") + 0.5) / H, (torch.arange(W, device="cuda") + 0.5) / W, indexing="ij")
    jitter = (torch.stack((x, y), -1)[None] + 0.005 * torch.randn(B, H, W, 2, generator=g, device="cuda")).contiguous()
    n = nrm().requires_grad_(True)
    if cfg == "texture":
        kd, ks4, p = rnd(B, H, W, 3).requires_grad_(True), rnd(B, H, W, 4).requires_grad_(True), nrm().requires_grad_(True)
        ops, leaves = [rast, jitter, kd, ks4[..., 0:3], n, p, None, None], [kd, ks4, n, p]
    else:
        T, J = rnd(B, H, W, 6).requires_grad_(True), rnd(B, H, W, 6).requires_grad_(True)
        ops, leaves = [rast, jitter, T[..., 0:3], T[..., 3:6], n, None, J[..., 0:3], J[..., 3:6]], [T, J, n]
    with torch.no_grad():
        shapes = {k: v.shape for k, v in jitter_taps(*ops).items()}
    G = {k: torch.randn(*s, generator=g, device="cuda") for k, s in shapes.items()}
    return ops, leaves, G


def fwd_bwd(impl, ops, leaves, G):
    def run():
        out = impl(*ops)
        return torch.autograd.grad(sum((out[k] * G[k]).sum() for k in out), leaves)
    return run


def agree(ops, leaves, G):
    """(buffers bit-identical except perturbed_nrm_grad, perturbed_nrm_grad max |difference|, worst gradient relative L2)"""
    a, b = jitter_taps(*ops), composition(*ops)
    same = all(torch.equal(a[k], b[k]) for k in ("kd_grad", "ks_grad", "normal_grad"))
    pd = float((a["perturbed_nrm_grad"] - b["perturbed_nrm_grad"]).abs().max()) if "perturbed_nrm_grad" in a else 0.0
    ga, gb = fwd_bwd(jitter_taps, ops, leaves, G)(), fwd_bwd(composition, ops, leaves, G)()
    return same, pd, max(float((x - y).norm() / y.norm()) for x, y in zip(ga, gb))


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
    return sorted(ts)[len(ts) // 2]


def alternate(arms, reps, inner, warmup):
    """{name: median ms} of each zero-argument callable of `arms`, their timings interleaved."""
    for f in arms.values():
        timed(f, 1, 1, warmup)
    samples = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            samples[k].append(timed(f, 1, inner, 0))
    return {k: sorted(v)[len(v) // 2] for k, v in samples.items()}


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
    assert torch.cuda.is_available(), "tapbench needs a GPU"
    res = {"card": card(), "reps": a.reps, "inner": a.inner, "sizes": {}}
    for B, H, W in ((8, 512, 512), (8, 800, 800)):
        row = {}
        for cfg in ("texture", "mlp"):
            ops, leaves, G = inputs(cfg, B, H, W)
            same, pd, gl2 = agree(ops, leaves, G)
            assert same and pd <= 1e-5 and gl2 < 1e-5, "%s: fused op and composition disagree (%s, %.3g, %.3g)" % (cfg, same, pd, gl2)
            det = [None if t is None else t.detach() for t in ops]
            runs = []
            for _ in range(2):
                with torch.no_grad():
                    fwd = alternate({"fused": lambda: jitter_taps(*det), "torch": lambda: composition(*det)}, a.reps, a.inner, a.warmup)
                fb = alternate({"fused": fwd_bwd(jitter_taps, ops, leaves, G), "torch": fwd_bwd(composition, ops, leaves, G)}, a.reps, a.inner,
                               a.warmup)
                runs.append({"fwd_ms": fwd, "fwd_bwd_ms": fb})
            row[cfg] = {"agree_perturbed_max_abs": pd, "agree_grad_rel_l2": gl2, "runs": runs}
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
