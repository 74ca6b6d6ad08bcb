"""Developer tool: CUDA-event timings of DMTet's geometry (csrc/dmtet.cu) against a plain-PyTorch composition of the same contract.

Grids: a procedural Kuhn grid of 64^3 cells (274 625 vertices, 1 572 864 tets: the scale of the reference's 128 grid) and the reference's
32 grid (tests/golden/tets_32.npz).  SDFs: the reference's initialisation rand - 0.1 (the large surface of the first iterations) and a
sphere of radius 0.3.  Timed (median of REPS after warm-up), each for the kernels and for the composition:
  fwd      marching_tets with grad enabled: count, the read-back of the counts, emit (the composition: occupancy masks, torch.unique of the
           valid tets' edges, boolean-mask indexing, the UV table rebuilt as the reference does)
  bwd      d pos and d sdf of a seeded upstream gradient of verts (the composition: autograd)
  reg      sdf_reg_loss over the grid's edges, forward + backward
The kernels' tables are built before timing (once per grid, as in training).  Prints the card name and power limit.
usage: python tools/dmtetbench.py [out.json]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
from dmtet_grids import grid32, kuhn_grid, ref_init_sdf, sphere_sdf
from nvdiffrecmc_b200.dmtet import marching_tets, sdf_reg_loss

dev = torch.device("cuda:0")
REPS = 20
BASE = [0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3]
TRI = torch.tensor([[-1] * 6, [1, 0, 2, -1, -1, -1], [4, 0, 3, -1, -1, -1], [1, 4, 2, 1, 3, 4], [3, 1, 5, -1, -1, -1], [2, 3, 0, 2, 5, 3],
                    [1, 4, 0, 1, 5, 4], [4, 2, 5, -1, -1, -1], [4, 5, 2, -1, -1, -1], [4, 1, 0, 4, 5, 1], [3, 2, 0, 3, 5, 2],
                    [1, 3, 5, -1, -1, -1], [4, 1, 2, 4, 3, 1], [3, 0, 4, -1, -1, -1], [2, 0, 1, -1, -1, -1], [-1] * 6], device=dev)
NTRI = torch.tensor([0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0], device=dev)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(dev)


def event_ms(fn, reps=REPS, warm=3):
    ts = []
    for k in range(reps + warm):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        if k >= warm:
            ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def torch_marching_tets(pos, sdf, tet):
    """The contract as a per-call PyTorch composition: masks, torch.unique of the valid tets' edges, gathers."""
    occ = sdf > 0
    occ4 = occ[tet]
    n = occ4.sum(-1)
    valid = (n > 0) & (n < 4)
    with torch.no_grad():
        e = torch.sort(tet[valid][:, BASE].reshape(-1, 2), dim=1)[0]
        ue, inv = torch.unique(e, dim=0, return_inverse=True)
        cross = occ[ue[:, 0]] != occ[ue[:, 1]]
        vid = torch.cumsum(cross.long(), 0) - 1
        vid[~cross] = -1
        a, b = ue[cross, 0], ue[cross, 1]
    sa, sb = sdf[a], sdf[b]
    D = sa + (-sb)
    verts = pos[a] * ((-sb) / D)[:, None] + pos[b] * (sa / D)[:, None]
    with torch.no_grad():
        emap = vid[inv].reshape(-1, 6)
        code = (occ4[valid].long() * torch.tensor([1, 2, 4, 8], device=dev)).sum(-1)
        nt = NTRI[code]
        one, two = nt == 1, nt == 2
        faces = torch.cat([torch.gather(emap[one], 1, TRI[code[one]][:, :3]).reshape(-1, 3),
                           torch.gather(emap[two], 1, TRI[code[two]]).reshape(-1, 3)])
        t = torch.arange(tet.shape[0], device=dev)[valid]
        tt = torch.cat([t[one], t[two].repeat_interleave(2)])
        k = torch.cat([torch.zeros_like(t[one]), torch.arange(2, device=dev).repeat(int(two.sum()))])
        uv_idx = torch.stack([4 * tt, 4 * tt + k + 1, 4 * tt + k + 2], -1)
        N = int(np.ceil(np.sqrt(tet.shape[0])))
        ax = torch.linspace(0, 1 - 1 / N, N, device=dev)
        y, x = torch.meshgrid(ax, ax, indexing="ij")
        p = 0.9 / N
        uvs = torch.stack([x, y, x + p, y, x + p, y + p, x, y + p], -1).view(-1, 2)
    return verts, faces, uvs, uv_idx


def torch_sdf_reg_loss(sdf, edges):
    s = sdf[edges.reshape(-1)].reshape(-1, 2)
    s = s[torch.sign(s[:, 0]) != torch.sign(s[:, 1])]
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    return bce(s[:, 0], (s[:, 1] > 0).float()) + bce(s[:, 1], (s[:, 0] > 0).float())


def bench_case(verts, tets, sdf):
    pos = torch.tensor(verts, device=dev, requires_grad=True)
    s = torch.tensor(sdf, device=dev, requires_grad=True)
    t = torch.tensor(tets, device=dev)
    edges = torch.unique(torch.sort(t[:, BASE].reshape(-1, 2), dim=1)[0], dim=0)
    out = {}
    for arm, mt, reg in (("kernels", marching_tets, sdf_reg_loss), ("torch", torch_marching_tets, torch_sdf_reg_loss)):
        v = mt(pos, s, t)[0]
        G = torch.randn(v.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        box = {}

        def fwd():
            box["v"] = mt(pos, s, t)[0]

        def bwd():
            torch.autograd.grad(box["v"], (pos, s), G, retain_graph=True)

        def reg_fb():
            torch.autograd.grad(reg(s, edges), s)
        fwd()
        out[arm] = {"fwd_ms": event_ms(fwd), "bwd_ms": event_ms(bwd), "reg_fwd_bwd_ms": event_ms(reg_fb)}
        out[arm]["verts"], out[arm]["faces"] = int(v.shape[0]), int(mt(pos, s, t)[1].shape[0])
    return out


def main():
    res = {"card": card(), "torch": torch.__version__, "cases": {}}
    print("[dmtetbench]", res["card"], flush=True)
    for gname, (verts, tets) in (("kuhn64", kuhn_grid(64)), ("grid32", grid32())):
        for sname, sdf in (("ref_init", ref_init_sdf(verts.shape[0], seed=0)), ("sphere", sphere_sdf(verts, 0.3))):
            r = bench_case(verts, tets, sdf)
            res["cases"]["%s/%s" % (gname, sname)] = r
            for arm in ("kernels", "torch"):
                print("  %-16s %-7s V %7d T %8d -> %7d verts %8d faces: fwd %7.3f ms  bwd %7.3f ms  reg fwd+bwd %7.3f ms" % (
                    gname + "/" + sname, arm, verts.shape[0], tets.shape[0], r[arm]["verts"], r[arm]["faces"], r[arm]["fwd_ms"], r[arm]["bwd_ms"],
                    r[arm]["reg_fwd_bwd_ms"]), flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
