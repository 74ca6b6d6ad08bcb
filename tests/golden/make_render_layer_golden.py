"""Generates tests/golden/ref_render_layer_db.npz by running the UNMODIFIED reference `render_layer` (render/render.py:172-253) on the CPU.

  * the reference module is imported through tests/refshade.py's `reference_render` (stub nvdiffrast, CPU redirection), unedited;
  * the stub's `dr.interpolate` is replaced by one with nvdiffrast's signature `(attr, rast, tri, rast_db=None, diff_attrs=None)`
    computing on the fp32 oracle of the derivatives (oracle/geometry.c: interpolate, out_da), with nvdiffrast's broadcast of a [1,V,C] attribute;
  * `shade` on the imported module is replaced by a function that captures its arguments (render_layer's G-buffer) and returns {};
  * `rast` is the oracle's closest hit (u, v = weights of vertices 0 / 1, z/w, id + 1) of a blob+torus scene seen by two perspective
    views at 24 x 32, and `rast_deriv` the oracle's rast_db of the clip-space vertices.

Stored: the mesh (verts, tris, v_tex, uv_idx), the clip-space pos [B,V,4], rast, rast_deriv and what render_layer passes to shade:
gb_texc, gb_texc_deriv and gb_depth (z0, z_grad).  This proves that the reference's own calls bind to the signature and layout of
`raster.interpolate(..., rast_db=, diff_attrs='all')`.  Nothing from the reference is copied into this repository.
    python tests/golden/make_render_layer_golden.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_render_layer_db.npz")
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

RES = (24, 32)
B = 2


def scene():
    """(verts, tris, v_tex, uv_idx, mtx [B,4,4]) in fp32 / int32."""
    from nvdiffrecmc_b200 import synth
    v, f = synth.scene_mesh("blob+torus", level=1)
    v, f = v.astype(np.float32), f.astype(np.int32)
    c = v - v.mean(0)
    v_tex = np.stack([0.5 + np.arctan2(c[:, 2], c[:, 0]) / (2 * np.pi), 0.5 + 0.4 * c[:, 1] / np.abs(c[:, 1]).max()], -1).astype(np.float32)
    proj = synth.perspective(aspect=RES[1] / RES[0], n=0.1, f=10.0).astype(np.float64)
    mtx = []
    for b in range(B):
        a = 0.8 * b + 0.4
        mv = np.eye(4)
        mv[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
        mv[2, 3] = -2.6
        mtx.append(proj @ mv)
    return v, f, v_tex, f.copy(), np.stack(mtx).astype(np.float32)


def oracle_rast(v, f, mtx):
    """rast [B,H,W,4] from the oracle's closest hit of each pixel's near-far segment (as k_rasterize un-projects it)."""
    from common import oracle
    sc = oracle().scene(v, f)
    H, W = RES
    ys, xs = np.meshgrid((np.arange(H, dtype=np.float32) + 0.5) / H * 2 - 1, (np.arange(W, dtype=np.float32) + 0.5) / W * 2 - 1, indexing="ij")
    rast = np.zeros((B, H, W, 4), np.float32)
    for b in range(B):
        inv = np.linalg.inv(mtx[b].astype(np.float64))
        near = np.stack([xs, ys, -np.ones_like(xs), np.ones_like(xs)], -1) @ inv.T
        far = np.stack([xs, ys, np.ones_like(xs), np.ones_like(xs)], -1) @ inv.T
        o = (near[..., :3] / near[..., 3:]).reshape(-1, 3).astype(np.float32); e = (far[..., :3] / far[..., 3:]).reshape(-1, 3).astype(np.float32)
        tid, tuv = sc.closest_hit(o, e - o)
        hit = tid >= 0
        p = (o + (e - o) * tuv[:, :1]).astype(np.float64)
        clip = np.concatenate([p, np.ones((p.shape[0], 1))], 1) @ mtx[b].astype(np.float64).T
        r = np.zeros((H * W, 4), np.float32)
        r[hit, 0] = 1 - tuv[hit, 1] - tuv[hit, 2]
        r[hit, 1] = tuv[hit, 1]
        r[hit, 2] = (clip[hit, 2] / clip[hit, 3]).astype(np.float32)
        r[hit, 3] = tid[hit] + 1
        rast[b] = r.reshape(H, W, 4)
    return rast


def oracle_interpolate(geo):
    """nvdiffrast's `interpolate` signature on the fp32 oracle of the derivatives (CPU tensors, forward only)."""
    def interpolate(attr, rast, tri, rast_db=None, diff_attrs=None):
        a = attr.detach().numpy()
        if a.ndim == 3 and a.shape[0] == 1:
            a = a[0]                                   # nvdiffrast broadcasts a [1,V,C] attribute over the minibatch
        r, t = rast.detach().numpy(), tri.detach().numpy()
        out = torch.from_numpy(geo.interpolate(a, t, r))
        if diff_attrs is None:
            return out, None
        assert rast_db is not None
        return out, torch.from_numpy(geo.interpolate_da(a, t, r, rast_db.detach().numpy(), diff_attrs))
    return interpolate


def generate():
    from oracle.geometry import geometry_oracle
    from refshade import reference_render
    geo = geometry_oracle()
    v, f, v_tex, uv_idx, mtx = scene()
    pos = np.einsum("bij,vj->bvi", mtx.astype(np.float64), np.concatenate([v, np.ones((v.shape[0], 1), np.float32)], 1)).astype(np.float32)
    rast = oracle_rast(v, f, mtx)
    rast_db = geo.rast_db(pos, f, rast)
    vt = torch.from_numpy(v)
    nrm = torch.nn.functional.normalize(vt - vt.mean(0), dim=-1)
    mesh = types.SimpleNamespace(v_pos=vt, t_pos_idx=torch.from_numpy(f).long(), v_nrm=nrm, t_nrm_idx=torch.from_numpy(f).long(),
                                 v_tng=torch.roll(nrm, 1, -1), t_tng_idx=torch.from_numpy(f).long(), v_tex=torch.from_numpy(v_tex),
                                 t_tex_idx=torch.from_numpy(uv_idx).long(), material=None)
    captured = {}

    def shade(FLAGS, rast, gb_depth, gb_pos, gb_geometric_normal, gb_normal, gb_tangent, gb_texc, gb_texc_deriv, *rest):
        captured.update(gb_depth=gb_depth, gb_texc=gb_texc, gb_texc_deriv=gb_texc_deriv)
        return {}

    empty = types.ModuleType("unused_backend")
    with reference_render(empty, empty) as (render, _light, _den):
        render.dr.interpolate = oracle_interpolate(geo)
        render.shade = shade
        with torch.no_grad():
            render.render_layer(None, torch.from_numpy(pos), torch.from_numpy(rast), torch.from_numpy(rast_db), mesh, None, None, list(RES), 1, False,
                                None, None, None, 1.0)
    d = {"verts": v, "tris": f, "v_tex": v_tex, "uv_idx": uv_idx, "mtx": mtx, "pos": pos, "rast": rast, "rast_deriv": rast_db}
    d.update({k: t.numpy() for k, t in captured.items()})
    return d


if __name__ == "__main__":
    d = generate()
    np.savez_compressed(OUT, **d)
    cov = int((d["rast"][..., 3] > 0).sum())
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", cov, "covered pixels; gb_depth", d["gb_depth"].shape, "gb_texc_deriv", d["gb_texc_deriv"].shape)
