"""Shared builders for the parity tests: seeded synthetic scenes (numpy) consumable by both the CPU
oracle and the CUDA product."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from nvdiffrecmc_b200 import synth  # noqa: E402

_ORACLE = {}


def oracle(f64=False):
    from oracle import Oracle
    if f64 not in _ORACLE:
        _ORACLE[f64] = Oracle(f64=f64)
    return _ORACLE[f64]


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def make_case(res=32, B=1, N=4, mesh="blob+torus", level=2, light="random", light_hw=(32, 64), seed=0, ks_mode="random",
              perm_rows=512, closest=None):
    """Returns a dict of numpy arrays describing one env_shade problem.
    closest(verts, tris, ro[n,3], rd[n,3]) -> (tri_id[n], tuv[n,3]) overrides the oracle's brute-force primary visibility."""
    o = oracle()
    v, f = synth.scene_mesh(mesh, level=level, seed=5 + seed)
    vn = synth.vertex_normals(v, f)
    scene = o.scene(v, f)
    gbs = []
    for b in range(B):
        mv = synth.orbit_view(0.7 * b + 0.3 * seed)
        campos, ro, rd = synth.primary_rays(mv, res)
        if closest is None:
            tid, tuv = scene.closest_hit(ro.reshape(-1, 3), rd.reshape(-1, 3))
        else:
            tid, tuv = closest(v, f, ro.reshape(-1, 3), rd.reshape(-1, 3))
        gbs.append(synth.assemble_gbuffer(v, f, vn, np.asarray(tid).reshape(res, res), np.asarray(tuv).reshape(res, res, 3), campos,
                                          seed=1 + b + 10 * seed, ks_mode=ks_mode))
    st = lambda k: np.stack([g[k] for g in gbs])
    view = st("view_pos").reshape(B, 1, 1, 3)
    pos, sn, tg, gn = st("pos"), st("smooth_nrm"), st("tangent"), st("geom_nrm")
    nrm = o.prepare_shading_normal(pos, view, None, sn, tg, gn)       # render.py:99
    mask = st("mask")
    nrm = nrm * (mask[..., None] > 0)
    ro = (pos + nrm * np.float32(0.001)).astype(np.float32)             # render.py:110
    if light == "random":
        base = synth.random_light(light_hw[0], seed=2 + seed)
        if light_hw[0] != light_hw[1]:
            base = np.ascontiguousarray(np.random.default_rng(2 + seed).uniform(0.25, 0.75, size=(light_hw[0], light_hw[1], 3)), np.float32)
    else:
        base = synth.hdr_light(light_hw[0], light_hw[1], seed=7 + seed)
    pdf, rows, cols = o.update_pdf(base)
    perms = synth.make_perms(N, seed=3 + seed, rows=perm_rows)
    return dict(verts=v, tris=f, scene=scene, mask=mask, ro=ro, pos=pos, nrm=nrm.astype(np.float32), view=view.astype(np.float32),
                kd=st("kd"), ks=st("ks"), depth=st("depth"), smooth_nrm=sn, tangent=tg, geom_nrm=gn,
                light=base, pdf=pdf, rows=rows, cols=cols, perms=perms, N=N, B=B, res=res)


# The renderutils ops with their oracle entry points:
# name, oracle forward, oracle backward, input channels, output channels, extras (f0, i0, i1), oracle kwargs
RU_OPS = [
    ("lambert", "lambert", "lambert_bwd", [3, 3], 1, (0.0, 0, 0), {}),
    ("frostbite", "frostbite_diffuse", "frostbite_diffuse_bwd", [3, 3, 3, 1], 1, (0.0, 0, 0), {}),
    ("fresnel", "fresnel_shlick", "fresnel_shlick_bwd", [3, 3, 1], 3, (0.0, 0, 0), {}),
    ("ndf", "ndf_ggx", "ndf_ggx_bwd", [1, 1], 1, (0.0, 0, 0), {}),
    ("lambda", "lambda_ggx", "lambda_ggx_bwd", [1, 1], 1, (0.0, 0, 0), {}),
    ("masking", "masking_smith", "masking_smith_bwd", [1, 1, 1], 1, (0.0, 0, 0), {}),
    ("specular", "pbr_specular", "pbr_specular_bwd", [3, 3, 3, 3, 1], 3, (0.08, 0, 0), {"min_roughness": 0.08}),
    ("bsdf", "pbr_bsdf", "pbr_bsdf_bwd", [3] * 6, 3, (0.08, 0, 0), {"min_roughness": 0.08, "bsdf": "lambert"}),
    ("bsdf", "pbr_bsdf", "pbr_bsdf_bwd", [3] * 6, 3, (0.08, 1, 0), {"min_roughness": 0.08, "bsdf": "frostbite"}),
    ("psn", "prepare_shading_normal", "prepare_shading_normal_bwd", [3] * 6, 3, (0.0, 1, 1), {"two_sided_shading": True, "opengl": True}),
    ("psn", "prepare_shading_normal", "prepare_shading_normal_bwd", [3] * 6, 3, (0.0, 0, 0), {"two_sided_shading": False, "opengl": False}),
]


def ru_edge_inputs(chans, out_c):
    """Renderutils inputs the reference tests never draw: zero vectors (safe-normalise guard), back-facing / grazing configurations,
    roughness at both ends of its clamp range, negative and > 1 values.  Returns ([1,6,8,c] inputs, [1,6,8,out_c] upstream gradient).
    Pixels (0,0) .. (0,2) hold 0, 1 and -1 in every channel, (1,0) and (1,1) hold 1e-6 and 1e4."""
    g = np.random.default_rng(11)
    shape = (1, 6, 8)
    ins = [g.normal(size=shape + (c,)).astype(np.float32) * (3.0 if c == 3 else 1.0) for c in chans]
    for a in ins:
        a[0, 0, 0] = 0.0                      # all-zero vectors / scalars
        a[0, 0, 1] = 1.0
        a[0, 0, 2] = -1.0
        a[0, 1, 0] = 1e-6
        a[0, 1, 1] = 1e4
    dout = g.uniform(size=shape + (out_c,)).astype(np.float32)
    return ins, dout


def env_shade_edge_case():
    """An env_shade problem with pixels the synthetic scenes never contain: zero shading normal, camera behind the surface (NdotV < 0),
    roughness 0 and 1 (min-roughness clamp), pure metal, black albedo, and a probe with a black row and black texels.
    Returns the make_case dict with those edits (pdf / rows / cols rebuilt for the edited probe); c["edge_px"][k] is the (b, y, x)
    index of edited pixel k: 0 zero normal, 1 flipped normal, 2-4 ks edits, 5-6 kd edits."""
    N = 4
    c = make_case(res=16, B=1, N=N, seed=4)
    m = c["mask"][0] > 0
    ys, xs = np.nonzero(m)
    assert len(ys) > 40
    nrm, kd, ks = c["nrm"].copy(), c["kd"].copy(), c["ks"].copy()
    px = [(0, ys[k], xs[k]) for k in range(7)]
    nrm[px[0]] = 0.0
    nrm[px[1]] = -nrm[px[1]]                                  # back-facing shading normal
    ks[px[2]] = [0.0, 0.0, 0.0]; ks[px[3]] = [0.0, 1.0, 1.0]; ks[px[4]] = [0.0, 0.08, 0.5]
    kd[px[5]] = 0.0; kd[px[6]] = 1.0
    light = c["light"].copy(); light[3] = 0.0; light[10, ::2] = 0.0
    pdf, rows, cols = oracle().update_pdf(light)
    c.update(nrm=nrm, kd=kd, ks=ks, light=light, pdf=pdf, rows=rows, cols=cols, edge_px=px)
    return c
