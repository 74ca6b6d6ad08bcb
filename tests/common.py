"""Shared builders for the parity tests: seeded synthetic scenes (numpy) consumable by both the CPU
oracle and the CUDA product."""
import ctypes as C
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from nvdiffrecmc_b200 import synth  # noqa: E402

def oracle(f64=False):
    from oracle import Oracle
    return Oracle.get(f64)


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def make_case(res=32, B=1, N=4, mesh="blob+torus", level=2, light="random", light_hw=(32, 64), seed=0, ks_mode="random",
              perm_rows=512, closest=None):
    """Returns a dict of numpy arrays describing one env_shade problem.  mesh: a synth.scene_mesh kind, or a (verts, tris) pair.
    closest(verts, tris, ro[n,3], rd[n,3]) -> (tri_id[n], tuv[n,3]) overrides the oracle's brute-force primary visibility."""
    o = oracle()
    v, f = synth.scene_mesh(mesh, level=level, seed=5 + seed) if isinstance(mesh, str) else mesh
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


# ------------------------------------------------------------------------------------------ rasterize: cameras and meshes
def frustum(l, r, b, t, n, f):
    """glFrustum: an off-axis (asymmetric) perspective projection."""
    return np.array([[2 * n / (r - l), 0, (r + l) / (r - l), 0], [0, 2 * n / (t - b), (t + b) / (t - b), 0],
                     [0, 0, -(f + n) / (f - n), -2 * f * n / (f - n)], [0, 0, -1, 0]], np.float64)


def ortho(l, r, b, t, n, f):
    """glOrtho: clip w is 1 everywhere."""
    return np.array([[2 / (r - l), 0, 0, -(r + l) / (r - l)], [0, 2 / (t - b), 0, -(t + b) / (t - b)],
                     [0, 0, -2 / (f - n), -(f + n) / (f - n)], [0, 0, 0, 1]], np.float64)


RASTER_CAMERAS = ["persp", "offaxis", "ortho", "wide", "inside", "behind", "away", "front", "singular"]


def raster_mtx(kind, B, aspect=1.0):
    """[B,4,4] fp32 clip matrices, a different one per view, around a mesh of radius ~1 at the origin.
      persp / offaxis / ortho / wide: orbit views through a symmetric, an asymmetric, an orthographic and a 1e-2 .. 1e3 frustum;
      inside:   the eye at the origin, inside the blob, with the near plane at 0.5, so it cuts the surface;
      behind:   the eye at the origin with a 160-degree field of view, so triangles at the image's edge have vertices behind the eye
                (clip w <= 0);
      away:     orbit eyes looking away from the mesh (every hit has t < 0);
      front:    eyes near (0, 0, 3) looking down -z (the `far` mesh's quad lies beyond their far plane);
      singular: view 0 is all zeros, the others have a zero w row."""
    out = []
    for b in range(B):
        ang, tilt = 0.7 * b + 0.3, -0.4 + 0.15 * b
        mv = synth.orbit_view(ang, tilt=tilt)
        if kind == "persp":
            m = synth.perspective(aspect=aspect, n=0.1, f=10.0).astype(np.float64) @ mv
        elif kind == "offaxis":
            m = frustum(-0.03 * aspect, 0.06 * aspect, -0.05, 0.035, 0.1, 10.0) @ mv
        elif kind == "ortho":
            m = ortho(-1.4 * aspect, 1.2 * aspect, -1.1, 1.5, 0.5, 6.0) @ mv
        elif kind == "wide":
            m = synth.perspective(aspect=aspect, n=1e-2, f=1e3).astype(np.float64) @ mv
        elif kind == "inside":
            rot = synth.orbit_view(ang, radius=0.0, tilt=tilt)
            m = synth.perspective(fovy=1.2, aspect=aspect, n=0.5, f=10.0).astype(np.float64) @ rot
        elif kind == "behind":
            rot = synth.orbit_view(ang, radius=0.0, tilt=tilt)
            m = synth.perspective(fovy=2.8, aspect=aspect, n=0.05, f=10.0).astype(np.float64) @ rot
        elif kind == "away":
            flip = np.diag([-1.0, 1.0, -1.0, 1.0])                   # a half turn about the eye's own y axis
            m = synth.perspective(aspect=aspect, n=0.1, f=10.0).astype(np.float64) @ flip @ mv
        elif kind == "front":                                          # eyes near (0, 0, 3), looking down -z
            m = synth.perspective(aspect=aspect, n=0.1, f=10.0).astype(np.float64) @ synth.orbit_view(0.05 * b, tilt=0.03 * b)
        elif kind == "singular":
            m = synth.perspective(aspect=aspect, n=0.1, f=10.0).astype(np.float64) @ mv
            m[3] = 0.0
            if b == 0:
                m[:] = 0.0
        else:
            raise ValueError(kind)
        out.append(m)
    return np.stack(out).astype(np.float32)


# ------------------------------------------------------------------------------------------ the per-element bar against the fp64 oracle
N_PERT = 4


def _ulp32(x):
    a = np.minimum(np.abs(np.asarray(x, np.float64)), np.finfo(np.float32).max).astype(np.float32)
    return np.nextafter(a, np.float32(np.inf)).astype(np.float64) - a.astype(np.float64)


def _perturb(x, rng):
    """Every element of the fp32 array x moved by one ulp up or down (seeded coin)."""
    x = np.asarray(x, np.float32)
    up = rng.random(x.shape) < 0.5
    return np.where(up, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf))).astype(np.float32)


def check_per_element(op, got, f64, f32, ins, K, names, seed=0, exempt=None, floor=None, tag="step-tail"):
    """got: the kernel's outputs (numpy); f64(ins) / f32(ins): the fp64 / fp32 oracle on the fp32 inputs `ins`, returning arrays of got's
    shapes in the same order; exempt: per output, a boolean mask of elements the caller checks by another rule (or None); floor: per
    output, a non-negative array R broadcastable to its shape (or None): the reduction floor, the most that summing the element's terms
    in another order can change it.  With r64 / r32 the fp64 / fp32 oracle and Delta the largest change of r64 over N_PERT seeded
    perturbations of every input element by +-1 fp32 ulp (a per-element sensitivity estimate), every finite element must satisfy
        |got - r64| <= K * max(Delta, |r32 - r64|) + R + 4 * ulp32(r64)
    and NaN / +-inf must sit where the fp32 oracle has them.  Returns the worst ratio (|got - r64| - R - 4 ulp) / max(Delta, |r32 - r64|)
    over all outputs; `tag` prefixes the printed per-output line."""
    r64 = [np.asarray(r, np.float64) for r in f64(ins)]
    r32 = [np.asarray(r, np.float64) for r in f32(ins)]
    rng = np.random.default_rng(1000 + seed)
    delta = [np.zeros_like(r) for r in r64]
    for _ in range(N_PERT):
        for d, r, rp in zip(delta, r64, f64([_perturb(x, rng) for x in ins])):
            np.fmax(d, np.abs(np.asarray(rp, np.float64) - r), out=d)
    worst = 0.0
    for k, (g, a, b, d) in enumerate(zip(got, r64, r32, delta)):
        name = "%s: %s" % (op, names[k])
        g = np.asarray(g, np.float64)
        assert g.shape == a.shape, (name, g.shape, a.shape)
        for pred, what in ((np.isnan, "NaN"), (np.isposinf, "+inf"), (np.isneginf, "-inf")):
            bad = pred(g) != pred(b)
            assert not bad.any(), "%s: %s at %d elements where the fp32 oracle disagrees (first %s: got %r, fp32 oracle %r)" % (
                name, what, int(bad.sum()), tuple(np.argwhere(bad)[0]), g[bad][0], b[bad][0])
        use = np.isfinite(g) & np.isfinite(a)
        if exempt is not None and exempt[k] is not None:
            use &= ~exempt[k]
        scale = np.maximum(d, np.abs(b - a))
        fl = 4.0 * _ulp32(a)
        if floor is not None and floor[k] is not None:
            fl = fl + np.nan_to_num(np.asarray(floor[k], np.float64), nan=0.0, posinf=0.0)
        err = np.abs(g - a)
        excess = np.maximum(err - fl, 0.0)
        ratio = np.divide(excess, scale, out=np.where(excess > 0, np.inf, 0.0), where=scale > 0)
        ratio = np.where(use, ratio, 0.0)
        r = float(ratio.max()) if ratio.size else 0.0
        worst = max(worst, r)
        bad = use & ~(err <= K * scale + fl)
        if bad.any():
            idx = np.argwhere(bad)[:3]
            fb = np.broadcast_to(fl, g.shape)
            ex = "; ".join("%s got %.9g r64 %.9g r32 %.9g Delta %.3g floor %.3g" % (tuple(i), g[tuple(i)], a[tuple(i)], b[tuple(i)], d[tuple(i)],
                                                                                    fb[tuple(i)]) for i in idx)
            raise AssertionError("%s: %d of %d elements beyond %g x max(Delta, |r32 - r64|) + R + 4 ulp (worst ratio %.3g): %s" % (
                name, int(bad.sum()), int(use.sum()), K, r, ex))
        print("[%s] %-60s worst ratio %.3g over %d elements" % (tag, name, r, int(use.sum())))
    return worst


# ------------------------------------------------------------------------------------------ per-element bars of the float-atomic scatters
U32 = 2.0 ** -24            # the unit roundoff of fp32


def _gamma(k):
    """gamma(k) = k u / (1 - k u), the relative bound of k fp32 roundings"""
    k = np.asarray(k, np.float64) * U32
    return k / (1.0 - k)


def check_scatter_fp32(op, got, r32, a32, n32, tag="scatter"):
    """A scatter whose terms the kernel computes bit for bit as the fp32 oracle does (d tex, hash-grid and MLP-texture d params,
    texel_fetch d tex): the two add the same n fp32 terms in different orders, so with r32 / a32 / n32 the fp32 oracle's sum, sum of
    absolute values and count of non-zero terms (terms="sum" / "abs" / "count"), every element must satisfy
        |got - r32| <= 2 gamma(n - 1) a32 (1 + gamma(n)),
    the deterministic bound of two summation orders (the factor covers the rounding of a32 itself).  Elements with n <= 2 are therefore
    bit-identical (fp addition is commutative) and checked as such; the zero pattern and NaN / +-inf must be the fp32 oracle's.  Prints and
    returns (worst |got - r32| / bound, largest n)."""
    got, r, a, n = (np.asarray(x, np.float64) for x in (got, r32, a32, n32))
    assert got.shape == r.shape == a.shape == n.shape, (op, got.shape, r.shape, a.shape, n.shape)
    for pred, what in ((np.isnan, "NaN"), (np.isposinf, "+inf"), (np.isneginf, "-inf")):
        bad = pred(got) != pred(r)
        assert not bad.any(), "%s: %s at %d elements where the fp32 oracle disagrees (first %s)" % (
            op, what, int(bad.sum()), tuple(np.argwhere(bad)[0]))
    fin = np.isfinite(r) & np.isfinite(a)
    zero = (got == 0) != (r == 0)
    assert not (zero & fin).any(), "%s: zero pattern differs from the fp32 oracle's at %d elements (first %s: got %r, fp32 oracle %r, " \
        "n %d)" % (op, int((zero & fin).sum()), tuple(np.argwhere(zero & fin)[0]), got[zero & fin][0], r[zero & fin][0], n[zero & fin][0])
    few = fin & (n <= 2) & (got != r)
    assert not few.any(), "%s: %d elements of at most two terms differ from the fp32 oracle (first %s: got %r, fp32 oracle %r, n %d)" % (
        op, int(few.sum()), tuple(np.argwhere(few)[0]), got[few][0], r[few][0], n[few][0])
    bound = 2.0 * _gamma(np.maximum(n - 1, 0)) * a * (1.0 + _gamma(n))
    err = np.abs(got - r)
    bad = fin & ~(err <= bound)
    ratio = np.where(fin, np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0), 0.0)
    worst = float(ratio.max()) if ratio.size else 0.0
    nmax = int(n[fin].max()) if fin.any() else 0
    if bad.any():
        ex = "; ".join("%s got %.9g r32 %.9g abs %.3g n %d bound %.3g" % (tuple(i), got[tuple(i)], r[tuple(i)], a[tuple(i)], n[tuple(i)],
                                                                            bound[tuple(i)]) for i in np.argwhere(bad)[:3])
        raise AssertionError("%s: %d of %d elements beyond 2 gamma(n-1) A (1 + gamma(n)) of the fp32 oracle (worst ratio %.3g): %s" % (
            op, int(bad.sum()), int(fin.sum()), worst, ex))
    print("[%s] %-60s worst ratio %.3g, largest n %d, over %d elements (%d of 1 or 2 terms, bit for bit)" % (
        tag, op, worst, nmax, int(fin.sum()), int((fin & (n > 0) & (n <= 2)).sum())))
    return worst, nmax


def texel_fetch_stats(T, idx, g):
    """texel_fetch's d tex [T,C] as the fp32 sum, abs sum and count of its terms g[i] (every i with 0 <= idx[i] < T), each a sequential
    scatter in i order (np.add.at is unbuffered)"""
    idx = np.asarray(idx).reshape(-1)
    g = np.asarray(g, np.float32).reshape(idx.size, -1)
    ok = (idx >= 0) & (idx < T)
    out = []
    for t in (g, np.abs(g), (g != 0).astype(np.float32)):
        d = np.zeros((T, g.shape[1]), np.float32)
        np.add.at(d, idx[ok], t[ok])
        out.append(d)
    return out


def scatter_floor(n64, a64):
    """The reduction floor of a scatter whose terms the kernel computes in its own order: n 2^-24 A with the fp64 oracle's count n and
    absolute sum A (terms="count" / "abs"): the most that adding the same n terms in another fp32 order can change the sum."""
    return np.asarray(n64, np.float64) * U32 * np.asarray(a64, np.float64)


def check_scatter_fp64(op, got, f64, f32, ins, stats, K=16, seed=0, tag="scatter"):
    """A scatter whose terms the kernel computes in its own order (rasterize / rast_db / antialias d pos, interpolate and
    interpolate_da d attr): check_per_element against the fp64 oracle, every element, with a reduction floor.
      f64(ins) / f32(ins): [the sum] of the fp64 / fp32 oracle;
      ins: the inputs the sensitivity Delta perturbs (pos or rast_db, and the upstream gradient; rast stays fixed);
      stats(f64): (count, abs) of the fp32 or fp64 oracle.
    The floor is scatter_floor(max(n32, n64), max(A32, A64)).  Where the two oracles count a different number of terms (an antialias
    pair or an e = 0 crossing decided differently, or a term exactly 0 in fp32 and tiny in fp64), the larger statistics bound the
    rounding of either precision's terms, and |r32 - r64| in check_per_element's scale covers the term one of them lacks; those
    elements are checked like the rest and counted in the printed line.  Rows (vertices) where the fp32 oracle has no term must be
    exactly 0.  Prints and returns (worst ratio, largest n, elements whose counts differ)."""
    got = np.asarray(got)
    n32, a32 = (np.asarray(x, np.float64) for x in stats(False))
    n64, a64 = (np.asarray(x, np.float64) for x in stats(True))
    differ = n32 != n64
    zero = (n32 == 0).all(-1)
    assert (got[zero] == 0).all(), "%s: %d rows are nonzero where the fp32 oracle has no term" % (op, int((got[zero] != 0).any(-1).sum()))
    floor = scatter_floor(np.maximum(n32, n64), np.maximum(a32, a64))
    worst = check_per_element(op, [got], f64, f32, ins, K, ["per element"], seed=seed, floor=[floor], tag=tag)
    nmax = int(np.maximum(n32, n64).max()) if n64.size else 0
    print("[%s] %-60s largest n %d; fp32 and fp64 count differently at %d elements (checked with the larger statistics)" % (
        tag, op, nmax, int(differ.sum())))
    return worst, nmax, int(differ.sum())


def _sample_px(B, H, W, n_rand=20000, seed=0, group=4):
    """Flat [B*H*W] pixel indices: rows 0, 1 and H-1 of views 0 and B-1, n_rand random pixels, and the last (ragged) `group`-pixel group."""
    n = B * H * W
    rows = [(b * H + h) * W + np.arange(W) for b in sorted({0, B - 1}) for h in sorted({0, min(1, H - 1), H - 1})]
    tail = np.arange(n - (n % group or group), n)
    return np.unique(np.concatenate(rows + [np.random.default_rng(seed).integers(0, n, n_rand), tail]))


def _take(x, grid, idx):
    """Pixels idx of x (numpy, broadcastable to grid + (C,)) as [1,1,K,C]."""
    x = np.asarray(x)
    C = x.shape[-1]
    return np.ascontiguousarray(np.broadcast_to(x, tuple(grid) + (C,)).reshape(-1, C)[idx]).reshape(1, 1, -1, C)


def same_bits(a, b):
    """bit-for-bit equality of two fp32 arrays (so +0 / -0 and NaN payloads count)"""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def nan_bits(a):
    """int32 bit patterns, every NaN mapped to one pattern: 'bit-identical' up to the NaN payload."""
    a = np.where(np.isnan(a), np.float32(np.nan), np.asarray(a, np.float32))
    return a.view(np.int32)


def pixel_grid_mesh(H, W, step=2, z=0.0, tilt=0.0, offset=0.5):
    """A planar grid for the identity clip matrix (orthographic, NDC = world) whose vertices lie exactly on pixel centres, as
    k_rasterize computes them in fp32, every `step` pixels: rays pass through vertices and along edges, where Moeller-Trumbore's
    closed bounds accept several triangles at the same t and the lowest id must win.  z = z0 + tilt * x.  offset = 1 puts the
    vertices half a pixel further, on pixel corners, so every grid line lies midway between two rows or columns of centres."""
    xs = ((np.arange(0, W, step, dtype=np.float32) + np.float32(offset)) / np.float32(W) * np.float32(2) - np.float32(1)).astype(np.float32)
    ys = ((np.arange(0, H, step, dtype=np.float32) + np.float32(offset)) / np.float32(H) * np.float32(2) - np.float32(1)).astype(np.float32)
    X, Y = np.meshgrid(xs, ys, indexing="ij")
    Z = (np.float32(z) + np.float32(tilt) * X).astype(np.float32)
    v = np.stack([X, Y, Z], -1).reshape(-1, 3).astype(np.float32)
    nx, ny = xs.size, ys.size
    idx = np.arange(nx * ny).reshape(nx, ny)
    a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    return v, f


def raster_mesh(kind):
    """(verts, tris) of the rasterize test meshes:
      blob+torus: synth.scene_mesh level 2;  icosphere: closed and convex (exactly two layers);
      dup:        blob+torus with every triangle twice (exact ties in t) and once more with reversed winding;
      degenerate: blob+torus with zero-area triangles (repeated and collinear vertices) between the real ones;
      single:     one triangle (T = 1);
      far:        blob+torus in front of a large quad 20 units from the orbit eyes, beyond their far plane at 10."""
    if kind == "blob+torus":
        return synth.scene_mesh("blob+torus", level=2)
    if kind == "icosphere":
        v, f = synth.icosphere(3)
        return v.astype(np.float32), f.astype(np.int32)
    v, f = synth.scene_mesh("blob+torus", level=2)
    if kind == "dup":
        return v, np.concatenate([f, f, f[:, ::-1]]).astype(np.int32)
    if kind == "degenerate":
        rng = np.random.default_rng(4)
        k = f.shape[0] // 4
        a = rng.integers(0, v.shape[0], (k, 2))
        rep = np.stack([a[:, 0], a[:, 0], a[:, 1]], -1)                          # two equal corners
        mid = ((v[a[:, 0]] + v[a[:, 1]]) * np.float32(0.5)).astype(np.float32)   # a corner on the segment of the other two
        col = np.stack([a[:, 0], v.shape[0] + np.arange(k), a[:, 1]], -1)
        pnt = np.repeat(a[:, :1], 3, 1)                                          # a single point
        bad = np.concatenate([rep, col, pnt])
        allf = np.concatenate([f, bad])
        order = rng.permutation(allf.shape[0])
        return np.concatenate([v, mid]).astype(np.float32), allf[order].astype(np.int32)
    if kind == "single":
        return np.array([[-0.9, -0.7, 0.2], [0.8, -0.5, -0.1], [0.1, 0.9, 0.0]], np.float32), np.array([[0, 1, 2]], np.int32)
    if kind == "far":
        q = np.array([[-40, -40, -17], [40, -40, -17], [40, 40, -17], [-40, 40, -17]], np.float32)
        return synth.merge((v, f), (q, np.array([[0, 1, 2], [0, 2, 3]], np.int32)))
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------ BVH builds at given triangle counts
# Triangle counts where the build changes shape (bvh.cu): 1-4 the tiny view, 5-8 an SAH root that may be a leaf run, 1024 the refit's
# CTA span, 4096 the radix sort's tile, 16 384 the last SAH size, 65 537 seventeen sort tiles.
BVH_SIZES = [1, 2, 3, 4, 5, 6, 7, 8, 9, 1023, 1024, 1025, 4095, 4096, 4097, 8192, 8193, 16384, 16385, 20481]
BVH_KINDS = ["coherent", "shuffled", "coincident", "planar"]
BVH_CASES = [(k, T) for T in BVH_SIZES for k in BVH_KINDS] + [("coincident", 65537)]
SAH_MAX_TRIS = 16384          # bvh.cu MCS_SAH_MAX_TRIS: 5 <= T <= this get the SAH shadow view
QSTACK = 100                  # envshade.cu MCS_QSTACK: the shadow-ray walker's stack


_SOURCE = {}


def _source_mesh(T):
    """A mesh of at least T triangles: blob level 5 (20 480), or the ~1.08 M-triangle grid above that."""
    key = "blob5" if T <= 20480 else "grid1m"
    if key not in _SOURCE:
        _SOURCE[key] = synth.blob_mesh(5) if key == "blob5" else synth.grid1m_mesh()
    return _SOURCE[key]


def _compact(v, f):
    used, inv = np.unique(f, return_inverse=True)
    return np.ascontiguousarray(v[used], np.float32), inv.reshape(f.shape).astype(np.int32)


def sized_mesh(kind, T, seed=0):
    """A mesh of exactly T triangles.
      coherent:   the first T triangles of a large mesh (input order close to Morton order);
      shuffled:   a random subset of it in random order, so that every key moves in every sort pass;
      coincident: a group of distinct triangles inscribed in one box (every axis has one vertex on each face), so they all have the
                  same box centre and Morton key 0, and their order comes from the sort's stability alone.  For T >= 3 two triangles
                  come first in the input: one two quantisation cells away in x (key 32: it differs from the group's only in the lowest
                  radix digit) and one at the far corner of the centroid bounds.  Moving those two shifts the group between passes;
                  with all keys equal every pass would see the same groups of 32, and four passes that each reversed them would
                  cancel.  T = 2: the far triangle and one of the group;
      planar:     cells of a plane at constant y, so the centroid extent in y is 0 (the Morton code's `ext > 0` branch) and the
                  quantisation grid has only the padding on that axis."""
    rng = np.random.default_rng(1000 * T + seed)
    if kind in ("coherent", "shuffled"):
        v, f = _source_mesh(T)
        f = f[:T] if kind == "coherent" else f[rng.permutation(f.shape[0])[:T]]
        return _compact(v, f)
    if kind == "coincident":
        lo, hi = np.float32([-0.5, -0.25, -0.75]), np.float32([0.75, 0.5, 0.25])
        far = np.float32([2.0, 2.0, 2.0])                           # offset of the far triangle's box: the centroid extent
        shift = np.zeros((T, 3), np.float32)                        # rows 0 .. T - n_group - 1: the two leading triangles
        if T == 2:
            shift[0] = far
        elif T >= 3:
            shift[0], shift[1] = [2.5 / 1024 * far[0], 0, 0], far
        r = lo + rng.uniform(0.05, 0.95, (T, 3)) * (hi - lo)
        a = np.stack([np.full(T, lo[0]), np.full(T, lo[1]), r[:, 2]], -1)
        b = np.stack([np.full(T, hi[0]), r[:, 1], np.full(T, lo[2])], -1)
        c = np.stack([r[:, 0], np.full(T, hi[1]), np.full(T, hi[2])], -1)
        v = (np.stack([a, b, c], 1) + shift[:, None, :]).reshape(-1, 3).astype(np.float32)
        return v, np.arange(3 * T, dtype=np.int32).reshape(T, 3)
    if kind == "planar":
        n = int(np.ceil(np.sqrt(T / 2.0)))
        v, f = synth.plane_mesh(y=-0.3, half=1.0, n=n)
        return _compact(v, f[:T])
    raise ValueError(kind)


def bvh_rays(n, seed, v):
    """Rays from around the mesh towards its centre; one in eight is axis-aligned (zero direction components: slab-test corner cases)."""
    rng = np.random.default_rng(seed)
    c = v.mean(0); ext = (v.max(0) - v.min(0)).max()
    ro = (c + rng.normal(size=(n, 3)) * ext * 0.7).astype(np.float32)
    tgt = (c + rng.normal(size=(n, 3)) * ext * 0.3).astype(np.float32)
    rd = tgt - ro
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    k = n // 8
    rd[:k] = np.eye(3, dtype=np.float32)[rng.integers(0, 3, k)] * rng.choice([-1.0, 1.0], (k, 1)).astype(np.float32)
    return ro, rd.astype(np.float32)


# ------------------------------------------------------------------------------------------ the shadow-ray view (bvh_export_shadow)
def walk_shadow_view(ctx):
    """Walk the exported view from node 0: 4-wide nodes as {node: [child slots]} in walk order (a node after its parent), each used
    slot ("run", first, count, ql, qh) or ("node", index, None, ql, qh); the triangle ids of the records; the grid; the max depth."""
    from nvdiffrecmc_b200.optixutils.ops import bvh_export_shadow
    g = {k: t.cpu().numpy() for k, t in bvh_export_shadow(ctx).items()}
    nq = g["nodes"].view(np.uint32)
    ids = g["tris"][:, 0, 3].copy().view(np.int32)
    nodes, depth, stack = {}, 0, [(0, 1)]
    while stack:
        i, d = stack.pop()
        assert i not in nodes, "node %d reached twice" % i
        depth = max(depth, d)
        lb = int(nq[i, 0, 3]) >> 28
        slots = []
        for c in range(4):
            rec = nq[i, c]
            ql, qh = rec[:3] & 0xFFFF, rec[:3] >> 16
            if (ql > qh).any():                      # unused slot: inverted box, flagged as a leaf
                assert (lb >> c) & 1 and (ql == 0xFFFF).all() and (qh == 0).all()
                continue
            payload = int(rec[3]) & 0x0FFFFFFF
            if (lb >> c) & 1:
                slots.append(("run", payload >> 3, (payload & 7) + 1, ql, qh))
            else:
                slots.append(("node", payload, None, ql, qh))
                stack.append((payload, d + 1))
        nodes[i] = slots
    return nodes, ids, g["qgrid"].astype(np.float64), depth


def shadow_subtree_bounds(nodes, ids, v, f):
    """(lo, hi) of the triangles under every node of a walked view, and the per-triangle boxes."""
    tv = v[f].astype(np.float64)                                     # [T, 3 verts, 3]
    tlo, thi = tv.min(1), tv.max(1)
    box = {}
    for i in reversed(list(nodes)):                                  # children were reached after their parents
        los, his = [], []
        for kind, a, n, _, _ in nodes[i]:
            lo, hi = (tlo[ids[a:a + n]].min(0), thi[ids[a:a + n]].max(0)) if kind == "run" else box[a]
            los.append(lo); his.append(hi)
        box[i] = (np.min(los, 0), np.max(his, 0))
    return box.__getitem__, tlo, thi


def shadow_stack_slots(nodes):
    """Stack entries the walker (envshade.cu:trace_queue) can touch on this view: every hit internal child is pushed and the last one
    popped at once, so below node v the stack holds sum(internal children - 1) over v's ancestors; a visit stores up to three more."""
    need, worst = {0: 0}, 0
    for i, slots in nodes.items():
        inner = [a for kind, a, _, _, _ in slots if kind == "node"]
        worst = max(worst, need[i] + 4)
        for a in inner:
            need[a] = need[i] + len(inner) - 1
    return worst


def lbvh_collapse_view(ex, T):
    """The view the walker must find when the shadow rays use the LBVH (T <= 4 or T > SAH_MAX_TRIS): node i holds the grandchildren of
    binary node i, a subtree of at most four triangles is one run.  {node: [(kind, first or index, count)]}, as walk_shadow_view."""
    if T <= 4:
        return {0: [("run", 0, T)]}
    left, right = ex["left"], ex["right"]
    span = np.zeros((2 * T - 1, 2), np.int64)
    span[T - 1:, 0] = span[T - 1:, 1] = np.arange(T)
    order, stack = [], [0]                  # sorted-triangle range of every internal node, children before parents
    while stack:
        i = stack.pop(); order.append(i)
        stack += [c for c in (left[i], right[i]) if c < T - 1]
    for i in reversed(order):
        span[i] = span[left[i], 0], span[right[i], 1]

    def code(c):
        n = span[c, 1] - span[c, 0] + 1
        return ("run", int(span[c, 0]), int(n)) if c >= T - 1 or n <= 4 else ("node", int(c), None)
    view, stack = {}, [0]
    while stack:
        i = stack.pop()
        slots = []
        for c in (left[i], right[i]):
            k = code(c)
            slots += [k] if k[0] == "run" else [code(left[c]), code(right[c])]
        view[i] = slots
        stack += [a for kind, a, _ in slots if kind == "node"]
    return view


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


# ------------------------------------------------------------------------------------------ the bilateral denoiser
def _radius(sigma):
    """denoising.cu:26,86: 2 * ceil(sigma * 2.5) + 1 with the product in double, sigma being an fp32 parameter."""
    return 2 * math.ceil(float(np.float32(sigma)) * 2.5) + 1


def _dn_both_paths(col, colB, nrm, zdz, gA, gB, sigma, dev):
    """Raw forward [B,H,W,4] and transposed filter [B,H,W,3] through the single- and two-signal entry points, once with contiguous
    signals (the TMA-staged kernel where the radius allows it) and once with the same values as strided views (the plain kernel).
    All paths must agree bit for bit (NaN payloads aside); returns (forward A, forward B, backward A, backward B)."""
    import torch
    from nvdiffrecmc_b200 import _lib as L
    from nvdiffrecmc_b200.optixutils.ops import _bilateral_denoiser_func, _bilateral_denoiser2_func
    t = lambda a: torch.tensor(a, device=dev)
    n, z = t(nrm), t(zdz)
    wide = lambda x: torch.cat([x, torch.zeros_like(x[..., :1])], -1)[..., :x.shape[-1]]
    res = {}
    for tag, view in (("contiguous", lambda x: x), ("strided", wide)):
        a, b, ga, gb = view(t(col)), view(t(colB)), view(t(gA)), view(t(gB))
        assert a.is_contiguous() == (tag == "contiguous")
        fa = _bilateral_denoiser_func.apply(a, n, z, sigma)
        f2a, f2b = _bilateral_denoiser2_func.apply(a, b, n, z, sigma)
        shape = tuple(col.shape[:3]) + (3,)
        ca, cb, c1 = torch.empty(shape, device=dev), torch.empty(shape, device=dev), torch.empty(shape, device=dev)
        L.check(L.lib().mcs_bilateral_bwd(C.byref(L.nhwc(n)), C.byref(L.nhwc(z)), float(sigma), C.byref(L.nhwc(ga)), c1.data_ptr(), L.stream_ptr()),
                "bilateral_denoiser (backward)")
        L.check(L.lib().mcs_bilateral_bwd2(C.byref(L.nhwc(n)), C.byref(L.nhwc(z)), float(sigma), C.byref(L.nhwc(ga)), C.byref(L.nhwc(gb)), ca.data_ptr(),
                                           cb.data_ptr(), L.stream_ptr()), "bilateral_denoiser2 (backward)")
        fa, c1 = fa.cpu().numpy(), c1.cpu().numpy()
        res[tag] = [x.cpu().numpy() for x in (f2a, f2b, ca, cb)]
        assert np.array_equal(nan_bits(fa), nan_bits(res[tag][0])) and np.array_equal(nan_bits(c1), nan_bits(res[tag][2])), tag
    for k, (x, y) in enumerate(zip(res["contiguous"], res["strided"])):
        assert np.array_equal(nan_bits(x), nan_bits(y)), "output %d: %d of %d values differ between the two kernels" % (
            k, (nan_bits(x) != nan_bits(y)).sum(), x.size)
    return res["contiguous"]


def _degenerate_guides(B, H, W, seed):
    """Piecewise-smooth guides with a zero normal inside the image, zero and negative depth gradients (each pixel is the centre of its
    own output and a tap of its neighbours', so both uses are covered), and depth steps along x and y."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    n = np.stack([np.full((H, W), 0.2), 0.1 * np.sin(xs * 0.3), np.ones((H, W))], -1)[None] + rng.normal(size=(B, H, W, 3)) * 0.05
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    n[0, H // 2, W // 3] = 0.0                                    # zero centre normal
    n[B - 1, 5, 7] = 0.0
    z = 1.0 + xs * 0.01 + ys * 0.005 + 0.5 * (xs >= W // 2) + 0.25 * (ys >= H // 3)       # depth steps
    z = np.broadcast_to(z, (B, H, W)) + rng.normal(size=(B, H, W)) * 1e-3
    dz = np.abs(rng.normal(size=(B, H, W))) * 0.02 + 0.001
    dz[0, 10:14, 20:25] = 0.0                                     # FLT_EPS guard, centre (forward) and tap (backward)
    dz[B - 1, H // 2 - 2:H // 2 + 2, W // 2 - 3:W // 2 + 3] = -0.01   # negative gradients straddling the depth step
    dz[0, H // 2, W // 3 + 1] = 0.0                               # next to the zero normal
    return n.astype(np.float32), np.stack([z, dz], -1).astype(np.float32)


def impulse_lattice(B, H, W, r, vals):
    """The impulse lattices of the denoiser's tap-by-tap tests.  With spacing S = 2r + 1, the lattice of offset (oy, ox) holds `vals` [C]
    at (oy + S i, ox + S j) and 0 elsewhere, so every pixel's (2r+1)^2 window holds exactly one lattice point: a filter's output there is
    that one tap's weight times `vals` (or 0 when the point lies outside the image).  The S^2 offsets together give every in-image tap of
    every pixel once.  Returns the lattices stacked offset-major along the batch, [S^2 B, H, W, C], and per offset, pixel of [B,H,W]:
    (dy, dx) of that pixel's lattice point, [S^2, B, H, W] each."""
    S = 2 * r + 1
    vals = np.asarray(vals, np.float32)
    sig = np.zeros((S, S, B, H, W, vals.shape[0]), np.float32)
    for oy in range(S):
        for ox in range(S):
            sig[oy, ox, :, oy::S, ox::S] = vals
    ys, xs = np.arange(H), np.arange(W)
    dy = (np.arange(S)[:, None] - ys[None, :] + r) % S - r             # [S(oy), H]
    dx = (np.arange(S)[:, None] - xs[None, :] + r) % S - r             # [S(ox), W]
    DY = np.broadcast_to(dy[:, None, None, :, None], (S, S, B, H, W)).reshape(S * S, B, H, W)
    DX = np.broadcast_to(dx[None, :, None, None, :], (S, S, B, H, W)).reshape(S * S, B, H, W)
    return sig.reshape(S * S * B, H, W, vals.shape[0]), DY, DX
