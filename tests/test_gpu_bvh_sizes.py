"""GPU: the BVH build at the triangle counts where its kernels change shape (tests/common.py BVH_SIZES: the radix sort's 4096-key tiles,
the refit's 1024-leaf CTA spans, the tiny and SAH shadow views), on four kinds of mesh, and one context rebuilt across those sizes.

At every size the LBVH must equal the oracle's bit for bit, the fp32-node queries must equal the oracle's predicate, and the shadow-ray
view (what env_shade's shadow rays walk) must hold every triangle once in boxes that contain it, with the records of the Morton-ordered
view and the topology of its size class: the LBVH grandchild collapse for T <= 4 and T > 16 384, an SAH tree of its own in between."""
import numpy as np
import pytest
import torch

from common import (BVH_CASES, QSTACK, SAH_MAX_TRIS, bvh_rays, lbvh_collapse_view, make_case, oracle, rel_l2, shadow_stack_slots,
                    shadow_subtree_bounds, sized_mesh, walk_shadow_view)

pytestmark = pytest.mark.gpu
NRAYS = 8192
BRUTE_MAX = 25000         # above this the oracle's LBVH traversal stands in for brute force (tests/test_oracle_bvh_sizes.py)


def _build(ctx, dev, v, f, rebuild=1):
    import nvdiffrecmc_b200.optixutils as ou
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=rebuild)


def _fresh(dev, v, f, refit_to=None):
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext()
    _build(ctx, dev, v, f)
    if refit_to is not None:
        _build(ctx, dev, refit_to, f, rebuild=0)
    return ctx


def _jitter(v, seed):
    ext = float((v.max(0) - v.min(0)).max())
    return (v + np.random.default_rng(seed).normal(size=v.shape) * 0.02 * ext).astype(np.float32)


def _export(ctx):
    from nvdiffrecmc_b200.optixutils.ops import bvh_export
    g = {k: t.cpu().numpy() for k, t in bvh_export(ctx).items()}
    g["morton"] = g["morton"].view(np.uint32)
    return g


def _check_lbvh(ctx, sc):
    g, r = _export(ctx), sc.export_lbvh()
    for k in ("morton", "prim", "left", "right", "lo", "hi"):
        assert np.array_equal(g[k], r[k]), "LBVH %s differs from the oracle's" % k
    return g


def _check_queries(ctx, dev, v, f, sc, seed):
    """trace_visibility and trace_closest on NRAYS rays against the oracle: bit-exact visibility, ids, and (t, u, v) of every hit."""
    import nvdiffrecmc_b200.optixutils as ou
    T = f.shape[0]
    ro, rd = bvh_rays(NRAYS, seed, v)
    tro, trd = torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)
    vis = ou.trace_visibility(ctx, tro, trd).cpu().numpy()
    ref = sc.visibility(ro, rd, mode="brute" if T <= BRUTE_MAX else "bvh")
    assert np.array_equal(vis, ref), "visibility: %d of %d rays differ" % ((vis != ref).sum(), NRAYS)
    tid, tuv = ou.trace_closest(ctx, tro, trd)
    tid, tuv = tid.cpu().numpy(), tuv.cpu().numpy()
    rid, rtuv = sc.closest_hit(ro, rd)
    assert np.array_equal(tid, rid), "closest hit: %d of %d ids differ" % ((tid != rid).sum(), NRAYS)
    hit = rid >= 0
    assert np.array_equal(tuv[hit].view(np.uint32), rtuv[hit].view(np.uint32))
    assert 0 < hit.mean() < 1
    return vis


def _records(v, f):
    """bvh.cu's triangle record of every original id: (v0, id as int bits), (v1 - v0, 0), (v2 - v0, 0) in fp32."""
    T = f.shape[0]
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    rec = np.zeros((T, 3, 4), np.float32)
    rec[:, 0, :3], rec[:, 1, :3], rec[:, 2, :3] = a, b - a, c - a
    rec[:, 0, 3] = np.arange(T, dtype=np.int32).view(np.float32)
    return rec


def _check_shadow_view(ctx, v, f, ex, kind):
    """The shadow-ray view against the mesh (v, f) and the context's own LBVH export ex."""
    from nvdiffrecmc_b200.optixutils.ops import bvh_export_shadow
    T = f.shape[0]
    nodes, ids, qg, depth = walk_shadow_view(ctx)
    assert np.array_equal(np.sort(ids), np.arange(T)), "triangle records are not a permutation of the mesh"
    tris = bvh_export_shadow(ctx)["tris"].cpu().numpy()
    assert np.array_equal(tris.view(np.uint32), _records(v, f)[ids].view(np.uint32)), "a record differs from its triangle's"
    seen = np.zeros(T, np.int32)
    for slots in nodes.values():
        for kind_, a, n, _, _ in slots:
            if kind_ == "run":
                assert a + n <= T
                seen[a:a + n] += 1
    assert (seen == 1).all(), "%d slots in no run, %d in several" % ((seen == 0).sum(), (seen > 1).sum())
    node_bounds, tlo, thi = shadow_subtree_bounds(nodes, ids, v, f)
    org, cell = qg[0:3], qg[3:6]
    for slots in nodes.values():
        for kind_, a, n, ql, qh in slots:
            lo, hi = (tlo[ids[a:a + n]].min(0), thi[ids[a:a + n]].max(0)) if kind_ == "run" else node_bounds(a)
            assert (org + ql * cell <= lo).all() and (org + qh * cell >= hi).all()
    # Stack: the walker can touch shadow_stack_slots entries.  Three pushes per level of depth bound that for any tree; triangles with
    # one common box make the SAH clustering merge one pair per round, a chain far deeper than the stack that never fills it.
    assert shadow_stack_slots(nodes) <= QSTACK
    if kind != "coincident":
        assert 3 * depth + 1 <= QSTACK
    # size class
    sah = 5 <= T <= SAH_MAX_TRIS
    assert max(n for slots in nodes.values() for kind_, a, n, _, _ in slots if kind_ == "run") <= (8 if sah else 4)
    view = {i: [s[:3] for s in slots] for i, slots in nodes.items()}
    if sah:
        if T >= 1000:
            assert view != lbvh_collapse_view(ex, T), "T = %d: the shadow rays walk the LBVH, not the SAH view" % T
    else:
        assert view == lbvh_collapse_view(ex, T), "T = %d: the shadow view is not the LBVH grandchild collapse" % T
        assert np.array_equal(ids, ex["prim"])


@pytest.mark.parametrize("kind,T", BVH_CASES)
def test_build_at_size(dev, kind, T):
    import nvdiffrecmc_b200.optixutils as ou
    v, f = sized_mesh(kind, T)
    assert f.shape[0] == T
    ctx = ou.OptiXContext()
    _build(ctx, dev, v, f)
    sc = oracle().scene(v, f)
    ex = _check_lbvh(ctx, sc)
    if kind == "coincident":                                        # the group sorts first, in input order
        g = T - 2 if T >= 3 else 1
        assert (ex["morton"][:g] == 0).all() and np.array_equal(ex["prim"][:g], np.arange(T - g, T))
    if kind == "planar" and T > 1:
        assert (ex["morton"] & 0x12492492 == 0).all()               # the y bits of every key are 0
    _check_queries(ctx, dev, v, f, sc, seed=T)
    _check_shadow_view(ctx, v, f, ex, kind)


@pytest.mark.parametrize("T", [4097, 5, 8, 9, 16384, 16385])
def test_refit_at_size(dev, T):
    """Built from jittered vertices, refitted (rebuild=0) to the true ones: the topology stays the jittered mesh's Morton order, the
    boxes, queries and the shadow view (whose SAH clustering is rerun on the refitted boxes) must follow the true vertices."""
    v, f = sized_mesh("shuffled", T, seed=1)
    ctx = _fresh(dev, _jitter(v, T), f, refit_to=v)
    sc = oracle().scene(v, f)
    ex = _export(ctx)
    _check_queries(ctx, dev, v, f, sc, seed=T + 1)
    _check_shadow_view(ctx, v, f, ex, "shuffled")


def _state(ctx, dev, v):
    """Everything a later query reads: LBVH export, visibility on 4096 rays, the shadow view as the walker reaches it (nodes, slots and
    records; slots of SAH nodes under a leaf run are never written, so the raw node array is not compared)."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.optixutils.ops import bvh_export_shadow
    ro, rd = bvh_rays(4096, 3, v)
    vis = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    nodes, ids, qg, _ = walk_shadow_view(ctx)
    view = {i: [(k, a, n, tuple(ql.tolist()), tuple(qh.tolist())) for k, a, n, ql, qh in s] for i, s in nodes.items()}
    sh = bvh_export_shadow(ctx)
    return dict(_export(ctx), vis=vis, view=view, ids=ids, qgrid=qg, tris=sh["tris"].cpu().numpy().view(np.uint32))


def test_one_context_across_sizes(dev):
    """Training rebuilds one context every iteration while DMTet changes the triangle count.  One context taken through sizes on both
    sides of every view boundary (and refitted twice) must hold what a fresh context builds from the same calls."""
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext()
    for step, (T, refit) in enumerate([(16385, False), (5, False), (4097, True), (1, False), (16384, False), (9, True), (20481, False),
                                       (3, False)]):
        v, f = sized_mesh("shuffled", T, seed=10 + step)
        v2 = _jitter(v, step) if refit else None
        _build(ctx, dev, v, f)
        if refit:
            _build(ctx, dev, v2, f, rebuild=0)
        got, want = _state(ctx, dev, v), _state(_fresh(dev, v, f, refit_to=v2), dev, v)
        for k in want:
            same = want[k] == got[k] if k == "view" else np.array_equal(want[k], got[k])
            assert same, "step %d (T = %d%s): %s differs from a fresh context" % (step, T, ", refitted" if refit else "", k)


def _occluder_scene(T, seed=0):
    """A ground quad (2 triangles) under T - 2 occluders of about equal total area; T = 1: one large ground triangle."""
    y0 = np.float32(-0.6)
    if T == 1:
        return np.float32([[-2, y0, -2], [2, y0, -2], [0, y0, 2]]), np.int32([[0, 2, 1]])
    v = [np.float32([[-1.2, y0, -1.2], [1.2, y0, -1.2], [1.2, y0, 1.2], [-1.2, y0, 1.2]])]
    f = [np.int32([[0, 2, 1], [0, 3, 2]])]
    n = T - 2
    if n:
        rng = np.random.default_rng(seed)
        c = np.stack([rng.uniform(-0.9, 0.9, n), rng.uniform(-0.3, 0.5, n), rng.uniform(-0.9, 0.9, n)], -1)
        size = 1.2 / np.sqrt(n)
        shape = np.float32([[-0.6, 0.0, -0.5], [0.6, 0.05, -0.4], [0.0, -0.05, 0.7]])
        v.append((c[:, None, :] + shape[None] * size).reshape(-1, 3))
        f.append(4 + np.arange(3 * n, dtype=np.int32).reshape(n, 3))
    return np.concatenate(v).astype(np.float32), np.concatenate(f).astype(np.int32)


@pytest.mark.parametrize("T", [1, 4, 5, 8, 9, 16384, 16385])
def test_shadow_rays_at_view_boundaries(dev, T):
    """env_shade's shadow rays through the tiny view (T <= 4), an SAH root that may be a leaf run (5-8), the SAH view at its largest size
    and the LBVH collapse just above it: env texel records and visibility bits bit-exact, radiance within 1e-4."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.optixutils.ops import env_shade_records
    N = 4
    v, f = _occluder_scene(T)
    assert f.shape[0] == T
    c = make_case(res=24, B=1, N=N, mesh=(v, f), seed=1)
    ctx = ou.OptiXContext()
    _build(ctx, dev, v, f)
    a = [torch.tensor(c[k], device=dev) for k in ("mask", "ro", "pos", "nrm", "view", "kd", "ks", "light", "pdf", "rows", "cols", "perms")]
    diff, spec, rec_t, rec_v = env_shade_records(ctx, *a, BSDF="pbr", n_samples_x=N, rnd_seed=11, shadow_scale=1.0)
    d_ref, s_ref, (rt, rv) = oracle().env_shade(c["scene"], c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"],
                                                c["pdf"], c["rows"], c["cols"], c["perms"], BSDF="pbr", n_samples_x=N, rnd_seed=11, records=True,
                                                vis_mode="brute" if T <= 4096 else "bvh")
    rec_t, rec_v = rec_t.cpu().numpy(), rec_v.cpu().numpy()
    assert np.array_equal(rec_t, rt), "env texel selection differs from the oracle (%d of %d rays)" % ((rec_t != rt).sum(), rt.size)
    traced = rec_v != 2
    assert np.array_equal(rec_v[traced], rv[traced]), "visibility bits differ from the oracle"
    assert traced[c["mask"] > 0].mean() > 0.2
    if T >= 3:
        assert 0.05 < rv[rv <= 1].mean() < 0.95                      # (255: pixels off the mesh)
    assert rel_l2(diff.cpu().numpy(), d_ref) < 1e-4 and rel_l2(spec.cpu().numpy(), s_ref) < 1e-4


def test_triangle_count_guard(dev):
    """More than 2^25 triangles do not fit the 28-bit child words of the quantised nodes: the build refuses before any device work and
    leaves the context's structure as it was.  The buffers are real and large enough, so a build that ran anyway could not fault."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200 import _lib as L
    v, f = sized_mesh("coherent", 9)
    ctx = _fresh(dev, v, f)
    before = _export(ctx)
    T = (1 << 25) + 1
    verts = torch.zeros(1, 3, dtype=torch.float32, device=dev)
    tris = torch.zeros(T, 3, dtype=torch.int32, device=dev)
    rc = L.lib().mcs_bvh_build(ctx.cpp_wrapper, verts.data_ptr(), 1, tris.data_ptr(), T, 1, L.stream_ptr())
    msg = L.lib().mcs_last_error() or b""
    assert rc != 0 and b"at most 2^25 triangles" in msg, msg
    after = _export(ctx)
    assert all(np.array_equal(before[k], after[k]) for k in before)
    ro, rd = bvh_rays(256, 0, v)
    vis = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    assert np.array_equal(vis, oracle().scene(v, f).visibility(ro, rd))
