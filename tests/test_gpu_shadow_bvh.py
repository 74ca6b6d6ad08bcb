"""GPU: the shadow-ray view (4-wide quantised nodes + triangle records in leaf order) that env_shade walks.  Meshes of 5 to 16 384
triangles get their own SAH topology (bvh.cu:k_ploc); larger ones keep the LBVH grandchild collapse.  Either way every triangle must
sit in exactly one leaf run, every quantised box must contain its subtree, and the walker's stack must suffice."""
import numpy as np
import pytest
import torch

from common import QSTACK, oracle
from common import shadow_subtree_bounds as _subtree_bounds
from common import walk_shadow_view as _walk
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _build(dev, v, f, rebuild_from=None):
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(v if rebuild_from is None else rebuild_from, device=dev), torch.tensor(f, device=dev), rebuild=1)
    if rebuild_from is not None:
        ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=0)
    return ctx


CASES = [("blob", 1), ("blob+torus", 4), ("bob-like", 4)]


@pytest.mark.parametrize("kind,level", CASES)
@pytest.mark.parametrize("refit", [False, True])
def test_every_triangle_in_exactly_one_leaf_run(dev, kind, level, refit):
    v, f = synth.scene_mesh(kind, level=level)
    v0 = (v * np.float32(0.97) - np.float32(0.02)).astype(np.float32) if refit else None
    nodes, ids, _, depth = _walk(_build(dev, v, f, rebuild_from=v0))
    T = f.shape[0]
    assert np.array_equal(np.sort(ids), np.arange(T)), "triangle records are not a permutation of the mesh"
    seen = np.zeros(T, np.int32)
    for slots in nodes.values():
        for kind_, a, n, _, _ in slots:
            if kind_ == "run":
                assert 1 <= n <= 8 and a + n <= T
                seen[a:a + n] += 1
    assert (seen == 1).all(), "%d slots in no run, %d in several" % ((seen == 0).sum(), (seen > 1).sum())
    assert 3 * depth + 1 <= QSTACK


@pytest.mark.parametrize("kind,level", CASES)
@pytest.mark.parametrize("refit", [False, True])
def test_quantised_boxes_contain_their_subtrees(dev, kind, level, refit):
    v, f = synth.scene_mesh(kind, level=level)
    v0 = (v * np.float32(0.97) - np.float32(0.02)).astype(np.float32) if refit else None
    nodes, ids, qg, _ = _walk(_build(dev, v, f, rebuild_from=v0))
    node_bounds, tlo, thi = _subtree_bounds(nodes, ids, v, f)
    org, cell = qg[0:3], qg[3:6]
    for slots in nodes.values():
        for kind_, a, n, ql, qh in slots:
            lo, hi = (tlo[ids[a:a + n]].min(0), thi[ids[a:a + n]].max(0)) if kind_ == "run" else node_bounds(a)
            assert (org + ql * cell <= lo).all() and (org + qh * cell >= hi).all()


def _area(lo, hi):
    d = hi - lo
    return d[0] * d[1] + d[1] * d[2] + d[2] * d[0]


def _sah_shadow(nodes, ids, v, f):
    node_bounds, tlo, thi = _subtree_bounds(nodes, ids, v, f)
    cost = 0.0
    for i, slots in nodes.items():
        cost += _area(*node_bounds(i))
        for kind_, a, n, _, _ in slots:
            if kind_ == "run":
                cost += n * _area(tlo[ids[a:a + n]].min(0), thi[ids[a:a + n]].max(0))
    return cost / _area(*node_bounds(0))


def _sah_lbvh_collapse(ex, v, f):
    """Same cost for the LBVH grandchild collapse (the view the shadow rays walked before): leaf runs = subtrees of <= 4 triangles."""
    T = f.shape[0]
    left, right, prim = ex["left"], ex["right"], ex["prim"]
    tv = v[f[prim]].astype(np.float64)
    tlo, thi = tv.min(1), tv.max(1)
    rng = {}

    def span(c):                                   # sorted-triangle range [a, b) of node c
        if c >= T - 1:
            return c - (T - 1), c - (T - 1) + 1
        if c not in rng:
            rng[c] = (span(left[c])[0], span(right[c])[1])
        return rng[c]

    def box(c):
        a, b = span(c)
        return tlo[a:b].min(0), thi[a:b].max(0)

    def is_run(c):
        a, b = span(c)
        return b - a <= 4
    cost, stack = 0.0, [0]
    while stack:
        i = stack.pop()
        cost += _area(*box(i))
        for c in (left[i], right[i]):
            for g in ((c,) if is_run(c) else (left[c], right[c])):
                if is_run(g):
                    a, b = span(g)
                    cost += (b - a) * _area(*box(g))
                else:
                    stack.append(g)
    return cost / _area(*box(0))


@pytest.mark.parametrize("kind,level", [("blob+torus", 4), ("bob-like", 4)])
def test_sah_cost_below_the_lbvh(dev, kind, level):
    import sys
    from nvdiffrecmc_b200.optixutils.ops import bvh_export
    sys.setrecursionlimit(10000)
    v, f = synth.scene_mesh(kind, level=level)
    ctx = _build(dev, v, f)
    nodes, ids, _, _ = _walk(ctx)
    ex = {k: t.cpu().numpy() for k, t in bvh_export(ctx).items()}
    new, old = _sah_shadow(nodes, ids, v, f), _sah_lbvh_collapse(ex, v, f)
    assert new < 0.97 * old, "SAH cost %.2f (shadow view) vs %.2f (LBVH collapse)" % (new, old)


def test_grid1m_visibility_matches_brute_force(dev):
    """1.08 M triangles: above the size that gets its own topology; the shadow view is the LBVH collapse and must still hold every
    triangle once, and the visibility mask must equal the brute-force loop."""
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh("grid1m", level=0)
    ctx = _build(dev, v, f)
    nodes, ids, _, depth = _walk(ctx)
    T = f.shape[0]
    seen = np.zeros(T, np.int32)
    for slots in nodes.values():
        for kind_, a, n, _, _ in slots:
            if kind_ == "run":
                seen[a:a + n] += 1
    assert (seen == 1).all() and np.array_equal(np.sort(ids), np.arange(T)) and 3 * depth + 1 <= QSTACK
    rng = np.random.default_rng(7)
    m = 1500
    lo, hi = v.min(0), v.max(0)
    ro = (lo + rng.uniform(size=(m, 3)) * (hi - lo)).astype(np.float32); ro[:, 1] = hi[1] * rng.uniform(0.2, 1.5, m).astype(np.float32)
    rd = rng.normal(size=(m, 3)).astype(np.float32); rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    vis = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    ref = oracle().scene(v, f).visibility(ro, rd, mode="brute")
    assert np.array_equal(vis, ref), "%d of %d rays differ" % ((vis != ref).sum(), m)
    assert 0.05 < ref.mean() < 0.95
