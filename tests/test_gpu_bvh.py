"""GPU parity: LBVH build + ray queries vs the oracle's canonical LBVH / brute-force predicate.
Integer structure (sorted Morton keys, primitive order, Karras children) and the visibility mask are
BIT-EXACT; node boxes are compared exactly too (same fp32 operations, min/max are order independent)."""
import numpy as np
import pytest
import torch

from common import bvh_rays as _rays
from common import oracle
from nvdiffrecmc_b200 import synth

pytestmark = pytest.mark.gpu


def _build(dev, v, f):
    import nvdiffrecmc_b200.optixutils as ou
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, torch.tensor(v, device=dev), torch.tensor(f, device=dev), rebuild=1)
    return ctx


@pytest.mark.parametrize("kind,level", [("blob", 1), ("blob+torus", 2), ("full", 3)])
def test_lbvh_structure_bit_exact(dev, kind, level):
    from nvdiffrecmc_b200.optixutils.ops import bvh_export
    v, f = synth.scene_mesh(kind, level=level)
    ctx = _build(dev, v, f)
    g = {k: t.cpu().numpy() for k, t in bvh_export(ctx).items()}
    r = oracle().scene(v, f).export_lbvh()
    assert np.array_equal(g["morton"].view(np.uint32), r["morton"])
    assert np.array_equal(g["prim"], r["prim"])
    assert np.array_equal(g["left"], r["left"]) and np.array_equal(g["right"], r["right"])
    assert np.array_equal(g["lo"], r["lo"]) and np.array_equal(g["hi"], r["hi"])


@pytest.mark.parametrize("kind,level,n", [("blob", 0, 20000), ("blob+torus", 2, 60000), ("full", 3, 60000)])
def test_visibility_mask_bit_exact(dev, kind, level, n):
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh(kind, level=level)
    ctx = _build(dev, v, f)
    ro, rd = _rays(n, 1, v)
    got = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    ref = oracle().scene(v, f).visibility(ro, rd, mode="brute")
    assert np.array_equal(got, ref), "%d of %d rays differ" % ((got != ref).sum(), n)
    assert 0.05 < ref.mean() < 0.95


def test_closest_hit_matches_brute_force(dev):
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh("blob+torus", level=2)
    ctx = _build(dev, v, f)
    ro, rd = _rays(30000, 2, v)
    tid, tuv = ou.trace_closest(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev))
    rid, rtuv = oracle().scene(v, f).closest_hit(ro, rd)
    assert np.array_equal(tid.cpu().numpy(), rid)
    hit = rid >= 0
    assert np.array_equal(tuv.cpu().numpy()[hit], rtuv[hit])


def test_single_triangle_and_degenerate(dev):
    import nvdiffrecmc_b200.optixutils as ou
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 2], [2, 2, 2], [2, 2, 2]], np.float32)
    for f in (np.array([[0, 1, 2]], np.int32), np.array([[0, 1, 2], [3, 4, 5], [0, 1, 2]], np.int32)):   # 1 tri; degenerate + duplicate tris
        ctx = _build(dev, v, f)
        ro = np.array([[0.2, 0.2, 1], [2, 2, 1], [0.2, 0.2, -1]], np.float32); rd = np.array([[0, 0, -1], [0, 0, -1], [0, 0, -1]], np.float32)
        got = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
        ref = oracle().scene(v, f).visibility(ro, rd)
        assert np.array_equal(got, ref) and list(ref) == [0, 1, 1]


def test_refit_equals_rebuild_visibility(dev):
    """rebuild=0 (OPTIX_BUILD_OPERATION_UPDATE, torch_bindings.cpp:57-59): same topology, new boxes."""
    import nvdiffrecmc_b200.optixutils as ou
    v, f = synth.scene_mesh("blob+torus", level=2)
    ctx = _build(dev, v, f)
    v2 = (v * np.float32(1.05) + np.float32(0.01)).astype(np.float32)
    ou.optix_build_bvh(ctx, torch.tensor(v2, device=dev), torch.tensor(f, device=dev), rebuild=0)
    ro, rd = _rays(20000, 3, v2)
    got = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    assert np.array_equal(got, oracle().scene(v2, f).visibility(ro, rd))
    with pytest.raises(RuntimeError, match="same triangle count"):
        ou.optix_build_bvh(ctx, torch.tensor(v2, device=dev), torch.tensor(f[:-1], device=dev), rebuild=0)


def test_million_triangle_mesh_matches_oracle_lbvh(dev):
    """BASELINE config 5 scale (1M triangles): structure and visibility stay bit-exact vs the oracle's canonical LBVH traversal
    (brute force is infeasible at this size; LBVH == brute force is established at small sizes on both sides)."""
    import nvdiffrecmc_b200.optixutils as ou
    from nvdiffrecmc_b200.optixutils.ops import bvh_export
    n = 724
    g = np.linspace(-1, 1, n + 1, dtype=np.float32)
    X, Z = np.meshgrid(g, g, indexing="ij")
    Y = (0.2 * np.sin(7 * X) * np.cos(5 * Z)).astype(np.float32)
    v = np.stack([X, Y, Z], -1).reshape(-1, 3)
    idx = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
    f = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([a, d, c], -1).reshape(-1, 3)]).astype(np.int32)
    assert f.shape[0] > 1_000_000
    ctx = _build(dev, v, f)
    sc = oracle().scene(v, f)
    got = {k: t.cpu().numpy() for k, t in bvh_export(ctx).items()}
    ref = sc.export_lbvh()
    assert np.array_equal(got["morton"].view(np.uint32), ref["morton"]) and np.array_equal(got["prim"], ref["prim"])
    assert np.array_equal(got["left"], ref["left"]) and np.array_equal(got["right"], ref["right"])
    assert np.array_equal(got["lo"], ref["lo"]) and np.array_equal(got["hi"], ref["hi"])
    rng = np.random.default_rng(5)
    m = 50000
    ro = rng.uniform(-1, 1, size=(m, 3)).astype(np.float32); ro[:, 1] = np.abs(ro[:, 1]) * 0.5 + 0.05
    rd = rng.normal(size=(m, 3)).astype(np.float32); rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    vis = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    assert np.array_equal(vis, sc.visibility(ro, rd, mode="bvh"))
    assert 0.1 < vis.mean() < 0.9


def _assert_structure(dev, v, f):
    from nvdiffrecmc_b200.optixutils.ops import bvh_export
    ctx = _build(dev, v, f)
    g = {k: t.cpu().numpy() for k, t in bvh_export(ctx).items()}
    r = oracle().scene(v, f).export_lbvh()
    assert np.array_equal(g["morton"].view(np.uint32), r["morton"]) and np.array_equal(g["prim"], r["prim"])
    assert np.array_equal(g["left"], r["left"]) and np.array_equal(g["right"], r["right"])
    assert np.array_equal(g["lo"], r["lo"]) and np.array_equal(g["hi"], r["hi"])
    return ctx


@pytest.mark.parametrize("kind,level", [("blob+torus", 4), ("bob-like", 4), ("blob+torus", 5)])
def test_structure_on_both_build_paths(dev, kind, level):
    """Sizes around the reference's meshes (bob 10 688, spot 5 856 triangles) and one above them.  Both must reproduce the oracle's LBVH bit for
    bit, and the visibility queries on its fp32 nodes must equal the oracle's LBVH traversal.  (The shadow rays walk a separate view:
    tests/test_gpu_shadow_bvh.py and tests/test_gpu_bvh_sizes.py.)"""
    v, f = synth.scene_mesh(kind, level=level)
    ctx = _assert_structure(dev, v, f)
    import nvdiffrecmc_b200.optixutils as ou
    ro, rd = _rays(20000, 3, v)
    vis = ou.trace_visibility(ctx, torch.tensor(ro, device=dev), torch.tensor(rd, device=dev)).cpu().numpy()
    assert np.array_equal(vis, oracle().scene(v, f).visibility(ro, rd, mode="bvh"))


def test_duplicate_morton_keys_break_ties_by_triangle_id(dev):
    """Coincident triangles (identical centroids => identical Morton codes): the order must be (key, triangle id), which the radix sort gets from stability."""
    v, f = synth.scene_mesh("blob", level=2)
    f2 = np.concatenate([f, f[::3], f[::5]]).astype(np.int32)
    _assert_structure(dev, v, f2)
