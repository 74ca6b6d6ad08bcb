"""CPU: the oracle's canonical LBVH traversal equals its brute-force predicate at the triangle counts and on the meshes of
tests/test_gpu_bvh_sizes.py, on the same rays.  That is what lets the GPU tests compare against the traversal where brute force is slow."""
import numpy as np
import pytest

from common import BVH_CASES, bvh_rays, sized_mesh

NRAYS = 8192              # tests/test_gpu_bvh_sizes.py NRAYS, seeded by T as there


@pytest.mark.parametrize("kind,T", BVH_CASES)
def test_lbvh_traversal_equals_brute_force(orc, kind, T):
    v, f = sized_mesh(kind, T)
    assert f.shape[0] == T
    sc = orc.scene(v, f)
    ro, rd = bvh_rays(NRAYS, T, v)
    brute = sc.visibility(ro, rd, mode="brute")
    lbvh = sc.visibility(ro, rd, mode="bvh")
    assert np.array_equal(lbvh, brute), "%d of %d rays differ" % ((lbvh != brute).sum(), NRAYS)
    assert 0 < brute.mean() < 1
