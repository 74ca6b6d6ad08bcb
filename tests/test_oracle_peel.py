"""CPU: the depth-peeling ray query (closest hit beyond sep(t_prev)) of the brute-force fp32 twin against every hit of each ray."""
import numpy as np
import pytest

from common import oracle
from nvdiffrecmc_b200 import synth
from oracle import peel_sep


def _rays(n, seed, v, spread=0.3):
    rng = np.random.default_rng(seed)
    c = v.mean(0); ext = (v.max(0) - v.min(0)).max()
    ro = (c + rng.normal(size=(n, 3)) * ext * 0.7).astype(np.float32)
    d = (c + rng.normal(size=(n, 3)) * ext * spread - ro)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return ro, d.astype(np.float32)


def _mesh(kind):
    if kind == "icosphere":
        v, f = synth.icosphere(3)
        return v.astype(np.float32), f.astype(np.int32)
    return synth.scene_mesh(kind, level=2)


@pytest.mark.parametrize("kind", ["blob+torus", "icosphere"])
def test_peel_lists_every_surface_once(kind):
    v, f = _mesh(kind)
    sc = oracle().scene(v, f)
    ro, rd = _rays(300, 7, v)
    layers = sc.peel(ro, rd, 16)
    assert (layers[-1][0] < 0).all(), "16 layers do not exhaust the scene"
    depth = np.zeros(ro.shape[0], int)
    for i in range(ro.shape[0]):
        listed = [(tuv[i, 0], tid[i]) for tid, tuv in layers if tid[i] >= 0]
        depth[i] = len(listed)
        t_l = np.array([t for t, _ in listed], np.float32)
        assert (np.diff(t_l) > 0).all()                                                   # strictly increasing t
        t_all, id_all = sc.all_hits(ro[i], rd[i])
        hits = dict(zip(id_all.tolist(), t_all.tolist()))
        for t, k in listed:
            assert hits.get(int(k)) == float(t)                                          # a brute-force hit, same t
        listed_ids = {int(k) for _, k in listed}
        for t, k in zip(t_all, id_all):
            if int(k) in listed_ids:
                continue
            before = t_l[t_l <= t]
            assert before.size > 0 and t <= peel_sep(before[-1]), (i, float(t), int(k))     # merged into the layer just before it
        # every layer is the smallest (t, id) beyond the previous layer's separation
        lo = np.float32(0)
        for t, k in listed:
            cand = [(tt, kk) for tt, kk in zip(t_all, id_all) if tt > lo]
            assert min(cand, key=lambda x: (x[0], x[1])) == (t, k)
            lo = peel_sep(t)
    assert depth.max() >= 2 and (depth == 0).any()


def test_rays_through_a_closed_sphere_have_two_layers():
    v, f = _mesh("icosphere")
    sc = oracle().scene(v, f)
    rng = np.random.default_rng(3)
    n = 2000
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    ro = (-3.0 * d + rng.uniform(-0.5, 0.5, size=(n, 3))).astype(np.float32)          # outside, aimed through the interior
    tgt = rng.uniform(-0.4, 0.4, size=(n, 3))
    rd = (tgt - ro); rd = (rd / np.linalg.norm(rd, axis=1, keepdims=True)).astype(np.float32)
    layers = sc.peel(ro, rd, 4)
    count = sum((tid >= 0).astype(int) for tid, _ in layers)
    assert (count == 2).all(), np.bincount(count)


def test_shared_edges_do_not_come_back_as_layers():
    """Rays aimed at the midpoints of an icosphere's edges: Moeller-Trumbore's closed bounds accept many of them on both triangles of
    the edge, a few ulp apart.  The separation merges the pair, so no ray sees more than the two surfaces of the sphere."""
    v, f = _mesh("icosphere")
    sc = oracle().scene(v, f)
    e = np.unique(np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1), axis=0)
    mid = ((v[e[:, 0]] + v[e[:, 1]]) * np.float32(0.5)).astype(np.float32)
    ro = np.broadcast_to(np.array([1.2, -0.8, 4.0], np.float32), mid.shape).copy()
    rd = (mid - ro).astype(np.float32)
    n_hits = np.array([sc.all_hits(ro[i], rd[i])[0].size for i in range(ro.shape[0])])
    count = sum((tid >= 0).astype(int) for tid, _ in sc.peel(ro, rd, 4))
    assert (n_hits == 3).sum() > 100                  # an edge hit twice on one side of the sphere
    assert count.max() == 2 and (count == 2).sum() > 0.7 * ro.shape[0]
