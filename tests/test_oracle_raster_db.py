"""CPU: the screen-space derivatives of row f2 (rast_db, interpolate's out_da and their adjoints) in the geometry oracle, against
finite differences, hand-computed affine cases and the adjoint identity; the C ABI's argument checks; the render_layer golden."""
import ctypes
import os

import numpy as np
import pytest

from oracle.raster_db import raster_db_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S_MIN = 1e-3        # pixels whose |S| (twice the clip-space area term) is below this are excluded from the finite-difference checks


def _ndc(i, n):
    return (i + 0.5) / n * 2 - 1


def _persp_soup(rng, T, behind=True):
    """T random perspective triangles [3T,4] (clip = P (p, 1), view-space z in [-4, -1]); with `behind`, triangle 0 has a vertex at w < 0."""
    p = np.concatenate([rng.uniform(-1.2, 1.2, (3 * T, 2)), rng.uniform(-4.0, -1.0, (3 * T, 1)), np.ones((3 * T, 1))], 1)
    if behind:
        p[0, 2] = 0.5
    n, f = 0.1, 10.0
    P = np.array([[1.3, 0, 0, 0], [0, 1.7, 0, 0], [0, 0, -(f + n) / (f - n), -2 * f * n / (f - n)], [0, 0, -1, 0]])
    pos = p @ P.T
    return pos, np.arange(3 * T, dtype=np.int32).reshape(T, 3)


def _bary(pos, tri, px, py):
    """(u, v) of the perspective-correct barycentrics at NDC (px, py), solved directly: sum b_i (x_i - px w_i, y_i - py w_i) = 0, sum b_i = 1."""
    q = pos[tri]
    M = np.stack([q[:, 0] - px * q[:, 3], q[:, 1] - py * q[:, 3], np.ones(3)])
    b = np.linalg.solve(M, [0.0, 0.0, 1.0])
    return b[0], b[1]


def _S(pos, tri, px, py):
    a = np.stack([pos[tri, 0] - px * pos[tri, 3], pos[tri, 1] - py * pos[tri, 3]], 1)
    cross = lambda p, q: p[0] * q[1] - p[1] * q[0]
    return sum(cross(a[(i + 1) % 3], a[(i + 2) % 3]) for i in range(3))


def _rast_ids(rng, B, H, W, T):
    r = np.zeros((B, H, W, 4))
    r[..., 3] = rng.integers(1, T + 1, (B, H, W))
    return r


def test_rast_db_matches_finite_differences():
    o = raster_db_oracle(f64=True)
    rng = np.random.default_rng(1)
    T, B, H, W = 6, 1, 9, 13
    pos, tris = _persp_soup(rng, T)
    assert (pos[:, 3] < 0).any()
    rast = _rast_ids(rng, B, H, W, T)
    db = o.rast_db(pos, tris, rast)
    h, checked = 1e-6, 0
    for y in range(H):
        for x in range(W):
            t = tris[int(rast[0, y, x, 3]) - 1]
            if abs(_S(pos, t, _ndc(x, W), _ndc(y, H))) < S_MIN:
                continue
            fd = []
            for dx, dy in ((h, 0), (0, h)):
                up = _bary(pos, t, _ndc(x + dx, W), _ndc(y + dy, H))
                dn = _bary(pos, t, _ndc(x - dx, W), _ndc(y - dy, H))
                fd.append([(up[0] - dn[0]) / (2 * h), (up[1] - dn[1]) / (2 * h)])
            ref = np.array([fd[0][0], fd[1][0], fd[0][1], fd[1][1]])          # (du/dX, du/dY, dv/dX, dv/dY)
            assert np.allclose(db[0, y, x], ref, rtol=1e-6, atol=1e-7 * np.abs(ref).max()), (y, x, db[0, y, x], ref)
            checked += 1
    assert checked > 0.9 * H * W


def test_rast_db_affine_is_the_hand_computed_constant():
    o = raster_db_oracle(f64=True)
    H, W = 5, 11                                        # H != W: a swapped 2/W and 2/H would show
    x0, y0, x1, y1, x2, y2 = -0.6, -0.5, 0.7, -0.2, 0.1, 0.8
    pos = np.array([[x0, y0, 0.3, 1.0], [x1, y1, -0.2, 1.0], [x2, y2, 0.5, 1.0]])
    rast = np.zeros((1, H, W, 4)); rast[..., 3] = 1
    S = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0)
    ref = np.array([2 / W * (y1 - y2) / S, 2 / H * (x2 - x1) / S, 2 / W * (y2 - y0) / S, 2 / H * (x0 - x2) / S])
    db = o.rast_db(pos, np.array([[0, 1, 2]]), rast)
    assert np.allclose(db.reshape(-1, 4), ref[None], rtol=1e-12, atol=0)


@pytest.mark.parametrize("batched", [False, True])
def test_rast_db_backward_matches_finite_differences(batched):
    o = raster_db_oracle(f64=True)
    rng = np.random.default_rng(3)
    T, B, H, W = 4, 2, 5, 7
    pos1, tris = _persp_soup(rng, T)
    pos = np.stack([pos1, pos1 + rng.normal(0, 0.02, pos1.shape)]) if batched else pos1
    rast = _rast_ids(rng, B, H, W, T)
    g = rng.normal(size=(B, H, W, 4))
    d = o.rast_db_bwd(pos, tris, rast, g)
    L = lambda p: float((o.rast_db(p, tris, rast) * g).sum())
    fd = np.zeros_like(pos)
    h = 1e-6
    for idx in np.ndindex(*pos.shape):
        pp, pm = pos.copy(), pos.copy()
        pp[idx] += h; pm[idx] -= h
        fd[idx] = (L(pp) - L(pm)) / (2 * h)
    assert np.abs(fd).max() > 0 and (d[..., 2] == 0).all()
    assert np.abs(d - fd).max() <= 1e-6 * np.abs(fd).max()


@pytest.mark.parametrize("diff_attrs", ["all", [2, 0, 2]])
def test_interpolate_da_adjoint_identity(diff_attrs):
    o = raster_db_oracle(f64=True)
    rng = np.random.default_rng(4)
    T, B, H, W, Cn = 5, 2, 6, 8, 3
    pos, tris = _persp_soup(rng, T)
    rast = _rast_ids(rng, B, H, W, T)
    rast[0, 0, :3, 3] = 0                                # background pixels
    attr = rng.normal(size=(B, 3 * T, Cn))
    db = o.rast_db(pos, tris, rast)
    out = o.interpolate_da(attr, tris, rast, db, diff_attrs)
    g = rng.normal(size=out.shape)
    d_attr, d_db = o.interpolate_da_bwd(attr, tris, rast, db, g, diff_attrs)
    lhs = float((g * out).sum())
    assert abs(float((d_attr * attr).sum()) - lhs) <= 1e-12 * abs(lhs) + 1e-14
    assert abs(float((d_db * db).sum()) - lhs) <= 1e-12 * abs(lhs) + 1e-14


def test_interpolate_da_of_one_hot_attributes():
    o = raster_db_oracle()
    rng = np.random.default_rng(5)
    T, B, H, W = 4, 1, 6, 7
    pos, tris = _persp_soup(rng, T, behind=False)
    rast = _rast_ids(rng, B, H, W, T).astype(np.float32)
    V = 3 * T
    attr = np.eye(V, dtype=np.float32)
    db = o.rast_db(pos, tris, rast)
    out = o.interpolate_da(attr, tris, rast, db).reshape(B, H, W, V, 2)
    for y in range(H):
        for x in range(W):
            i0, i1, i2 = tris[int(rast[0, y, x, 3]) - 1]
            d = db[0, y, x]
            ref = np.zeros((V, 2), np.float32)
            ref[i0] = d[[0, 1]]; ref[i1] = d[[2, 3]]; ref[i2] = [-(d[0] + d[2]), -(d[1] + d[3])]
            assert np.array_equal(out[0, y, x], ref)


def test_zeros_for_background_ids_beyond_T_and_degenerate_triangles():
    for o in (raster_db_oracle(), raster_db_oracle(f64=True)):
        rng = np.random.default_rng(6)
        T, H, W = 3, 4, 5
        pos, tris = _persp_soup(rng, T, behind=False)
        pos[6:9] = pos[6]                                # triangle 2: three equal vertices, S == 0 exactly
        rast = np.zeros((1, H, W, 4)); rast[..., 3] = 1
        rast[0, 0, :, 3] = 0                             # background
        rast[0, 1, :, 3] = T + 1                         # id >= T
        rast[0, 2, :, 3] = 3                             # degenerate
        db = o.rast_db(pos, tris, rast)
        assert (db[0, :3] == 0).all() and (np.abs(db[0, 3]) > 0).all()
        attr = rng.normal(size=(3 * T, 2))
        out = o.interpolate_da(attr, tris, rast, db)
        assert (out[0, :3] == 0).all() and (np.abs(out[0, 3]) > 0).any()
        g = np.ones((1, H, W, 4))
        assert (o.rast_db_bwd(pos, tris, rast, g)[6:9] == 0).all()
        d_attr, d_db = o.interpolate_da_bwd(attr, tris, rast, db, np.ones(out.shape))
        assert (d_db[0, :2] == 0).all() and (np.abs(d_db[0, 3]) > 0).any()


def test_cabi_argument_checks_without_a_device():
    from nvdiffrecmc_b200 import _lib
    l = _lib.lib()
    N, F = None, 64                                      # F: a non-null address that is never dereferenced (validation fails first)
    idx = lambda *k: (ctypes.c_int32 * len(k))(*k)
    calls = [
        (lambda: l.mcs_rast_db(N, 0, 3, N, 1, N, 1, 2, 2, N, N), b"mcs_rast_db: bad arguments"),
        (lambda: l.mcs_rasterize_bwd_db(F, 0, 3, F, 1, F, 1, 2, 2, F, N, F, N), b"mcs_rasterize_bwd_db: bad arguments"),
        (lambda: l.mcs_interpolate_da_fwd(F, 0, 3, 3, F, 1, F, N, 1, 2, 2, 3, N, F, N), b"bad arguments"),
        (lambda: l.mcs_interpolate_da_fwd(F, 0, 3, 3, F, 1, F, F, 1, 2, 2, 2, N, F, N), b"must equal C"),
        (lambda: l.mcs_interpolate_da_fwd(F, 0, 3, 3, F, 1, F, F, 1, 2, 2, 2, idx(0, 3), F, N), b"out of range"),
        (lambda: l.mcs_interpolate_da_fwd(F, 0, 3, 3, F, 1, F, F, 1, 2, 2, 2, idx(-1, 0), F, N), b"out of range"),
        (lambda: l.mcs_interpolate_da_fwd(F, 0, 3, 3, F, 1, F, F, 1, 2, 2, 33, idx(*([0] * 33)), F, N), b"1 to 32"),
        (lambda: l.mcs_interpolate_da_fwd(F, 0, 3, 3, F, 1, F, F, 1, 2, 2, 1, idx(0), N, N), b"null output"),
        (lambda: l.mcs_interpolate_da_bwd(F, 0, 3, 3, F, 1, F, F, 1, 2, 2, 1, idx(0), F, N, N, N), b"null gradient pointer"),
    ]
    for call, frag in calls:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0 and frag in msg, msg


@pytest.mark.skipif(not os.path.isdir("/root/reference/render"), reason="the reference checkout is not available")
def test_render_layer_golden_regenerates_bit_identically():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_render_layer_golden as mk
    finally:
        sys.path.remove(os.path.join(ROOT, "tests", "golden"))
    d = mk.generate()
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_render_layer_db.npz"))
    assert sorted(g.files) == sorted(d)
    for k in g.files:
        assert g[k].dtype == d[k].dtype and np.array_equal(g[k], d[k]), k
    # the reference reads channels 2:3 and 3:4 of clip_pos_deriv, i.e. dy_clip/dX and dy_clip/dY under nvdiffrast's layout
    geo = raster_db_oracle()
    da = geo.interpolate_da(d["pos"], d["tris"], d["rast"], d["rast_deriv"])
    clip = geo.interpolate(d["pos"], d["tris"], d["rast"])
    eps = np.float32(1e-5)
    z0 = np.maximum(clip[..., 2:3], eps) / np.maximum(clip[..., 3:4], eps)
    z1 = np.maximum(clip[..., 2:3] + np.abs(da[..., 2:3]), eps) / np.maximum(clip[..., 3:4] + np.abs(da[..., 3:4]), eps)
    assert np.array_equal(d["gb_depth"], np.concatenate([z0, np.abs(z1 - z0)], -1))
    assert (d["gb_depth"][..., 1] > 0).sum() > 300
