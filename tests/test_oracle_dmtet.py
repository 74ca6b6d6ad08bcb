"""CPU: the DMTet oracle (oracle/dmtet.c) against the reference's own marching_tets / sdf_reg_loss (tests/golden/ref_dmtet.npz), its fp64
build against finite differences and the analytic regulariser gradient, and the argument checks of the Python API and the C entries."""
import ctypes
import os

import numpy as np
import pytest

from dmtet_grids import GOLDEN, grid32, kuhn_grid, load_dmtet_golden, ref_all_edges
from oracle.dmtet import dmtet_oracle

CASES = ("init", "sphere0", "nonfinite")


@pytest.fixture(scope="module")
def golden():
    return load_dmtet_golden()


@pytest.fixture(scope="module")
def tables32():
    v, idx = grid32()
    return dmtet_oracle().tables(idx, v.shape[0])


def same(a, b):
    """Equal values (-0 == +0), NaN where the other has NaN."""
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def close(a, b, tol=1e-6):
    """Relative L2 over the entries finite in both, with the same zero set and the same non-finite entries."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert np.array_equal(fa, fb) and np.array_equal(a[~fa], b[~fb], equal_nan=True), "different non-finite entries"
    assert np.array_equal(a[fa] == 0, b[fb] == 0), "different zero sets"
    d = np.linalg.norm(a[fa] - b[fb])
    n = np.linalg.norm(b[fb])
    assert d <= tol * max(n, 1e-30), "rel L2 %.3e" % (d / max(n, 1e-30))


def test_static_tables_are_the_reference_edge_list(tables32):
    tb = tables32
    v, idx = grid32()
    assert np.array_equal(tb["edges"], ref_all_edges(idx))
    pairs = np.sort(idx[:, [0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3]].reshape(-1, 6, 2), -1)
    assert np.array_equal(tb["edges"][tb["tet_edges"]], pairs)
    off, adj = tb["v2e_offsets"], tb["v2e_edges"]
    assert off[0] == 0 and off[-1] == 2 * len(tb["edges"])
    for vtx in (0, 17, 3000, v.shape[0] - 1):
        rows = adj[off[vtx]:off[vtx + 1]]
        assert np.all(np.diff(rows) > 0) and np.array_equal(rows, np.nonzero((tb["edges"] == vtx).any(1))[0])


@pytest.mark.parametrize("case", CASES)
def test_fp32_oracle_reproduces_the_reference(golden, tables32, case):
    o = dmtet_oracle()
    v, idx = grid32()
    g = golden[case]
    verts, faces, uvs, uv_idx, _ = o.marching_tets(v, g["sdf"], idx, tables32)
    assert same(verts, g["verts"])
    assert np.array_equal(faces, g["faces"]) and np.array_equal(uv_idx, g["uv_idx"])
    assert uvs.shape == golden["uvs_shape"] and np.array_equal(uvs[:64].view(np.int32), golden["uvs_head"].view(np.int32))
    assert np.array_equal(golden["codec"].uvs_digest(uvs), golden["uvs_sha256"])
    d_pos, d_sdf = o.backward(v, g["sdf"], idx, g["d_verts"], tables32)
    close(d_pos, g["d_pos"])
    close(d_sdf, g["d_sdf"])
    edges = ref_all_edges(idx)
    loss, m = o.sdf_reg_loss(g["sdf"], edges)
    ref = float(g["reg_loss"])
    assert (np.isnan(loss) and np.isnan(ref)) or abs(loss - ref) <= 1e-6 * abs(ref)
    close(o.sdf_reg_loss_bwd(g["sdf"], edges, g["reg_d_loss"]), g["reg_d_sdf"])


def _away_from_zero(n, seed, margin=0.05):
    r = np.random.default_rng(seed)
    s = r.uniform(margin, 1.0, n) * np.where(r.random(n) < 0.5, -1.0, 1.0)
    return s


def test_fp64_gradients_match_finite_differences():
    o = dmtet_oracle(f64=True)
    verts, tets = kuhn_grid(3)
    V = verts.shape[0]
    r = np.random.default_rng(5)
    pos = verts.astype(np.float64) + r.uniform(-0.05, 0.05, verts.shape)
    sdf = _away_from_zero(V, 6)
    tb = o.tables(tets, V)
    v0 = o.marching_tets(pos, sdf, tets, tb)[0]
    G = r.standard_normal(v0.shape)
    L = lambda p, s: float((o.marching_tets(p, s, tets, tb)[0] * G).sum())
    d_pos, d_sdf = o.backward(pos, sdf, tets, G, tb)
    h = 1e-6
    for i in r.choice(V, 12, replace=False):
        sp, sm = sdf.copy(), sdf.copy()
        sp[i] += h; sm[i] -= h
        assert abs((L(pos, sp) - L(pos, sm)) / (2 * h) - d_sdf[i]) <= 1e-6 * (1 + abs(d_sdf[i]))
        for c in range(3):
            pp, pm = pos.copy(), pos.copy()
            pp[i, c] += h; pm[i, c] -= h
            assert abs((L(pp, sdf) - L(pm, sdf)) / (2 * h) - d_pos[i, c]) <= 1e-6 * (1 + abs(d_pos[i, c]))
    assert (d_sdf != 0).any() and (d_sdf == 0).any()


def test_fp64_regulariser_gradient_is_the_analytic_form():
    o = dmtet_oracle(f64=True)
    verts, tets = kuhn_grid(3)
    V = verts.shape[0]
    sdf = np.random.default_rng(8).standard_normal(V)
    sdf[::7] = 0.0
    edges = o.tables(tets, V)["edges"]
    loss, M = o.sdf_reg_loss(sdf, edges)
    s = sdf[edges]
    sg = np.sign(s)
    mask = sg[:, 0] != sg[:, 1]
    assert M == mask.sum() > 0
    sig = lambda x: 1 / (1 + np.exp(-x))
    bce = lambda x, y: np.log1p(np.exp(-np.abs(x))) + np.maximum(x, 0) - x * y
    a, b = s[mask, 0], s[mask, 1]
    assert abs(loss - (bce(a, b > 0).mean() + bce(b, a > 0).mean())) <= 1e-12
    want = np.zeros(V)
    np.add.at(want, edges[mask, 0], (sig(a) - (b > 0)) * 0.75 / M)
    np.add.at(want, edges[mask, 1], (sig(b) - (a > 0)) * 0.75 / M)
    assert np.abs(o.sdf_reg_loss_bwd(sdf, edges, 0.75) - want).max() <= 1e-14
    # no sign change: NaN loss (the mean of nothing) and a zero gradient
    pos_only = np.abs(sdf) + 1.0
    assert np.isnan(o.sdf_reg_loss(pos_only, edges)[0]) and not o.sdf_reg_loss_bwd(pos_only, edges).any()


def test_golden_generator_reproduces_the_fixture(golden):
    mk = golden["codec"]
    if not os.path.exists(mk.REF):
        pytest.skip("the reference checkout is not present")
    d = mk.generate()
    frozen = dict(np.load(os.path.join(GOLDEN, "ref_dmtet.npz")))
    assert sorted(d) == sorted(frozen)
    for k in d:
        assert same(np.asarray(d[k]), frozen[k]) and np.asarray(d[k]).dtype == frozen[k].dtype, k


def test_python_api_rejects_bad_arguments_before_any_launch():
    import torch
    from nvdiffrecmc_b200.dmtet import marching_tets, sdf_reg_loss
    pos, sdf, tet = torch.zeros(8, 3), torch.zeros(8), torch.zeros(2, 4, dtype=torch.int64)
    bad = [
        (marching_tets, (pos.double(), sdf, tet)), (marching_tets, (pos[:, :2], sdf, tet)), (marching_tets, (pos, sdf[:7], tet)),
        (marching_tets, (pos, sdf.half(), tet)), (marching_tets, (pos, sdf, tet.float())), (marching_tets, (pos, sdf, tet[:, :3])),
        (marching_tets, (pos, sdf, tet[:0])), (sdf_reg_loss, (sdf[:, None], tet[:, :2])), (sdf_reg_loss, (sdf, tet)),
        (sdf_reg_loss, (sdf, tet[:, :2].short())), (sdf_reg_loss, (sdf.double(), tet[:, :2])),
    ]
    for fn, args in bad:
        with pytest.raises(ValueError):
            fn(*args)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            marching_tets(pos, sdf, tet)


def test_c_entries_check_their_arguments_before_any_launch():
    import torch
    from nvdiffrecmc_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("the calls would launch on the fake pointers")
    l = _lib.lib()
    N, P = None, 0x10000
    calls = [
        ("mcs_dmtet_count", lambda: l.mcs_dmtet_count(N, 1, P, 4, P, 1, P, P, P, P, N), b"null argument"),
        ("mcs_dmtet_count", lambda: l.mcs_dmtet_count(P, 1, P, 0, P, 1, P, P, P, P, N), b"bad sizes"),
        ("mcs_dmtet_count", lambda: l.mcs_dmtet_count(P, 1, P + 4, 4, P, 1, P, P, P, P, N), b"misaligned"),
        ("mcs_dmtet_emit", lambda: l.mcs_dmtet_emit(P, 3, 1, P, 1, P, 4, P, P, 1, P, P, P, P, N, P, N), b"null argument"),
        ("mcs_dmtet_emit", lambda: l.mcs_dmtet_emit(P, -3, 1, P, 1, P, 4, P, P, 1, P, P, P, P, P, P, N), b"bad sizes"),
        ("mcs_dmtet_bwd", lambda: l.mcs_dmtet_bwd(P, 3, 1, P, 1, 8, P, 4, P, P, P, N, P, P, N), b"null argument"),
        ("mcs_dmtet_bwd", lambda: l.mcs_dmtet_bwd(P, 3, 1, P, 1, 0, P, 4, P, P, P, P, P, P, N), b"bad sizes"),
        ("mcs_sdf_reg_fwd", lambda: l.mcs_sdf_reg_fwd(P, 1, N, 4, P, P, P, N), b"null argument"),
        ("mcs_sdf_reg_fwd", lambda: l.mcs_sdf_reg_fwd(P, -1, P, 4, P, P, P, N), b"bad sizes"),
        ("mcs_sdf_reg_bwd", lambda: l.mcs_sdf_reg_bwd(P, 1, 8, P, P, P, N, P, P, N), b"null argument"),
        ("mcs_sdf_reg_bwd", lambda: l.mcs_sdf_reg_bwd(P, 1, 0, P, P, P, P, P, P, N), b"bad sizes"),
    ]
    for name, call, frag in calls:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0 and frag in msg and name[len("mcs_"):].encode() in msg, (name, msg)
    assert l.mcs_dmtet_workspace_bytes(0, 5) < 0
    assert l.mcs_dmtet_workspace_bytes(2048, 2049) == 8 * (1 + 1 + 2)
    assert l.mcs_sdf_reg_num_partials(0) == 1 and l.mcs_sdf_reg_num_partials(4097) == 2
