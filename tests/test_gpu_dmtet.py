"""GPU: nvdiffrecmc_b200.dmtet against the reference's own marching_tets / sdf_reg_loss (tests/golden/ref_dmtet.npz) and bit for bit
against the fp32 oracle (oracle/dmtet.c) -- on the 64^3 Kuhn grid, at the scan's tile boundaries, on one tet, on non-finite and
boundary SDFs and on empty surfaces -- plus equivalent inputs, the table cache, sdf_reg_loss against the fp64 oracle and in a CUDA
graph, and the host synchronisations of each pass."""
import warnings

import numpy as np
import pytest
import torch

from dmtet_grids import grid32, kuhn_grid, load_dmtet_golden, ref_init_sdf, sphere_sdf
from oracle.dmtet import dmtet_oracle

pytestmark = pytest.mark.gpu

TILE = 2048          # MCS_DMTET_TILE
RES = 32
CASES = ("init", "sphere0", "nonfinite")


def _np(t):
    return t.detach().cpu().numpy()


def bits_equal(a, b):
    """Same bits, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32))


def close(a, b, tol=1e-6):
    """Relative L2 over the entries finite in both, with the same zero set and the same non-finite entries."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert np.array_equal(fa, fb) and np.array_equal(a[~fa], b[~fb], equal_nan=True), "different non-finite entries"
    assert np.array_equal(a[fa] == 0, b[fb] == 0), "different zero sets"
    n = max(np.linalg.norm(b[fb]), 1e-30)
    assert np.linalg.norm(a[fa] - b[fb]) <= tol * n, "rel L2 %.3e" % (np.linalg.norm(a[fa] - b[fb]) / n)


def run(dev, pos, sdf, tet, G=None, seed=0):
    """marching_tets forward + backward of the upstream gradient G (seeded normal if None) -> dict of numpy arrays."""
    from nvdiffrecmc_b200.dmtet import marching_tets
    p = torch.as_tensor(pos, device=dev).requires_grad_(True) if not torch.is_tensor(pos) else pos
    s = torch.as_tensor(sdf, device=dev).requires_grad_(True) if not torch.is_tensor(sdf) else sdf
    t = torch.as_tensor(tet, device=dev) if not torch.is_tensor(tet) else tet
    verts, faces, uvs, uv_idx = marching_tets(p, s, t)
    if G is None:
        G = np.random.default_rng(seed).standard_normal(tuple(verts.shape)).astype(np.float32)
    d_pos, d_sdf = torch.autograd.grad(verts, (p, s), torch.as_tensor(G, device=dev))
    return {"verts": _np(verts), "faces": _np(faces), "uvs": _np(uvs), "uv_idx": _np(uv_idx), "d_pos": _np(d_pos), "d_sdf": _np(d_sdf),
            "G": G, "dtypes": (verts.dtype, faces.dtype, uvs.dtype, uv_idx.dtype)}


def check_oracle(dev, pos, sdf, tet, seed=0):
    pos = np.ascontiguousarray(pos, np.float32); sdf = np.ascontiguousarray(sdf, np.float32)
    r = run(dev, pos, sdf, tet, seed=seed)
    o = dmtet_oracle()
    tb = o.tables(tet, pos.shape[0])
    verts, faces, uvs, uv_idx, _ = o.marching_tets(pos, sdf, tet, tb)
    assert bits_equal(r["verts"], verts)
    assert np.array_equal(r["faces"], faces) and np.array_equal(r["uv_idx"], uv_idx)
    assert bits_equal(r["uvs"], uvs)
    d_pos, d_sdf = o.backward(pos, sdf, tet, r["G"], tb)
    assert bits_equal(r["d_pos"], d_pos) and bits_equal(r["d_sdf"], d_sdf)
    return r


@pytest.fixture(scope="module")
def golden():
    return load_dmtet_golden()


@pytest.mark.parametrize("case", CASES)
def test_reproduces_the_reference_fixture(dev, golden, case):
    from nvdiffrecmc_b200.dmtet import marching_tets
    v, idx = grid32()
    g = golden[case]
    r = run(dev, v, g["sdf"], idx, G=g["d_verts"])
    assert np.array_equal(r["verts"], g["verts"], equal_nan=True)
    assert np.array_equal(r["faces"], g["faces"]) and np.array_equal(r["uv_idx"], g["uv_idx"])
    assert r["uvs"].shape == golden["uvs_shape"] and np.array_equal(r["uvs"][:64].view(np.int32), golden["uvs_head"].view(np.int32))
    assert np.array_equal(golden["codec"].uvs_digest(r["uvs"]), golden["uvs_sha256"])
    assert r["dtypes"] == (torch.float32, torch.int64, torch.float32, torch.int64)
    close(r["d_pos"], g["d_pos"])
    close(r["d_sdf"], g["d_sdf"])
    # d deform through getMesh's deformation, run on the GPU, against the chain rule on the reference's d pos
    deform = torch.tensor(golden["deform"], device=dev, requires_grad=True)
    verts = marching_tets(torch.tensor(v, device=dev) + 2 / (RES * 2) * torch.tanh(deform), torch.tensor(g["sdf"], device=dev),
                          torch.tensor(idx, device=dev))[0]
    verts.backward(torch.tensor(g["d_verts"], device=dev))
    t = np.tanh(golden["deform"].astype(np.float64))
    close(_np(deform.grad), g["d_pos"].astype(np.float64) * (2 / (2 * RES)) * (1 - t * t))


@pytest.mark.parametrize("sdf_kind", ["ref_init", "sphere"])
def test_kuhn64_bit_for_bit_with_the_oracle(dev, sdf_kind):
    verts, tets = kuhn_grid(64)
    assert verts.shape[0] == 274625 and tets.shape[0] == 1572864
    sdf = ref_init_sdf(verts.shape[0], seed=3) if sdf_kind == "ref_init" else sphere_sdf(verts)
    r = check_oracle(dev, verts, sdf, tets)
    assert r["verts"].shape[0] > 1000 and r["faces"].shape[0] > 1000


def _prefix_edges(tets):
    """E of every tet prefix: E(k) = number of distinct edges among the first k tets."""
    t = np.sort(tets[:, [0, 1, 0, 2, 0, 3, 1, 2, 1, 3, 2, 3]].reshape(-1, 6, 2), -1)
    keys = t[..., 0].astype(np.int64) * (tets.max() + 1) + t[..., 1]
    _, first = np.unique(keys.reshape(-1), return_index=True)
    return np.searchsorted(np.sort(first // 6), np.arange(tets.shape[0] + 1), side="left")


def _grid_with(T=None, E=None):
    """A grid of exactly T tets (a prefix of a Kuhn grid), or exactly E edges (a prefix padded with tets (x, x, x, x) on fresh vertices,
    one edge each)."""
    verts, tets = kuhn_grid(14)
    if T is not None:
        tets = tets[:T]
    else:
        pe = _prefix_edges(tets)
        k = int(np.searchsorted(pe, E, side="right") - 1)
        pad = E - int(pe[k])
        V = verts.shape[0]
        extra = np.repeat(np.arange(V, V + pad)[:, None], 4, 1)
        verts = np.concatenate([verts, np.random.default_rng(1).uniform(-0.5, 0.5, (pad, 3)).astype(np.float32)])
        tets = np.concatenate([tets[:k], extra])
    used = np.unique(tets)
    remap = np.full(verts.shape[0], -1, np.int64); remap[used] = np.arange(used.size)
    return verts[used], remap[tets]


@pytest.mark.parametrize("n", [TILE - 1, TILE, TILE + 1, 5 * TILE + 3])
@pytest.mark.parametrize("what", ["T", "E"])
def test_scan_tile_boundaries(dev, what, n):
    verts, tets = _grid_with(**{what: n})
    if what == "T":
        assert tets.shape[0] == n
    else:
        assert dmtet_oracle().tables(tets, verts.shape[0])["edges"].shape[0] == n
    sdf = np.random.default_rng(n).standard_normal(verts.shape[0]).astype(np.float32)
    check_oracle(dev, verts, sdf, tets, seed=n)


def test_single_tet_every_occupancy_code(dev):
    pos = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    tet = np.array([[0, 1, 2, 3]])
    for code in range(1, 15):
        sdf = np.array([0.7 if code >> k & 1 else -0.4 - 0.1 * k for k in range(4)], np.float32)
        r = check_oracle(dev, pos, sdf, tet, seed=code)
        assert r["faces"].shape[0] == (2 if bin(code).count("1") == 2 else 1)


def test_single_crossing_edge(dev):
    pos = np.array([[0, 0, 0], [1, 2, 3]], np.float32)
    r = check_oracle(dev, pos, np.array([0.25, -0.75], np.float32), np.array([[0, 1, 1, 1]]))
    assert r["verts"].shape == (1, 3) and r["faces"].shape == (1, 3)


@pytest.mark.parametrize("kind", ["zeros", "neg_zeros", "nan", "inf", "huge"])
def test_edge_sdfs_bit_for_bit_with_the_oracle(dev, kind):
    verts, tets = kuhn_grid(10)
    V = verts.shape[0]
    rng = np.random.default_rng(7)
    sdf = rng.standard_normal(V).astype(np.float32)
    pick = rng.random(V) < 0.25
    if kind == "zeros":
        sdf[pick] = 0.0
    elif kind == "neg_zeros":
        sdf[pick] = -0.0
    elif kind == "nan":
        sdf[pick] = np.nan
    elif kind == "inf":
        sdf[pick] = np.where(rng.random(pick.sum()) < 0.5, np.inf, -np.inf)
    else:                                       # +-3e38: D = sa - sb overflows where both ends are huge with opposite signs
        sdf = np.where(rng.random(V) < 0.5, 3e38, -3e38).astype(np.float32)
        sdf[pick] = rng.standard_normal(pick.sum())
    check_oracle(dev, verts, sdf, tets, seed=11)


@pytest.mark.parametrize("sign", [1.0, -1.0, 0.0])
def test_empty_surface(dev, sign):
    from nvdiffrecmc_b200.dmtet import marching_tets
    verts, tets = kuhn_grid(4)
    sdf = torch.full((verts.shape[0],), sign, device=dev, requires_grad=True)
    pos = torch.tensor(verts, device=dev, requires_grad=True)
    v, f, uvs, uv_idx = marching_tets(pos, sdf, torch.tensor(tets, device=dev))
    assert v.shape == (0, 3) and v.dtype == torch.float32 and v.requires_grad
    assert f.shape == (0, 3) and f.dtype == torch.int64 and uv_idx.shape == (0, 3) and uv_idx.dtype == torch.int64
    assert bits_equal(_np(uvs), dmtet_oracle().uvs(tets.shape[0]))
    v.sum().backward()
    assert not pos.grad.any() and not sdf.grad.any()


def test_equivalent_inputs_and_reproducibility(dev):
    verts, tets = kuhn_grid(12)
    V = verts.shape[0]
    sdf = sphere_sdf(verts, 0.31)
    base = run(dev, verts, sdf, tets)
    again = run(dev, verts, sdf, tets, G=base["G"])
    as32 = run(dev, verts, sdf, tets.astype(np.int32), G=base["G"])
    wide = torch.zeros(V, 7, device=dev); wide[:, 2:5] = torch.tensor(verts, device=dev)
    col = torch.zeros(V, 3, device=dev); col[:, 1] = torch.tensor(sdf, device=dev)
    p, s = wide[:, 2:5].requires_grad_(True), col[:, 1].requires_grad_(True)
    assert not p.is_contiguous() and not s.is_contiguous()
    strided = run(dev, p, s, tets, G=base["G"])
    for other in (again, as32, strided):
        for k in ("verts", "faces", "uvs", "uv_idx", "d_pos", "d_sdf"):
            assert bits_equal(other[k], base[k]), k


def test_no_grad_and_single_input_grads(dev):
    from nvdiffrecmc_b200.dmtet import marching_tets
    verts, tets = kuhn_grid(6)
    pos = torch.tensor(verts, device=dev, requires_grad=True)
    sdf = torch.tensor(sphere_sdf(verts, 0.27), device=dev, requires_grad=True)
    t = torch.tensor(tets, device=dev)
    with torch.no_grad():
        v = marching_tets(pos, sdf, t)[0]
    assert not v.requires_grad and v.grad_fn is None
    v2 = marching_tets(pos.detach(), sdf, t)[0]
    v2.sum().backward()
    assert pos.grad is None and sdf.grad is not None and torch.equal(v, v2.detach())


def test_table_cache(dev):
    from nvdiffrecmc_b200.dmtet import marching_tets
    va, ta = kuhn_grid(5)
    vb, tb = kuhn_grid(7)
    sa, sb = sphere_sdf(va, 0.3), sphere_sdf(vb, 0.3)
    ta_d, tb_d = torch.tensor(ta, device=dev), torch.tensor(tb, device=dev)
    o = dmtet_oracle()
    for _ in range(2):              # two grids used alternately
        for v, t, s, td in ((va, ta, sa, ta_d), (vb, tb, sb, tb_d)):
            out = marching_tets(torch.tensor(v, device=dev), torch.tensor(s, device=dev), td)
            ref = o.marching_tets(v, s, t)
            assert bits_equal(_np(out[0]), ref[0]) and np.array_equal(_np(out[1]), ref[1]) and bits_equal(_np(out[2]), ref[2])
    # an in-place edit of the index tensor rebuilds the tables
    ta_d[:, [1, 2]] = ta_d[:, [2, 1]].clone()
    edited = ta[:, [0, 2, 1, 3]]
    out = marching_tets(torch.tensor(va, device=dev), torch.tensor(sa, device=dev), ta_d)
    ref = o.marching_tets(va, sa, edited)
    assert bits_equal(_np(out[0]), ref[0]) and np.array_equal(_np(out[1]), ref[1])
    # indices outside [0, V) are refused when the tables are built
    bad = ta_d.clone(); bad[3, 2] = va.shape[0]
    with pytest.raises(ValueError):
        marching_tets(torch.tensor(va, device=dev), torch.tensor(sa, device=dev), bad)
    from nvdiffrecmc_b200.dmtet import sdf_reg_loss
    with pytest.raises(ValueError):
        sdf_reg_loss(torch.tensor(sa, device=dev), torch.tensor([[0, va.shape[0]]], device=dev))


def _reg(dev, sdf, edges, d_loss=1.0):
    from nvdiffrecmc_b200.dmtet import sdf_reg_loss
    s = torch.tensor(sdf, device=dev, requires_grad=True)
    loss = sdf_reg_loss(s, torch.as_tensor(edges, device=dev))
    assert loss.shape == () and loss.dtype == torch.float32
    g, = torch.autograd.grad(loss, s, torch.tensor(d_loss, device=dev))
    return float(loss.detach()), _np(g)


@pytest.mark.parametrize("kind", ["ref_init", "sphere_zeros", "nonfinite", "kuhn64"])
def test_sdf_reg_loss_against_the_fp64_oracle(dev, kind):
    if kind == "kuhn64":
        verts, tets = kuhn_grid(64)
        sdf = ref_init_sdf(verts.shape[0], seed=4)
    else:
        verts, tets = grid32()
        rng = np.random.default_rng(9)
        sdf = ref_init_sdf(verts.shape[0], seed=5) if kind == "ref_init" else sphere_sdf(verts, 0.4)
        if kind == "sphere_zeros":
            sdf[rng.random(sdf.size) < 0.2] = 0.0
            sdf[rng.random(sdf.size) < 0.05] = -0.0
    edges = dmtet_oracle().tables(tets, verts.shape[0])["edges"]
    if kind == "nonfinite":         # NaN has sign 0, so a NaN next to 0 is not masked; inf keeps the loss finite or inf
        sdf[np.random.default_rng(3).random(sdf.size) < 0.02] = np.inf
    o64 = dmtet_oracle(f64=True)
    loss, g = _reg(dev, sdf, edges.astype(np.int64), 0.7)
    ref, M = o64.sdf_reg_loss(sdf.astype(np.float64), edges)
    assert M > 0
    if np.isfinite(ref):
        assert abs(loss - ref) <= 1e-6 * abs(ref)
    else:
        assert loss == ref or (np.isnan(loss) and np.isnan(ref))
    close(g, o64.sdf_reg_loss_bwd(sdf.astype(np.float64), edges, 0.7))


def test_sdf_reg_loss_without_sign_changes_is_nan_with_zero_gradient(dev):
    verts, tets = kuhn_grid(4)
    edges = dmtet_oracle().tables(tets, verts.shape[0])["edges"]
    for sdf in (np.full(verts.shape[0], 0.5, np.float32), np.zeros(verts.shape[0], np.float32)):
        loss, g = _reg(dev, sdf, edges)
        assert np.isnan(loss) and not g.any()


def test_sdf_reg_loss_in_a_cuda_graph(dev):
    from nvdiffrecmc_b200.dmtet import sdf_reg_loss
    verts, tets = grid32()
    sdf = torch.tensor(ref_init_sdf(verts.shape[0], seed=6), device=dev, requires_grad=True)
    edges = torch.tensor(dmtet_oracle().tables(tets, verts.shape[0])["edges"], device=dev, dtype=torch.int64)
    d_loss = torch.tensor(0.3, device=dev)

    def step():
        loss = sdf_reg_loss(sdf, edges)
        g, = torch.autograd.grad(loss, sdf, d_loss)
        return loss.detach(), g

    eager = [v.clone() for v in step()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])


def test_host_synchronisations(dev):
    from nvdiffrecmc_b200.dmtet import marching_tets, sdf_reg_loss
    verts, tets = kuhn_grid(16)
    pos = torch.tensor(verts, device=dev, requires_grad=True)
    sdf = torch.tensor(ref_init_sdf(verts.shape[0], seed=8), device=dev, requires_grad=True)
    t = torch.tensor(tets, device=dev)
    edges = torch.tensor(dmtet_oracle().tables(tets, verts.shape[0])["edges"], device=dev, dtype=torch.int64)
    v = marching_tets(pos, sdf, t)[0]                    # builds and caches the tables
    sdf_reg_loss(sdf, edges).backward()
    G = torch.randn(v.shape, device=dev)
    torch.cuda.synchronize()

    def warnings_of(fn):
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        return out, [x for x in w if "synchroniz" in str(x.message)]

    (v, f, uvs, uv_idx), w = warnings_of(lambda: marching_tets(pos, sdf, t))
    assert len(w) == 1, [str(x.message) for x in w]
    _, w = warnings_of(lambda: torch.autograd.grad(v, (pos, sdf), G))
    assert w == []
    _, w = warnings_of(lambda: torch.autograd.grad(sdf_reg_loss(sdf, edges), sdf))
    assert w == []
