"""CPU: the hash-grid encoding's level table, the oracle's indices, adjoints and precision, the C ABI's argument checks and the config
checks of `nvdiffrecmc_b200.tinycudann.Encoding` (all without a GPU); in the build container, the reference's render/mlptexture.py
imports with that module as `tinycudann` and its frozen output regenerates bit for bit."""
import ctypes
import os
import sys

import numpy as np
import pytest

from oracle.hashgrid import REF_CONFIG, hashgrid_oracle
from nvdiffrecmc_b200 import _lib
from nvdiffrecmc_b200.tinycudann import level_table

HERE = os.path.dirname(os.path.abspath(__file__))
HAVE_REF = os.path.exists("/root/reference/render/mlptexture.py")
EDGE = {"otype": "HashGrid", "n_levels": 5, "log2_hashmap_size": 9, "base_resolution": 4, "per_level_scale": 2.0}
PADDED = {"otype": "HashGrid", "n_levels": 3, "log2_hashmap_size": 10, "base_resolution": 5, "per_level_scale": 1.5}


def _table(cfg):
    return level_table(cfg["n_levels"], cfg["log2_hashmap_size"], cfg["base_resolution"], cfg["per_level_scale"])


def test_reference_config_level_table():
    t = _table(REF_CONFIG)
    assert t["res"][:5] == [16, 24, 34, 49, 71]
    assert t["dense_mask"] == 0b11111
    sizes = np.diff(t["offset"])
    assert list(sizes[:5]) == [4096, 13824, 39304, 117656, 357912]
    assert list(sizes[5:]) == [1 << 19] * 11
    assert t["offset"][-1] == 6299960 and 2 * t["offset"][-1] == 12599920
    assert t["scale"][0] == 15.0


def test_edge_config_level_tables():
    t = _table(EDGE)
    assert t["res"] == [4, 8, 16, 32, 64]
    assert list(np.diff(t["offset"])) == [64, 512, 512, 512, 512]       # 4^3 dense, 8^3 = 2^9 exact fit (dense), then hashed
    assert t["dense_mask"] == 0b11
    t = _table(PADDED)
    assert t["res"] == [5, 8, 12]                                        # scale 4, 6.5, 10.25
    assert list(np.diff(t["offset"])) == [128, 512, 1024]               # 125 padded to 128; 512; 12^3 = 1728 > 2^10 hashed
    assert t["dense_mask"] == 0b11


@pytest.mark.parametrize("cfg", [REF_CONFIG, EDGE, PADDED, dict(EDGE, base_resolution=1300, n_levels=2, per_level_scale=1.7)])
def test_oracle_level_table_matches_the_product(cfg):
    a, b = hashgrid_oracle().levels(cfg), _table(cfg)
    assert [int(v) for v in a["offset"]] == b["offset"] and [int(v) for v in a["res"]] == b["res"]
    assert a["scale"].tolist() == [float(np.float32(s)) for s in b["scale"]] and a["dense_mask"] == b["dense_mask"]


def _index_params(lv):
    """params whose entry e holds (e, 1): y0 = sum_c w_c idx_c, y1 = sum_c w_c"""
    n = int(lv["offset"][-1])
    p = np.zeros((n, 2), np.float32)
    for l in range(lv["n_levels"]):
        o0, o1 = int(lv["offset"][l]), int(lv["offset"][l + 1])
        p[o0:o1, 0] = np.arange(o1 - o0)
    p[:, 1] = 1
    return p.reshape(-1)


def _hash(cx, cy, cz, size):
    M = 0xFFFFFFFF
    return ((cx & M) ^ ((cy * 2654435761) & M) ^ ((cz * 805459861) & M)) % size


def test_hand_computed_indices():
    o = hashgrid_oracle()
    lv = o.levels(EDGE)                       # scales 3, 7, 15, 31, 63
    p = _index_params(lv)
    # x = 0.5: p_d = scale / 2 + 0.5 is an integer at every level, t = 0, only corner 0 has weight
    y = o.forward(np.full((1, 3), 0.5), p, lv)[0]
    assert y[0] == 2 + 2 * 4 + 2 * 16                                   # dense, res 4, g = 2
    assert y[2] == 4 + 4 * 8 + 4 * 64                                   # dense, res 8, g = 4
    assert y[4] == _hash(8, 8, 8, 512) and y[6] == _hash(16, 16, 16, 512) and y[8] == _hash(32, 32, 32, 512)
    assert np.all(y[1::2] == 1)
    # x = 0 at level 0: p = 0.5, g = 0, t = 1/2: w_c = 1/8 for the cell's corners (0|1) + 4 (0|1) + 16 (0|1)
    y = o.forward(np.zeros((1, 3)), p, lv)[0]
    assert y[0] == 0.125 * sum(a + 4 * b + 16 * c for a in (0, 1) for b in (0, 1) for c in (0, 1))
    # x = 1 at level 0: p = 3.5, g = 3, the upper corner 4 == res aliases into the next row and wraps modulo 64
    y = o.forward(np.ones((1, 3)), p, lv)[0]
    assert y[0] == 0.125 * sum((a + 4 * b + 16 * c) % 64 for a in (3, 4) for b in (3, 4) for c in (3, 4))
    # a hashed level with t = 1/2 at every dimension (level 2: x = 0, p = 0.5)
    assert y[1] == 1.0
    y = o.forward(np.zeros((1, 3)), p, lv)[0]
    assert y[4] == 0.125 * sum(_hash(a, b, c, 512) for a in (0, 1) for b in (0, 1) for c in (0, 1))
    # negative coordinates wrap as uint32 (x = -0.5 at level 0: p = -1, g = -1 -> 2^32 - 1)
    y = o.forward(np.full((1, 3), -0.5), p, lv)[0]
    g = (1 << 32) - 1
    assert y[0] == (g + g * 4 + g * 16) % (1 << 32) % 64


def _away_from_faces(x, lv, margin=1e-3):
    ok = np.ones(len(x), bool)
    for s in lv["scale"]:
        p = float(s) * x + 0.5
        t = p - np.floor(p)
        ok &= np.all((t > margin) & (t < 1 - margin), axis=1)
    return x[ok]


def test_fp64_dx_matches_finite_differences():
    o = hashgrid_oracle(f64=True)
    lv = o.levels(EDGE)
    rng = np.random.default_rng(0)
    params = rng.uniform(-1, 1, 2 * int(lv["offset"][-1]))
    x = _away_from_faces(rng.uniform(0, 1, (400, 3)), lv)[:100]
    dy = rng.normal(size=(len(x), 2 * lv["n_levels"]))
    _, dx = o.backward(x, params, lv, dy, want_params=False)
    h = 1e-7
    fd = np.zeros_like(x)
    for d in range(3):
        e = np.zeros(3); e[d] = h
        fd[:, d] = ((o.forward(x + e, params, lv) - o.forward(x - e, params, lv)) * dy).sum(1) / (2 * h)
    assert len(x) >= 50
    assert np.abs(dx - fd).max() <= 1e-6 * np.abs(fd).max()


def test_fp64_adjoint_identity():
    """The encoding is linear in the params: <d params, p> = <dy, y(p)>."""
    o = hashgrid_oracle(f64=True)
    for cfg in (EDGE, PADDED):
        lv = o.levels(cfg)
        rng = np.random.default_rng(1)
        p = rng.uniform(-1, 1, 2 * int(lv["offset"][-1]))
        x = rng.uniform(-0.5, 1.5, (3000, 3))
        dy = rng.normal(size=(len(x), 2 * lv["n_levels"]))
        dy[::3] = 0
        dp, _ = o.backward(x, p, lv, dy, want_x=False)
        lhs, rhs = float(dp @ p), float((dy * o.forward(x, p, lv)).sum())
        assert abs(lhs - rhs) <= 1e-12 * abs(rhs)


def test_fp32_oracle_agrees_with_fp64():
    """To 1e-6 relative L2 on the coarse levels.  The fp32 error grows with the level's scale: p = scale * x + 0.5 is rounded to
    fp32, so at scale 63 (p up to 64, ulp 7.6e-6) the fractions t carry about 4x the error of scale 16; the bound scales with it."""
    o32, o64 = hashgrid_oracle(), hashgrid_oracle(f64=True)
    rl2 = lambda a, b: np.linalg.norm(a - b) / np.linalg.norm(b)
    for cfg in (PADDED, EDGE):
        lv = o32.levels(cfg)
        rng = np.random.default_rng(2)
        p = rng.uniform(-1, 1, 2 * int(lv["offset"][-1])).astype(np.float32)
        x = _away_from_faces(rng.uniform(0, 1, (3000, 3)).astype(np.float32), lv, 1e-2)
        dy = rng.normal(size=(len(x), 2 * lv["n_levels"])).astype(np.float32)
        tol = [1e-6 * max(1.0, float(s) / 16) for s in lv["scale"]]
        y32, y64 = o32.forward(x, p, lv), o64.forward(x, p, lv)
        for l in range(lv["n_levels"]):
            assert rl2(y32[:, 2 * l:2 * l + 2], y64[:, 2 * l:2 * l + 2]) <= tol[l], (cfg, l)
        dp32, dx32 = o32.backward(x, p, lv, dy)
        dp64, dx64 = o64.backward(x, p, lv, dy)
        assert rl2(dx32, dx64) <= max(tol) and rl2(dp32, dp64) <= max(tol)


def _c_levels(cfg, **override):
    from nvdiffrecmc_b200.tinycudann import _c_levels
    lv = _c_levels(_table(cfg))
    for k, v in override.items():
        if isinstance(v, tuple):
            getattr(lv, k)[v[0]] = v[1]
        else:
            setattr(lv, k, v)
    return lv


def test_entry_points_reject_bad_arguments_without_a_device():
    l = _lib.lib()
    N = None
    P = ctypes.c_void_p(256)              # never dereferenced: validation fails first
    good = _c_levels(EDGE)
    bad = [
        ("null x", lambda: l.mcs_hashgrid_fwd(N, 4, P, ctypes.byref(good), P, N), b"null pointer"),
        ("null params", lambda: l.mcs_hashgrid_fwd(P, 4, N, ctypes.byref(good), P, N), b"null pointer"),
        ("null levels", lambda: l.mcs_hashgrid_fwd(P, 4, P, N, P, N), b"null pointer"),
        ("null out", lambda: l.mcs_hashgrid_fwd(P, 4, P, ctypes.byref(good), N, N), b"null pointer"),
        ("n < 0", lambda: l.mcs_hashgrid_fwd(P, -1, P, ctypes.byref(good), P, N), b"n must be >= 0"),
        ("0 levels", lambda: l.mcs_hashgrid_fwd(P, 4, P, ctypes.byref(_c_levels(EDGE, n_levels=0)), P, N), b"n_levels must be in 1..16"),
        ("17 levels", lambda: l.mcs_hashgrid_fwd(P, 4, P, ctypes.byref(_c_levels(EDGE, n_levels=17)), P, N), b"n_levels must be in 1..16"),
        ("offset not a multiple of 8", lambda: l.mcs_hashgrid_fwd(P, 4, P, ctypes.byref(_c_levels(EDGE, offset=(2, 580))), P, N), b"multiple of 8"),
        ("decreasing offsets", lambda: l.mcs_hashgrid_fwd(P, 4, P, ctypes.byref(_c_levels(EDGE, offset=(2, 8))), P, N), b"not increasing"),
        ("empty level", lambda: l.mcs_hashgrid_fwd(P, 4, P, ctypes.byref(_c_levels(EDGE, offset=(2, 64))), P, N), b"size 0"),
        ("misaligned params", lambda: l.mcs_hashgrid_fwd(P, 4, ctypes.c_void_p(260), ctypes.byref(good), P, N), b"8-byte aligned"),
        ("bwd null d_out", lambda: l.mcs_hashgrid_bwd(P, 4, P, ctypes.byref(good), N, P, P, N), b"null pointer"),
        ("bwd no gradient", lambda: l.mcs_hashgrid_bwd(P, 4, P, ctypes.byref(good), P, N, N, N), b"both null"),
        ("bwd n < 0", lambda: l.mcs_hashgrid_bwd(P, -3, P, ctypes.byref(good), P, P, N, N), b"n must be >= 0"),
        ("bwd 17 levels", lambda: l.mcs_hashgrid_bwd(P, 4, P, ctypes.byref(_c_levels(EDGE, n_levels=17)), P, P, P, N), b"n_levels"),
    ]
    for name, call, frag in bad:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0, name
        assert frag in msg, (name, msg)
    # n = 0 succeeds without launching anything
    assert l.mcs_hashgrid_fwd(P, 0, P, ctypes.byref(good), P, N) == 0
    assert l.mcs_hashgrid_bwd(P, 0, P, ctypes.byref(good), P, P, P, N) == 0


@pytest.mark.parametrize("n_input_dims, change", [
    (3, {"otype": "Frequency"}), (3, {"otype": "DenseGrid"}), (2, {}), (3, {"n_features_per_level": 4}),
    (3, {"interpolation": "Smoothstep"}), (3, {"n_levels": 0}), (3, {"n_levels": 17}), (3, {"per_level_scale": float("nan")}),
    (3, {"base_resolution": -1}), (3, {"log2_hashmap_size": 40})])
def test_unsupported_configs_raise_value_error(n_input_dims, change):
    from nvdiffrecmc_b200.tinycudann import Encoding
    with pytest.raises(ValueError):
        Encoding(n_input_dims, dict(REF_CONFIG, **change))


def test_unsupported_dtype_raises_value_error():
    import torch
    from nvdiffrecmc_b200.tinycudann import Encoding
    with pytest.raises(ValueError, match="fp32"):
        Encoding(3, REF_CONFIG, dtype=torch.float16)


@pytest.mark.skipif(not HAVE_REF, reason="the reference checkout is only present in the build container")
def test_reference_mlptexture_imports_with_this_package_as_tinycudann():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_mlptexture_golden
    import nvdiffrecmc_b200.tinycudann as ours
    with make_mlptexture_golden.reference_mlptexture(ours) as mod:
        assert mod.tcnn is ours
        assert callable(mod.MLPTexture3D)


@pytest.mark.skipif(not HAVE_REF, reason="the reference checkout is only present in the build container")
def test_mlptexture_golden_regenerates_bit_identically():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_mlptexture_golden
    g = make_mlptexture_golden.generate()
    d = np.load(os.path.join(HERE, "golden", "ref_mlptexture.npz"))
    assert sorted(g) == sorted(d.files)
    for k in d.files:
        assert g[k].dtype == d[k].dtype and np.array_equal(g[k], d[k]), k
