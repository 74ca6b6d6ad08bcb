"""CPU: the MLP texture's contract (csrc/mlptexture.cu) as the oracle restates it -- the fixed exp, the fp64 adjoints against finite
differences, the fp32 oracle against the reference's own MLPTexture3D (tests/golden/ref_mlptexture.npz) -- the C ABI's argument checks
and the drop-in's configuration checks, all without a GPU; where the reference checkout exists, the drop-in's constructor signature and
the reference instance's state_dict layout."""
import ctypes
import inspect
import os
import re
import sys

import numpy as np
import pytest

from common import rel_l2
from oracle import REAL
from oracle.hashgrid import REF_CONFIG, init_params
from oracle.mlptexture import SOURCES, MlpTextureOracle, mlptexture_oracle
from nvdiffrecmc_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
HAVE_REF = os.path.exists("/root/reference/render/mlptexture.py")
SMALL = {"otype": "HashGrid", "n_levels": 16, "log2_hashmap_size": 7, "base_resolution": 2, "per_level_scale": 1.3}
# the state_dict layout of the reference's MLPTexture3D(channels=6) (hidden 2); tests/test_gpu_mlptexture.py checks the drop-in against it
REF_STATE = {"encoder.params": (12599920,), "net.net.0.weight": (32, 32), "net.net.2.weight": (32, 32), "net.net.4.weight": (6, 32)}


def test_signature_table_names_exactly_the_exports():
    """Every function oracle/mlptexture.c exports (its own and those of the hashgrid.c it includes) has a declared signature, and the
    library loads once per precision with it."""
    names = []
    for src in SOURCES:
        text = re.sub(r"/\*.*?\*/", "", open(src).read(), flags=re.S)
        names += re.findall(r"^(?!static\b)[A-Za-z_][\w \*]*?\b((?:hg|mlt)_\w+)\s*\([^;{]*\)\s*\{", text, re.M)
    assert len(names) >= 7 and sorted(MlpTextureOracle.SIGS) == sorted(names)
    for f64 in (False, True):
        o = mlptexture_oracle(f64)
        assert o is mlptexture_oracle(f64) and o.f64 == f64
        for name, (args, res) in MlpTextureOracle.SIGS.items():
            fn = getattr(o.lib, name)
            assert fn.restype is res and list(fn.argtypes) == [o.real if a is REAL else a for a in args], name


def _ulp_distance(a, b):
    """|a - b| in float32 ulps (both finite, same sign convention by integer ordering)."""
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_exp_is_within_2_ulp_of_double_exp():
    o = mlptexture_oracle()
    x = np.concatenate([np.linspace(-104, 89, 2_000_001, dtype=np.float32),
                        np.float32(88.72283935546875) - np.arange(64, dtype=np.float32) * np.float32(7.62939453125e-06)])
    y = o.exp(x)
    with np.errstate(over="ignore"):
        ref = np.exp(x.astype(np.float64)).astype(np.float32)      # exp rounded twice (double, then fp32): within 1 ulp of exp
    assert np.array_equal(np.isinf(y), np.isinf(ref))
    fin = np.isfinite(ref)
    assert _ulp_distance(y[fin], ref[fin]).max() <= 2
    assert o.exp(np.float32(0.0))[()] == 1.0
    assert o.exp(np.float32(89.0))[()] == np.inf and o.exp(np.float32(np.inf))[()] == np.inf
    assert o.exp(np.float32(-104.0))[()] == 0.0 and o.exp(np.float32(-np.inf))[()] == 0.0
    assert np.isnan(o.exp(np.float32(np.nan))[()])


def _texture(rng, C, hidden, lv, scale=0.5):
    params = rng.uniform(-1, 1, 2 * int(lv["offset"][-1]))
    ws = [rng.normal(0, scale, (32, 32)) for _ in range(hidden)] + [rng.normal(0, scale, (C, 32))]
    aabb = np.array([[-1.0, -0.5, -0.8], [1.1, 0.9, 0.7]])
    mm = np.stack([rng.uniform(-0.5, 0.2, C), rng.uniform(0.5, 1.5, C)])
    return params, ws, aabb, mm


def _clean_points(o, rng, n, lv, aabb, params, ws, mm):
    """Points well inside the AABB, away from every level's cell faces and every ReLU kink (|pre-activation| > 1e-3)."""
    x = rng.uniform(0.05, 0.95, (n * 8, 3))
    ok = np.ones(len(x), bool)
    for s in lv["scale"]:
        p = float(s) * x + 0.5
        f = p - np.floor(p)
        ok &= np.all((f > 1e-3) & (f < 1 - 1e-3), axis=1)
    x = x[ok]
    t = aabb[0] + x * (aabb[1] - aabb[0])
    _, e = o.mlptex_forward(t, aabb, mm, params, lv, ws)
    v, keep = e, np.ones(len(t), bool)
    for w in ws[:-1]:
        pre = v @ w.T
        keep &= np.all(np.abs(pre) > 1e-3, axis=1)
        v = np.maximum(pre, 0)
    return t[keep][:n]


@pytest.mark.parametrize("C,hidden", [(3, 1), (6, 2), (2, 4)])
def test_fp64_oracle_agrees_with_finite_differences(C, hidden):
    o = mlptexture_oracle(f64=True)
    lv = o.levels(SMALL)
    rng = np.random.default_rng(C * 10 + hidden)
    params, ws, aabb, mm = _texture(rng, C, hidden, lv)
    t = _clean_points(o, rng, 40, lv, aabb, params, ws, mm)
    assert len(t) >= 20
    g = rng.normal(size=(len(t), C))
    f = lambda tt=t, pp=params, ww=ws: float((o.mlptex_forward(tt, aabb, mm, pp, lv, ww)[0] * g).sum())
    dp, dt, dw = o.mlptex_backward(t, aabb, mm, params, lv, ws, g)
    h = 1e-6
    fd = np.zeros_like(t)
    for d in range(3):
        e = np.zeros(3); e[d] = h
        fd[:, d] = [(f(t + np.where(np.arange(len(t))[:, None] == i, e, 0)) - f(t - np.where(np.arange(len(t))[:, None] == i, e, 0))) / (2 * h)
                    for i in range(len(t))]
    assert np.abs(dt - fd).max() <= 1e-6 * max(1.0, np.abs(fd).max())
    for l, w in enumerate(ws):
        for (j, k) in [(0, 0), (w.shape[0] - 1, 31), (w.shape[0] // 2, 7)]:
            wp, wm = [x.copy() for x in ws], [x.copy() for x in ws]
            wp[l][j, k] += h; wm[l][j, k] -= h
            num = (f(ww=wp) - f(ww=wm)) / (2 * h)
            assert abs(dw[l][j, k] - num) <= 1e-6 * max(1.0, abs(num)), (l, j, k)
    nz = np.nonzero(dp)[0]
    for q in rng.choice(nz, 12, replace=False):
        pp, pm = params.copy(), params.copy()
        pp[q] += h; pm[q] -= h
        num = (f(pp=pp) - f(pp=pm)) / (2 * h)
        assert abs(dp[q] - num) <= 1e-6 * max(1.0, abs(num)), q


def test_fp32_oracle_reproduces_the_reference_mlptexture():
    """ref_mlptexture.npz is the reference's own MLPTexture3D with its hooks: x128 on d params, d points and d W unscaled."""
    d = np.load(os.path.join(HERE, "golden", "ref_mlptexture.npz"))
    o = mlptexture_oracle()
    lv = o.levels(REF_CONFIG)
    p = init_params(2 * int(lv["offset"][-1]))
    assert np.array_equal(p[:8], d["params_head"])
    ws = [d["w0"], d["w1"], d["w2"]]
    out, _ = o.mlptex_forward(d["points"], d["aabb"], d["min_max"], p, lv, ws)
    assert rel_l2(out.reshape(d["out"].shape), d["out"]) <= 1e-5
    dp, dt, dw = o.mlptex_backward(d["points"], d["aabb"], d["min_max"], p, lv, ws, d["dout"])
    assert rel_l2(dt.reshape(d["d_points"].shape), d["d_points"]) <= 1e-4
    for k in range(3):
        assert rel_l2(dw[k], d["d_w%d" % k]) <= 1e-4, k
    ref = np.zeros_like(p)
    ref[d["params_grad_idx"]] = d["params_grad_val"]
    assert rel_l2(dp * 128, ref) <= 1e-4


def test_entry_points_reject_bad_arguments_without_a_device():
    from nvdiffrecmc_b200.tinycudann import _c_levels, level_table
    l = _lib.lib()
    N = None
    P = ctypes.c_void_p(256)              # never dereferenced: validation fails first
    lv = _c_levels(level_table(16, 19, 16, REF_CONFIG["per_level_scale"]))
    lv8 = _c_levels(level_table(8, 19, 16, 2.0))
    W = (ctypes.c_void_p * 5)(256, 256, 256, 256, 256)
    W0 = (ctypes.c_void_p * 5)(256, None, 256, 256, 256)
    D = (ctypes.c_void_p * 5)(256, 256, 256, 256, 256)
    Dn = (ctypes.c_void_p * 5)()
    by = ctypes.byref
    fwd = lambda t=P, n=4, aabb=P, mm=P, p=P, lvv=lv, h=2, C=6, w=W, out=P, enc=P: l.mcs_mlptex_fwd(t, n, aabb, mm, p, by(lvv) if lvv else N, h, C,
                                                                                                   w, out, enc, N)
    bwd = lambda t=P, n=4, p=P, h=2, C=6, w=W, enc=P, g=P, dp=P, dt=P, dw=D, ws=P: l.mcs_mlptex_bwd(t, n, P, P, p, by(lv), h, C, w, enc, g, dp, dt, dw,
                                                                                                  ws, N)
    bad = [
        ("null t", lambda: fwd(t=N), b"null pointer"),
        ("null aabb", lambda: fwd(aabb=N), b"null pointer"),
        ("null min_max", lambda: fwd(mm=N), b"null pointer"),
        ("null params", lambda: fwd(p=N), b"null pointer"),
        ("null levels", lambda: fwd(lvv=None), b"null pointer"),
        ("null weight", lambda: fwd(w=W0), b"weights[1]"),
        ("null out", lambda: fwd(out=N), b"null pointer"),
        ("n < 0", lambda: fwd(n=-1), b"n must be >= 0"),
        ("hidden 0", lambda: fwd(h=0), b"hidden must be in 1..4"),
        ("hidden 5", lambda: fwd(h=5), b"hidden must be in 1..4"),
        ("channels 0", lambda: fwd(C=0), b"channels must be in 1..8"),
        ("channels 9", lambda: fwd(C=9), b"channels must be in 1..8"),
        ("8 levels", lambda: fwd(lvv=lv8), b"16 levels"),
        ("misaligned params", lambda: fwd(p=ctypes.c_void_p(260)), b"8-byte aligned"),
        ("misaligned enc", lambda: fwd(enc=ctypes.c_void_p(264)), b"16-byte aligned"),
        ("bwd null enc", lambda: bwd(enc=N), b"null pointer"),
        ("bwd null d_out", lambda: bwd(g=N), b"null pointer"),
        ("bwd no gradient", lambda: bwd(dp=N, dt=N, dw=Dn), b"no gradient requested"),
        ("bwd null workspace", lambda: bwd(ws=N), b"workspace"),
        ("bwd misaligned workspace", lambda: bwd(ws=ctypes.c_void_p(260)), b"16-byte aligned"),
        ("bwd misaligned d_params", lambda: bwd(dp=ctypes.c_void_p(260)), b"8-byte aligned"),
        ("bwd n < 0", lambda: bwd(n=-3), b"n must be >= 0"),
        ("bwd hidden 5", lambda: bwd(h=5), b"hidden"),
    ]
    for name, call, frag in bad:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0, name
        assert frag in msg, (name, msg)
    assert fwd(n=0) == 0 and fwd(n=0, enc=N) == 0
    assert bwd(n=0, dw=Dn) == 0
    assert l.mcs_mlptex_workspace_bytes(1025, 2, 6) == 2 * (2 * 1024 + 6 * 32) * 4
    assert l.mcs_mlptex_workspace_bytes(0, 2, 6) == 0 and l.mcs_mlptex_workspace_bytes(4, 5, 6) < 0


@pytest.mark.parametrize("kw", [{"internal_dims": 64}, {"hidden": 0}, {"hidden": 5}, {"channels": 0}, {"channels": 9}])
def test_unsupported_configs_raise_value_error(kw):
    from nvdiffrecmc_b200.mlptexture import MLPTexture3D
    with pytest.raises(ValueError, match="supported: internal_dims 32, hidden 1..4, channels 1..8"):
        MLPTexture3D(np.zeros((2, 3), np.float32), **kw)


@pytest.mark.skipif(not HAVE_REF, reason="the reference checkout is only present in the build container")
def test_constructor_signature_and_state_dict_layout_equal_the_reference():
    import torch
    from nvdiffrecmc_b200.mlptexture import MLPTexture3D
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_mlptexture_golden
    with make_mlptexture_golden.reference_mlptexture(make_mlptexture_golden.oracle_tinycudann()) as mt:
        assert inspect.signature(MLPTexture3D.__init__) == inspect.signature(mt.MLPTexture3D.__init__)
        ref = mt.MLPTexture3D(torch.tensor([[0.0] * 3, [1.0] * 3]), channels=6, min_max=[torch.zeros(6), torch.ones(6)])
        assert {k: tuple(v.shape) for k, v in ref.state_dict().items()} == REF_STATE
