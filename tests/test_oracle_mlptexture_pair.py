"""CPU: MLPTexture3D.sample_pair's contract as the oracle states it -- two single calls and one add -- checked against those calls bit for
bit (fp32), against finite differences (fp64) and against the reference's render.py:63-64 (tests/golden/ref_mlptexture_pair.npz); and the
pair entry points' argument checks without a device."""
import ctypes
import os

import numpy as np
import pytest

from common import rel_l2
from oracle.hashgrid import REF_CONFIG, init_params
from oracle.mlptexture import mlptexture_oracle
from mlptexture_pair_oracle import pair_backward, pair_forward
from nvdiffrecmc_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
SMALL = {"otype": "HashGrid", "n_levels": 16, "log2_hashmap_size": 7, "base_resolution": 2, "per_level_scale": 1.3}
AABB = np.array([[-1.0, -0.5, -0.8], [1.1, 0.9, 0.7]])


def _texture(rng, C, hidden, lv, scale=0.5):
    params = rng.uniform(-1, 1, 2 * int(lv["offset"][-1]))
    ws = [rng.normal(0, scale, (32, 32)) for _ in range(hidden)] + [rng.normal(0, scale, (C, 32))]
    mm = np.stack([rng.uniform(-0.5, 0.2, C), rng.uniform(0.5, 1.5, C)])
    return params, ws, mm


@pytest.mark.parametrize("C,hidden", [(1, 1), (6, 2), (8, 4)])
def test_fp32_pair_is_two_calls_and_one_add(C, hidden):
    o = mlptexture_oracle()
    lv = o.levels(REF_CONFIG)
    rng = np.random.default_rng(C + hidden)
    params, ws, mm = _texture(rng, C, hidden, lv)
    n = 700
    t = (AABB[0] + rng.uniform(-0.2, 1.2, (n, 3)) * (AABB[1] - AABB[0])).astype(np.float32)
    off = rng.normal(0, 0.01, (n, 3)).astype(np.float32)
    off[::7] = 0.0
    g, gj = rng.normal(size=(n, C)).astype(np.float32), rng.normal(size=(n, C)).astype(np.float32)
    tj = t + off
    assert tj.dtype == np.float32
    out, enc = o.mlptex_forward(t, AABB, mm, params, lv, ws)
    out_j, enc_j = o.mlptex_forward(tj, AABB, mm, params, lv, ws)
    for a, b in zip(pair_forward(o, t, off, AABB, mm, params, lv, ws), (out, enc, out_j, enc_j)):
        assert a.dtype == np.float32 and np.array_equal(a, b)
    dp, dt, dw = o.mlptex_backward(t, AABB, mm, params, lv, ws, g)
    dpj, dtj, dwj = o.mlptex_backward(tj, AABB, mm, params, lv, ws, gj)
    p_dp, p_dt, p_do, p_dw = pair_backward(o, t, off, AABB, mm, params, lv, ws, g, gj)
    assert np.array_equal(p_dt, dt + dtj) and np.array_equal(p_do, dtj)
    assert np.array_equal(p_dp, dp + dpj)
    for a, x, y in zip(p_dw, dw, dwj):
        assert a.dtype == np.float32 and np.array_equal(a, x + y)
    q = pair_backward(o, t, off, AABB, mm, params, lv, ws, g, gj, want_params=False, want_t=False, want_w=False)
    assert q[0] is None and q[1] is None and q[3] is None and np.array_equal(q[2], dtj)


def test_fp64_pair_gradients_agree_with_finite_differences():
    o = mlptexture_oracle(f64=True)
    lv = o.levels(SMALL)
    rng = np.random.default_rng(5)
    C = 3
    params, ws, mm = _texture(rng, C, 2, lv)
    # points well inside the AABB whose plain and jittered points are away from every level's cell faces and every ReLU kink
    x = rng.uniform(0.05, 0.95, (400, 3))
    off = rng.normal(0, 0.01, (400, 3))
    ok = np.ones(len(x), bool)
    for xx in (x, x + off / (AABB[1] - AABB[0])):
        for s in lv["scale"]:
            f = float(s) * xx + 0.5
            f = f - np.floor(f)
            ok &= np.all((f > 1e-3) & (f < 1 - 1e-3), axis=1)
        v = o.mlptex_forward(AABB[0] + xx * (AABB[1] - AABB[0]), AABB, mm, params, lv, ws)[1]
        for w in ws[:-1]:
            pre = v @ w.T
            ok &= np.all(np.abs(pre) > 1e-3, axis=1)
            v = np.maximum(pre, 0)
    t = (AABB[0] + x * (AABB[1] - AABB[0]))[ok][:25]
    off = off[ok][:25]
    assert len(t) >= 20
    g, gj = rng.normal(size=(len(t), C)), rng.normal(size=(len(t), C))

    def f(tt, oo):
        out, _, out_j, _ = pair_forward(o, tt, oo, AABB, mm, params, lv, ws)
        return float((out * g).sum() + (out_j * gj).sum())

    _, dt, do, _ = pair_backward(o, t, off, AABB, mm, params, lv, ws, g, gj)
    h = 1e-6
    for grad, wrt in ((dt, 0), (do, 1)):
        fd = np.zeros_like(t)
        for i in range(len(t)):
            for d in range(3):
                e = np.zeros_like(t); e[i, d] = h
                args_p = (t + e, off) if wrt == 0 else (t, off + e)
                args_m = (t - e, off) if wrt == 0 else (t, off - e)
                fd[i, d] = (f(*args_p) - f(*args_m)) / (2 * h)
        assert np.abs(grad - fd).max() <= 1e-6 * max(1.0, np.abs(fd).max()), wrt


def test_fp32_oracle_reproduces_the_reference_pair():
    """ref_mlptexture_pair.npz is render.py:63-64 run on the reference's own MLPTexture3D with its hooks, with the bars of
    test_oracle_mlptexture.py."""
    d = np.load(os.path.join(HERE, "golden", "ref_mlptexture_pair.npz"))
    o = mlptexture_oracle()
    lv = o.levels(REF_CONFIG)
    p = init_params(2 * int(lv["offset"][-1]))
    assert np.array_equal(p[:8], d["params_head"])
    ws = [d["w0"], d["w1"], d["w2"]]
    out, _, out_j, _ = pair_forward(o, d["gb_pos"], d["noise"], d["aabb"], d["min_max"], p, lv, ws)
    assert rel_l2(out.reshape(d["out"].shape), d["out"]) <= 1e-5
    assert rel_l2(out_j.reshape(d["out_jit"].shape), d["out_jit"]) <= 1e-5
    dp, dt, _, dw = pair_backward(o, d["gb_pos"], d["noise"], d["aabb"], d["min_max"], p, lv, ws, d["dout"], d["dout_jit"])
    assert rel_l2(dt.reshape(d["d_gb_pos"].shape), d["d_gb_pos"]) <= 1e-4
    for k in range(3):
        assert rel_l2(dw[k], d["d_w%d" % k]) <= 1e-4, k
    ref = np.zeros_like(p)
    ref[d["params_grad_idx"]] = d["params_grad_val"]
    assert rel_l2(dp * 128, ref) <= 1e-4


def test_pair_entry_points_reject_bad_arguments_without_a_device():
    from nvdiffrecmc_b200.tinycudann import _c_levels, level_table
    l = _lib.lib()
    N = None
    P = ctypes.c_void_p(256)              # never dereferenced: validation fails first
    lv = _c_levels(level_table(16, 19, 16, REF_CONFIG["per_level_scale"]))
    W = (ctypes.c_void_p * 5)(256, 256, 256, 256, 256)
    D = (ctypes.c_void_p * 5)(256, 256, 256, 256, 256)
    Dn = (ctypes.c_void_p * 5)()
    by = ctypes.byref
    fwd = lambda t=P, off=P, n=4, h=2, C=6, out=P, oj=P, enc=P, ej=P: l.mcs_mlptex_pair_fwd(t, off, n, P, P, P, by(lv), h, C, W, out, oj, enc,
                                                                                           ej, N)
    bwd = lambda off=P, n=4, enc=P, ej=P, g=P, gj=P, dp=P, dt=P, do=P, dw=D, ws=P: l.mcs_mlptex_pair_bwd(P, off, n, P, P, P, by(lv), 2, 6, W,
                                                                                                        enc, ej, g, gj, dp, dt, do, dw, ws, N)
    bad = [
        ("null t", lambda: fwd(t=N), b"null pointer"),
        ("null offset", lambda: fwd(off=N), b"null pointer (offset)"),
        ("null out", lambda: fwd(out=N), b"null pointer (out / out_jit)"),
        ("null out_jit", lambda: fwd(oj=N), b"null pointer (out / out_jit)"),
        ("misaligned enc_jit", lambda: fwd(ej=ctypes.c_void_p(264)), b"16-byte aligned"),
        ("hidden 5", lambda: fwd(h=5), b"hidden must be in 1..4"),
        ("channels 9", lambda: fwd(C=9), b"channels must be in 1..8"),
        ("n < 0", lambda: fwd(n=-1), b"n must be >= 0"),
        ("bwd null offset", lambda: bwd(off=N), b"null pointer (offset)"),
        ("bwd null enc", lambda: bwd(enc=N), b"null pointer (enc / enc_jit)"),
        ("bwd null enc_jit", lambda: bwd(ej=N), b"null pointer (enc / enc_jit)"),
        ("bwd misaligned enc_jit", lambda: bwd(ej=ctypes.c_void_p(264)), b"16-byte aligned"),
        ("bwd no gradient", lambda: bwd(dp=N, dt=N, do=N, dw=Dn), b"no gradient requested"),
        ("bwd null workspace", lambda: bwd(ws=N), b"workspace"),
        ("bwd misaligned workspace", lambda: bwd(ws=ctypes.c_void_p(260)), b"16-byte aligned"),
        ("bwd misaligned d_params", lambda: bwd(dp=ctypes.c_void_p(260)), b"8-byte aligned"),
    ]
    for name, call, frag in bad:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0, name
        assert frag in msg, (name, msg)
    assert fwd(n=0) == 0 and fwd(n=0, enc=N, ej=N) == 0
    assert bwd(n=0, dw=Dn) == 0 and bwd(n=0, dw=Dn, g=N, gj=N) == 0
    assert bwd(n=0, dp=N, dt=N, dw=Dn) == 0                     # d offset alone is a gradient


def test_sample_pair_raises_value_errors_before_any_launch():
    import torch
    from nvdiffrecmc_b200.mlptexture import MLPTexture3D
    tex = MLPTexture3D.__new__(MLPTexture3D)          # the argument checks run before anything touches the device
    torch.nn.Module.__init__(tex)
    _lib.LAUNCHES.clear()
    for texc, off, frag in [(torch.zeros(4, 3), torch.zeros(5, 3), "differ in shape"),
                            (torch.zeros(4, 2), torch.zeros(4, 2), r"\[\.\.\., 3\]"),
                            (torch.zeros(4, 3, dtype=torch.int32), torch.zeros(4, 3), "texc must be a floating-point"),
                            (torch.zeros(4, 3), torch.zeros(4, 3, dtype=torch.int64), "offset must be a floating-point"),
                            (torch.zeros(4, 3), torch.zeros(4, 3, device="meta"), "offset is on meta")]:
        with pytest.raises(ValueError, match=frag):
            tex.sample_pair(texc, off)
    assert not _lib.LAUNCHES
