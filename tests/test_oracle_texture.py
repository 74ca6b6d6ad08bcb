"""CPU: the filtered texture look-up's oracle (adjoints by finite differences and the adjoint identity, fp32 against fp64, the
deterministic log2, agreement with torch grid_sample, the level of detail at integer levels and at zero derivatives, non-finite and
huge uv), the C ABI's argument checks and the Python interface's ValueErrors (all without a GPU); in the build container, the frozen
output of the reference's Texture2D / EnvironmentLight regenerates bit for bit."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from oracle.texture import chain_shapes, texture_oracle
from nvdiffrecmc_b200 import _lib
from nvdiffrecmc_b200.raster import texture

HERE = os.path.dirname(os.path.abspath(__file__))
HAVE_REF = os.path.exists("/root/reference/render/texture.py")
LML = "linear-mipmap-linear"


def _chain(rng, H, W, C, n_levels, Bt=1):
    return [rng.normal(size=(Bt, h, w, C)) for h, w in chain_shapes(H, W, n_levels)]


def _fracs_ok(uv, levels, margin):
    """pixels whose bilinear fractions stay `margin` away from texel boundaries on every level"""
    ok = np.ones(uv.shape[:3], bool)
    for t in levels:
        for d, n in ((0, t.shape[2]), (1, t.shape[1])):
            x = uv[..., d] * n - 0.5
            f = x - np.floor(x)
            ok &= (f > margin) & (f < 1 - margin)
    return ok


def _lam(da, W0, H0):
    a, b, c, d = da[..., 0] * W0, da[..., 1] * W0, da[..., 2] * H0, da[..., 3] * H0
    A, B, C = a * a + c * c, b * b + d * d, a * b + c * d
    M = (A + B) / 2 + np.sqrt(((A - B) / 2) ** 2 + C * C)
    with np.errstate(divide="ignore"):
        return 0.5 * np.log2(M)


def _case(seed, B=2, h=6, w=7, H=24, W=40, C=3, n_levels=5, Bt=1):
    """fp64 inputs whose fractions and lambda stay away from the non-differentiable points; lambda spans every level"""
    rng = np.random.default_rng(seed)
    levels = _chain(rng, H, W, C, n_levels, Bt)
    uv = rng.uniform(-0.4, 1.4, (B, h, w, 2))
    # general (anisotropic, sheared) footprints of about 2^s texels, s in [-1, L + 1]
    s = rng.uniform(-1, n_levels, (B, h, w))
    J = rng.normal(size=(B, h, w, 4)) * (2.0 ** s)[..., None]
    da = J / np.array([W, W, H, H])
    return levels, uv, da


def test_fp64_d_uv_and_d_uv_da_match_finite_differences():
    o = texture_oracle(f64=True)
    for boundary in ("wrap", "clamp"):
        levels, uv, da = _case(1)
        L = len(levels) - 1
        lam = _lam(da, 40, 24)
        keep = _fracs_ok(uv, levels, 0.02) & (np.abs(lam - np.round(lam)) > 0.02) & (np.abs(lam) > 0.02)
        g = np.random.default_rng(2).normal(size=uv.shape[:3] + (3,))
        _, duv, dda = o.backward(levels, uv, da, g, LML, boundary)
        h = 1e-7
        f = lambda u, d: (o.forward(levels, u, d, LML, boundary) * g).sum(-1)
        for k in range(2):
            e = np.zeros(2); e[k] = h
            fd = (f(uv + e, da) - f(uv - e, da)) / (2 * h)
            assert np.abs(duv[..., k] - fd)[keep].max() <= 1e-6 * np.abs(fd[keep]).max(), (boundary, k)
        inner = keep & (lam > 0.02) & (lam < L - 0.02)
        for k in range(4):
            e = np.zeros(4); e[k] = h * np.abs(da[..., k]).max()
            fd = (f(uv, da + e) - f(uv, da - e)) / (2 * e[k])
            assert np.abs(dda[..., k] - fd)[inner].max() <= 1e-5 * np.abs(fd[inner]).max(), (boundary, k)
            assert np.abs(fd[inner]).max() > 0
        assert inner.sum() >= 20 and (lam[keep] > L).any() and (lam[keep] < 0).any()
        assert np.all(dda[~inner & keep & ((lam < 0) | (lam > L))] == 0)


@pytest.mark.parametrize("boundary", ["wrap", "clamp"])
@pytest.mark.parametrize("Bt", [1, 2])
def test_fp64_adjoint_identity_per_level(boundary, Bt):
    """The look-up is linear in the texels: <d tex_k, T_k> = <g, out(T with only level k)> for every level k."""
    o = texture_oracle(f64=True)
    levels, uv, da = _case(3, Bt=Bt)
    g = np.random.default_rng(4).normal(size=uv.shape[:3] + (3,))
    g[0, ::2] = 0
    dt, _, _ = o.backward(levels, uv, da, g, LML, boundary)
    for k, t in enumerate(levels):
        only = [x if j == k else np.zeros_like(x) for j, x in enumerate(levels)]
        rhs = float((g * o.forward(only, uv, da, LML, boundary)).sum())
        assert abs(float((dt[k] * t).sum()) - rhs) <= 1e-12 * max(1.0, abs(rhs)), k


def test_fp32_oracle_agrees_with_fp64():
    o32, o64 = texture_oracle(), texture_oracle(f64=True)
    rl2 = lambda a, b: np.linalg.norm(a - b) / np.linalg.norm(b)
    levels, uv, da = _case(5, C=4)
    uv = uv[_fracs_ok(uv, levels, 0.01)][None, None]
    lam = _lam(_case(5, C=4)[2], 40, 24)
    da = _case(5, C=4)[2][_fracs_ok(_case(5, C=4)[1], levels, 0.01)][None, None]
    g = np.random.default_rng(6).normal(size=uv.shape[:3] + (4,))
    for boundary in ("wrap", "clamp"):
        assert rl2(o32.forward(levels, uv, da, LML, boundary), o64.forward(levels, uv, da, LML, boundary)) <= 1e-5
        a, b = o32.backward(levels, uv, da, g, LML, boundary), o64.backward(levels, uv, da, g, LML, boundary)
        for k in range(len(levels)):
            if np.any(b[0][k]):
                assert rl2(a[0][k], b[0][k]) <= 1e-5, k
        assert rl2(a[1], b[1]) <= 1e-4 and rl2(a[2], b[2]) <= 1e-4
    assert lam.size


def test_deterministic_log2_against_double():
    """Within 1.5 ulp of the correctly rounded result over normal and subnormal arguments; exact at powers of two."""
    o = texture_oracle()
    rng = np.random.default_rng(0)
    x = (rng.uniform(0.5, 1.0, 100000) * 2.0 ** rng.integers(-148, 128, 100000)).astype(np.float32)
    x = np.concatenate([x[np.isfinite(x) & (x > 0)], np.linspace(0.5, 2.0, 50001, dtype=np.float32)])
    ref = np.log2(x.astype(np.float64))
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    assert (np.abs(o.log2(x).astype(np.float64) - ref) / ulp).max() <= 1.5
    p = np.float32(2.0) ** np.arange(-149, 128).astype(np.float32)
    assert np.array_equal(o.log2(p), np.arange(-149, 128).astype(np.float32))
    s = o.log2(np.array([0.0, np.inf, -1.0, np.nan], np.float32))
    assert s[0] == -np.inf and s[1] == np.inf and np.isnan(s[2]) and np.isnan(s[3])


def test_linear_matches_grid_sample():
    """clamp == grid_sample(bilinear, border, align_corners=False); wrap == grid_sample on a circularly padded texture."""
    o = texture_oracle()
    rng = np.random.default_rng(7)
    tex = rng.normal(size=(2, 9, 13, 3)).astype(np.float32)
    uv = rng.uniform(-0.3, 1.3, (2, 8, 10, 2)).astype(np.float32)
    gs = lambda t, u, pad: torch.nn.functional.grid_sample(torch.from_numpy(t).permute(0, 3, 1, 2), torch.from_numpy(u) * 2 - 1, mode="bilinear",
                                                           padding_mode=pad, align_corners=False).permute(0, 2, 3, 1).numpy()
    assert np.abs(o.forward([tex], uv, None, "linear", "clamp") - gs(tex, uv, "border")).max() <= 1e-5
    uvw = rng.uniform(0, 1, (2, 8, 10, 2)).astype(np.float32)
    padded = np.pad(tex, ((0, 0), (1, 1), (1, 1), (0, 0)), mode="wrap")
    uvp = ((uvw.astype(np.float64) * [13, 9] + 1) / [15, 11]).astype(np.float32)
    assert np.abs(o.forward([tex], uvw, None, "linear", "wrap") - gs(padded, uvp, "zeros")).max() <= 1e-5
    # wrap is periodic: shifting uv by whole textures picks the same texels
    assert np.abs(o.forward([tex], uvw + 3, None, "linear", "wrap") - o.forward([tex], uvw, None, "linear", "wrap")).max() <= 1e-5


def test_integer_lambda_gives_that_level_and_zero_derivatives_give_level_0():
    o = texture_oracle()
    rng = np.random.default_rng(8)
    levels = [t.astype(np.float32) for t in _chain(rng, 32, 64, 2, 6)]
    uv = rng.uniform(0, 1, (1, 4, 5, 2)).astype(np.float32)
    g = rng.normal(size=(1, 4, 5, 2)).astype(np.float32)
    for k in range(6):
        da = np.zeros((1, 4, 5, 4), np.float32)
        da[..., 0] = np.float32(2.0 ** k / 64)             # a = 2^k texels, M = 4^k, lambda = k exactly
        for boundary in ("wrap", "clamp"):
            out = o.forward(levels, uv, da, LML, boundary)
            assert np.array_equal(out, o.forward([levels[k]], uv, None, "linear", boundary)), k
            dt, duv, dda = o.backward(levels, uv, da, g, LML, boundary)
            assert not np.any(dda) and all(not np.any(dt[j]) for j in range(6) if j != k)
    da = np.zeros((1, 4, 5, 4), np.float32)
    out = o.forward(levels, uv, da, LML, "wrap")
    assert np.array_equal(out, o.forward(levels[:1], uv, None, "linear", "wrap"))
    dt, duv, dda = o.backward(levels, uv, da, g, LML, "wrap")
    assert np.all(dda == 0) and np.all(np.isfinite(duv)) and not any(np.any(t) for t in dt[1:])


def test_non_finite_and_huge_uv_stay_in_bounds():
    """Every tap is clamped or wrapped into the level, so an out-of-range read cannot happen: finite huge uv give a convex combination of
    texels, and NaN / Inf uv and uv_da return (values unspecified) without touching memory outside the levels."""
    o = texture_oracle()
    rng = np.random.default_rng(9)
    levels = [t.astype(np.float32) for t in _chain(rng, 5, 7, 3, 3)]
    special = np.array([np.nan, np.inf, -np.inf, 3e9, -3e9, 1e38, -1e38, 2.0 ** 31, -(2.0 ** 31), 0.5], np.float32)
    uv = np.stack(np.meshgrid(special, special, indexing="ij"), -1)[None]
    da = np.broadcast_to(np.array([np.nan, np.inf, 1e30, 0.0], np.float32)[[0, 1, 2, 3]], uv.shape[:3] + (4,)).copy()
    da[0, ::2] = 0
    finite = (np.abs(uv) <= 3e9).all(-1)               # u * W stays finite in fp32 (1e38 * 7 does not)
    lo, hi = min(t.min() for t in levels), max(t.max() for t in levels)
    for boundary in ("wrap", "clamp"):
        out = o.forward(levels, uv, da, LML, boundary)
        o.backward(levels, uv, da, np.ones_like(out), LML, boundary)
        lin = o.forward(levels, uv, None, "linear", boundary)
        assert np.all((lin[finite] >= lo - 1e-5) & (lin[finite] <= hi + 1e-5))


def _c_levels(n=3, C=4, H=8, W=16, **override):
    lv = _lib.mcs_texture_levels()
    lv.n_levels, lv.C = n, C
    for k, (h, w) in enumerate(chain_shapes(H, W, n)):
        lv.ptr[k], lv.h[k], lv.w[k], lv.batch_stride[k] = 256 * (k + 1), h, w, 0
    for key, v in override.items():
        if isinstance(v, tuple):
            getattr(lv, key)[v[0]] = v[1]
        else:
            setattr(lv, key, v)
    return ctypes.byref(lv)


def test_entry_points_reject_bad_arguments_without_a_device():
    l = _lib.lib()
    N = None
    P = ctypes.c_void_p(256)              # never dereferenced: validation fails first
    D = (ctypes.c_void_p * 3)(256, 256, 256)
    fwd = lambda lv=None, uv=P, da=P, B=1, H=4, W=4, f=1, b=0, out=P: l.mcs_texture_fwd(lv or _c_levels(), uv, da, B, H, W, f, b, out, N)
    bwd = lambda lv=None, uv=P, da=P, f=1, g=P, dt=D, du=P, dd=P: l.mcs_texture_bwd(lv or _c_levels(), uv, da, 1, 4, 4, f, 0, g, dt, du, dd, N)
    bad = [
        ("null levels", lambda: l.mcs_texture_fwd(N, P, P, 1, 4, 4, 1, 0, P, N), b"null pointer"),
        ("null uv", lambda: fwd(uv=N), b"null pointer"),
        ("null uv_da in lml", lambda: fwd(da=N), b"uv_da is required"),
        ("null out", lambda: fwd(out=N), b"null pointer"),
        ("bad filter", lambda: fwd(f=2), b"unknown filter_mode"),
        ("bad boundary", lambda: fwd(b=5), b"unknown boundary_mode"),
        ("negative size", lambda: fwd(B=-1), b"must be >= 0"),
        ("0 levels", lambda: fwd(lv=_c_levels(n_levels=0)), b"n_levels must be in 1..16"),
        ("17 levels", lambda: fwd(lv=_c_levels(n_levels=17)), b"n_levels must be in 1..16"),
        ("0 channels", lambda: fwd(lv=_c_levels(C=0)), b"C must be >= 1"),
        ("null level", lambda: fwd(lv=_c_levels(ptr=(1, None))), b"null pointer (level 1)"),
        ("empty level", lambda: fwd(lv=_c_levels(h=(0, 0))), b"level 0 has size"),
        ("wrong level size", lambda: fwd(lv=_c_levels(w=(2, 5))), b"level 2 is"),
        ("bad batch stride", lambda: fwd(lv=_c_levels(batch_stride=(1, 7))), b"batch_stride"),
        ("mixed batch strides", lambda: fwd(lv=_c_levels(batch_stride=(0, 128 * 4))), b"minibatch"),
        ("misaligned level", lambda: fwd(lv=_c_levels(ptr=(0, 258))), b"not 4-byte aligned"),
        ("misaligned uv_da", lambda: fwd(da=ctypes.c_void_p(264)), b"16-byte aligned"),
        ("bwd null d_out", lambda: bwd(g=N), b"null pointer"),
        ("bwd no gradient", lambda: bwd(dt=N, du=N, dd=N), b"no gradient requested"),
        ("bwd only d_uv_da in linear", lambda: bwd(f=0, dt=N, du=N), b"no gradient requested"),
        ("bwd misaligned d_uv_da", lambda: bwd(dd=ctypes.c_void_p(260)), b"16-byte aligned"),
        ("bwd misaligned d_tex", lambda: bwd(dt=(ctypes.c_void_p * 3)(256, 258, 256)), b"d_tex[1]"),
    ]
    for name, call, frag in bad:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0, name
        assert frag in msg, (name, msg)
    # an empty pixel grid succeeds without launching anything
    assert fwd(B=0) == 0 and l.mcs_texture_bwd(_c_levels(), P, P, 2, 0, 3, 1, 1, P, D, P, P, N) == 0


def _bad_calls():
    t = lambda *s: torch.zeros(*s)
    tex, uv, da = t(1, 8, 16, 3), t(2, 4, 5, 2), t(2, 4, 5, 4)
    mip = [t(1, 4, 8, 3), t(1, 2, 4, 3)]
    return [
        ("nearest", dict(tex=tex, uv=uv, filter_mode="nearest")),
        ("linear-mipmap-nearest", dict(tex=tex, uv=uv, uv_da=da, mip=mip, filter_mode="linear-mipmap-nearest")),
        ("zero boundary", dict(tex=tex, uv=uv, boundary_mode="zero")),
        ("cube boundary", dict(tex=tex, uv=uv, boundary_mode="cube")),
        ("mip_level_bias", dict(tex=tex, uv=uv, uv_da=da, mip=mip, mip_level_bias=t(2, 4, 5))),
        ("max_mip_level", dict(tex=tex, uv=uv, uv_da=da, mip=mip, max_mip_level=2)),
        ("mipmap without uv_da", dict(tex=tex, uv=uv, mip=mip, filter_mode=LML)),
        ("mipmap without mip", dict(tex=tex, uv=uv, uv_da=da)),
        ("tex rank", dict(tex=t(8, 16, 3), uv=uv)),
        ("tex dtype", dict(tex=tex.double(), uv=uv)),
        ("tex empty channels", dict(tex=t(1, 8, 16, 0), uv=uv)),
        ("uv rank", dict(tex=tex, uv=t(4, 5, 2))),
        ("uv channels", dict(tex=tex, uv=t(2, 4, 5, 3))),
        ("uv dtype", dict(tex=tex, uv=uv.half())),
        ("uv_da shape", dict(tex=tex, uv=uv, uv_da=t(2, 4, 5, 2), mip=mip)),
        ("uv_da pixels", dict(tex=tex, uv=uv, uv_da=t(2, 4, 6, 4), mip=mip)),
        ("minibatch", dict(tex=t(3, 8, 16, 3), uv=uv)),
        ("mip size", dict(tex=tex, uv=uv, uv_da=da, mip=[t(1, 4, 7, 3)])),
        ("mip channels", dict(tex=tex, uv=uv, uv_da=da, mip=[t(1, 4, 8, 2)])),
        ("mip minibatch", dict(tex=tex, uv=uv, uv_da=da, mip=[t(2, 4, 8, 3)])),
        ("mip rank", dict(tex=tex, uv=uv, uv_da=da, mip=[t(4, 8, 3)])),
        ("17 levels", dict(tex=t(1, 1, 1 << 16, 1), uv=uv, uv_da=da, mip=[t(1, 1, max(1, (1 << 16) >> k), 1) for k in range(1, 17)])),
    ]


@pytest.mark.parametrize("name, kw", _bad_calls(), ids=[c[0] for c in _bad_calls()])
def test_bad_inputs_raise_value_error_before_any_launch(name, kw):
    _lib.LAUNCHES.clear()
    with pytest.raises(ValueError):
        texture(**kw)
    assert not _lib.LAUNCHES


def test_valid_cpu_tensors_are_refused_not_computed():
    with pytest.raises(RuntimeError, match="CUDA"):
        texture(torch.zeros(1, 1, 1, 3), torch.zeros(1, 2, 2, 2), torch.zeros(1, 2, 2, 4))


@pytest.mark.skipif(not HAVE_REF, reason="the reference checkout is only present in the build container")
def test_texture_golden_regenerates_bit_identically():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_texture_golden
    g = make_texture_golden.generate()
    d = np.load(os.path.join(HERE, "golden", "ref_texture2d.npz"))
    assert sorted(g) == sorted(d.files)
    for k in d.files:
        assert g[k].dtype == d[k].dtype and np.array_equal(g[k], d[k]), k
