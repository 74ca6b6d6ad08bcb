"""CPU: the oracle's restatement of Texture2D's automatic mip chain (oracle/mipchain.c) against torch and against the reference's own
texture2d_mip (render/texture.py:20-30, run unmodified where the reference checkout exists), and the argument checks of the four C entry
points of the chain."""
import ctypes
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from common import rel_l2
from oracle.mipchain import mip_shapes, mipchain_oracle
from nvdiffrecmc_b200 import _lib

REF = "/root/reference/render/texture.py"
SHAPES = [(1024, 1024, 4), (32, 96, 4), (24, 40, 3), (13, 29, 1), (64, 16, 7), (2, 2, 1)]


def _pool(x):
    return torch.nn.functional.avg_pool2d(torch.from_numpy(x).permute(0, 3, 1, 2), (2, 2)).permute(0, 2, 3, 1).contiguous().numpy()


def same_bits(a, b):
    """equal bit for bit, every NaN equal to every other (their sign and payload are not part of the contract)"""
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def _base(rng, Bt, H, W, C):
    """normal texels with NaN, +Inf and -Inf sprinkled in"""
    x = rng.normal(size=(Bt, H, W, C)).astype(np.float32)
    m = rng.random(x.shape)
    x[m < 0.002] = np.nan
    x[(m >= 0.002) & (m < 0.004)] = np.inf
    x[(m >= 0.004) & (m < 0.006)] = -np.inf
    return x


@pytest.mark.parametrize("Bt", [1, 2])
@pytest.mark.parametrize("H,W,C", SHAPES)
def test_chain_forward_is_avg_pool2d(H, W, C, Bt):
    base = _base(np.random.default_rng(H * W + C + Bt), Bt, H, W, C)
    got = mipchain_oracle().forward(base)
    assert [g.shape[1:3] for g in got] == mip_shapes(H, W)[1:]
    prev = base
    for k, g in enumerate(got, 1):
        prev = _pool(prev)
        assert same_bits(g, prev), k


def _grads(rng, Bt, H, W, C, absent=(0, 2)):
    return [None if k in absent else rng.normal(size=(Bt, h, w, C)).astype(np.float32) for k, (h, w) in enumerate(mip_shapes(H, W))]


def _reference_fold(shape, grads):
    """d base of the reference's automatic chain (texture2d_mip, unmodified) for the per-level gradients grads (None = none), its
    dr.texture on the fp32 oracle and its torch.linspace on the CPU, as make_texture_golden.py runs it."""
    from golden.make_texture_golden import oracle_texture
    from refshade import reference_render
    linspace = torch.linspace

    def cpu_linspace(*a, **k):
        if str(k.get("device", "")).startswith("cuda"):
            k["device"] = "cpu"
        return linspace(*a, **k)

    empty = type(sys)("unused_backend")
    with reference_render(empty, empty):
        tex_mod = importlib.import_module("render.texture")
        tex_mod.dr.texture = oracle_texture()
        torch.linspace = cpu_linspace
        try:
            base = torch.zeros(shape, requires_grad=True)
            mips = [base]
            while mips[-1].shape[1] > 1 and mips[-1].shape[2] > 1:
                mips.append(tex_mod.texture2d_mip.apply(mips[-1]))
            loss = sum((m * torch.from_numpy(g)).sum() for m, g in zip(mips, grads) if g is not None)
            return torch.autograd.grad(loss, base)[0].numpy()
        finally:
            torch.linspace = linspace


needs_ref = pytest.mark.skipif(not os.path.exists(REF), reason="needs the reference checkout")


@needs_ref
@pytest.mark.parametrize("H,W,C,exact", [(1024, 1024, 1, True), (64, 16, 7, True), (32, 96, 4, False)])
def test_fold_is_the_reference_backward(H, W, C, exact):
    """Power-of-two sides: the reference's arithmetic bit for bit.  32 x 96 (even at every level): torch.linspace's grid is an ulp off the
    texel centres at the levels whose sides are not powers of two.  (The reference's backward samples with a one-image grid, so it only
    runs for Bt = 1.)"""
    rng = np.random.default_rng(H + W + C)
    for absent in ((0, 2), ()):
        grads = _grads(rng, 1, H, W, C, absent)
        got = mipchain_oracle().fold(grads, (1, H, W, C))
        ref = _reference_fold((1, H, W, C), grads)
        if exact:
            assert same_bits(got, ref)
        else:
            assert rel_l2(got, ref) <= 1e-6 and not np.array_equal(got, ref)


@needs_ref
@pytest.mark.parametrize("H,W", [(24, 40), (48, 80), (13, 29)])
def test_reference_backward_fails_on_an_odd_pooled_level(H, W):
    """The behaviour mip_chain's backward keeps: a level pooled from an odd side has no backward in the reference."""
    grads = _grads(np.random.default_rng(0), 1, H, W, 2, absent=())
    with pytest.raises(RuntimeError, match="invalid gradient"):
        _reference_fold((1, H, W, 2), grads)


def test_clamp_is_torch_clamp():
    rng = np.random.default_rng(1)
    levels = [_base(rng, 2, h, w, 4) for h, w in [(16, 8), (8, 4), (4, 2), (2, 1), (1, 1)]]
    levels[0][0, 0, 0] = [0.0, -0.0, 0.25, 1.0]
    lo = np.array([0.0, 0.1, np.nan, 0.5], np.float32)
    hi = np.array([1.0, 0.9, 0.5, 0.25], np.float32)           # channel 3: lo > hi, torch returns hi
    got = mipchain_oracle().clamp(levels, lo, hi)
    for g, x in zip(got, levels):
        ref = torch.from_numpy(x.copy())
        for c in range(4):
            ref[..., c].clamp_(min=torch.tensor(lo[c]), max=torch.tensor(hi[c]))
        assert same_bits(g, ref.numpy())


def test_normalize_is_safe_normalize():
    """Within 2 ulp of util.safe_normalize on the CPU, whose vectorised division rounds differently; the kernels are held to the oracle
    bit for bit and to the device's safe_normalize within 1 ulp."""
    rng = np.random.default_rng(2)
    levels = [_base(rng, 1, h, w, 3) * np.float32(10.0) ** rng.integers(-25, 20, (1, h, w, 1)).astype(np.float32) for h, w in [(64, 32), (32, 16)]]
    levels[1][0, 0, :4] = [[0, 0, 0], [1e-12, 0, 0], [3, 4, 0], [-0.0, 0, 2]]
    got = mipchain_oracle().normalize(levels)
    for g, x in zip(got, levels):
        t = torch.from_numpy(x)
        ref = (t / torch.sqrt(torch.clamp(torch.sum(t * t, -1, keepdim=True), min=1e-20))).numpy()
        assert np.array_equal(np.isnan(g), np.isnan(ref))
        fin = np.isfinite(ref) & np.isfinite(g)
        ulp = np.abs(g[fin].view(np.int32).astype(np.int64) - ref[fin].view(np.int32).astype(np.int64))
        assert ulp.max() <= 2
        assert g[~fin & ~np.isnan(g)].tobytes() == ref[~fin & ~np.isnan(ref)].tobytes()
    small = np.float32(1e-12) / np.sqrt(np.float32(1e-20))              # below eps the length is sqrt(1e-20)
    assert same_bits(got[1][0, 0, :4], np.array([[0, 0, 0], [small, 0, 0], [0.6, 0.8, 0], [-0.0, 0, 1]], np.float32))


# ---- the C entry points refuse bad tables before any launch ------------------------------------------------------------------------

FAKE = 0x10000          # an aligned address that is never dereferenced: every call below fails its checks first


def _table(shapes, C=4, ptrs=None, stride=True):
    lv = _lib.mcs_texture_levels()
    lv.n_levels, lv.C = len(shapes), C
    for k, (h, w) in enumerate(shapes):
        lv.ptr[k] = FAKE if ptrs is None else ptrs[k]
        lv.h[k], lv.w[k], lv.batch_stride[k] = h, w, h * w * C if stride else 0
    return lv


def _n_levels(lv, n):
    lv.n_levels = n
    return lv


def _bad_calls():
    l, s = _lib.lib(), None
    chain = [(32, 32), (16, 16), (8, 8)]
    r = ctypes.byref
    fwd = lambda lv, Bt=1: l.mcs_mip_chain_fwd(r(lv), Bt, s)
    bwd = lambda lv, d=FAKE, Bt=1: l.mcs_mip_chain_bwd(r(lv), Bt, d, s)
    clamp = lambda lv, lo=FAKE, hi=FAKE: l.mcs_mip_clamp(r(lv), 1, lo, hi, s)
    norm = lambda lv: l.mcs_mip_normalize(r(lv), 1, s)
    return [
        ("fwd: null table", lambda: l.mcs_mip_chain_fwd(None, 1, s), b"null pointer (level table)"),
        ("fwd: one level", lambda: fwd(_table(chain[:1])), b"n_levels must be in 2..16 (got 1)"),
        ("fwd: 17 levels", lambda: fwd(_n_levels(_table([(1 << 16 >> k, 1 << 16 >> k) for k in range(16)]), 17)), b"n_levels must be in 2..16 (got 17)"),
        ("fwd: not halved", lambda: fwd(_table([(32, 32), (16, 16), (8, 7)])), b"level 2 is 8 x 7, which is not the 2 x 2 pool of level 1"),
        ("fwd: pooled past 1", lambda: fwd(_table([(2, 8), (1, 4), (1, 2)])), b"level 2 is 1 x 2, which is not the 2 x 2 pool of level 1"),
        ("fwd: null level", lambda: fwd(_table(chain, ptrs=[FAKE, None, FAKE])), b"null pointer (level 1)"),
        ("fwd: unaligned", lambda: fwd(_table(chain, ptrs=[FAKE, FAKE + 2, FAKE])), b"level 1 is not 4-byte aligned"),
        ("fwd: Bt 0", lambda: fwd(_table(chain), 0), b"Bt must be in 1..65535"),
        ("fwd: shared level, Bt 2", lambda: fwd(_table(chain, stride=False), 2), b"batch_stride"),
        ("fwd: C 0", lambda: fwd(_table(chain, C=0)), b"C must be >= 1"),
        ("bwd: no gradient", lambda: bwd(_table(chain, ptrs=[None] * 3)), b"null pointer (no level given)"),
        ("bwd: null d_base", lambda: bwd(_table(chain), None), b"null pointer (d_base)"),
        ("bwd: not halved", lambda: bwd(_table([(32, 32), (15, 16)])), b"level 1 is 15 x 16"),
        ("clamp: null bounds", lambda: clamp(_table(chain), hi=None), b"null pointer (lo / hi)"),
        ("clamp: off the layout", lambda: clamp(_table([(8, 2), (4, 1), (1, 1)])), b"level 2 is 1 x 1, expected 2 x 1"),
        ("clamp: null level", lambda: clamp(_table(chain, ptrs=[FAKE, FAKE, None])), b"null pointer (level 2)"),
        ("normalize: C 4", lambda: norm(_table(chain)), b"C must be 3 (got 4)"),
        ("normalize: no levels", lambda: norm(_table([])), b"n_levels must be in 1..16 (got 0)"),
    ]


@pytest.mark.parametrize("case", range(len(_bad_calls())), ids=[c[0] for c in _bad_calls()])
def test_entry_points_refuse_bad_tables(case):
    """Each chain entry point validates its table and pointers before launching and names the problem through its status and
    mcs_last_error().  The tables point at a fake address, so this runs where no kernel can launch."""
    if torch.cuda.is_available():
        pytest.skip("the calls would launch on the fake pointers")
    name, call, frag = _bad_calls()[case]
    rc = call()
    msg = _lib.lib().mcs_last_error() or b""
    assert rc != 0, name
    assert frag in msg, (name, msg)


def test_launch_count_of_the_chain_forward():
    l = _lib.lib()
    assert [l.mcs_mip_chain_fwd_launches(n) for n in (1, 2, 6, 7, 11, 12, 16)] == [0, 1, 1, 2, 2, 3, 3]
