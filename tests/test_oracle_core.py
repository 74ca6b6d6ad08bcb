"""CPU: self-consistency of the oracle pieces that the reference cannot pin (SURVEY 8c: no test, no golden vector and no
CPU-runnable path exists for env_shade / BVH / visibility): deterministic math accuracy, PCG stream, CDF sampling,
LBVH == brute force, estimator sanity (white furnace, analytic irradiance), finite-difference check of the hand-derived
adjoints, and the multi-GPU batch-offset rule."""
import math

import numpy as np
import pytest

from common import make_case, oracle, rel_l2
from nvdiffrecmc_b200 import synth


def test_det_math_accuracy():
    o = oracle()
    rng = np.random.default_rng(0)
    a = np.concatenate([rng.uniform(-7, 7, 20000), np.linspace(-2 * np.pi, 2 * np.pi, 1001)]).astype(np.float32)
    s, c = o.det_sincos(a)
    assert np.abs(s - np.sin(a.astype(np.float64))).max() < 3e-7 and np.abs(c - np.cos(a.astype(np.float64))).max() < 3e-7
    y, x = rng.normal(size=20000).astype(np.float32), rng.normal(size=20000).astype(np.float32)
    assert np.abs(o.det_atan2(y, x) - np.arctan2(y.astype(np.float64), x.astype(np.float64))).max() < 6e-7
    assert o.det_atan2(np.float32([0, 0, 1, -1]), np.float32([0, -1, 0, 0])).tolist() == pytest.approx([0, math.pi, math.pi / 2, -math.pi / 2], abs=1e-6)
    x = np.concatenate([rng.uniform(-1, 1, 20000), [-1, 1, 0, 0.5, -0.5]]).astype(np.float32)
    assert np.abs(o.det_acos(x) - np.arccos(x.astype(np.float64))).max() < 6e-7


def test_pcg_stream_matches_an_independent_numpy_restatement():
    """kernel.cu:30-45"""
    import ctypes as C
    o = oracle()

    def rand_pcg(s):
        s = np.uint32(s)
        with np.errstate(over="ignore"):
            word = np.uint32(((s >> np.uint32((s >> np.uint32(28)) + np.uint32(4))) ^ s) * np.uint32(277803737))
            ns = np.uint32(s * np.uint32(747796405) + np.uint32(2891336453))
        return np.uint32((word >> np.uint32(22)) ^ word), ns
    for seed in (0, 1, 12345, 2**31 - 1, 0xFFFFFFFF):
        st = C.c_uint32(seed)
        exp_s = np.uint32(seed)
        for _ in range(5):
            got = o.lib.orc_rand_pcg(C.byref(st))
            exp, exp_s = rand_pcg(exp_s)
            assert got == int(exp) and st.value == int(exp_s)
        a, _ = rand_pcg(np.uint32(seed)); b, _ = rand_pcg(np.uint32(77))
        assert o.lib.orc_hash_pcg(seed, 77) == int(a ^ b)


def test_update_pdf_matches_light_py_formulas():
    """render/light.py:46-59 restated with numpy float64"""
    rng = np.random.default_rng(1)
    base = rng.uniform(0, 2, (12, 20, 3)).astype(np.float32)
    base[3] = 0          # an all-black row: cols stays 0 (the `> 0` guard, light.py:58)
    pdf, rows, cols = oracle().update_pdf(base)
    Y = (np.arange(12) + 0.5) / 12
    p = base.max(-1).astype(np.float64) * np.sin(Y * np.pi)[:, None]
    p /= p.sum()
    c = np.cumsum(p, 1); r = np.cumsum(c[:, -1])
    c = c / np.where(c[:, -1:] > 0, c[:, -1:], 1); r = r / r[-1]
    assert rel_l2(pdf, p) < 1e-6 and rel_l2(cols, c) < 1e-6 and rel_l2(rows, r) < 1e-6
    assert cols[3].max() == 0 and abs(rows[-1] - 1) < 1e-6


@pytest.mark.parametrize("kind,level", [("blob", 1), ("blob+torus", 2), ("full", 2)])
def test_canonical_lbvh_equals_brute_force(kind, level):
    o = oracle()
    v, f = synth.scene_mesh(kind, level=level)
    sc = o.scene(v, f)
    rng = np.random.default_rng(2)
    ro = rng.normal(size=(20000, 3)).astype(np.float32); rd = rng.normal(size=(20000, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    rd[:500] = np.eye(3, dtype=np.float32)[rng.integers(0, 3, 500)]
    a = sc.visibility(ro, rd, "brute"); b, cnt = sc.visibility(ro, rd, "bvh", return_counters=True)
    assert np.array_equal(a, b) and 0.05 < a.mean() < 0.95 and cnt[0] > 0
    lb = sc.export_lbvh()
    assert sorted(lb["prim"].tolist()) == list(range(f.shape[0])) and (np.diff(lb["morton"].astype(np.int64)) >= 0).all()
    # every internal box contains its children
    T = f.shape[0]
    for i in range(T - 1):
        for c in (lb["left"][i], lb["right"][i]):
            assert (lb["lo"][i] <= lb["lo"][c]).all() and (lb["hi"][i] >= lb["hi"][c]).all()


def _furnace_case(N, res=12):
    c = make_case(res=res, B=1, N=N, mesh="blob", level=1, light_hw=(16, 32))
    c["light"] = np.ones_like(c["light"])
    c["pdf"], c["rows"], c["cols"] = oracle().update_pdf(c["light"])
    return c


def test_white_furnace_diffuse():
    """Constant radiance L=1, no occluders, Lambert: E = int L cos/pi = 1 for every covered pixel (MIS estimator is unbiased)."""
    N = 8
    c = _furnace_case(N)
    o = oracle()
    d, s = o.env_shade(None, c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"],
                       c["perms"], BSDF="diffuse", n_samples_x=N, rnd_seed=3)
    m = c["mask"] > 0
    nl = np.linalg.norm(c["nrm"][m], axis=-1)
    est = d[m][:, 0] / nl          # the Lambert term uses the un-normalised shading normal (bent normals are shorter than 1)
    assert abs(est.mean() - 1.0) < 0.01 and est.std() < 0.15
    assert (s == 0).all()
    assert (d[~m] == 0).all()


def test_visibility_halves_irradiance_under_a_half_space_occluder():
    """A huge plane through the shading point's horizon... simpler: shadow_scale blends V (kernel.cu:420): out(ss) is affine in ss."""
    N = 4
    c = make_case(res=16, B=1, N=N, seed=3)
    o = oracle()
    run = lambda ss: o.env_shade(c["scene"], c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"],
                                 c["cols"], c["perms"], n_samples_x=N, rnd_seed=1, shadow_scale=ss)
    d0, d1, dh = run(0.0)[0], run(1.0)[0], run(0.5)[0]
    assert rel_l2(dh, 0.5 * (d0 + d1)) < 1e-6 and d1.sum() < d0.sum()
    unocc = o.env_shade(None, c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"],
                        c["perms"], n_samples_x=N, rnd_seed=1)[0]
    assert np.array_equal(unocc, d0)


def test_f32_and_f64_oracles_agree_statistically():
    N = 8
    c = make_case(res=16, B=1, N=N, seed=1)
    a = oracle().env_shade(None, c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"],
                           c["perms"], n_samples_x=N, rnd_seed=2)
    b = oracle(True).env_shade(None, c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"],
                               c["perms"], n_samples_x=N, rnd_seed=2)
    # different libm on the decision path => a few samples land in neighbouring texels; aggregates must still agree closely
    assert rel_l2(a[0], b[0]) < 2e-2 and abs(a[0].sum() / b[0].sum() - 1) < 2e-3


@pytest.mark.parametrize("bsdf", ["pbr", "diffuse"])
def test_hand_derived_adjoints_vs_finite_differences(bsdf):
    """fp64 oracle: d<out, w>/d(param) by central differences vs orc_env_shade backward.  The Monte-Carlo sample set is held fixed
    through the test-only `sampling_gbuffer` override, because the reference's gradients deliberately ignore the dependence of the
    samples on the parameters (and drop the visibility boundary term, kernel.cu:97-99)."""
    N = 3
    o = oracle(True)
    c = make_case(res=8, B=1, N=N, seed=5)
    c["scene"] = o.scene(c["verts"], c["tris"])          # fp64 scene for the fp64 oracle
    samp = (c["pos"], c["nrm"], c["kd"], c["ks"])
    rng = np.random.default_rng(0)
    wd, ws = rng.uniform(0, 1, c["pos"].shape), rng.uniform(0, 1, c["pos"].shape)

    def f(pos, nrm, kd, ks, light):
        d, s = o.env_shade(c["scene"], c["mask"], c["ro"], pos, nrm, c["view"], kd, ks, light, c["pdf"], c["rows"], c["cols"], c["perms"],
                           BSDF=bsdf, n_samples_x=N, rnd_seed=4, sampling_gbuffer=samp)
        return float((d * wd).sum() + (s * ws).sum())
    base = [np.asarray(c[k], np.float64) for k in ("pos", "nrm", "kd", "ks", "light")]
    g = o.env_shade(c["scene"], c["mask"], c["ro"], *base[:2], c["view"], *base[2:4], base[4], c["pdf"], c["rows"], c["cols"], c["perms"], BSDF=bsdf,
                    n_samples_x=N, rnd_seed=4, grads=(wd, ws), sampling_gbuffer=samp)
    g = dict(zip(("pos", "nrm", "kd", "ks", "light"), g))
    for idx, name in enumerate(("pos", "nrm", "kd", "ks", "light")):
        direction = rng.normal(size=base[idx].shape)
        if name != "light":
            direction *= (c["mask"] > 0)[..., None]
        eps = 1e-6
        p_plus = [b.copy() for b in base]; p_minus = [b.copy() for b in base]
        p_plus[idx] += eps * direction; p_minus[idx] -= eps * direction
        fd = (f(*p_plus) - f(*p_minus)) / (2 * eps)
        an = float((g[name] * direction).sum())
        if bsdf == "diffuse" and name in ("pos", "kd", "ks"):
            assert an == 0.0 and abs(fd) < 1e-9          # Lambert-only modes touch the normal and the light only
        else:
            assert abs(fd - an) <= 2e-5 * max(abs(an), abs(fd)) + 1e-9, "%s: fd %.8e analytic %.8e" % (name, fd, an)


def test_batch_offset_reproduces_the_full_batch_random_stream():
    N = 2
    c = make_case(res=8, B=2, N=N, seed=2)
    o = oracle()
    full = o.env_shade(c["scene"], c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"], c["rows"], c["cols"],
                       c["perms"], n_samples_x=N, rnd_seed=9)
    s = slice(1, 2)
    part = o.env_shade(c["scene"], c["mask"][s], c["ro"][s], c["pos"][s], c["nrm"][s], c["view"][s], c["kd"][s], c["ks"][s], c["light"], c["pdf"],
                       c["rows"], c["cols"], c["perms"], n_samples_x=N, rnd_seed=9, batch_offset=1)
    assert np.array_equal(full[0][s], part[0]) and np.array_equal(full[1][s], part[1])
    other = o.env_shade(c["scene"], c["mask"][s], c["ro"][s], c["pos"][s], c["nrm"][s], c["view"][s], c["kd"][s], c["ks"][s], c["light"], c["pdf"],
                        c["rows"], c["cols"], c["perms"], n_samples_x=N, rnd_seed=9, batch_offset=0)
    assert not np.array_equal(other[0], part[0])


def test_cdf_bisection_is_upper_bound():
    """kernel.cu:144-154 bisects with a fixed iteration count.  For any non-decreasing CDF (plateaus, non-power-of-two sizes) it
    returns exactly min(upper_bound(x), size-1); the CUDA product relies on this to find the same index with a 4-ary search."""
    rng = np.random.default_rng(0)

    def ref(cdf, x):
        lo, hi = 0, len(cdf) - 1
        m = int(math.ceil(math.log2(np.float32(hi)))) + 1
        for _ in range(m):
            mid = (lo + hi) // 2
            if x >= cdf[mid]:
                lo = mid
            if x < cdf[mid]:
                hi = mid
        return hi

    def four_ary(cdf, x):             # integer logic of csrc/envshade.cu:sample_cdf
        lo, hi = 0, len(cdf) - 1
        steps, span = 1, len(cdf) - 1
        while span > 0:
            steps += 1; span //= 4
        for _ in range(steps):
            span = hi - lo
            m1, m2, m3 = lo + (span >> 2), lo + (span >> 1), lo + ((3 * span) >> 2)
            if span > 0:
                if x < cdf[m1]: hi = m1
                elif x < cdf[m2]: lo, hi = m1 + 1, m2
                elif x < cdf[m3]: lo, hi = m2 + 1, m3
                else: lo = m3 + 1
                lo = min(lo, hi)
        return hi
    for _ in range(400):
        n = int(rng.choice([2, 3, 5, 16, 17, 31, 32, 100, 256, 257, 1000, 1024, 2048]))
        p = rng.random(n) ** rng.choice([1, 4, 16])
        if rng.random() < 0.5:
            p[rng.random(n) < 0.3] = 0
        if p.sum() == 0:
            p[0] = 1
        cdf = np.cumsum(p.astype(np.float32), dtype=np.float32); cdf = (cdf / cdf[-1]).astype(np.float32)
        for x in np.concatenate([rng.random(12).astype(np.float32), cdf[rng.integers(0, n, 4)], [np.float32(0), np.float32(0.99999994)]]):
            x = min(np.float32(x), np.float32(0.99999994))
            ub = min(int(np.searchsorted(cdf, x, side="right")), n - 1)
            assert ref(cdf, x) == ub == four_ary(cdf, x)


@pytest.mark.parametrize("f64", [False, True])
def test_env_shade_abs_terms_bounds_every_sum(f64):
    """abs_terms accumulates |term| for every per-ray term: the result bounds the plain sum elementwise (rounding is monotone, so this
    holds exactly in fp32 too), and where every term is >= 0 -- radiance and, for non-negative upstream gradients, the light gradient,
    with a non-negative probe -- it is the plain sum itself.  The gradients of pos / nrm / ks have terms of both signs: there A is larger."""
    o = oracle(f64)
    c = make_case(res=16, B=1, N=4, seed=4)
    assert (c["light"] >= 0).all()
    args = (o.scene(c["verts"], c["tris"]), c["mask"], c["ro"], c["pos"], c["nrm"], c["view"], c["kd"], c["ks"], c["light"], c["pdf"],
            c["rows"], c["cols"], c["perms"])
    g = np.random.default_rng(5)
    dg, sg = [g.uniform(0, 1, size=c["pos"].shape).astype(np.float32) for _ in range(2)]
    kw = dict(BSDF="pbr", n_samples_x=4, rnd_seed=3, shadow_scale=0.5)
    fwd, fwd_a = o.env_shade(*args, **kw), o.env_shade(*args, abs_terms=True, **kw)
    bwd, bwd_a = o.env_shade(*args, grads=(dg, sg), **kw), o.env_shade(*args, grads=(dg, sg), abs_terms=True, **kw)
    for name, r, a in zip(("diff", "spec", "pos", "nrm", "kd", "ks", "light"), fwd + bwd, fwd_a + bwd_a):
        assert (a >= np.abs(r)).all(), name
    for name, r, a in zip(("diff", "spec", "light"), fwd + bwd[4:], fwd_a + bwd_a[4:]):
        assert np.array_equal(a, r) and a.max() > 0, name
    for name, r, a in zip(("pos", "nrm", "ks"), (bwd[0], bwd[1], bwd[3]), (bwd_a[0], bwd_a[1], bwd_a[3])):
        assert (a > np.abs(r) * 1.5).mean() > 0.05, name          # cancellation between rays: the floor is not the sum
