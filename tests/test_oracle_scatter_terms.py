"""CPU: the `terms` mode of every oracle entry point that scatters -- d tex, hash-grid and MLP-texture d params, rasterize / rast_db /
antialias d pos, interpolate and interpolate_da d attr -- in both precisions.  terms="sum" sums exactly what the entry points summed before
they took the mode (tests/golden/scatter_sums.npz); "abs" bounds the sum elementwise and equals it where every term is >= 0; "count"
equals a count made independently in numpy; the one-writer outputs (d uv, d uv_da, d x, d t, d W, d color, d rast_db) do not depend on
the mode.  The GPU tests build their per-element bars from these statistics (tests/common.py: check_scatter_fp32 / scatter_floor)."""
import os

import numpy as np
import pytest

from oracle.geometry import geometry_oracle
from oracle.hashgrid import REF_CONFIG, hashgrid_oracle
from oracle.mlptexture import mlptexture_oracle
from oracle.texture import texture_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
EDGE = {"otype": "HashGrid", "n_levels": 5, "log2_hashmap_size": 9, "base_resolution": 4, "per_level_scale": 2.0}
LML = "linear-mipmap-linear"
PREC = pytest.mark.parametrize("f64", [False, True], ids=["fp32", "fp64"])


def _golden():
    return np.load(os.path.join(HERE, "golden", "scatter_sums.npz"))


def _same(a, b, f64):
    a, b = np.asarray(a), np.asarray(b)
    it = np.int64 if f64 else np.int32
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(it), b.view(it))


def _three(fn):
    """fn(terms) for the three modes -> (sum, abs, count)"""
    return tuple(fn(t) for t in ("sum", "abs", "count"))


def _check_stats(s, a, n):
    s, a, n = (np.asarray(x, np.float64) for x in (s, a, n))
    assert (a >= np.abs(s)).all(), "abs below |sum| at %d elements" % (a < np.abs(s)).sum()
    assert (n == np.round(n)).all() and (n >= 0).all()
    assert ((n == 0) == (a == 0)).all(), "count and abs disagree on which elements have terms"
    assert (s[n == 0] == 0).all()


# ------------------------------------------------------------------------------------------ texture
def _tex_case(d):
    return [d["tex_l%d" % k] for k in range(3)], d["tex_uv"], d["tex_da"], d["tex_g"]


@PREC
@pytest.mark.parametrize("filt,bnd", [(LML, "wrap"), ("linear", "clamp")])
def test_texture_terms(f64, filt, bnd):
    d = _golden()
    o = texture_oracle(f64)
    levels, uv, da, g = _tex_case(d)
    res = _three(lambda t: o.backward(levels, uv, da, g, filt, bnd, terms=t))
    sfx = "_f64" if f64 else "_f32"
    for k, x in enumerate(res[0][0]):
        assert _same(x, d["tex_%s_%s_l%d%s" % (filt, bnd, k, sfx)], f64), k
    for r in res[1:]:                                     # d uv and d uv_da do not depend on the mode
        assert _same(r[1], res[0][1], f64) and (r[2] is None or _same(r[2], res[0][2], f64))
    for s, a, n in zip(res[0][0], res[1][0], res[2][0]):
        _check_stats(s, a, n)
    assert max(float(n.max()) for n in res[2][0]) >= 3
    pos = np.abs(g)                                       # every term >= 0: abs is the sum
    for s, a in zip(o.backward(levels, uv, da, pos, filt, bnd)[0], o.backward(levels, uv, da, pos, filt, bnd, terms="abs")[0]):
        assert _same(s, a, f64)


@PREC
@pytest.mark.parametrize("bnd", ["wrap", "clamp"])
def test_texture_count_equals_numpy(f64, bnd):
    """'linear' on one 8 x 12 level: each pixel's four taps, computed in numpy; a tap whose bilinear weight or gradient is 0 adds nothing"""
    d = _golden()
    o = texture_oracle(f64)
    tex, uv, g = d["tex_l0"], d["tex_uv"].copy(), d["tex_g"]
    uv[0, 2, :3] = [0.5 / 12 * 3, 0.5 / 8 * 5]            # texel centres: fx = fy = 0, three of the four taps have weight 0
    n = o.backward([tex], uv, None, g, "linear", bnd, terms="count")[0][0]
    H, W, C = tex.shape[1:]
    ref = np.zeros(tex.shape, np.float64)
    x, y = uv[..., 0].astype(o.dt) * o.dt(W) - o.dt(0.5), uv[..., 1].astype(o.dt) * o.dt(H) - o.dt(0.5)
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    fx, fy = x - np.floor(x), y - np.floor(y)
    fix = (lambda i, m: np.clip(i, 0, m - 1)) if bnd == "clamp" else (lambda i, m: i % m)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        w = (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
        for c in range(C):
            live = (w != 0) & (g[..., c] != 0)
            np.add.at(ref[0, :, :, c], (fix(y0 + dy, H)[live], fix(x0 + dx, W)[live]), 1)
    assert np.array_equal(n, ref)


# ------------------------------------------------------------------------------------------ hash grid and MLP texture
@PREC
def test_hashgrid_terms(f64):
    d = _golden()
    o = hashgrid_oracle(f64)
    lv = o.levels(EDGE)
    x, p, g = d["hg_x"], d["hg_p"], d["hg_g"]
    res = _three(lambda t: o.backward(x, p, lv, g, terms=t))
    assert _same(res[0][0], d["hg_dp" + ("_f64" if f64 else "_f32")], f64)
    assert all(_same(r[1], res[0][1], f64) for r in res[1:])          # d x
    _check_stats(res[0][0], res[1][0], res[2][0])
    a, b = 2 * int(lv["offset"][2]), 2 * int(lv["offset"][3])
    assert not res[2][0][a:b].any()                                   # level 2's gradient is 0: no terms
    assert _same(o.backward(x, p, lv, np.abs(g), want_x=False)[0], o.backward(x, p, lv, np.abs(g), want_x=False, terms="abs")[0], f64)


@PREC
def test_hashgrid_count_equals_numpy(f64):
    """Points away from every cell face (all eight corner weights non-zero), indices computed in numpy"""
    o = hashgrid_oracle(f64)
    lv = o.levels(EDGE)
    rng = np.random.default_rng(5)
    x = rng.uniform(0, 1, (4000, 3)).astype(np.float32)
    for s in lv["scale"]:
        t = float(s) * x.astype(np.float64) + 0.5
        t -= np.floor(t)
        x = x[((t > 1e-3) & (t < 1 - 1e-3)).all(1)]
    assert len(x) > 300
    g = rng.normal(size=(len(x), 2 * lv["n_levels"])).astype(np.float32)
    g[::3, 2] = 0.0                                                   # feature 0 of level 1
    g[1::3, 6:8] = 0.0                                                # all of level 3: the point adds nothing there
    n = o.backward(x, np.zeros(2 * int(lv["offset"][-1]), np.float32), lv, g, want_x=False, terms="count")[0].reshape(-1, 2)
    ref = np.zeros(n.shape, np.float64)
    M = 0xFFFFFFFF
    for l in range(lv["n_levels"]):
        s, res, size = float(lv["scale"][l]), int(lv["res"][l]), int(lv["offset"][l + 1] - lv["offset"][l])
        cell = np.floor(s * x.astype(np.float64) + 0.5).astype(np.int64)
        for c in range(8):
            cx, cy, cz = (cell[:, k] + ((c >> k) & 1) for k in range(3))
            if (lv["dense_mask"] >> l) & 1:
                h = ((cx + cy * res + cz * res * res) & M) % size
            else:
                h = ((cx & M) ^ ((cy * 2654435761) & M) ^ ((cz * 805459861) & M)) % size
            for f in range(2):
                live = g[:, 2 * l + f] != 0
                np.add.at(ref[:, f], int(lv["offset"][l]) + h[live], 1)
    assert np.array_equal(n, ref)


@PREC
def test_mlptexture_passes_the_mode_through(f64):
    d = _golden()
    m = mlptexture_oracle(f64)
    lv = m.levels(REF_CONFIG)
    p = np.random.default_rng(7).uniform(-1, 1, 2 * int(lv["offset"][-1])).astype(np.float32)
    aabb = np.array([[-1, -1, -1], [1, 1, 1]], np.float32)
    mm = np.array([[-0.1, 0.0, 0.2], [0.9, 1.0, 1.1]], np.float32)
    res = _three(lambda t: m.mlptex_backward(d["mt_t"], aabb, mm, p, lv, [d["mt_w0"], d["mt_w1"]], d["mt_g"], terms=t))
    sfx = "_f64" if f64 else "_f32"
    nz = np.flatnonzero(res[0][0])
    assert np.array_equal(nz, d["mt_dp_idx" + sfx]) and _same(res[0][0][nz], d["mt_dp_val" + sfx], f64)
    for r in res[1:]:                                                 # d t and d W
        assert _same(r[1], res[0][1], f64) and all(_same(a, b, f64) for a, b in zip(r[2], res[0][2]))
    _check_stats(res[0][0], res[1][0], res[2][0])
    assert res[2][0].max() >= 2
    # the encoder's count is the hash grid's on the clamped, normalised points with the MLP's d encoding as the upstream gradient:
    # every (point, level, corner, feature) whose weight and d encoding are non-zero
    xc = np.clip((d["mt_t"] - aabb[0]) / (aabb[1] - aabb[0]), 0, 1).astype(np.float32)
    h = hashgrid_oracle(f64)
    assert np.array_equal(res[2][0] != 0, h.backward(xc, p, lv, np.ones((len(xc), 32), np.float32), want_x=False, terms="count")[0] != 0)


# ------------------------------------------------------------------------------------------ geometry
def _geo(d):
    return d["geo_pos"], d["geo_tris"], d["geo_rast"]


@PREC
@pytest.mark.parametrize("tag", ["batched", "shared"])
def test_geometry_terms_sum_equals_the_golden(f64, tag):
    d = _golden()
    g = geometry_oracle(f64)
    pos, tris, rast = _geo(d)
    P = pos if tag == "batched" else pos[0]
    A = d["geo_attr"] if tag == "batched" else d["geo_attr"][0]
    sfx = "_%s%s" % (tag, "_f64" if f64 else "_f32")
    ops = {
        "raster": lambda t: g.raster_bwd(P, tris, rast, d["geo_g4"], terms=t),
        "rast_db": lambda t: g.rast_db_bwd(P, tris, rast, d["geo_h4"], terms=t),
        "aa": lambda t: g.antialias_bwd(d["geo_color"], rast, P, tris, d["geo_gc"], terms=t)[1],
        "da": lambda t: g.interpolate_da_bwd(A, tris, rast, d["geo_h4"], d["geo_gda"], [3, 0, 3], terms=t)[0],
    }
    for name, fn in ops.items():
        s, a, n = _three(fn)
        assert _same(s, d[name + sfx], f64), name
        _check_stats(s, a, n)
        assert n.max() >= 2, name
    dc = [g.antialias_bwd(d["geo_color"], rast, P, tris, d["geo_gc"], terms=t)[0] for t in ("sum", "abs", "count")]
    ddb = [g.interpolate_da_bwd(A, tris, rast, d["geo_h4"], d["geo_gda"], [3, 0, 3], terms=t)[1] for t in ("sum", "abs", "count")]
    assert all(_same(x, dc[0], f64) for x in dc) and all(_same(x, ddb[0], f64) for x in ddb)


def _interp_numpy(attr_shape, tris, rast, g, dt, terms):
    """d attr of interpolate scattered in numpy in pixel, channel, vertex order (np.add.at is sequential in index order)"""
    ids = rast[..., 3].astype(np.int64).reshape(-1) - 1
    m = (ids >= 0) & (ids < tris.shape[0])
    B = rast.shape[0]
    px = np.nonzero(m)[0]
    b = px // (rast[0, ..., 0].size)
    u, v = rast.reshape(-1, 4)[px, 0].astype(dt), rast.reshape(-1, 4)[px, 1].astype(dt)
    w = np.stack([u, v, (dt(1) - u) - v], -1)                               # [P, 3]
    gg = g.reshape(-1, g.shape[-1])[px].astype(dt)                         # [P, C]
    t = w[:, None, :] * gg[:, :, None]                                     # [P, C, 3]
    t = {"sum": t, "abs": np.abs(t), "count": (t != 0).astype(dt)}[terms]
    tri = tris[ids[px]]                                                    # [P, 3]
    Cn = attr_shape[-1]
    V = attr_shape[-2]
    row = np.broadcast_to(tri[:, None, :], t.shape) + (b[:, None, None] * V if len(attr_shape) == 3 else 0)
    ch = np.broadcast_to(np.arange(Cn)[None, :, None], t.shape)
    d = np.zeros((B * V if len(attr_shape) == 3 else V, Cn), dt)
    np.add.at(d, (row.reshape(-1), ch.reshape(-1)), t.reshape(-1))
    return d.reshape(attr_shape)


@PREC
@pytest.mark.parametrize("tag", ["batched", "shared"])
def test_interpolate_bwd_attr_equals_the_numpy_scatter(f64, tag):
    """The sequential scatter in the same order gives the same bits in every mode, and with u, v >= 0, u + v <= 1 and g >= 0 abs is
    the sum."""
    d = _golden()
    g = geometry_oracle(f64)
    _, tris, rast = _geo(d)
    shape = d["geo_attr"].shape if tag == "batched" else d["geo_attr"].shape[1:]
    gc = d["geo_g4"].copy()
    gc[0, 1] = 0.0
    for t in ("sum", "abs", "count"):
        got = g.interpolate_bwd_attr(shape, tris, rast, gc, terms=t)
        assert _same(got, _interp_numpy(shape, tris, rast, gc, g.dt, t), f64), t
    s, a, n = _three(lambda t: g.interpolate_bwd_attr(shape, tris, rast, gc, terms=t))
    _check_stats(s, a, n)
    pos = np.abs(gc)
    assert _same(g.interpolate_bwd_attr(shape, tris, rast, pos), g.interpolate_bwd_attr(shape, tris, rast, pos, terms="abs"), f64)


@PREC
def test_raster_and_interpolate_da_counts_equal_numpy(f64):
    """rasterize d pos: every covered pixel with S != 0 adds one term to x, y and w of its three vertices (generic inputs: none is 0);
    interpolate_da d attr: one term per pixel and selected attribute to each vertex, the third one's counted when a0 or a1 is non-zero."""
    d = _golden()
    g = geometry_oracle(f64)
    pos, tris, rast = _geo(d)
    B = rast.shape[0]
    ids = rast[..., 3].astype(np.int64).reshape(B, -1) - 1
    n = g.raster_bwd(pos, tris, rast, d["geo_g4"], terms="count")
    ref = np.zeros(pos.shape, np.float64)
    for b in range(B):
        live = ids[b][(ids[b] >= 0) & (ids[b] < tris.shape[0])]
        for k in range(3):
            np.add.at(ref[b], (tris[live, k], slice(None)), [1, 1, 0, 1])
    uv = g.raster_bary(pos, tris, rast).reshape(B, -1, 2)
    assert np.array_equal(n, ref) and (uv[(ids >= 0) & (ids < tris.shape[0])] != 0).all()
    sel = [3, 0, 3]
    h = d["geo_h4"].copy()
    h[0, 0, :, :2] = 0.0                                  # a0 = 0 on row 0 of view 0: the third vertex still has a1's term
    gda = d["geo_gda"].copy()
    gda[1, 2] = 0.0                                       # a0 = a1 = 0 on row 2 of view 1
    n = g.interpolate_da_bwd(d["geo_attr"], tris, rast, h, gda, sel, terms="count")[0]
    ref = np.zeros(d["geo_attr"].shape, np.float64)
    gX, gY = gda[..., 0::2].astype(g.dt), gda[..., 1::2].astype(g.dt)
    a0 = gX * h[..., 0:1] + gY * h[..., 1:2]
    a1 = gX * h[..., 2:3] + gY * h[..., 3:4]
    for b in range(B):
        for p in range(ids.shape[1]):
            i = ids[b, p]
            if i < 0 or i >= tris.shape[0]:
                continue
            for k, c in enumerate(sel):
                x0, x1 = a0.reshape(B, -1, 3)[b, p, k], a1.reshape(B, -1, 3)[b, p, k]
                ref[b, tris[i, 0], c] += x0 != 0
                ref[b, tris[i, 1], c] += x1 != 0
                ref[b, tris[i, 2], c] += (x0 != 0) or (x1 != 0)
    assert np.array_equal(n, ref)


@PREC
def test_interpolate_da_third_vertex_abs_is_the_sum_of_both_terms(f64):
    """a0 = -a1 exactly in every pixel: the third vertex's sum is 0 and its abs is |a0| + |a1| = 2 |a0| per pixel"""
    d = _golden()
    g = geometry_oracle(f64)
    _, tris, rast = _geo(d)
    tri1 = np.array([[0, 1, 2]], np.int32)
    r = rast.copy()
    r[..., 3] = 1.0                                        # every pixel on the one triangle
    h = d["geo_h4"].copy()
    h[..., 2:] = -h[..., :2]                               # rast_db's v row = -(its u row): a1 = -a0
    attr = d["geo_attr"][0][:3]
    gda = d["geo_gda"][..., :2]
    s, a, n = _three(lambda t: g.interpolate_da_bwd(attr, tri1, r, h, gda, [1], terms=t)[0])
    a0 = gda[..., 0].astype(g.dt) * h[..., 0].astype(g.dt) + gda[..., 1].astype(g.dt) * h[..., 1].astype(g.dt)
    assert s[2, 1] == 0 and s[0, 1] == -s[1, 1] != 0
    assert a[0, 1] == a[1, 1] and a[2, 1] == 2 * a[0, 1] and n[2, 1] == n[0, 1] == (a0 != 0).sum()
