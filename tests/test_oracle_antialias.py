"""CPU: the oracle's restatement of the geometry-gradient ops (rasterize / interpolate backward, edge adjacency, analytic antialias).
Adjacency against a plain dictionary construction, hand-derived adjoints against fp64 finite differences, and the antialias semantics
against geometry: on one large triangle the antialiased coverage sums to the triangle's screen area and its gradient is the area's."""
import numpy as np
import pytest

from common import rel_l2
from nvdiffrecmc_b200 import synth
from oracle.geometry import geometry_oracle


@pytest.fixture(scope="module")
def geo():
    return geometry_oracle()


@pytest.fixture(scope="module")
def geo64():
    return geometry_oracle(f64=True)


def dict_topology(f):
    edges = {}
    for t, tri in enumerate(f):
        for k in range(3):
            a, b = int(tri[k]), int(tri[(k + 1) % 3])
            edges.setdefault((min(a, b), max(a, b)), []).append(t)
    adj = np.empty(f.shape, np.int32)
    for t, tri in enumerate(f):
        for k in range(3):
            a, b = int(tri[k]), int(tri[(k + 1) % 3])
            lst = edges[(min(a, b), max(a, b))]
            adj[t, k] = -1 if len(lst) == 1 else (-2 if len(lst) >= 3 else (lst[1] if lst[0] == t else lst[0]))
    return adj


def _meshes():
    ico = synth.icosphere(3)
    bt = synth.scene_mesh("blob+torus", level=2)
    out = {"icosphere3": (ico[0].astype(np.float32), ico[1].astype(np.int32)), "blob+torus": bt}
    rng = np.random.default_rng(3)
    for name in list(out):
        v, f = out[name]
        keep = rng.random(f.shape[0]) > 0.1
        out[name + "-holes"] = (v, f[keep])
    out["fan"] = (np.zeros((5, 3), np.float32), np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [2, 1, 4]], np.int32))
    return out


@pytest.mark.parametrize("name", ["icosphere3", "blob+torus", "icosphere3-holes", "blob+torus-holes", "fan"])
def test_topology_matches_dict_construction(geo, name):
    v, f = _meshes()[name]
    adj = geo.aa_topology(f)
    assert np.array_equal(adj, dict_topology(f))
    if name == "fan":
        assert adj[0, 0] == -2 and adj[1, 0] == -2 and adj[2, 0] == -2 and adj[3, 0] == 0 and adj[0, 1] == 3
    if name.endswith("holes"):
        assert (adj == -1).any()
    else:
        assert (adj >= 0).all() or name == "fan"
    # only the set of triangles on an edge matters: a permuted triangle list gives the permuted answer
    perm = np.random.default_rng(1).permutation(f.shape[0])
    inv = np.argsort(perm)
    adj_p = geo.aa_topology(f[perm])
    mapped = np.where(adj_p >= 0, perm[np.maximum(adj_p, 0)], adj_p)
    assert np.array_equal(mapped[inv], adj)


# ------------------------------------------------------------------------------------------------ a CPU z-buffer for the tests
def _perspective(fovy=0.7854, n=0.1, f=10.0):
    y = np.tan(fovy / 2)
    return np.array([[1 / y, 0, 0, 0], [0, 1 / -y, 0, 0], [0, 0, -(f + n) / (f - n), -(2 * f * n) / (f - n)], [0, 0, -1, 0]])


def _view(ang, dist=3.0):
    mv = np.eye(4)
    mv[:3, :3] = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
    mv[2, 3] = -dist
    return _perspective() @ mv


def zbuffer(pos, f, H, W):
    """rast [B,H,W,4] (u, v, z/w, id + 1) of clip-space vertices pos [B,V,4] by brute force (fp64)."""
    pos = np.asarray(pos, np.float64)
    B = pos.shape[0]
    px = (np.arange(W) + 0.5) / W * 2 - 1
    py = (np.arange(H) + 0.5) / H * 2 - 1
    PX, PY = np.meshgrid(px, py)
    rast = np.zeros((B, H, W, 4))
    depth = np.full((B, H, W), np.inf)
    for b in range(B):
        for t, tri in enumerate(f):
            q = pos[b, tri]
            if (q[:, 3] <= 0).any():
                continue
            ax = q[:, 0][:, None, None] - PX * q[:, 3][:, None, None]
            ay = q[:, 1][:, None, None] - PY * q[:, 3][:, None, None]
            s0 = ax[1] * ay[2] - ay[1] * ax[2]; s1 = ax[2] * ay[0] - ay[2] * ax[0]; s2 = ax[0] * ay[1] - ay[0] * ax[1]
            S = s0 + s1 + s2
            with np.errstate(divide="ignore", invalid="ignore"):
                u, v = s0 / S, s1 / S
                w2 = 1 - u - v
                inside = (S != 0) & (u >= 0) & (v >= 0) & (w2 >= 0)
                zw = (u * q[0, 2] + v * q[1, 2] + w2 * q[2, 2]) / (u * q[0, 3] + v * q[1, 3] + w2 * q[2, 3])
            m = inside & (zw < depth[b]) & (zw > -1)
            depth[b][m] = zw[m]
            rast[b][m] = np.stack([u[m], v[m], zw[m], np.full(m.sum(), t + 1.0)], -1)
    return rast


def _scene(B=2, res=24, level=1):
    v, f = synth.icosphere(level)
    v = v * (1 + 0.15 * np.sin(3 * v[:, :1]) * np.cos(2 * v[:, 1:2]))       # not a sphere: some edges face away, some do not
    f = f.astype(np.int32)
    vh = np.concatenate([v, np.ones((v.shape[0], 1))], 1)
    pos = np.stack([vh @ _view(0.4 + 0.9 * b).T for b in range(B)])
    return pos, f, zbuffer(pos, f, res, res)


def _fd(fn, x, eps=1e-6):
    g = np.zeros_like(x)
    for idx in np.ndindex(x.shape):
        xp = x.copy(); xp[idx] += eps
        xm = x.copy(); xm[idx] -= eps
        g[idx] = (fn(xp) - fn(xm)) / (2 * eps)
    return g


def test_barycentrics_adjoint_matches_finite_differences(geo64):
    pos, f, rast = _scene()
    uv = geo64.raster_bary(pos, f, rast)
    m = rast[..., 3] > 0
    assert m.sum() > 300
    assert np.abs(uv[m] - rast[m][:, :2]).max() < 1e-9            # the z-buffer's barycentrics are the formula's
    g = np.random.default_rng(0).standard_normal(rast.shape[:3] + (2,))
    d_rast = np.concatenate([g, np.ones_like(g)], -1)              # z/w and id channels carry no gradient
    for p in (pos, pos[0]):                                        # [B,V,4] and a shared [V,4]
        r = rast if p.ndim == 3 else rast[:1]
        dr = d_rast if p.ndim == 3 else d_rast[:1]
        ana = geo64.raster_bwd(p, f, r, dr)
        num = _fd(lambda x: float((geo64.raster_bary(x, f, r) * dr[..., :2]).sum()), p)
        assert rel_l2(ana, num) < 1e-6


def test_interpolate_rast_adjoint_matches_numpy(geo64):
    pos, f, rast = _scene()
    rng = np.random.default_rng(1)
    attr = rng.random((pos.shape[1], 5))
    g = rng.standard_normal(rast.shape[:3] + (5,))
    d = geo64.interpolate_bwd_rast(attr, f, rast, g)
    ids = rast[..., 3].astype(np.int64) - 1
    A = attr[f[np.maximum(ids, 0)]]                                  # [B,H,W,3,5]
    ref = np.stack([((A[..., 0, :] - A[..., 2, :]) * g).sum(-1), ((A[..., 1, :] - A[..., 2, :]) * g).sum(-1)], -1) * (ids >= 0)[..., None]
    assert np.abs(d[..., :2] - ref).max() < 1e-12 and (d[..., 2:] == 0).all()


@pytest.mark.parametrize("C", [1, 3])
def test_antialias_adjoints_match_finite_differences(geo64, C):
    pos, f, rast = _scene()
    rng = np.random.default_rng(2)
    color = rng.random(rast.shape[:3] + (C,))
    g = rng.standard_normal(color.shape)
    adj = geo64.aa_topology(f)
    out = geo64.antialias(color, rast, pos, f, adj)
    assert np.abs(out - color).max() > 1e-3                          # some pixels are blended
    dc, dp = geo64.antialias_bwd(color, rast, pos, f, g, adj)
    assert np.abs(dp).max() > 0
    num_p = _fd(lambda x: float((geo64.antialias(color, rast, x, f, adj) * g).sum()), pos)
    assert rel_l2(dp, num_p) < 1e-6
    num_c = _fd(lambda x: float((geo64.antialias(x, rast, pos, f, adj) * g).sum()), color)
    assert rel_l2(dc, num_c) < 1e-6


# ------------------------------------------------------------------------------------------------ area property
def _screen_area(pos, H, W):
    X = (pos[:, 0] / pos[:, 3] + 1) * W / 2
    Y = (pos[:, 1] / pos[:, 3] + 1) * H / 2
    return 0.5 * ((X[1] - X[0]) * (Y[2] - Y[0]) - (X[2] - X[0]) * (Y[1] - Y[0]))


def _random_triangle(rng, H, W):
    while True:
        ndc = rng.uniform(-0.9, 0.9, (3, 2))
        pix = (ndc + 1) * np.array([W, H]) / 2
        if min(np.linalg.norm(pix[k] - pix[(k + 1) % 3]) for k in range(3)) < 100:
            continue
        w = rng.uniform(0.5, 2.0, 3)
        z = rng.uniform(-0.5, 0.5, 3) * w
        return np.concatenate([ndc * w[:, None], z[:, None], w[:, None]], 1)


def test_antialias_area_property(geo64):
    """Coverage mask of one large triangle on background, antialiased: the sum is the exact screen area (+-1 % from the one-row
    discretisation per edge) and its gradient the analytic area gradient (+-5 %), over random triangles, perspective w and both windings."""
    rng = np.random.default_rng(7)
    H = W = 256
    f = np.array([[0, 1, 2]], np.int32)
    errs_a, errs_g = [], []
    for trial in range(8):
        pos = _random_triangle(rng, H, W)
        if trial % 2:
            pos = pos[[0, 2, 1]]
        rast = zbuffer(pos[None], f, H, W)
        mask = (rast[..., 3:4] > 0).astype(np.float64)
        out = geo64.antialias(mask, rast, pos, f)
        area = abs(_screen_area(pos, H, W))
        errs_a.append(abs(out.sum() - area) / area)
        _, dp = geo64.antialias_bwd(mask, rast, pos, f, np.ones_like(mask))
        ana = _fd(lambda x: abs(_screen_area(x, H, W)), pos, eps=1e-7)
        errs_g.append(rel_l2(dp, ana))
    assert max(errs_a) < 0.01, errs_a
    assert max(errs_g) < 0.05, errs_g
