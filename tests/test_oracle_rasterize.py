"""CPU: the oracle's restatement of k_invert4 / k_rasterize (oracle/mcoracle.c orc_invert4, orc_rasterize).  The fp32 build is the
one the GPU is held to bit for bit (tests/test_gpu_rasterize_exact.py); here the inverse is checked against numpy, and the fp64 build
against the geometry it stands for: hit points on the pixel rays, barycentrics of the clip-space triangle, depths inside the frustum,
and peel layers beyond the previous layer's separation."""
import numpy as np
import pytest

from common import oracle, pixel_grid_mesh, raster_mesh, raster_mtx
from oracle import peel_sep
from oracle.geometry import geometry_oracle
from nvdiffrecmc_b200 import synth


def _well_conditioned(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        m = rng.normal(size=(4, 4)) + 3.0 * np.eye(4)
        if np.linalg.cond(m) < 8:
            out.append(m)
    return np.stack(out).astype(np.float32)


def test_invert4_within_one_ulp_of_numpy():
    o = oracle()
    m = np.concatenate([_well_conditioned(300, 1), raster_mtx("persp", 8), raster_mtx("offaxis", 8), raster_mtx("ortho", 8)])
    got = o.invert4(m)
    ref = np.linalg.inv(m.astype(np.float64))
    assert got.dtype == np.float32
    ulp = np.spacing(np.abs(ref.astype(np.float32)))
    tiny = np.abs(ref) < 1e-6 * np.abs(ref).max(axis=(1, 2), keepdims=True)           # entries that are zero in exact arithmetic
    err = np.abs(got.astype(np.float64) - ref)
    assert (err[~tiny] <= ulp[~tiny]).all(), err[~tiny].max()
    assert (err[tiny] <= 1e-6 * np.abs(ref).max()).all()


def test_invert4_exact_cases():
    o = oracle()
    rng = np.random.default_rng(2)
    perms = np.stack([np.eye(4, dtype=np.float32)[rng.permutation(4)] for _ in range(12)])
    assert np.array_equal(o.invert4(perms), perms.transpose(0, 2, 1))
    diag = np.stack([np.diag(rng.uniform(0.1, 10, 4) * rng.choice([-1, 1], 4)) for _ in range(12)]).astype(np.float32)
    ref = np.zeros_like(diag)
    for k in range(4):
        ref[:, k, k] = (1.0 / diag[:, k, k].astype(np.float64)).astype(np.float32)    # double rounding is exact for a quotient of floats
    assert np.array_equal(o.invert4(diag), ref)
    pd = (perms * np.exp2(rng.integers(-6, 7, (12, 1, 4)))).astype(np.float32)          # permutation times powers of two
    assert np.array_equal(o.invert4(pd), np.linalg.inv(pd.astype(np.float64)).astype(np.float32))
    m = _well_conditioned(20, 3)
    for e in (-5, 3):                                                                   # scaling by 2^e scales the inverse by 2^-e
        assert np.array_equal(o.invert4(m * np.float32(2.0 ** e)), o.invert4(m) * np.float32(2.0 ** -e))


def test_invert4_singular_is_not_finite():
    o = oracle()
    m = raster_mtx("singular", 3)                       # all zeros, then a zero w row
    zc = raster_mtx("persp", 1)[0].copy(); zc[:, 1] = 0  # a zero column
    inv = o.invert4(np.concatenate([m, zc[None]]))
    for k in range(inv.shape[0]):
        assert not np.isfinite(inv[k]).any(), (k, inv[k])


def _geom(f64, mesh, cam, B=2, res=(40, 56)):
    o = oracle(f64)
    v, f = raster_mesh(mesh)
    mtx = raster_mtx(cam, B, aspect=res[1] / res[0])
    return o, o.scene(v, f), v, f, mtx, res


@pytest.mark.parametrize("cam", ["persp", "offaxis", "ortho", "wide", "inside"])
def test_hit_points_reproject_to_pixel_centres(cam):
    o, sc, v, f, mtx, (H, W) = _geom(True, "blob+torus", cam)
    rast, t = sc.rasterize(mtx, (H, W))
    tid = rast[..., 3].astype(np.int64) - 1
    hit = tid >= 0
    assert hit.sum() > 300
    w = np.stack([rast[..., 0], rast[..., 1], 1.0 - rast[..., 0] - rast[..., 1]], -1)   # weights of vertices 0, 1, 2
    p = np.einsum("bhwk,bhwkc->bhwc", w, v.astype(np.float64)[f[np.maximum(tid, 0)]])
    clip = np.einsum("bij,bhwj->bhwi", mtx.astype(np.float64), np.concatenate([p, np.ones(p.shape[:-1] + (1,))], -1))
    ndc = clip[..., :2] / clip[..., 3:]
    px = (np.arange(W) + 0.5) / W * 2 - 1; py = (np.arange(H) + 0.5) / H * 2 - 1
    assert np.abs(ndc[..., 0] - px[None, None, :])[hit].max() < 1e-9
    assert np.abs(ndc[..., 1] - py[None, :, None])[hit].max() < 1e-9
    assert np.abs(rast[..., 2] - clip[..., 2] / clip[..., 3])[hit].max() < 1e-9        # z/w of that point
    assert (rast[~hit] == 0).all() and np.isinf(t[~hit]).all() and (t[hit] > 0).all()


@pytest.mark.parametrize("cam", ["persp", "offaxis", "ortho"])
def test_barycentrics_are_those_of_the_clip_space_triangle(cam):
    o, sc, v, f, mtx, res = _geom(True, "blob+torus", cam)
    rast, _ = sc.rasterize(mtx, res)
    pos = np.einsum("bij,vj->bvi", mtx.astype(np.float64), np.concatenate([v, np.ones((v.shape[0], 1))], 1))
    uv = geometry_oracle(f64=True).raster_bary(pos, f, rast)
    tid = rast[..., 3].astype(np.int64) - 1
    hit = tid >= 0
    # grazing pixels (ray nearly in the triangle's plane) are ill-conditioned in both formulas; compare the others
    tv = v.astype(np.float64)[f[np.maximum(tid, 0)]]
    n = np.cross(tv[..., 1, :] - tv[..., 0, :], tv[..., 2, :] - tv[..., 0, :])
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    inv = np.linalg.inv(mtx.astype(np.float64))
    H, W = res
    px = (np.arange(W) + 0.5) / W * 2 - 1; py = (np.arange(H) + 0.5) / H * 2 - 1
    X, Y = np.meshgrid(px, py)
    near = np.einsum("bij,hwj->bhwi", inv, np.stack([X, Y, -np.ones_like(X), np.ones_like(X)], -1))
    far = np.einsum("bij,hwj->bhwi", inv, np.stack([X, Y, np.ones_like(X), np.ones_like(X)], -1))
    d = far[..., :3] / far[..., 3:] - near[..., :3] / near[..., 3:]
    cosang = np.abs((n * d).sum(-1)) / np.linalg.norm(d, axis=-1)
    ok = hit & (cosang > 0.05)
    assert ok.sum() > 300 and ok.sum() > 0.9 * hit.sum()
    assert np.abs(rast[..., :2] - uv)[ok].max() < 1e-9


@pytest.mark.parametrize("cam", ["persp", "wide", "ortho", "inside"])
def test_depth_lies_in_the_frustum_and_grows_along_the_ray(cam):
    o, sc, v, f, mtx, res = _geom(True, "blob+torus", cam)
    t_state, prev_z, n_layers = None, None, 0
    for k in range(12):
        rast, t_new = sc.rasterize(mtx, res, t_state)
        hit = rast[..., 3] > 0
        if not hit.any():
            break
        n_layers += 1
        z = rast[..., 2]
        assert (z[hit] >= -1 - 1e-12).all() and (z[hit] <= 1 + 1e-12).all()            # the whole mesh lies between near and far
        if t_state is not None:
            assert not (hit & np.isinf(t_state)).any()
            both = hit & (prev_z != 0)
            assert (t_new[hit] > t_state[hit] * (1 + 2.0 ** -16)).all()                   # beyond sep(t_prev)
            assert (z[both] > prev_z[both]).all()
        t_state, prev_z = t_new, np.where(hit, z, 0.0)
    assert n_layers >= 3


def test_peel_layers_fp32_beyond_separation():
    o, sc, v, f, mtx, res = _geom(False, "blob+torus", "persp", B=3)
    t_state = None
    layers = 0
    while True:
        rast, t_new = sc.rasterize(mtx, res, t_state)
        assert rast.dtype == np.float32 and t_new.dtype == np.float32
        hit = rast[..., 3] > 0
        if t_state is not None:
            fin = np.isfinite(t_state) & hit
            assert (t_new[fin] > peel_sep(t_state[fin])).all()
            assert np.isinf(t_new[~hit]).all()
        if not hit.any():
            break
        t_state = t_new
        layers += 1
        assert layers < 16
    assert layers >= 3
    # layer 0 is the plain closest hit on the same rays: the peel query with t_after = 0
    r0, _ = sc.rasterize(mtx, res)
    r1, _ = sc.rasterize(mtx, res, np.zeros(r0.shape[:3], np.float32))
    assert np.array_equal(r0, r1)


def test_pixel_subset_equals_full_image():
    o, sc, v, f, mtx, res = _geom(False, "blob+torus", "offaxis", B=3)
    full, t_full = sc.rasterize(mtx, res)
    px = np.random.default_rng(0).choice(full[..., 0].size, 500, replace=False)
    sub, t_sub = sc.rasterize(mtx, res, px=px)
    assert np.array_equal(sub, full.reshape(-1, 4)[px]) and np.array_equal(t_sub, t_full.reshape(-1)[px])
    full2, _ = sc.rasterize(mtx, res, t_full)
    sub2, _ = sc.rasterize(mtx, res, t_sub, px=px)
    assert np.array_equal(sub2, full2.reshape(-1, 4)[px])


def test_pixel_aligned_grid_ties_go_to_the_lowest_id():
    H, W = 33, 47
    v, f = pixel_grid_mesh(H, W)
    sc = oracle().scene(v, f)
    rast, t = sc.rasterize(np.eye(4, dtype=np.float32)[None], (H, W))
    tid = rast[0, ..., 3].astype(np.int64) - 1
    ys, xs = np.nonzero(tid >= 0)
    assert ys.size > 0.8 * (H - 1) * (W - 1)
    for y, x in zip(ys[::7], xs[::7]):
        px = ((np.float32(x) + np.float32(0.5)) / np.float32(W) * np.float32(2) - np.float32(1))
        py = ((np.float32(y) + np.float32(0.5)) / np.float32(H) * np.float32(2) - np.float32(1))
        ts, ids = sc.all_hits(np.float32([px, py, -1]), np.float32([0, 0, 2]))
        assert ids.size >= 1 and tid[y, x] == ids[ts == ts[0]].min()
    # vertices on even pixel centres: many pixels are hit by more than one triangle at the same t
    multi = sum(sc.all_hits(np.float32([((x + 0.5) / W) * 2 - 1, ((y + 0.5) / H) * 2 - 1, -1]), np.float32([0, 0, 2]))[0].size > 1
                for y in range(0, H - 1, 2) for x in range(0, W - 1, 2))
    assert multi > 50


def test_surface_beyond_the_far_plane_is_returned():
    """k_rasterize searches the line of the near-far segment (t up to 1e16), so a surface beyond the far plane is a hit with
    z/w > 1; nvdiffrast would clip it."""
    sc = oracle().scene(*raster_mesh("far"))
    rast, t = sc.rasterize(raster_mtx("front", 2), (32, 32))
    far = rast[..., 3] > 0
    beyond = far & (rast[..., 2] > 1)
    assert beyond.sum() > 200 and (t[beyond] > 1).all()
    assert (rast[..., 3][beyond] > raster_mesh("blob+torus")[1].shape[0]).all()        # the quad's two triangles come last


def test_near_plane_cuts_the_surface_for_an_eye_inside_the_mesh():
    """The `inside` camera's near plane (0.5 from an eye inside the blob) passes through the surface: surface closer than the near
    plane is not returned, so a nearer near plane changes what those pixels see."""
    v, f = raster_mesh("blob+torus")
    sc = oracle().scene(v, f)
    m = raster_mtx("inside", 2)
    rot = np.stack([synth.orbit_view(0.7 * b + 0.3, radius=0.0, tilt=-0.4 + 0.15 * b) for b in range(2)])
    m_near = (synth.perspective(fovy=1.2, n=0.05, f=10.0).astype(np.float64) @ rot).astype(np.float32)
    a, ta = sc.rasterize(m, (40, 40))
    b, tb = sc.rasterize(m_near, (40, 40))
    assert (a[..., 3] != b[..., 3]).sum() > 20
