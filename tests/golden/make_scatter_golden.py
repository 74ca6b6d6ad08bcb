"""Freeze the oracle's scattered gradients -- d tex, d params (hash grid and MLP texture), rasterize / rast_db / antialias d pos and
interpolate_da d attr -- on small seeded cases, in both precisions, into scatter_sums.npz.  The file was written before the oracle's
scatter entry points took their `terms` argument, so tests/test_oracle_scatter_terms.py can check that terms="sum" (the default) still
sums exactly what they summed.  Run from the repository root: python tests/golden/make_scatter_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle.geometry import geometry_oracle  # noqa: E402
from oracle.hashgrid import REF_CONFIG, hashgrid_oracle  # noqa: E402
from oracle.mlptexture import mlptexture_oracle  # noqa: E402
from oracle.texture import chain_shapes, texture_oracle  # noqa: E402

EDGE = {"otype": "HashGrid", "n_levels": 5, "log2_hashmap_size": 9, "base_resolution": 4, "per_level_scale": 2.0}


def inputs():
    """The seeded inputs of every case (numpy, fp32 / int32)."""
    rng = np.random.default_rng(2024)
    d = {}
    # texture: a 3-level chain of 8 x 12, C = 3, signed gradients
    for k, (h, w) in enumerate(chain_shapes(8, 12, 3)):
        d["tex_l%d" % k] = rng.normal(size=(1, h, w, 3)).astype(np.float32)
    d["tex_uv"] = rng.uniform(-0.3, 1.3, (2, 5, 7, 2)).astype(np.float32)
    d["tex_da"] = (rng.normal(size=(2, 5, 7, 4)) * 2.0 ** rng.uniform(-1, 3, (2, 5, 7, 1)) / np.array([12, 12, 8, 8])).astype(np.float32)
    d["tex_g"] = rng.normal(size=(2, 5, 7, 3)).astype(np.float32)
    d["tex_g"][0, 1] = 0.0
    # hash grid: 300 points of a 5-level grid, level 2's gradient zero
    d["hg_x"] = rng.uniform(-0.1, 1.1, (300, 3)).astype(np.float32)
    lv = hashgrid_oracle().levels(EDGE)
    d["hg_p"] = rng.uniform(-1, 1, 2 * int(lv["offset"][-1])).astype(np.float32)
    d["hg_g"] = rng.normal(size=(300, 10)).astype(np.float32)
    d["hg_g"][:, 4:6] = 0.0
    # MLP texture: 64 points, one hidden layer, C = 3, the reference's grid
    d["mt_t"] = rng.uniform(-1.2, 1.2, (64, 3)).astype(np.float32)
    d["mt_w0"] = rng.normal(0, 0.4, (32, 32)).astype(np.float32)
    d["mt_w1"] = rng.normal(0, 0.4, (3, 32)).astype(np.float32)
    d["mt_g"] = rng.normal(size=(64, 3)).astype(np.float32)
    # geometry: 12 random triangles over a 2 x 6 x 9 image with a synthetic rast (background, ids >= T, random barycentrics and depth)
    V, T, B, H, W = 20, 12, 2, 6, 9
    pos = np.concatenate([rng.uniform(-1, 1, (B, V, 2)), rng.uniform(-0.5, 0.5, (B, V, 1)), rng.uniform(0.5, 2, (B, V, 1))], -1)
    d["geo_pos"] = pos.astype(np.float32)
    d["geo_tris"] = rng.integers(0, V, (T, 3)).astype(np.int32)
    rast = np.concatenate([rng.uniform(0, 0.5, (B, H, W, 2)), rng.uniform(0, 1, (B, H, W, 1)), rng.integers(0, T + 3, (B, H, W, 1))], -1)
    d["geo_rast"] = rast.astype(np.float32)
    d["geo_attr"] = rng.uniform(-1, 1, (B, V, 4)).astype(np.float32)
    d["geo_g4"] = rng.normal(size=(B, H, W, 4)).astype(np.float32)
    d["geo_h4"] = rng.normal(size=(B, H, W, 4)).astype(np.float32)
    d["geo_color"] = rng.uniform(0, 1, (B, H, W, 3)).astype(np.float32)
    d["geo_gc"] = rng.normal(size=(B, H, W, 3)).astype(np.float32)
    d["geo_gda"] = rng.normal(size=(B, H, W, 6)).astype(np.float32)
    return d


def outputs(d, f64):
    """Every scattered gradient of the cases, from the oracle at one precision: {name: array}; the MLP texture's d params as the indices
    and values of its non-zero entries."""
    sfx = "_f64" if f64 else "_f32"
    out = {}
    levels = [d["tex_l%d" % k] for k in range(3)]
    o = texture_oracle(f64)
    for filt, bnd in (("linear-mipmap-linear", "wrap"), ("linear", "clamp")):
        dt, _, _ = o.backward(levels, d["tex_uv"], d["tex_da"], d["tex_g"], filt, bnd)
        for k, x in enumerate(dt):
            out["tex_%s_%s_l%d%s" % (filt, bnd, k, sfx)] = x
    h = hashgrid_oracle(f64)
    out["hg_dp" + sfx] = h.backward(d["hg_x"], d["hg_p"], h.levels(EDGE), d["hg_g"], want_x=False)[0]
    m = mlptexture_oracle(f64)
    lv = m.levels(REF_CONFIG)
    p = np.random.default_rng(7).uniform(-1, 1, 2 * int(lv["offset"][-1])).astype(np.float32)
    aabb = np.array([[-1, -1, -1], [1, 1, 1]], np.float32)
    mm = np.array([[-0.1, 0.0, 0.2], [0.9, 1.0, 1.1]], np.float32)
    dp = m.mlptex_backward(d["mt_t"], aabb, mm, p, lv, [d["mt_w0"], d["mt_w1"]], d["mt_g"], want_t=False, want_w=False)[0]
    nz = np.flatnonzero(dp)
    out["mt_dp_idx" + sfx], out["mt_dp_val" + sfx] = nz.astype(np.int64), dp[nz]
    g = geometry_oracle(f64)
    pos, tris, rast = d["geo_pos"], d["geo_tris"], d["geo_rast"]
    for tag, P in (("batched", pos), ("shared", pos[0])):
        out["raster_%s%s" % (tag, sfx)] = g.raster_bwd(P, tris, rast, d["geo_g4"])
        out["rast_db_%s%s" % (tag, sfx)] = g.rast_db_bwd(P, tris, rast, d["geo_h4"])
        dc, dpos = g.antialias_bwd(d["geo_color"], rast, P, tris, d["geo_gc"])
        out["aa_%s%s" % (tag, sfx)] = dpos
    for tag, A in (("batched", d["geo_attr"]), ("shared", d["geo_attr"][0])):
        da, _ = g.interpolate_da_bwd(A, tris, rast, d["geo_h4"], d["geo_gda"], [3, 0, 3])
        out["da_%s%s" % (tag, sfx)] = da
    return out


if __name__ == "__main__":
    d = inputs()
    res = dict(d)
    for f64 in (False, True):
        res.update(outputs(d, f64))
    path = os.path.join(HERE, "scatter_sums.npz")
    np.savez_compressed(path, **res)
    print("wrote %s: %d arrays, %d bytes" % (path, len(res), os.path.getsize(path)))
