"""GPU: every float-atomic gradient per element, on the inputs where scatters go wrong -- signed, zero-mean upstream gradients summed into
hot spots, warp groups that are full, ragged, non-contiguous or straddle two images, and interpolate_da's cancelling third-vertex term.

Two rules (tests/common.py):
  * d tex (texture, texel_fetch) and d params (hash grid, MLP texture): the kernel adds the fp32 oracle's own terms in another order, so
    each element is within 2 gamma(n - 1) A (1 + gamma(n)) of the fp32 oracle and bit-identical where it has at most two terms
    (check_scatter_fp32);
  * d pos of rasterize, rast_db and antialias and d attr of interpolate and interpolate_da: the kernel computes its terms in its own
    order, so each element is held to the fp64 oracle with the reduction floor n 2^-24 A (check_scatter_fp64).
Each output prints its worst ratio and largest n.  The geometry ops take rast as an input, so the cases build it directly: one triangle
under every pixel (every lane of every warp has the same key), or ids that alternate lane by lane.

Which cases can see which failure.  Both bars grow with n, so a wrong term is visible where n is small next to the term's share of A:
  * a lost or doubled lane of a warp group: with signed gradients, the lost terms of the biggest hot spots (n ~ 5e4 per vertex) random-walk
    to less than the floor, so the small warp shapes carry it (full, ragged, non-contiguous and straddling groups of a few to 32 lanes);
    with one-signed gradients the lost terms add up coherently (1/32 of A against a floor of n 2^-24 A ~ 3e-3 A), so the one-triangle
    case also runs with positive upstream gradients, and the hash grid's hot cell groups 32 lanes on its dense levels;
  * a wrong tap or weight of the texture and a wrong feature of the hash grid: every element with one or two terms is bit for bit
    (the ragged texture shapes, the unique texels of texel_fetch, the hash grid's sparse entries);
  * a dropped item of texel_fetch: its bench case gives every odd pixel a texel of its own."""
import numpy as np
import pytest
import torch

from common import check_scatter_fp32, check_scatter_fp64, texel_fetch_stats
from oracle.geometry import geometry_oracle
from oracle.hashgrid import REF_CONFIG, hashgrid_oracle
from oracle.mlptexture import mlptexture_oracle
from oracle.texture import chain_shapes, texture_oracle
from nvdiffrecmc_b200 import _lib as L

pytestmark = pytest.mark.gpu
LML = "linear-mipmap-linear"
EDGE = {"otype": "HashGrid", "n_levels": 5, "log2_hashmap_size": 9, "base_resolution": 4, "per_level_scale": 2.0}


def _t(dev, a):
    return torch.tensor(np.ascontiguousarray(a), device=dev)


# ------------------------------------------------------------------------------------------ texture
# (B, H, W): the 512^2 hot spot, B H W % 32 = 1 and 31, and widths that are not a multiple of the kernel's 8 x 4 warp tile
TEX_SHAPES = [(1, 512, 512), (1, 33, 33), (1, 31, 33), (3, 13, 17)]


@pytest.mark.parametrize("bnd", ["wrap", "clamp"])
@pytest.mark.parametrize("shape", TEX_SHAPES, ids=["%dx%dx%d" % s for s in TEX_SHAPES])
def test_texture_hot_spot_signed(dev, shape, bnd):
    """A 4 x 4 chain (4x4, 2x2, 1x1) under the whole image: thousands of signed terms per texel at 512^2; C = 7 with the channel group
    4-5 exactly zero (no reduction issued for it) and one level-0-only region (blend fraction 0)."""
    from nvdiffrecmc_b200.raster import texture
    B, H, W = shape
    rng = np.random.default_rng(H * W + (bnd == "clamp"))
    C = 7
    levels = [rng.normal(size=(1, h, w, C)).astype(np.float32) for h, w in chain_shapes(4, 4, 3)]
    ys, xs = np.meshgrid((np.arange(H) + 0.5) / H, (np.arange(W) + 0.5) / W, indexing="ij")
    uv = np.broadcast_to(np.stack([xs, ys], -1), (B, H, W, 2)).astype(np.float32).copy()
    uv += rng.normal(size=uv.shape).astype(np.float32) * np.float32(0.01)
    da = (rng.normal(size=(B, H, W, 4)) * 2.0 ** rng.uniform(-1, 3, (B, H, W, 1)) / 4).astype(np.float32)
    da[:, : H // 4] = 0.0                                             # lambda 0: level 0 alone
    g = rng.normal(size=(B, H, W, C)).astype(np.float32)
    g[..., 4:6] = 0.0
    g[:, :, : W // 5] = 0.0
    t = [_t(dev, x).requires_grad_(True) for x in levels]
    y = texture(t[0], _t(dev, uv), _t(dev, da), mip=t[1:], filter_mode=LML, boundary_mode=bnd)
    y.backward(_t(dev, g))
    o = texture_oracle()
    rt = [o.backward(levels, uv, da, g, LML, bnd, want_uv=False, want_uv_da=False, terms=m)[0] for m in ("sum", "abs", "count")]
    for k in range(3):
        check_scatter_fp32("texture %s %s d tex level %d" % ("x".join(map(str, shape)), bnd, k), t[k].grad.cpu().numpy(), rt[0][k], rt[1][k],
                           rt[2][k], tag="scatter")
    assert not t[0].grad[..., 4:6].any()
    if shape == (1, 512, 512):
        assert rt[2][2].max() > 1e5 and rt[2][0].max() > 1e4


# ------------------------------------------------------------------------------------------ hash grid and MLP texture
@pytest.mark.parametrize("cfg", [EDGE, REF_CONFIG], ids=["edge", "ref"])
def test_hashgrid_hot_cell_and_faces(dev, cfg):
    """2^18 points inside one cell of the finest dense level (full-warp groups on every dense level), a quarter of them on cell faces of
    the coarser levels, signed gradients, level 1 and the second feature of level 3 zero (the scatter's skip)."""
    from nvdiffrecmc_b200.tinycudann import Encoding
    o = hashgrid_oracle()
    lv = o.levels(cfg)
    dense = [l for l in range(lv["n_levels"]) if (lv["dense_mask"] >> l) & 1]
    s = float(lv["scale"][dense[-1]])
    n = 1 << 18
    rng = np.random.default_rng(len(dense))
    c = np.floor(0.37 * s + 0.5) / s                                           # a cell centre of the finest dense level
    x = (c + rng.uniform(-0.45, 0.45, (n, 3)) / s).astype(np.float32)
    face = (np.round(float(lv["scale"][0]) * 0.37 + 0.5) - 0.5) / float(lv["scale"][0])
    k = rng.integers(0, 4, (n, 3))
    x[k == 0] = np.float32(face)
    x[: 4096] = x[0]                                                            # one exact hot point
    enc = Encoding(3, cfg)
    p = rng.uniform(-1, 1, enc.params.numel()).astype(np.float32)
    with torch.no_grad():
        enc.params.copy_(torch.from_numpy(p))
    dy = rng.normal(size=(n, 2 * lv["n_levels"])).astype(np.float32)
    dy[:, 2:4] = 0.0
    dy[:, 7] = 0.0
    enc(_t(dev, x)).backward(_t(dev, dy))
    r = [o.backward(x, p, lv, dy, want_x=False, terms=m)[0] for m in ("sum", "abs", "count")]
    what = "hashgrid %s d params" % ("edge" if cfg is EDGE else "ref")
    nmax = check_scatter_fp32(what, enc.params.grad.cpu().numpy(), *r, tag="scatter")[1]
    assert nmax >= 4096 and not r[2][2 * int(lv["offset"][1]):2 * int(lv["offset"][2])].any()


def test_mlptexture_one_position(dev):
    """Every point at one position (a warp group of 32 on every dense level) and signed gradients."""
    from nvdiffrecmc_b200.mlptexture import MLPTexture3D
    aabb = np.array([[-1.0, -0.5, -0.8], [1.1, 0.9, 0.7]], np.float32)
    n, Cn = 65536 + 17, 6
    torch.manual_seed(0)
    tex = MLPTexture3D(_t(dev, aabb), channels=Cn, min_max=[torch.zeros(Cn, device=dev), torch.ones(Cn, device=dev)])
    rng = np.random.default_rng(3)
    with torch.no_grad():
        tex.encoder.params.copy_(torch.from_numpy(rng.uniform(-1, 1, tex.encoder.params.numel()).astype(np.float32)))
        for w in tex.net.weights():
            w.copy_(torch.from_numpy(rng.normal(0, 0.4, tuple(w.shape)).astype(np.float32)))
    t = np.broadcast_to(np.float32([0.13, 0.2, -0.31]), (n, 3)).copy()
    g = rng.normal(size=(n, Cn)).astype(np.float32)
    g[::7] = 0.0
    tex.sample(_t(dev, t)).backward(_t(dev, g))
    mo = mlptexture_oracle()
    lv = mo.levels(REF_CONFIG)
    ws = [w.detach().cpu().numpy() for w in tex.net.weights()]
    p = tex.encoder.params.detach().cpu().numpy()
    mm = np.stack([tex.min_max[0].cpu().numpy(), tex.min_max[1].cpu().numpy()])
    r = [mo.mlptex_backward(t, aabb, mm, p, lv, ws, g, want_t=False, want_w=False, terms=m)[0] for m in ("sum", "abs", "count")]
    nmax = check_scatter_fp32("mlptexture d params (one position)", tex.encoder.params.grad.cpu().numpy(), r[0] * 128, r[1] * 128, r[2],
                              tag="scatter")[1]
    assert nmax > 50000


# ------------------------------------------------------------------------------------------ texel_fetch
@pytest.mark.parametrize("shape", [(8, 512, 512), (1, 33, 1), (1, 63, 1)], ids=["bench", "ragged1", "ragged31"])
def test_texel_fetch(dev, shape):
    """bench shape: even pixels onto 64 hot texels (~16 k signed terms each), odd pixels onto a texel of their own (one term, bit for
    bit); the ragged shapes leave B H W % 32 = 1 and 31."""
    from nvdiffrecmc_b200.raster import texel_fetch
    rng = np.random.default_rng(shape[1])
    n = int(np.prod(shape))
    i = np.arange(n)
    idx = np.where(i % 2 == 0, (i // 2) % 64, 64 + i // 2).reshape(shape).astype(np.int64)
    T, Cn = 64 + (n + 1) // 2, 4
    tex = _t(dev, rng.normal(size=(T, Cn)).astype(np.float32)).requires_grad_(True)
    g = rng.normal(size=shape + (Cn,)).astype(np.float32)
    g[..., 3] = 0.0
    texel_fetch(tex, _t(dev, idx)).backward(_t(dev, g))
    s, a, cnt = texel_fetch_stats(T, idx, g)
    nmax = check_scatter_fp32("texel_fetch d tex %s" % "x".join(map(str, shape)), tex.grad.cpu().numpy(), s, a, cnt, tag="scatter")[1]
    assert nmax == (16384 if n == 1 << 21 else 1)


# ------------------------------------------------------------------------------------------ geometry
def _bar(what, got, fn, ins):
    o = lambda f64: geometry_oracle(f64=f64)
    return check_scatter_fp64(what, got, lambda x: [fn(o(True), x, "sum")], lambda x: [fn(o(False), x, "sum")], ins,
                              lambda f64: (fn(o(f64), ins, "count"), fn(o(f64), ins, "abs")), tag="scatter")


def _big_triangle(B, batched):
    """one perspective triangle whose NDC image covers [-1, 1]^2 (vertices at NDC (-1.05, -1.05), (3.5, -1.05), (-1.05, 3.5))"""
    ndc = np.array([[-1.05, -1.05], [3.5, -1.05], [-1.05, 3.5]])
    w = np.array([1.0, 1.3, 0.8])
    pos = np.concatenate([ndc * w[:, None], np.array([[0.1], [0.2], [0.3]]) * w[:, None], w[:, None]], 1)
    pos = np.stack([pos * (1 + 0.05 * b) for b in range(B)]) if batched else pos
    return pos.astype(np.float32), np.array([[0, 1, 2]], np.int32)


def _mesh(rng, B, batched, T=6):
    """T random perspective triangles over the image (w in [0.7, 1.6]), V = 3 T + 2 (two unused vertices)"""
    V = 3 * T + 2
    p = np.concatenate([rng.uniform(-1.6, 1.6, (V, 2)), rng.uniform(-0.3, 0.3, (V, 1))], 1)
    w = rng.uniform(0.7, 1.6, (V, 1))
    pos = np.concatenate([p * w, w], 1)
    if batched:
        pos = np.stack([pos * rng.uniform(0.9, 1.1, (V, 1)) for _ in range(B)])
    return pos.astype(np.float32), rng.permutation(V - 2)[: 3 * T].reshape(T, 3).astype(np.int32)


def _rast(rng, B, H, W, ids):
    """[B,H,W,4] rast: barycentrics in the triangle, depth, id + 1 from `ids`"""
    u = rng.uniform(0, 1, (B, H, W))
    v = rng.uniform(0, 1, (B, H, W)) * (1 - u)
    return np.stack([u, v, rng.uniform(0.1, 0.9, (B, H, W)), ids], -1).astype(np.float32)


def _alternating_ids(B, H, W, T):
    """lane by lane: triangle 0, background, an id >= T, triangle 1, triangle 0, ...: every warp group is non-contiguous"""
    i = np.arange(B * H * W).reshape(B, H, W)
    return np.choose(i % 5, [1, 0, T + 1 + i % 3, 2, 1]).astype(np.float32)


def _geometry_ops(dev, what, pos, tris, rast, rng, db_cancel=False, aa=True, positive=False):
    """rasterize d pos (d rast, and d rast + d rast_db in one launch), interpolate d attr ([V,C] or [B,V,C] like pos), interpolate_da
    d attr and antialias d pos, each per element against the fp64 oracle.  positive: every upstream gradient >= 0 (one-signed), so
    that the terms of a warp group add up coherently."""
    from nvdiffrecmc_b200.raster import antialias, antialias_topology, interpolate
    B, H, W = rast.shape[:3]
    batched = pos.ndim == 3
    V = pos.shape[-2]
    pt, ft, rt = _t(dev, pos), _t(dev, tris), _t(dev, rast)
    draw = (lambda shape: np.abs(rng.normal(size=shape)).astype(np.float32)) if positive else (
        lambda shape: rng.normal(size=shape).astype(np.float32))
    g, h = draw((B, H, W, 4)), draw((B, H, W, 4))
    g[..., 2:] = 0.0
    # rasterize d pos: the C entry points on this rast (as rasterize's backward calls them)
    r_bwd = lambda o, x, t: o.raster_bwd(x[0], tris, rast, x[1], terms=t)
    both_bwd = lambda o, x, t: r_bwd(o, x[:2], t) + o.rast_db_bwd(x[0], tris, rast, x[2], terms=t)
    pa = (pt.data_ptr(), V * 4 if batched else 0, V, ft.data_ptr(), tris.shape[0], rt.data_ptr(), B, H, W)
    one, two = torch.zeros_like(pt), torch.zeros_like(pt)
    gt, ht = _t(dev, g), _t(dev, h)
    L.check(L.lib().mcs_rasterize_bwd(*pa, gt.data_ptr(), one.data_ptr(), L.stream_ptr()), "rasterize (backward)")
    L.check(L.lib().mcs_rasterize_bwd_db(*pa, gt.data_ptr(), ht.data_ptr(), two.data_ptr(), L.stream_ptr()), "rasterize_db (backward)")
    _bar(what + ": rasterize d pos", one.cpu().numpy(), r_bwd, [pos, g])
    _bar(what + ": rasterize_db d pos", two.cpu().numpy(), both_bwd, [pos, g, h])
    # interpolate d attr
    Cn = 5
    attr = rng.uniform(-1, 1, ((B,) if batched else ()) + (V, Cn)).astype(np.float32)
    a = _t(dev, attr).requires_grad_(True)
    gi = draw((B, H, W, Cn))
    gi[..., 2] = 0.0
    interpolate(a, rt, ft)[0].backward(_t(dev, gi))
    _bar(what + ": interpolate d attr", a.grad.cpu().numpy(), lambda o, x, t: o.interpolate_bwd_attr(attr.shape, tris, rast, x[0], terms=t),
         [gi])
    # interpolate_da d attr
    db = rng.normal(size=(B, H, W, 4)).astype(np.float32)
    if db_cancel:                                     # a1 = -(1 + 2^-10 r) a0: the third vertex's term cancels down to ~1e-3 of |a0|
        db[..., 2:] = (-db[..., :2] * (1 + rng.uniform(-1, 1, (B, H, W, 1)) * 2.0 ** -10)).astype(np.float32)
    sel = [4, 0, 4]
    a2 = _t(dev, attr).requires_grad_(True)
    _, da = interpolate(a2, rt, ft, rast_db=_t(dev, db), diff_attrs=sel)
    gda = draw(tuple(da.shape))
    da.backward(_t(dev, gda))
    nmax = _bar(what + ": interpolate_da d attr", a2.grad.cpu().numpy(),
                lambda o, x, t: o.interpolate_da_bwd(attr, tris, rast, x[0], x[1], sel, terms=t)[0], [db, gda])[1]
    # antialias d pos
    if aa:
        col = rng.uniform(-1, 2, (B, H, W, 3)).astype(np.float32)
        gc = rng.normal(size=col.shape).astype(np.float32)
        p = _t(dev, pos).requires_grad_(True)
        antialias(_t(dev, col), rt, p, ft, antialias_topology(ft)).backward(_t(dev, gc))
        _bar(what + ": antialias d pos", p.grad.cpu().numpy(),
             lambda o, x, t: o.antialias_bwd(col, rast, x[0], tris, x[1], scatter=True, terms=t)[1], [pos, gc])
    return nmax


@pytest.mark.parametrize("sign", ["signed", "positive"])
@pytest.mark.parametrize("batched", [False, True], ids=["shared_pos", "batched_pos"])
def test_one_triangle_under_every_pixel(dev, batched, sign):
    """every lane of every warp has the same key (image, triangle): groups of 32 and n = H W (B H W with one [V,4] pos) per vertex;
    signed, zero-mean upstream gradients, or one-signed ones, under which a lost or doubled lane adds up over the whole image"""
    rng = np.random.default_rng(1 + batched + 2 * (sign == "positive"))
    B, H, W = 2, 256, 192
    pos, tris = _big_triangle(B, batched)
    rast = _rast(rng, B, H, W, np.ones((B, H, W)))
    nmax = _geometry_ops(dev, "one triangle %s %s" % ("[B,V,4]" if batched else "[V,4]", sign), pos, tris, rast, rng, aa=False,
                         positive=sign == "positive")
    assert nmax >= H * W
    # S != 0 everywhere: the triangle covers the image
    assert (geometry_oracle().raster_bary(pos, tris, rast) != 0).all(-1).mean() > 0.99


def test_interpolate_da_cancelling_third_vertex(dev):
    """rast_db with (du/dX, du/dY) = -(dv/dX, dv/dY)(1 + 2^-10 r): a0 ~ -a1 in every pixel, so the third vertex's sum -(A0 + A1) of
    the group sums is ~1e-3 of its floor's |a0| + |a1|"""
    rng = np.random.default_rng(9)
    pos, tris = _big_triangle(2, False)
    _geometry_ops(dev, "cancelling rast_db", pos, tris, _rast(rng, 2, 96, 64, np.ones((2, 96, 64))), rng, db_cancel=True, aa=False)


# (B, H, W): B H W % 32 = 1 and 31; H W % 32 != 0, so warps straddle two images
WARP_SHAPES = [(1, 11, 3), (1, 7, 9), (3, 13, 17), (4, 5, 7)]


@pytest.mark.parametrize("batched", [False, True], ids=["shared_pos", "batched_pos"])
@pytest.mark.parametrize("shape", WARP_SHAPES, ids=["%dx%dx%d" % s for s in WARP_SHAPES])
def test_warp_shapes(dev, shape, batched):
    """ragged last warps and warps across two images of one triangle id (B H W % 32, H W % 32 != 0), both with one triangle under every
    pixel and with ids alternating lane by lane between two triangles, background and ids >= T; antialias on a random mesh's ids"""
    B, H, W = shape
    rng = np.random.default_rng(B * H * W + batched)
    pos, tris = _big_triangle(B, batched)
    _geometry_ops(dev, "%dx%dx%d one triangle" % shape, pos, tris, _rast(rng, B, H, W, np.ones((B, H, W))), rng, aa=False)
    pos, tris = _mesh(rng, B, batched)
    ids = _alternating_ids(B, H, W, tris.shape[0])
    _geometry_ops(dev, "%dx%dx%d alternating ids" % shape, pos, tris, _rast(rng, B, H, W, ids), rng)
    rnd = rng.integers(0, tris.shape[0] + 3, (B, H, W)).astype(np.float32)
    _geometry_ops(dev, "%dx%dx%d random ids" % shape, pos, tris, _rast(rng, B, H, W, rnd), rng)
