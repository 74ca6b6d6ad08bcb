"""Developer tool: tiny end-to-end pass of every kernel family, meant to run under compute-sanitizer
(memcheck / racecheck / initcheck) -- SURVEY.md section 5 "race detection"."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from common import make_case
import nvdiffrecmc_b200.optixutils as ou
import nvdiffrecmc_b200.renderutils as ru

dev = torch.device("cuda:0")
for N in (4, 9):
    c = make_case(res=12, B=2, N=N, perm_rows=64)
    t = lambda k: torch.tensor(c[k], device=dev)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, t("verts"), t("tris"), 1)
    pos, kd, ks, light = [t(k).requires_grad_(True) for k in ("pos", "kd", "ks", "light")]
    nrm = ru.prepare_shading_normal(pos, t("view"), None, t("smooth_nrm"), t("tangent"), t("geom_nrm"))
    d, s = ou.optix_env_shade(ctx, t("mask"), t("ro"), pos, nrm, t("view"), kd, ks, light, t("pdf"), t("rows"), t("cols"), n_samples_x=N, rnd_seed=3,
                              perms=t("perms"))
    zdz = torch.stack([t("depth"), torch.full_like(t("depth"), 0.01)], -1)
    a, b = ou.bilateral_denoiser2(d, s, torch.nn.functional.normalize(nrm.detach() + 1e-6, dim=-1), zdz, 1.0)
    loss = ru.image_loss(a * kd + b, torch.rand_like(a), loss="l1", tonemapper="log_srgb")
    loss.backward()
    ou.optix_build_bvh(ctx, t("verts"), t("tris"), 0)
    v = ou.trace_visibility(ctx, t("ro").reshape(-1, 3), torch.nn.functional.normalize(torch.randn(c["ro"].size // 3, 3, device=dev), dim=-1))
    pts = ru.xfm_points(t("verts")[None], torch.rand(2, 4, 4, device=dev))
    # strided operands: channel-strided points, a transposed matrix, a stride-0 upstream gradient; per-partial weighted loss backward
    ps = t("verts").t().contiguous()[None].transpose(1, 2).requires_grad_(True)
    ru.xfm_vectors(ps, torch.rand(2, 4, 4, device=dev).transpose(1, 2)).backward(torch.rand(1, ps.shape[1], 3, device=dev).expand(2, -1, 3))
    from nvdiffrecmc_b200.renderutils.ops import _image_loss_func
    parts = _image_loss_func.apply(torch.rand(2, 12, 12, 4, device=dev, requires_grad=True)[..., :3], torch.rand(1, 12, 12, 3, device=dev), "relmse", "log_srgb")
    (parts * torch.rand_like(parts)).sum().backward()
    # re-tracing backward (decorrelated seeds), update_pdf, rasterize / interpolate
    d2, s2 = ou.optix_env_shade(ctx, t("mask"), t("ro"), pos, nrm.detach().requires_grad_(True), t("view"), kd, ks, light, t("pdf"), t("rows"), t("cols"), n_samples_x=N, rnd_seed=None,
                                perms=t("perms"))
    (d2.sum() + s2.sum()).backward()
    from nvdiffrecmc_b200.light import EnvironmentLight
    from nvdiffrecmc_b200.raster import rasterize, interpolate
    lg = EnvironmentLight(light.detach())
    proj = torch.tensor([[2.4, 0, 0, 0], [0, -2.4, 0, 0], [0, 0, -1.02, -0.2], [0, 0, -1, 0]], device=dev)
    mv = torch.eye(4, device=dev); mv[2, 3] = -3.0
    rast = rasterize(ctx, (proj @ mv)[None], (24, 24))
    att = t("verts").clone().requires_grad_(True)
    interpolate(att, rast, t("tris"))[0].sum().backward()
# round 2: records entry point (MODE 2), fused shade tail, texel fetch, device-side seed
from nvdiffrecmc_b200.optixutils.ops import env_shade_records, shade_combine
from nvdiffrecmc_b200.raster import texel_fetch
env_shade_records(ctx, t("mask"), t("ro"), t("pos"), nrm.detach(), t("view"), t("kd"), t("ks"), t("light"), t("pdf"), t("rows"), t("cols"), t("perms"), n_samples_x=N, rnd_seed=1)
seed_t = torch.full((1,), 7, dtype=torch.int32, device=dev)
ou.optix_env_shade(ctx, t("mask"), t("ro"), t("pos"), nrm.detach(), t("view"), t("kd"), t("ks"), t("light"), t("pdf"), t("rows"), t("cols"), n_samples_x=N, rnd_seed=seed_t, perms=t("perms"))
a4 = (torch.rand(2, 12, 12, 4, device=dev) + 0.5).requires_grad_(True)
shade_combine(a4, a4 * 1.5, t("kd"), t("ks")).sum().backward()
tex = torch.rand(64, 3, device=dev, requires_grad=True)
texel_fetch(tex, torch.randint(0, 64, (2, 12, 12), device=dev)).sum().backward()
# geometry gradients: rasterize backward, interpolate backward to rast (no attribute gradient), edge adjacency, antialias fwd / bwd
from nvdiffrecmc_b200.raster import rasterize, interpolate, antialias, antialias_topology
mg = (proj @ mv)[None]
posg = ru.xfm_points(t("verts")[None], mg).detach().requires_grad_(True)
rg = rasterize(ctx, mg, (24, 24), pos=posg, tri=t("tris"))
ig, _ = interpolate(t("verts"), rg, t("tris"))
antialias(torch.cat([ig, rg[..., 3:4].clamp(0, 1)], -1), rg, posg, t("tris")).sum().backward()
antialias(torch.rand(1, 24, 24, 1, device=dev), rg.detach(), posg.detach()[0], t("tris"), antialias_topology(t("tris")))
# depth peeling: three layers with a backward through each, and the ray-level query beyond a bound
from nvdiffrecmc_b200.raster import DepthPeeler
posp = posg.detach().clone().requires_grad_(True)
with DepthPeeler(ctx, mg, (24, 24), posp, t("tris")) as peeler:
    layers = [peeler.rasterize_next_layer()[0] for _ in range(3)]
sum(antialias(rl[..., 3:4].clamp(0, 1), rl, posp, t("tris")).sum() + rl[..., :2].sum() for rl in layers).backward()
ou.trace_closest(ctx, t("ro").reshape(-1, 3), torch.randn(c["ro"].size // 3, 3, device=dev), t_after=torch.rand(c["ro"].size // 3, device=dev))
# hash-grid encoding: forward, d params + d x, d params only, on a padded dense level, an exact-fit level and hashed levels
from nvdiffrecmc_b200.tinycudann import Encoding
enc = Encoding(3, {"otype": "HashGrid", "n_levels": 5, "log2_hashmap_size": 9, "base_resolution": 5, "per_level_scale": 1.5})
xh = (torch.rand(1000, 3, device=dev) * 2 - 0.5).requires_grad_(True)
enc(xh).sum().backward()
enc(xh.detach()).sum().backward()
# fused MLP texture: forward, backward with d texc (points across two d W chunks), backward without d texc, no_grad forward
from nvdiffrecmc_b200.mlptexture import MLPTexture3D
mlt = MLPTexture3D(torch.tensor([[-1.0] * 3, [1.0] * 3], device=dev), channels=6, min_max=[torch.zeros(6, device=dev), torch.ones(6, device=dev)])
tm = (torch.rand(1500, 3, device=dev) * 2.4 - 1.2).requires_grad_(True)
mlt.sample(tm).sum().backward()
mlt.sample(tm.detach()).sum().backward()
with torch.no_grad():
    mlt.sample(tm)
# filtered texture look-up: 'linear' / 'clamp' on a per-batch 3-channel texture, 'linear-mipmap-linear' / 'wrap' on a custom 4-channel chain
from nvdiffrecmc_b200.raster import texture
uvt = (torch.rand(2, 9, 11, 2, device=dev) * 1.6 - 0.3).requires_grad_(True)
dat = (torch.randn(2, 9, 11, 4, device=dev) * 0.2).requires_grad_(True)
texture(torch.rand(2, 5, 7, 3, device=dev, requires_grad=True), uvt, filter_mode="linear", boundary_mode="clamp").sum().backward()
mipc = [torch.rand(1, max(1, 12 >> k), max(1, 20 >> k), 4, device=dev, requires_grad=True) for k in range(5)]
texture(mipc[0], uvt, dat, mip=mipc[1:]).sum().backward()
torch.cuda.synchronize()
print("sanitize workload ok", float(loss), int(v.sum()), tuple(pts.shape))
