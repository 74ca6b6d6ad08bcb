"""GPU: raster.composite (csrc/composite.cu) against the reference's composite_buffer restated with raster.antialias and the same topology on
the same device (render/render.py:284-291, 321-330): forward bit for bit, gradients of every buffer, the background and pos, one launch
per layer each way, no host sync, CUDA-graph capture, edge cases, argument errors and the full 8 x 512^2 size; and
material_smoothness_grad with the 5-channel kd_grad of a 4-channel kd."""
import numpy as np
import pytest
import torch

import nvdiffrecmc_b200._lib as L
import nvdiffrecmc_b200.regularizer as R
from nvdiffrecmc_b200 import synth
from nvdiffrecmc_b200.raster import DepthPeeler, antialias, antialias_topology, composite

pytestmark = pytest.mark.gpu

PASS1 = [(k, 4) for k in ("shaded", "z_grad", "normal", "geometric_normal", "kd", "ks", "kd_grad", "ks_grad", "normal_grad", "diffuse_light",
                          "specular_light")]
PASS2 = [(k, 5 if k == "kd_grad" else c) for k, c in PASS1] + [("perturbed_nrm", 4), ("perturbed_nrm_grad", 4)]
SPEC = PASS2 + [("mono", 1), ("wide", 7)]                          # render_mesh's pass-2 set plus a C = 1 and a C = 7 buffer
STRIDED = ("normal", "kd_grad", "wide")


def _scene(dev, B, res, n_layers, dist=3.0):
    """Peeled layers of the blob+torus scene from B views: (rasts, pos [B,V,4], tri, topology)."""
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    v, f = synth.scene_mesh("blob+torus", level=2)
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    proj = synth.perspective(aspect=res[1] / res[0], n=0.1, f=10.0).astype(np.float64)
    mtx = []
    for b in range(B):
        ang, tilt = 0.7 * b + 0.3, 0.2 * b - 0.1
        ry = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
        rx = np.array([[1, 0, 0], [0, np.cos(tilt), -np.sin(tilt)], [0, np.sin(tilt), np.cos(tilt)]])
        mv = np.eye(4)
        mv[:3, :3] = rx @ ry
        mv[2, 3] = -dist
        mtx.append(proj @ mv)
    mtx = torch.tensor(np.stack(mtx).astype(np.float32), device=dev)
    with DepthPeeler(ctx, mtx, res) as p:
        rasts = [p.rasterize_next_layer()[0] for _ in range(n_layers)]
    pos = ru.xfm_points(vt[None], mtx).detach()
    return rasts, pos, ft, antialias_topology(ft)


def _buffers(rasts, spec, seed, nonfinite=True, strided=STRIDED):
    """Per layer a dict of [B,H,W,C] buffers: values in [-0.5, 1.5], alphas random fractions with exact 0, 0.5 and 1 (covered pixels with
    alpha 0 among them); with nonfinite, a NaN alpha and an inf colour on some uncovered pixels.  Keys in `strided` are non-dense views."""
    dev = rasts[0].device
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *shape: torch.rand(*shape, generator=g, device=dev)
    out = []
    for rast in rasts:
        B, H, W = rast.shape[:3]
        unc = rast[..., 3] <= 0
        bufs = {}
        for key, C in spec:
            x = rnd(B, H, W, C) * 2 - 0.5
            a, pick = rnd(B, H, W), (rnd(B, H, W) * 6).floor()
            a = torch.where(pick == 0, 0.0, torch.where(pick == 1, 0.5, torch.where(pick == 2, 1.0, a)))
            if nonfinite:
                a = torch.where(unc & (rnd(B, H, W) < 0.05), float("nan"), a)
                if C > 1:
                    x[..., 0] = torch.where(unc & (rnd(B, H, W) < 0.05), float("inf"), x[..., 0])
            x[..., C - 1] = a
            if key in strided:
                wide = torch.full((B, H, W, C + 3), float("nan"), device=rast.device)
                wide[..., 2:2 + C] = x
                x = wide[..., 2:2 + C]
            bufs[key] = x
        out.append(bufs)
    return out


def _layers(rasts, bufs):
    return [(b, r) for b, r in zip(bufs, rasts)]


def _chain(layers, pos, tri, topo, background=None):
    """The reference's composite_buffer(key, layers, bg, True) for every key, with raster.antialias."""
    out = {}
    for key in layers[0][0]:
        accum = background[key] if background and key in background else torch.zeros_like(layers[0][0][key])
        for buffers, rast in reversed(layers):
            b = buffers[key]
            alpha = (rast[..., -1:] > 0).float() * b[..., -1:]
            accum = torch.lerp(accum, torch.cat((b[..., :-1], torch.ones_like(b[..., -1:])), dim=-1), alpha)
            accum = antialias(accum.contiguous(), rast, pos, tri, topo)
        out[key] = accum
    return out


def _bits(a, b, what):
    """Bit for bit, every NaN counted as one pattern."""
    a, b = a.detach(), b.detach()
    na, nb = torch.isnan(a), torch.isnan(b)
    same = (torch.where(na, float("nan"), a).view(torch.int32) == torch.where(nb, float("nan"), b).view(torch.int32))
    if not bool(same.all()):
        k = tuple(int(i) for i in torch.nonzero(~same)[0])
        raise AssertionError("%s: %d of %d elements differ, first at %s (got %r, chain %r)" % (
            what, int((~same).sum()), same.numel(), k, float(a[k]), float(b[k])))


def _values(a, b, what):
    """Equal values (+0 == -0) with NaN in the same places: the chain's gradients pass through autograd's accumulation of slice
    gradients, which adds +0 to each."""
    a, b = a.detach(), b.detach()
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "%s: NaN at %d vs %d places" % (what, int(na.sum()), int(nb.sum()))
    diff = ~na & (a != b)
    assert not bool(diff.any()), "%s: %d elements differ (got %r, chain %r)" % (what, int(diff.sum()), float(a[diff][0]), float(b[diff][0]))


def _close(a, b, tol, what):
    a, b = a.detach(), b.detach()
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb), "%s: NaN at %d vs %d places" % (what, int(na.sum()), int(nb.sum()))
    a, b = a[~na].double(), b[~nb].double()
    e = float((a - b).norm() / max(float(b.norm()), 1e-30))
    assert e <= tol, "%s: rel-L2 %.3e" % (what, e)
    return e


def _grads(fn, layers, pos, tri, topo, background, G, pos_grad=True):
    out = fn(layers, pos, tri, topo, background)
    keys = list(out)
    ins = [b[k] for b, _ in layers for k in keys] + [background[k] for k in background] + ([pos] if pos_grad else [])
    gs = torch.autograd.grad([out[k] for k in keys], ins, grad_outputs=[G[k] for k in keys])
    n = len(keys) * len(layers)
    return out, gs[:n], gs[n:n + len(background)], (gs[-1] if pos_grad else None)


def _product(layers, pos, tri, topo, background):
    return composite(layers, pos, tri, background=background, topology=topo)


def _check_backward(layers, pos, tri, topo, bg, seed, pos_grad=True):
    keys = list(layers[0][0])
    g = torch.Generator(device=pos.device).manual_seed(seed)
    G = {k: torch.rand(layers[0][0][k].shape, generator=g, device=pos.device) * 2 - 1 for k in keys}
    got = _grads(_product, layers, pos, tri, topo, bg, G, pos_grad)
    ref = _grads(_chain, layers, pos, tri, topo, bg, G, pos_grad)
    for k in keys:
        _bits(got[0][k], ref[0][k], "forward %s" % k)
    worst = 0.0
    for i, (a, b) in enumerate(zip(got[1], ref[1])):
        what = "layer %d d %s" % (i // len(keys), keys[i % len(keys)])
        _values(a[..., :-1], b[..., :-1], what)
        worst = max(worst, _close(a[..., -1], b[..., -1], 1e-6, what + " alpha"))
    for a, b, k in zip(got[2], ref[2], bg):
        _values(a, b, "d background %s" % k)
    if pos_grad:
        assert torch.isfinite(ref[3]).all() and ref[3].abs().max() > 0
        e = _close(got[3], ref[3], 1e-5, "d pos")
        print("d alpha worst rel-L2 %.2e, d pos rel-L2 %.2e" % (worst, e))
    return got


# ---- 1. forward, bit for bit
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n_layers", [1, 2, 4])
def test_forward_bit_for_bit(dev, n_layers, B):
    rasts, pos, tri, topo = _scene(dev, B, (40, 56), n_layers)
    layers = _layers(rasts, _buffers(rasts, SPEC, seed=n_layers + 10 * B))
    bg = {"shaded": torch.rand(B, 40, 56, 4, device=dev), "wide": torch.rand(B, 40, 56, 7, device=dev)}
    for p in (pos, pos[0]):
        got, ref = composite(layers, p, tri, background=bg, topology=topo), _chain(layers, p, tri, topo, bg)
        assert list(got) == [k for k, _ in SPEC]
        for k in got:
            _bits(got[k], ref[k], k)
    nan = sum(int(torch.isnan(got[k]).sum()) for k in got)
    blended = sum(int(((got[k] != layers[0][0][k]) & (rasts[0][..., 3:4] > 0)).sum()) for k in got)
    print("L %d B %d: %d NaN outputs, %d covered outputs blended" % (n_layers, B, nan, blended))
    assert nan > 0 and blended > 1000


def test_lerp_equals_torch_lerp(dev):
    """One triangle id under every pixel: no antialias pairs, so the output is the kernel's lerp alone."""
    rasts, pos, tri, topo = _scene(dev, 2, (64, 96), 1)
    rast = torch.zeros_like(rasts[0])
    rast[..., 3] = 1.0
    g = torch.Generator().manual_seed(5)
    buf = torch.rand(2, 64, 96, 6, generator=g) * 4 - 2
    w = torch.rand(2, 64, 96, generator=g)
    w[0, :8] = torch.rand(8, 96, generator=g) * 3 - 1                  # weights outside [0, 1]
    w[0, 8, :4] = torch.tensor([0.5, -0.5, float("nan"), 0.4999999])
    buf[..., 5] = w
    buf, bg = buf.to(dev), (torch.rand(2, 64, 96, 6, generator=g) * 4 - 2).to(dev)
    got = composite([({"x": buf}, rast)], pos, tri, background={"x": bg}, topology=topo)["x"]
    ref = torch.lerp(bg, torch.cat((buf[..., :-1], torch.ones_like(buf[..., -1:])), -1), buf[..., -1:])
    _bits(got, ref, "lerp")
    frac = (w > 0) & (w < 1) & (w != 0.5)
    assert frac.sum() > 10000 and (w.abs() < 0.5).any() and (w.abs() >= 0.5).any()     # both of torch's branches at fractional weights


# ---- 2. backward against torch autograd through the chain
@pytest.mark.parametrize("batched_pos", [True, False], ids=["pos_BV4", "pos_V4"])
@pytest.mark.parametrize("n_layers", [1, 3])
def test_backward_against_the_chain(dev, n_layers, batched_pos):
    rasts, pos, tri, topo = _scene(dev, 2, (40, 56), n_layers)
    p = (pos if batched_pos else pos[0]).clone().requires_grad_(True)
    for nonfinite in (False, True):
        bufs = _buffers(rasts, SPEC, seed=3 + n_layers, nonfinite=nonfinite)
        for b in bufs:
            for k in b:
                b[k].requires_grad_(True)
        bg = {"shaded": torch.rand(2, 40, 56, 4, device=dev, requires_grad=True), "mono": torch.rand(2, 40, 56, 1, device=dev, requires_grad=True)}
        _check_backward(_layers(rasts, bufs), p, tri, topo, bg, seed=n_layers, pos_grad=not nonfinite)


# ---- 3. launches, sync, graph capture, no_grad
def _finite_case(dev, n_layers=3, res=(40, 56)):
    rasts, pos, tri, topo = _scene(dev, 2, res, n_layers)
    bufs = _buffers(rasts, PASS2, seed=7, nonfinite=False)
    for b in bufs:
        for k in b:
            b[k].requires_grad_(True)
    bg = {"shaded": torch.rand(2, *res, 4, device=dev, requires_grad=True)}
    return _layers(rasts, bufs), pos.clone().requires_grad_(True), tri, topo, bg


def test_one_launch_per_layer_each_way_and_no_sync(dev):
    layers, pos, tri, topo, bg = _finite_case(dev, n_layers=3)
    G = [torch.rand(2, 40, 56, c, device=dev) for _, c in PASS2]
    torch.cuda.synchronize()
    before = L.LAUNCHES.copy()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = composite(layers, pos, tri, background=bg, topology=topo)
        torch.autograd.backward(list(out.values()), G)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    delta = {k: v - before.get(k, 0) for k, v in L.LAUNCHES.items() if v != before.get(k, 0)}
    assert delta == {"composite_fwd": 3, "composite_bwd": 3}, delta
    assert pos.grad.abs().max() > 0 and bg["shaded"].grad.abs().max() > 0


def test_no_grad_forward_equals_grad_forward(dev):
    layers, pos, tri, topo, bg = _finite_case(dev, n_layers=4)
    a = composite(layers, pos, tri, background=bg, topology=topo)
    with torch.no_grad():
        b = composite(layers, pos, tri, background=bg, topology=topo)
    for k in a:
        assert a[k].grad_fn is not None and b[k].grad_fn is None
        _bits(b[k], a[k], k)


def test_cuda_graph_replay_equals_eager(dev):
    layers, pos, tri, topo, bg = _finite_case(dev, n_layers=2)
    ins = [b[k] for b, _ in layers for k in b] + [bg["shaded"], pos]
    G = [torch.rand(2, 40, 56, c, device=dev) for _, c in PASS2]

    def run():
        out = composite(layers, pos, tri, background=bg, topology=topo)
        return [o.detach().clone() for o in out.values()] + [g.clone() for g in torch.autograd.grad(list(out.values()), ins, G)]

    eager = run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            run()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    for t in captured:
        t.fill_(-7.0)
    graph.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(captured[:-1], eager[:-1])):
        _bits(a, b, "output or gradient %d" % i)
    _close(captured[-1], eager[-1], 1e-6, "d pos")                    # float atomics: order-dependent


# ---- 4. edge cases
def test_deeper_layers_all_background(dev):
    rasts, pos, tri, topo = _scene(dev, 2, (40, 56), 2)
    rasts = rasts + [torch.zeros_like(rasts[0])] * 2
    layers = _layers(rasts, _buffers(rasts, PASS1, seed=11, nonfinite=False))
    for b, _ in layers:
        for k in b:
            b[k].requires_grad_(True)
    _check_backward(layers, pos.clone().requires_grad_(True), tri, topo, {"shaded": torch.rand(2, 40, 56, 4, device=dev, requires_grad=True)}, 1)


def test_fully_covered_image(dev):
    rasts, pos, tri, topo = _scene(dev, 2, (40, 56), 2)
    full = rasts[0].clone()
    unc = full[..., 3] <= 0
    full[..., 3] = torch.where(unc, 1.0, full[..., 3])
    full[..., 2] = torch.where(unc, 0.5, full[..., 2])
    rasts = [full, rasts[1]]
    assert (rasts[0][..., 3] > 0).all()
    layers = _layers(rasts, _buffers(rasts, PASS1, seed=12))
    for b, _ in layers:
        for k in b:
            b[k].requires_grad_(True)
    _check_backward(layers, pos.clone().requires_grad_(True), tri, topo, {}, 2, pos_grad=False)
    cov = rasts[0][..., 3] > 0
    assert ((layers[0][0]["kd"][..., 3] == 0) & cov).any()          # covered pixels with alpha 0


@pytest.mark.parametrize("res", [(1, 1), (1, 37), (29, 1)], ids=["1x1", "1xW", "Hx1"])
def test_degenerate_images(dev, res):
    rasts, pos, tri, topo = _scene(dev, 2, res, 2, dist=2.0)
    layers = _layers(rasts, _buffers(rasts, SPEC, seed=13))
    for b, _ in layers:
        for k in b:
            b[k].requires_grad_(True)
    _check_backward(layers, pos.clone().requires_grad_(True), tri, topo, {"wide": torch.rand(2, *res, 7, device=dev, requires_grad=True)}, 3,
                    pos_grad=False)


def test_sixteen_buffers(dev):
    rasts, pos, tri, topo = _scene(dev, 2, (40, 56), 2)
    spec = [("b%d" % k, 1 + k % 6) for k in range(16)]
    layers = _layers(rasts, _buffers(rasts, spec, seed=14, nonfinite=False, strided=("b3", "b9")))
    for b, _ in layers:
        for k in b:
            b[k].requires_grad_(True)
    _check_backward(layers, pos.clone().requires_grad_(True), tri, topo, {"b15": torch.rand(2, 40, 56, 4, device=dev, requires_grad=True)}, 4)


# ---- 5. errors
def test_argument_errors_raise_before_any_launch(dev):
    rasts, pos, tri, topo = _scene(dev, 2, (16, 24), 2)
    bufs = _buffers(rasts, PASS1[:3], seed=15, nonfinite=False)
    layers = _layers(rasts, bufs)
    x = bufs[0]["shaded"]
    one = lambda **kw: [({**bufs[0], **kw}, rasts[0])]
    cases = [
        ("layers", lambda: composite([], pos, tri)),
        ("layers", lambda: composite([(bufs[0], rasts[0]), ({"shaded": x}, rasts[1])], pos, tri)),           # keys differ between layers
        ("layers", lambda: composite([({"a": x[..., :0]}, rasts[0])], pos, tri)),                            # C = 0
        ("layers", lambda: composite([({"b%d" % k: x for k in range(17)}, rasts[0])], pos, tri)),          # 17 buffers
        ("layers", lambda: composite(one(shaded=torch.rand(2, 16, 25, 4, device=dev)), pos, tri)),         # W mismatch
        ("layers", lambda: composite(one(shaded=torch.rand(1, 16, 24, 4, device=dev)), pos, tri)),         # B mismatch
        ("layers", lambda: composite(one(shaded=x.cpu()), pos, tri)),                                      # CPU tensor
        ("layers", lambda: composite(one(shaded=x.double()), pos, tri)),                                   # not fp32
        ("layers", lambda: composite([(bufs[0], rasts[0]), (bufs[1], rasts[1][:, :8])], pos, tri)),        # rast H mismatch
        ("layers", lambda: composite([(bufs[0], rasts[0]), ({**bufs[1], "z_grad": bufs[1]["z_grad"][..., :3]}, rasts[1])], pos, tri)),
        ("pos", lambda: composite(layers, pos.cpu(), tri)),
        ("pos", lambda: composite(layers, pos[..., :3], tri)),
        ("pos", lambda: composite(layers, pos[:1].repeat(3, 1, 1), tri)),
        ("pos", lambda: composite(layers, pos.double(), tri)),
        ("tri", lambda: composite(layers, pos, tri.long())),
        ("tri", lambda: composite(layers, pos, tri[:0])),
        ("background", lambda: composite(layers, pos, tri, background={"albedo": x})),
        ("background", lambda: composite(layers, pos, tri, background={"shaded": x[:1]})),
        ("background", lambda: composite(layers, pos, tri, background={"shaded": x.cpu()})),
        ("background", lambda: composite(layers, pos, tri, background={"shaded": x[..., :3]})),
        ("topology", lambda: composite(layers, pos, tri, topology=topo[:-1])),
        ("topology", lambda: composite(layers, pos, tri, topology=topo.long())),
    ]
    for name, call in cases:
        before = L.LAUNCHES.copy()
        with pytest.raises(ValueError, match=name):
            call()
        assert L.LAUNCHES == before, name


# ---- 6. full size
def test_full_size_pass2_eight_layers(dev):
    """8 x 512^2, 8 peeled layers of the bench mesh, pass 2's buffer set (5-channel kd_grad)."""
    import bench
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    B, res = 8, (512, 512)
    mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32),
                       device=dev)
    with DepthPeeler(ctx, mtx, res) as p:
        rasts = [p.rasterize_next_layer()[0] for _ in range(8)]
    pos = ru.xfm_points(vt[None], mtx).detach().requires_grad_(True)
    topo = antialias_topology(ft)
    bufs = _buffers(rasts, PASS2, seed=16, nonfinite=False, strided=("normal",))
    for b in bufs:
        for k in b:
            b[k].requires_grad_(True)
    bg = {"shaded": torch.rand(B, *res, 4, device=dev, requires_grad=True)}
    _check_backward(_layers(rasts, bufs), pos, ft, topo, bg, seed=6)


# ---- 7. material_smoothness_grad with a 5-channel kd_grad
def _smooth_inputs(dev, shape=(3, 37, 53), seed=0):
    g = torch.Generator().manual_seed(seed)
    kd5 = (torch.rand(*shape, 5, generator=g) * 0.3).to(dev)
    kd5[0, 0, :4, 4] = torch.tensor([0.0, 1.0, 0.5, 0.25])[:shape[2]]
    ks, nr = [(torch.rand(*shape, 4, generator=g) * 0.2).to(dev) for _ in range(2)]
    return kd5, ks, nr


def _smooth_check(kd5, ks, nr, lam=(0.25, 0.1, 0.05)):
    a = [kd5.detach().clone().requires_grad_(True), ks.clone().requires_grad_(True), nr.clone().requires_grad_(True)]
    b = [kd5.detach()[..., [0, 1, 2, 4]].clone().requires_grad_(True), ks.clone().requires_grad_(True), nr.clone().requires_grad_(True)]
    la, lb = R.material_smoothness_grad(*a, *lam), R.material_smoothness_grad(*b, *lam)
    la.backward(torch.tensor(1.5, device=kd5.device))
    lb.backward(torch.tensor(1.5, device=kd5.device))
    _bits(la, lb, "loss")
    assert a[0].grad.shape == kd5.shape
    _bits(a[0].grad[..., [0, 1, 2, 4]], b[0].grad, "d kd_grad")
    assert (a[0].grad[..., 3] == 0).all() and not torch.signbit(a[0].grad[..., 3]).any()
    _bits(a[1].grad, b[1].grad, "d ks_grad")
    _bits(a[2].grad, b[2].grad, "d nrm_grad")
    with torch.no_grad():
        _bits(R.material_smoothness_grad(kd5, ks, nr, *lam), lb, "no_grad loss")


def test_smoothness_five_channel_kd_grad(dev):
    _smooth_check(*_smooth_inputs(dev))
    kd5, ks, nr = _smooth_inputs(dev, (1, 1, 1), seed=1)           # one pixel: the 4-channel operands would take the float4 path
    _smooth_check(kd5, ks, nr)


def test_smoothness_five_channel_strided(dev):
    kd5, ks, nr = _smooth_inputs(dev, (2, 40, 56), seed=2)
    wide = torch.full((2, 40, 56, 9), float("nan"), device=dev)
    wide[..., 3:8] = kd5
    _smooth_check(wide[..., 3:8], ks, nr)
    _smooth_check(kd5.transpose(1, 2).contiguous().transpose(1, 2), ks, nr)


def test_smoothness_from_jitter_taps_with_a_four_channel_kd(dev):
    rasts, _, _, _ = _scene(dev, 2, (40, 56), 1)
    g = torch.Generator().manual_seed(3)
    mk = lambda c: torch.rand(2, 40, 56, c, generator=g).to(dev)
    kd = mk(4).requires_grad_(True)
    ks, nrm = mk(3).requires_grad_(True), mk(3).requires_grad_(True)
    jit = mk(2)
    taps = R.jitter_taps(rasts[0], jit, kd, ks, nrm)
    assert taps["kd_grad"].shape[-1] == 5
    loss = R.material_smoothness_grad(taps["kd_grad"], taps["ks_grad"], taps["normal_grad"], 0.25, 0.1, 0.05)
    loss.backward()
    kd4 = taps["kd_grad"].detach()[..., [0, 1, 2, 4]]
    ref = R.material_smoothness_grad(kd4, taps["ks_grad"].detach(), taps["normal_grad"].detach(), 0.25, 0.1, 0.05)
    _bits(loss, ref, "loss")
    assert torch.isfinite(kd.grad).all() and kd.grad.abs().max() > 0 and ks.grad.abs().max() > 0


def test_smoothness_other_kd_grad_channel_counts_raise(dev):
    x = torch.rand(2, 8, 9, 4, device=dev)
    for c in (3, 6):
        before = L.LAUNCHES.copy()
        with pytest.raises(ValueError, match="kd_grad"):
            R.material_smoothness_grad(torch.rand(2, 8, 9, c, device=dev), x, x)
        assert L.LAUNCHES == before
    with pytest.raises(ValueError, match="ks_grad"):
        R.material_smoothness_grad(x, torch.rand(2, 8, 9, 5, device=dev), x)
    with pytest.raises(ValueError, match="nrm_grad"):
        R.material_smoothness_grad(torch.rand(2, 8, 9, 5, device=dev), x, torch.rand(2, 8, 10, 4, device=dev))
