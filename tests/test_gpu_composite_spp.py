"""GPU: raster.composite with spp > 1 (csrc/composite.cu, supersampled) against render_mesh's supersampled tail restated in torch with
raster.antialias on the same device: render_layer's nearest upscale of MSAA-shaded buffers (render/render.py:247-250), the background's
upscale (:313-319), composite_buffer per key and avg_pool_nhwc (:321-330).  Forward bit for bit, gradients of every buffer, the background
and pos, spp = 1 against the default call, one launch per layer each way, no host sync, no_grad, CUDA-graph capture, edge cases, the
pass-2 set at output 8 x 256^2 and buffers interpolated on rast[:, ::spp, ::spp] of a real peel."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import nvdiffrecmc_b200._lib as L
from nvdiffrecmc_b200 import synth
from nvdiffrecmc_b200.raster import DepthPeeler, antialias_topology, composite, interpolate
from test_gpu_composite import PASS2, SPEC, _bits, _buffers, _chain, _close, _layers, _scene, _values

pytestmark = pytest.mark.gpu

RES = (48, 72)                      # full resolution: a multiple of 1, 2, 3 and 4


def _up(x, H, W):
    """scale_img_nhwc(x, (H, W), mag='nearest'): F.interpolate in NCHW, back to contiguous NHWC; full-resolution tensors pass through."""
    if tuple(x.shape[1:3]) == (H, W):
        return x
    return F.interpolate(x.permute(0, 3, 1, 2), (H, W), mode="nearest").permute(0, 2, 3, 1).contiguous()


def _pool(x, spp):
    """avg_pool_nhwc(x, spp)"""
    return F.avg_pool2d(x.permute(0, 3, 1, 2), spp).permute(0, 2, 3, 1).contiguous()


def _chain_ss(layers, pos, tri, topo, background, spp):
    """render_mesh's tail for spp: upscale every buffer and the backgrounds, composite_buffer per key, then avg_pool_nhwc."""
    H, W = layers[0][1].shape[1:3]
    full = [({k: _up(t, H, W) for k, t in b.items()}, r) for b, r in layers]
    bg = {k: _up(t, H, W) for k, t in (background or {}).items()}
    out = _chain(full, pos, tri, topo, bg)
    return {k: _pool(t, spp) if spp > 1 else t for k, t in out.items()}


def _msaa_buffers(rasts, spec, seed, spp, msaa, **kw):
    """_buffers at output resolution (from the nearest-minified rast, as render_layer shades with msaa) or at full resolution."""
    return _buffers([r[:, ::spp, ::spp] for r in rasts] if msaa else rasts, spec, seed, **kw)


def _grads(fn, layers, pos, bg, G, pos_grad):
    out = fn(layers, pos, bg)
    keys = list(out)
    ins = [b[k] for b, _ in layers for k in keys] + [bg[k] for k in bg] + ([pos] if pos_grad else [])
    gs = torch.autograd.grad([out[k] for k in keys], ins, grad_outputs=[G[k] for k in keys])
    n = len(keys) * len(layers)
    return out, gs[:n], gs[n:n + len(bg)], (gs[-1] if pos_grad else None)


def _check_backward(layers, pos, tri, topo, bg, seed, spp, pos_grad=True):
    keys = list(layers[0][0])
    B, H, W = layers[0][1].shape[:3]
    g = torch.Generator(device=pos.device).manual_seed(seed)
    G = {k: torch.rand(B, H // spp, W // spp, layers[0][0][k].shape[3], generator=g, device=pos.device) * 2 - 1 for k in keys}
    got = _grads(lambda ls, p, b: composite(ls, p, tri, background=b, topology=topo, spp=spp), layers, pos, bg, G, pos_grad)
    ref = _grads(lambda ls, p, b: _chain_ss(ls, p, tri, topo, b, spp), layers, pos, bg, G, pos_grad)
    for k in keys:
        assert got[0][k].shape == (B, H // spp, W // spp, G[k].shape[3])
        _bits(got[0][k], ref[0][k], "forward %s" % k)
    worst = 0.0
    for i, (a, b) in enumerate(zip(got[1], ref[1])):
        what = "layer %d d %s" % (i // len(keys), keys[i % len(keys)])
        _values(a[..., :-1], b[..., :-1], what)
        worst = max(worst, _close_nf(a[..., -1], b[..., -1], 1e-6, what + " alpha"))
    for a, b, k in zip(got[2], ref[2], bg):
        _values(a, b, "d background %s" % k)
    e = None
    if pos_grad:
        assert torch.isfinite(ref[3]).all() and ref[3].abs().max() > 0
        e = _close(got[3], ref[3], 1e-5, "d pos")
    print("spp %d: d alpha worst rel-L2 %.2e, d pos rel-L2 %s" % (spp, worst, "-" if e is None else "%.2e" % e))
    return got


def _close_nf(a, b, tol, what):
    """_close on the finite elements, the others identical: with MSAA an inf colour is read by every covered pixel of its block, and
    its alpha's gradient sums to the same inf in both."""
    a, b = a.detach(), b.detach()
    fa, fb = torch.isfinite(a), torch.isfinite(b)
    assert torch.equal(fa, fb), "%s: non-finite at %d vs %d places" % (what, int((~fa).sum()), int((~fb).sum()))
    _values(a[~fa], b[~fb], what + " (non-finite)")
    return _close(a[fa], b[fb], tol, what)


def _requires_grad(bufs):
    for b in bufs:
        for k in b:
            b[k].requires_grad_(True)
    return bufs


# ---- 1. forward, bit for bit
@pytest.mark.parametrize("msaa", [True, False], ids=["msaa", "fullres"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n_layers", [1, 3, 8])
@pytest.mark.parametrize("spp", [1, 2, 3, 4])
def test_forward_bit_for_bit(dev, spp, n_layers, B, msaa):
    rasts, pos, tri, topo = _scene(dev, B, RES, n_layers)
    layers = _layers(rasts, _msaa_buffers(rasts, SPEC, n_layers + 10 * B + 100 * spp, spp, msaa))
    Ho, Wo = RES[0] // spp, RES[1] // spp
    bg = {"shaded": torch.rand(B, Ho, Wo, 4, device=dev), "wide": torch.rand(B, Ho, Wo, 7, device=dev)}
    for p in (pos, pos[0]):
        for background in (bg, None):
            got, ref = composite(layers, p, tri, background=background, topology=topo, spp=spp), _chain_ss(layers, p, tri, topo, background, spp)
            assert list(got) == [k for k, _ in SPEC]
            for k in got:
                assert got[k].shape == (B, Ho, Wo, dict(SPEC)[k])
                _bits(got[k], ref[k], k)
    nan = sum(int(torch.isnan(got[k]).sum()) for k in got)
    print("spp %d L %d B %d msaa %d: %d NaN outputs" % (spp, n_layers, B, msaa, nan))
    assert nan > 0


# ---- 2. backward against torch autograd through the chain
@pytest.mark.parametrize("batched_pos", [True, False], ids=["pos_BV4", "pos_V4"])
@pytest.mark.parametrize("msaa", [True, False], ids=["msaa", "fullres"])
@pytest.mark.parametrize("n_layers", [1, 3])
@pytest.mark.parametrize("spp", [2, 3])
def test_backward_against_the_chain(dev, spp, n_layers, msaa, batched_pos):
    rasts, pos, tri, topo = _scene(dev, 2, RES, n_layers)
    p = (pos if batched_pos else pos[0]).clone().requires_grad_(True)
    Ho, Wo = RES[0] // spp, RES[1] // spp
    for nonfinite in (False, True):
        bufs = _requires_grad(_msaa_buffers(rasts, SPEC, 3 + n_layers, spp, msaa, nonfinite=nonfinite))
        bg = {"shaded": torch.rand(2, Ho, Wo, 4, device=dev, requires_grad=True), "mono": torch.rand(2, Ho, Wo, 1, device=dev, requires_grad=True)}
        _check_backward(_layers(rasts, bufs), p, tri, topo, bg, n_layers, spp, pos_grad=not nonfinite)


def test_spp1_equals_the_default_call(dev):
    rasts, pos, tri, topo = _scene(dev, 2, RES, 3)
    layers = _layers(rasts, _requires_grad(_buffers(rasts, SPEC, seed=21, nonfinite=False)))
    pos = pos.clone().requires_grad_(True)
    bg = {"shaded": torch.rand(2, *RES, 4, device=dev, requires_grad=True)}
    ins = [b[k] for b, _ in layers for k in b] + [bg["shaded"]]
    G = [torch.rand(2, *RES, c, device=dev) for _, c in SPEC]
    a = composite(layers, pos, tri, background=bg, topology=topo)
    b = composite(layers, pos, tri, background=bg, topology=topo, spp=1)
    for k in a:
        _bits(b[k], a[k], k)
    ga, gb = torch.autograd.grad(list(a.values()), ins, G), torch.autograd.grad(list(b.values()), ins, G)
    for i, (x, y) in enumerate(zip(gb, ga)):
        _bits(x, y, "gradient %d" % i)


# ---- 3. launches, sync, graph capture, no_grad
def _finite_case(dev, spp=2, n_layers=3, msaa=True):
    rasts, pos, tri, topo = _scene(dev, 2, RES, n_layers)
    bufs = _requires_grad(_msaa_buffers(rasts, PASS2, 7, spp, msaa, nonfinite=False))
    bg = {"shaded": torch.rand(2, RES[0] // spp, RES[1] // spp, 4, device=dev, requires_grad=True)}
    return _layers(rasts, bufs), pos.clone().requires_grad_(True), tri, topo, bg


def test_one_launch_per_layer_each_way_and_no_sync(dev):
    layers, pos, tri, topo, bg = _finite_case(dev, n_layers=3)
    G = [torch.rand(2, RES[0] // 2, RES[1] // 2, c, device=dev) for _, c in PASS2]
    torch.cuda.synchronize()
    before = L.LAUNCHES.copy()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = composite(layers, pos, tri, background=bg, topology=topo, spp=2)
        torch.autograd.backward(list(out.values()), G)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    delta = {k: v - before.get(k, 0) for k, v in L.LAUNCHES.items() if v != before.get(k, 0)}
    assert delta == {"composite_fwd": 3, "composite_bwd": 3}, delta
    assert pos.grad.abs().max() > 0 and bg["shaded"].grad.abs().max() > 0


@pytest.mark.parametrize("msaa", [True, False], ids=["msaa", "fullres"])
def test_no_grad_forward_equals_grad_forward(dev, msaa):
    layers, pos, tri, topo, bg = _finite_case(dev, spp=2, n_layers=4, msaa=msaa)
    a = composite(layers, pos, tri, background=bg, topology=topo, spp=2)
    with torch.no_grad():
        b = composite(layers, pos, tri, background=bg, topology=topo, spp=2)
    for k in a:
        assert a[k].grad_fn is not None and b[k].grad_fn is None
        _bits(b[k], a[k], k)


def test_cuda_graph_replay_equals_eager(dev):
    layers, pos, tri, topo, bg = _finite_case(dev, spp=2, n_layers=2)
    ins = [b[k] for b, _ in layers for k in b] + [bg["shaded"], pos]
    G = [torch.rand(2, RES[0] // 2, RES[1] // 2, c, device=dev) for _, c in PASS2]

    def run():
        out = composite(layers, pos, tri, background=bg, topology=topo, spp=2)
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
@pytest.mark.parametrize("spp", [2, 3])
@pytest.mark.parametrize("out_res", [(1, 1), (1, 37), (29, 1)], ids=["1x1", "1xW", "Hx1"])
def test_degenerate_outputs(dev, out_res, spp):
    res = (out_res[0] * spp, out_res[1] * spp)
    rasts, pos, tri, topo = _scene(dev, 2, res, 2, dist=2.0)
    for msaa in (True, False):
        layers = _layers(rasts, _requires_grad(_msaa_buffers(rasts, SPEC, 13, spp, msaa)))
        _check_backward(layers, pos.clone().requires_grad_(True), tri, topo, {"wide": torch.rand(2, *out_res, 7, device=dev, requires_grad=True)},
                        3, spp, pos_grad=False)


def test_sixteen_buffers(dev):
    rasts, pos, tri, topo = _scene(dev, 2, RES, 2)
    spec = [("b%d" % k, 1 + k % 6) for k in range(16)]
    for spp, msaa in ((2, True), (4, False)):
        layers = _layers(rasts, _requires_grad(_msaa_buffers(rasts, spec, 14, spp, msaa, nonfinite=False, strided=("b3", "b9"))))
        bg = {"b15": torch.rand(2, RES[0] // spp, RES[1] // spp, 4, device=dev, requires_grad=True)}
        _check_backward(layers, pos.clone().requires_grad_(True), tri, topo, bg, 4, spp)


# ---- 5. the pass-2 set at output 8 x 256^2
def test_full_size_pass2_eight_layers_spp2(dev):
    """Output 8 x 256^2 (rast 8 x 512^2), spp 2, 8 peeled layers of the bench mesh, pass 2's MSAA buffer set (5-channel kd_grad)."""
    import bench
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    v, f, _ = bench.build_scene_numpy(bench.WORKLOAD, 0)
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    B, spp, res = 8, 2, (512, 512)
    mtx = torch.tensor(np.stack([synth.perspective(n=0.1, f=10.0) @ synth.orbit_view(2 * np.pi * b / B) for b in range(B)]).astype(np.float32),
                       device=dev)
    with DepthPeeler(ctx, mtx, res) as p:
        rasts = [p.rasterize_next_layer()[0] for _ in range(8)]
    pos = ru.xfm_points(vt[None], mtx).detach().requires_grad_(True)
    topo = antialias_topology(ft)
    bufs = _requires_grad(_msaa_buffers(rasts, PASS2, 16, spp, True, nonfinite=False, strided=("normal",)))
    bg = {"shaded": torch.rand(B, 256, 256, 4, device=dev, requires_grad=True)}
    _check_backward(_layers(rasts, bufs), pos, ft, topo, bg, 6, spp)


# ---- 6. buffers interpolated at the shading resolution of a real peel
@pytest.mark.parametrize("spp", [2, 3])
def test_interpolated_msaa_buffers_of_a_peel(dev, spp):
    """render_layer's MSAA glue: interpolate on rast[:, ::spp, ::spp] of each peeled layer, pos requiring grad through the peel,
    interpolate and the compositing."""
    import nvdiffrecmc_b200.optixutils as ou
    import nvdiffrecmc_b200.renderutils as ru
    v, f = synth.scene_mesh("blob+torus", level=2)
    vt, ft = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    ctx = ou.OptiXContext()
    ou.optix_build_bvh(ctx, vt, ft, rebuild=1)
    B, res = 2, RES
    mtx = torch.tensor(np.stack([synth.perspective(aspect=res[1] / res[0], n=0.1, f=10.0) @ synth.orbit_view(0.9 * b + 0.3)
                                 for b in range(B)]).astype(np.float32), device=dev)
    pos = ru.xfm_points(vt[None], mtx).detach().requires_grad_(True)
    g = torch.Generator(device=dev).manual_seed(spp)
    attrs = {"kd": torch.rand(vt.shape[0], 4, generator=g, device=dev), "nrm": torch.rand(vt.shape[0], 3, generator=g, device=dev)}
    for a in attrs.values():
        a[:, -1] = a[:, -1] * 0.8 + 0.1                               # alphas inside (0, 1)
        a.requires_grad_(True)
    topo = antialias_topology(ft)
    Ho, Wo = res[0] // spp, res[1] // spp
    bg = {"kd": torch.rand(B, Ho, Wo, 4, generator=g, device=dev, requires_grad=True)}
    G = {k: torch.rand(B, Ho, Wo, a.shape[1], generator=g, device=dev) * 2 - 1 for k, a in attrs.items()}

    def run(fn):
        with DepthPeeler(ctx, mtx, res, pos, ft) as p:
            rasts = [p.rasterize_next_layer()[0] for _ in range(3)]
        layers = [({k: interpolate(a, r[:, ::spp, ::spp], ft)[0] for k, a in attrs.items()}, r) for r in rasts]
        out = fn(layers)
        keys = list(out)
        ins = [*attrs.values(), bg["kd"], pos]
        return out, torch.autograd.grad([out[k] for k in keys], ins, [G[k] for k in keys])

    got, ggot = run(lambda ls: composite(ls, pos, ft, background=bg, topology=topo, spp=spp))
    ref, gref = run(lambda ls: _chain_ss(ls, pos, ft, topo, bg, spp))
    for k in got:
        _bits(got[k], ref[k], k)
    for a, b, what in zip(ggot, gref, ["d attr kd", "d attr nrm", "d background kd", "d pos"]):
        assert torch.isfinite(b).all() and b.abs().max() > 0, what
        _close(a, b, 1e-5, what)
