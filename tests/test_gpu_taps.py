"""GPU: jitter_taps (csrc/taps.cu) against the fp32 oracle (oracle/taps.c) -- forward and one-writer gradients bit for bit, scattered
gradients per element under check_scatter_fp32 --, against the reference's lines composed from raster.texture and torch autograd, and
against the reference's own shade() frozen in tests/golden/ref_jitter_taps.npz; edge inputs, no_grad and CUDA-graph capture."""
import numpy as np
import pytest
import torch

from common import check_scatter_fp32, nan_bits
from oracle.taps import taps_oracle
from taps_cases import ARGS, random_case
from test_oracle_taps import CASES, GOLDEN_BAR, golden_case
from nvdiffrecmc_b200 import _lib, raster
from nvdiffrecmc_b200.regularizer import jitter_taps

pytestmark = pytest.mark.gpu
DEV = "cuda"
ONE_WRITER = ["kd_jitter", "ks_jitter"]


def to_dev(args, strided=False):
    """Device copies; with `strided`, kd is a channel-sliced view, ks the [..., 0:3] slice of a 4-channel sample and gb_normal a
    transposed layout, as shade() hands them over."""
    out = []
    for name, a in zip(ARGS, args):
        if a is None:
            out.append(None)
            continue
        t = torch.tensor(np.asarray(a, np.float32), device=DEV)
        if strided and name == "ks":
            t = torch.cat([t, torch.rand_like(t[..., :1])], -1)[..., 0:3]
        elif strided and name == "kd":
            t = torch.cat([torch.rand_like(t[..., :1]), t], -1)[..., 1:]
        elif strided and name == "gb_normal":
            t = t.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)
        out.append(t)
    return out


def leaves(ops):
    return [None if t is None else (t.detach().requires_grad_(True) if i >= 2 else t) for i, t in enumerate(ops)]


def run(ops, G):
    """jitter_taps forward and the gradients of sum_k <G_k, buffer_k> -> (buffers, {operand: gradient}) as numpy"""
    ops = leaves(ops)
    out = jitter_taps(*ops)
    loss = sum((out[k] * G[k]).sum() for k in out)
    need = [(n, t) for n, t in zip(ARGS, ops) if t is not None and t.requires_grad]
    gr = torch.autograd.grad(loss, [t for _, t in need])
    return {k: v.detach().cpu().numpy() for k, v in out.items()}, {n: g.cpu().numpy() for (n, _), g in zip(need, gr)}


def upstream(fwd, seed):
    rng = np.random.default_rng(seed)
    return {k: rng.normal(size=v.shape).astype(np.float32) for k, v in fwd.items()}


def check_vs_oracle(tag, args, strided=False, seed=0):
    o = taps_oracle()
    want = o.forward(*args)
    G = upstream(want, seed)
    got_f, got_g = run(to_dev(args, strided), {k: torch.tensor(v, device=DEV) for k, v in G.items()})
    assert sorted(got_f) == sorted(want)
    for k in want:
        assert np.array_equal(nan_bits(got_f[k]), nan_bits(want[k])), "%s: %s differs from the fp32 oracle at %d elements" % (
            tag, k, int((nan_bits(got_f[k]) != nan_bits(want[k])).sum()))
    s, a, n = (o.backward(*args, G, terms=t) for t in ("sum", "abs", "count"))
    assert sorted(got_g) == sorted(s)
    for k in got_g:
        if k in ONE_WRITER:
            assert np.array_equal(nan_bits(got_g[k]), nan_bits(s[k])), "%s: d %s differs from the fp32 oracle" % (tag, k)
        else:
            check_scatter_fp32("%s d %s" % (tag, k), got_g[k], s[k], a[k], n[k], tag="taps")
    return got_f, got_g


CONFIGS = {"tex_kd3": (3, False, False), "tex_kd4_nrm": (4, True, False), "mlp_kd3": (3, False, True), "mlp_kd4_nrm": (4, True, True)}
SIZES = [(2, 13, 19), (1, 1, 1), (2, 33, 31), (3, 16, 24)]


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_matches_fp32_oracle(cfg, size):
    ckd, pn, mlp = CONFIGS[cfg]
    args = random_case(np.random.default_rng(10 * list(CONFIGS).index(cfg) + SIZES.index(size)), *size, ckd, pn, mlp)
    check_vs_oracle("%s %s" % (cfg, size), args, strided=size == (3, 16, 24))


def _centre_jitter(B, H, W, dx=0.0):
    yy, xx = np.meshgrid((np.arange(H) + 0.5) / H, (np.arange(W) + 0.5 + dx) / W, indexing="ij")
    return np.broadcast_to(np.stack([xx, yy], -1), (B, H, W, 2)).astype(np.float32).copy()


def edge_case(kind):
    rng = np.random.default_rng(3)
    B, H, W = 2, 8, 16
    args = random_case(rng, B, H, W, 4, True, False)
    if kind == "outside":                      # jitter far outside [0, 1]: every tap clamps to the border texels
        args[1] = rng.uniform(-1.5, 2.5, (B, H, W, 2)).astype(np.float32)
    elif kind == "empty":
        args[0][..., 3] = 0
    elif kind == "full":
        args[0][..., 3] = 1
    elif kind == "tie":                        # jitter at the pixel centres of power-of-two sides: fx = fy = 0, every tap == its value
        args[1] = _centre_jitter(B, H, W)
    elif kind == "degenerate_nrm":             # zero-length perturbed normals, and taps that cancel sn(p) exactly (the 1e-20 clamp)
        args[1] = _centre_jitter(B, H, W, dx=1.0)
        p = np.broadcast_to(rng.normal(size=(B, H, 1, 3)), (B, H, W, 3)) * np.where(np.arange(W) % 2, -1.0, 1.0)[None, None, :, None]
        p = p.copy()
        p[:, ::3, ::5] = 0
        args[5] = p
    elif kind == "nan_red":                    # NaN in ks's red channel, which the [0, 1, 1] mask multiplies by 0: the buffer stays NaN
        args[3][:, ::2, ::3, 0] = np.nan
    return args


@pytest.mark.parametrize("kind", ["outside", "empty", "full", "tie", "degenerate_nrm", "nan_red"])
def test_edge_inputs(kind):
    args = edge_case(kind)
    f, g = check_vs_oracle(kind, args)
    if kind == "empty":
        assert not f["kd_grad"][..., :4].any() and not g["gb_normal"].any()
    if kind == "tie":
        assert not f["kd_grad"][..., :4].any() and not g["kd"][..., :3].any() and not g["ks"].any()
    if kind == "degenerate_nrm":
        assert np.isfinite(g["perturbed_nrm"]).all() and np.abs(g["perturbed_nrm"]).max() > 1e6       # the clamp's 1 / 1e-10
    if kind == "nan_red":
        assert np.isnan(f["ks_grad"][:, ::2, ::3, 0]).all() and np.isfinite(g["ks"]).all()


def test_hot_case_8x512():
    args = random_case(np.random.default_rng(9), 8, 512, 512, 3, True, False, sigma=0.005)
    check_vs_oracle("8x512^2", args)


# ---- the reference's lines (render.py:50-97), with raster.texture as dr.texture and torch autograd ----
def sn(x):
    return x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=1e-20))


def composition(rast, jitter, kd, ks, gb_normal, perturbed_nrm=None, kd_jitter=None, ks_jitter=None):
    tex = lambda t: raster.texture(t.contiguous(), jitter, filter_mode='linear', boundary_mode='clamp')
    mask = (rast[..., -1:] > 0).float()
    grad_weight = mask * tex(mask)
    m011 = torch.tensor([0, 1, 1], dtype=torch.float32, device=DEV)[None, None, None, :]
    if kd_jitter is not None:
        kd_grad = torch.abs(kd_jitter - kd)
        ks_grad = torch.abs(ks_jitter - ks) * m011
    else:
        kd_grad = torch.abs(tex(kd) - kd) * grad_weight
        ks_grad = torch.abs(tex(ks) - ks) * m011 * grad_weight
    alpha = kd[..., 3:4] if kd.shape[-1] == 4 else torch.ones_like(kd[..., 0:1])
    nrm_grad = torch.abs(tex(gb_normal) - gb_normal) * grad_weight
    out = {"kd_grad": torch.cat((kd_grad, alpha), -1), "ks_grad": torch.cat((ks_grad, alpha), -1), "normal_grad": torch.cat((nrm_grad, alpha), -1)}
    if perturbed_nrm is not None:
        pg = 1.0 - sn(sn(tex(perturbed_nrm)) + sn(perturbed_nrm))[..., 2:3]
        out["perturbed_nrm_grad"] = torch.cat((pg.repeat(1, 1, 1, 3) * grad_weight, alpha), -1)
    return out


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_matches_torch_composition(cfg):
    """kd_grad, ks_grad, normal_grad bit for bit; perturbed_nrm_grad within 4 ulp of 1 (torch's 3-element sums may take another order);
    kd, ks and gb_normal gradients within the per-element scatter bar of the fp32 oracle's terms (the composition adds the same terms);
    perturbed_nrm's within that bar plus 1024 * 2^-24 of the terms' absolute sum A.  torch sums the three products of each dot, of g_l and
    of repeat's backward in its own order, and the two normalisations in series amplify that: in sn's adjoint gy / l and 2 g_d x cancel
    along x, so a term's rounding is relative to summands larger than the term (measured on an H100: up to 390 * 2^-24 A)."""
    ckd, pn, mlp = CONFIGS[cfg]
    args = random_case(np.random.default_rng(21), 2, 33, 31, ckd, pn, mlp)
    ops = to_dev(args)
    o = taps_oracle()
    G = upstream(o.forward(*args), 4)
    Gd = {k: torch.tensor(v, device=DEV) for k, v in G.items()}
    got_f, got_g = run(ops, Gd)
    lv = leaves(ops)
    ref = composition(*lv)
    need = [(n, t) for n, t in zip(ARGS, lv) if t is not None and t.requires_grad]
    rg = dict(zip([n for n, _ in need], torch.autograd.grad(sum((ref[k] * Gd[k]).sum() for k in ref), [t for _, t in need])))
    for k in ("kd_grad", "ks_grad", "normal_grad"):
        assert np.array_equal(nan_bits(got_f[k]), nan_bits(ref[k].detach().cpu().numpy())), k
    if pn:
        err = np.abs(got_f["perturbed_nrm_grad"] - ref["perturbed_nrm_grad"].detach().cpu().numpy())
        assert err.max() <= 4 * 2.0 ** -23, err.max()
    a, n = (o.backward(*args, G, terms=t) for t in ("abs", "count"))
    for k in got_g:
        r = rg[k].cpu().numpy()
        if k in ONE_WRITER:
            assert np.array_equal(nan_bits(got_g[k]), nan_bits(r)), k
        elif k == "perturbed_nrm":
            bound = 1024 * 2.0 ** -24 * a[k] + 2 * (n[k] * 2.0 ** -24) * a[k]
            err = np.abs(got_g[k] - r)
            assert (err <= bound).all(), (k, float((err / np.maximum(bound, 1e-30)).max()))
            print("[taps] composition d perturbed_nrm: worst error %.3g of A * 2^-24" % float((err / np.maximum(a[k], 1e-30)).max() * 2.0 ** 24))
        else:
            check_scatter_fp32("composition d %s" % k, got_g[k], r, a[k], n[k], tag="taps")


@pytest.mark.parametrize("case", CASES)
def test_matches_reference_golden(case):
    args, G, want_fwd, want_bwd = golden_case(case)
    f, g = run(to_dev(args), {k: torch.tensor(v, device=DEV) for k, v in G.items()})
    for k in want_fwd:
        assert np.abs(f[k] - want_fwd[k]).max() <= GOLDEN_BAR, k
    assert sorted(g) == sorted(want_bwd)
    for k in want_bwd:
        assert np.abs(g[k] - want_bwd[k]).max() <= GOLDEN_BAR, k


def test_no_grad_saves_nothing():
    ops = leaves(to_dev(random_case(np.random.default_rng(1), 2, 9, 11, 4, True, False)))
    with torch.no_grad():
        out = jitter_taps(*ops)
    assert all(v.grad_fn is None and not v.requires_grad for v in out.values())
    out = jitter_taps(*[None if t is None else t.detach() for t in ops])
    assert all(v.grad_fn is None for v in out.values())
    with_grad = jitter_taps(*ops)
    assert all(v.grad_fn is not None for v in with_grad.values())


def test_one_launch_each_way():
    ops = leaves(to_dev(random_case(np.random.default_rng(2), 2, 9, 11, 3, True, False)))
    before = dict(_lib.LAUNCHES)
    out = jitter_taps(*ops)
    sum(v.sum() for v in out.values()).backward()
    assert _lib.LAUNCHES["jitter_taps_fwd"] - before.get("jitter_taps_fwd", 0) == 1
    assert _lib.LAUNCHES["jitter_taps_bwd"] - before.get("jitter_taps_bwd", 0) == 1


@pytest.mark.parametrize("name", ["kd", "jitter", "perturbed_nrm", "ks_jitter"])
def test_shape_and_device_errors(name):
    args = random_case(np.random.default_rng(3), 2, 9, 11, 3, True, True)
    ops = dict(zip(ARGS, to_dev(args)))
    ops[name] = ops[name][:, :8]
    before = sum(_lib.LAUNCHES.values())
    with pytest.raises(ValueError, match="%s has B,H,W" % name):
        jitter_taps(**ops)
    ops = dict(zip(ARGS, to_dev(args)))
    ops[name] = ops[name].cpu()
    with pytest.raises(ValueError, match="%s must be a CUDA tensor" % name):
        jitter_taps(**ops)
    assert sum(_lib.LAUNCHES.values()) == before


def test_jitter_requiring_grad_raises():
    ops = dict(zip(ARGS, to_dev(random_case(np.random.default_rng(4), 1, 5, 6, 3, False, False))))
    ops["jitter"].requires_grad_(True)
    with pytest.raises(ValueError, match="jitter is a constant"):
        jitter_taps(**ops)
    ops["jitter"].requires_grad_(False)
    ops["rast"].requires_grad_(True)                 # rasterize's output: only its coverage test is read
    jitter_taps(**ops)


def test_cuda_graph_replays_like_eager():
    args = random_case(np.random.default_rng(6), 2, 40, 56, 4, True, False)
    ops = leaves(to_dev(args))
    o = taps_oracle()
    G = upstream(o.forward(*args), 8)
    Gd = {k: torch.tensor(v, device=DEV) for k, v in G.items()}
    need = [t for t in ops[2:] if t is not None]

    def step():
        out = jitter_taps(*ops)
        return out, torch.autograd.grad(sum((out[k] * Gd[k]).sum() for k in out), need)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager_out, eager_g = step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_g = step()
    graph.replay()
    torch.cuda.synchronize()
    for k in eager_out:
        assert np.array_equal(nan_bits(g_out[k].detach().cpu().numpy()), nan_bits(eager_out[k].detach().cpu().numpy())), k
    a, n = (o.backward(*args, G, terms=t) for t in ("abs", "count"))
    for name, ge, gg in zip(["kd", "ks", "gb_normal", "perturbed_nrm"], eager_g, g_g):
        check_scatter_fp32("graph d %s" % name, gg.cpu().numpy(), ge.cpu().numpy(), a[name], n[name], tag="taps")
