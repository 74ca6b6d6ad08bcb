"""Freeze the reference's image-space regularisers (render/regularizer.py:15-49, imported UNMODIFIED from the reference checkout and run
on the CPU) into tests/golden/ref_regularizer.npz: inputs, losses and every gradient for a fixed upstream gradient.

`render/regularizer.py` imports `nvdiffrast.torch` and, through `render.util` / `render.mesh`, `imageio` and `tinycudann`; none of them is
used by the three functions, so each is an empty stub here.  The three functions make no "cuda" factory call.

Two cases per function, [2,24,40,4] each:
  * "finite": exact RGB ties (greyscale and two-way), value(x) exactly at eps = fl32(0.001), diffuse luma + specular luma exactly at eps,
    lit values at 0, at 65535 and above, log(u + 1) just below and just above the sRGB threshold (and on it, where fl32 log reaches it),
    alpha 0, 1 and fractional, negative lights, black references;
  * "nonfinite": the same with one NaN and one +-inf pixel in the operands (lambda_nrm = 0 meets an inf: the reference's loss is NaN).
Run: python tests/golden/make_regularizer_golden.py   (only where the reference checkout exists)
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

REF_ROOT = "/root/reference"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_regularizer.npz")
SHAPE = (2, 24, 40)
G = np.float32(0.75)                       # the upstream gradient of every loss
EPS = np.float32(0.001)
SRGB_T = np.float32(0.0031308)
LAMBDAS = {"shading_loss": {"finite": (0.15, 0.0025), "nonfinite": (0.15, 0.0025)},
           "material_smoothness_grad": {"finite": (0.1, 0.05, 0.025), "nonfinite": (0.25, 0.1, 0.0)},
           "chroma_loss": {"finite": (0.025,), "nonfinite": (0.025,)}}
ARGS = {"shading_loss": ("diffuse_light", "specular_light", "color_ref"), "material_smoothness_grad": ("kd_grad", "ks_grad", "nrm_grad"),
        "chroma_loss": ("kd", "color_ref")}


def reference_regularizer():
    """render.regularizer of the reference checkout, imported with stubbed nvdiffrast / imageio / tinycudann."""
    stubs = {"nvdiffrast": types.ModuleType("nvdiffrast"), "nvdiffrast.torch": types.ModuleType("nvdiffrast.torch"),
             "imageio": types.ModuleType("imageio"), "tinycudann": types.ModuleType("tinycudann")}
    stubs["nvdiffrast"].torch = stubs["nvdiffrast.torch"]
    saved = {k: sys.modules.get(k) for k in list(stubs) + [k for k in sys.modules if k == "render" or k.startswith("render.")]}
    for k in saved:
        sys.modules.pop(k, None)
    sys.modules.update(stubs)
    sys.path.insert(0, REF_ROOT)
    try:
        return importlib.import_module("render.regularizer")
    finally:
        sys.path.remove(REF_ROOT)
        for k in [k for k in sys.modules if k == "render" or k.startswith("render.")] + list(stubs):
            sys.modules.pop(k, None)
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v


def _luma32(x):
    x = np.asarray(x, np.float32)
    return ((x[..., 0] + x[..., 1]) + x[..., 2]) / np.float32(3)


def _grey_at(target):
    """A float32 c with luma((c, c, c)) == target exactly (the nearest such c found by stepping ulps)."""
    c = np.float32(target)
    for _ in range(64):
        l = _luma32([c, c, c])
        if l == target:
            return c
        c = np.nextafter(c, np.float32(np.inf) if l < target else np.float32(-np.inf))
    raise AssertionError("no grey value with luma %r" % target)


def _srgb_edge_values():
    """Lit values u (float32) with torch.log(u + 1) just below, just above and (if fl32 log reaches it) on the sRGB threshold: u + 1 steps
    through the float32 neighbours of exp(threshold), and u = (u + 1) - 1 is exact."""
    y0 = np.float32(np.exp(np.float64(SRGB_T)))
    ys = [y0]
    for _ in range(8):
        ys = [np.nextafter(ys[0], np.float32(0))] + ys + [np.nextafter(ys[-1], np.float32(2))]
    us = (np.array(ys, np.float32) - np.float32(1)).astype(np.float32)
    L = torch.log(torch.from_numpy(us) + 1).numpy()
    below, above, on = us[L < SRGB_T][-1:], us[L > SRGB_T][:1], us[L == SRGB_T][:1]
    return np.concatenate([below, on, above]).astype(np.float32)


def make_inputs(case):
    """{function: {argument: [2,24,40,4] float32}} for one case."""
    rng = np.random.default_rng(11 if case == "finite" else 12)
    B, H, W = SHAPE
    alpha = (rng.random((B, H, W)) < 0.8).astype(np.float32)
    alpha[:, :, 0] = 0.0
    alpha[:, 1, :] = 1.0
    alpha[:, 2, ::3] = 0.5
    ref = np.concatenate([rng.random((B, H, W, 3)), alpha[..., None]], -1).astype(np.float32)
    diff = np.concatenate([rng.uniform(-0.1, 1.5, (B, H, W, 3)), alpha[..., None]], -1).astype(np.float32)
    spec = np.concatenate([rng.uniform(-0.05, 0.6, (B, H, W, 3)), alpha[..., None]], -1).astype(np.float32)
    kd = np.concatenate([rng.random((B, H, W, 3)), alpha[..., None]], -1).astype(np.float32)
    kdg, ksg, nrg = (np.concatenate([np.abs(rng.normal(0, s, (B, H, W, 3))), alpha[..., None]], -1).astype(np.float32)
                     for s in (0.1, 0.05, 0.2))
    px = iter([(b, h, w) for b in range(B) for h in (3, 4, 5, 6) for w in range(1, W)])

    def put(arr, rgb, a=1.0):
        p = next(px)
        arr[p] = np.array(list(rgb) + [a], np.float32)
        return p

    # --- ties and eps in value(): color_ref and kd
    for rgb in ([0.5, 0.5, 0.5], [0.7, 0.7, 0.2], [0.2, 0.9, 0.9], [0.9, 0.3, 0.9], [0, 0, 0], [EPS, EPS / 2, EPS], [EPS / 4, EPS, EPS],
                [EPS, EPS, EPS], [np.nextafter(EPS, np.float32(0)), 0.0, 0.0], [1.0, 1.0, 1.0]):
        p = put(ref, rgb)
        kd[p] = ref[p]
        p = put(kd, rgb)
        ref[p] = [0.3, 0.6, 0.1, 1.0]
    # --- shading: greyscale lights equal to a greyscale reference (|img - tgt| = 0), luma sums at eps, lit values at 0 / 65535 / above,
    #     the sRGB threshold, negative lights
    for rgb in ([0.5, 0.5, 0.5], [0.25, 0.25, 0.25]):
        p = put(diff, rgb); spec[p] = [0, 0, 0, 1]; ref[p] = diff[p]
    g = _grey_at(EPS)
    p = put(diff, [g, g, g]); spec[p] = [0, 0, 0, 1]
    g2 = _grey_at(np.float32(0.0006))
    p = put(diff, [g2, g2, g2])
    sv = np.float32(EPS - _luma32(diff[p][:3]))               # the specular luma that brings the sum to eps exactly
    sg = _grey_at(sv)
    spec[p] = [sg, sg, sg, 1]
    assert np.float32(_luma32(diff[p][:3]) + _luma32(spec[p][:3])) == EPS
    p = put(diff, [g2, g2, g2]); spec[p] = [sg, sg, np.nextafter(sg, np.float32(0)), 1]      # just below eps
    p = put(diff, [0, 0, 0]); spec[p] = [0, 0, 0, 1]
    p = put(diff, [0, 0, 0], a=0.0); spec[p] = [0.2, 0.2, 0.2, 0]
    p = put(diff, [65535, 65535, 65535]); spec[p] = [0, 0, 0, 1]; ref[p] = [1, 1, 1, 1]
    p = put(diff, [70000, 60000, 80000]); spec[p] = [10, 10, 10, 1]
    for u in _srgb_edge_values():
        g = _grey_at(u)
        p = put(diff, [g, g, g]); spec[p] = [0, 0, 0, 1]
        p = put(ref, [u, u / 2, u / 4])                       # the reference's value on the threshold
    p = put(diff, [-0.3, -0.2, -0.4]); spec[p] = [-0.1, 0.05, -0.2, 1]
    p = put(diff, [-0.3, 0.1, 0.1]); spec[p] = [0.2, 0.1, 0.0, 1]
    # --- material smoothness: zero jitter, alpha 0 with non-zero jitter
    for arr in (kdg, ksg, nrg):
        arr[0, 7, 3] = [0, 0, 0, 1]
        arr[0, 7, 4] = [0.3, 0.1, 0.2, 0]
    if case == "nonfinite":
        diff[1, 8, 5, 1] = np.nan
        spec[1, 9, 7, 0] = np.inf
        ref[0, 8, 9, 2] = np.nan
        kd[0, 10, 11, 1] = np.nan
        kd[1, 10, 12, 0] = -np.inf
        kdg[1, 11, 3, 2] = np.nan
        nrg[0, 11, 4, 0] = np.inf
        ksg[1, 12, 5, 3] = -np.inf
    return {"shading_loss": dict(diffuse_light=diff, specular_light=spec, color_ref=ref),
            "material_smoothness_grad": dict(kd_grad=kdg, ks_grad=ksg, nrm_grad=nrg),
            "chroma_loss": dict(kd=kd, color_ref=ref)}


def run_reference(reg, fn, ins, lambdas):
    """(loss, {argument: gradient}) of the reference function on the CPU; color_ref is a constant."""
    ts = {k: torch.from_numpy(v.copy()).requires_grad_(k != "color_ref") for k, v in ins.items()}
    loss = getattr(reg, fn)(*[ts[k] for k in ARGS[fn]], *lambdas)
    loss.backward(torch.tensor(G))
    return loss.detach().numpy().astype(np.float32), {k: t.grad.numpy() for k, t in ts.items() if k != "color_ref"}


def generate():
    reg = reference_regularizer()
    out = {"G": np.array(G, np.float32)}
    for case in ("finite", "nonfinite"):
        inputs = make_inputs(case)
        for fn, ins in inputs.items():
            lam = LAMBDAS[fn][case]
            loss, grads = run_reference(reg, fn, ins, lam)
            pre = "%s/%s/" % (fn, case)
            out[pre + "lambdas"] = np.array(lam, np.float64)
            out[pre + "loss"] = loss
            for k, v in ins.items():
                out[pre + k] = v
            for k, v in grads.items():
                out[pre + "d_" + k] = v
    return out


if __name__ == "__main__":
    data = generate()
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, "%d arrays" % len(data))
    for k, v in data.items():
        if k.endswith("/loss"):
            print("  %-40s %r" % (k, float(v)))
