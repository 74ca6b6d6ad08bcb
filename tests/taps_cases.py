"""Operands of the jittered regulariser taps (jitter_taps, oracle/taps.c) shared by the CPU and GPU tests: numpy, in the argument order of
jitter_taps."""
import numpy as np

ARGS = ["rast", "jitter", "kd", "ks", "gb_normal", "perturbed_nrm", "kd_jitter", "ks_jitter"]


def random_case(rng, B, H, W, ckd, pn, mlp, cover=0.7, sigma=0.05):
    rast = np.zeros((B, H, W, 4), np.float32)
    rast[..., 3] = (rng.random((B, H, W)) < cover) * 5.0
    yy, xx = np.meshgrid((np.arange(H) + 0.5) / H, (np.arange(W) + 0.5) / W, indexing="ij")
    jit = (np.stack([xx, yy], -1)[None] + rng.normal(0, sigma, (B, H, W, 2))).astype(np.float32)
    kd, ks, n = rng.random((B, H, W, ckd)), rng.random((B, H, W, 3)), rng.normal(size=(B, H, W, 3))
    p = rng.normal(size=(B, H, W, 3)) + [0, 0, 1.0] if pn else None
    kdj = rng.random((B, H, W, ckd)) if mlp else None
    ksj = rng.random((B, H, W, 3)) if mlp else None
    return [rast, jit, kd, ks, n, p, kdj, ksj]
