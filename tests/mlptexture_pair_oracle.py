"""MLPTexture3D.sample_pair's contract stated on the CPU oracle of the single sample (oracle/mlptexture.py) -- TEST INFRASTRUCTURE.

The pair is two single calls plus one add: the jittered point is t + offset, and d params, d t and d W are the two calls' sums, each add
made in the oracle build's precision; d offset is the jittered call's d t.  No C of its own."""
import numpy as np


def _jittered(o, t, offset):
    return np.asarray(t, o.dt).reshape(-1, 3) + np.asarray(offset, o.dt).reshape(-1, 3)      # one add in the build's precision


def pair_forward(o, t, offset, aabb, min_max, params, lv, weights):
    """(out, enc, out_jit, enc_jit): o.mlptex_forward at t and at t + offset."""
    out, enc = o.mlptex_forward(t, aabb, min_max, params, lv, weights)
    out_jit, enc_jit = o.mlptex_forward(_jittered(o, t, offset), aabb, min_max, params, lv, weights)
    return out, enc, out_jit, enc_jit


def pair_backward(o, t, offset, aabb, min_max, params, lv, weights, d_out, d_out_jit, want_params=True, want_t=True, want_offset=True,
                  want_w=True, terms="sum"):
    """(d params or None, d t or None, d offset or None, [d W per layer] or None): o.mlptex_backward at t with d_out and at t + offset
    with d_out_jit (true gradients, no x128 on d params; terms as mlptex_backward's)."""
    a = o.mlptex_backward(t, aabb, min_max, params, lv, weights, d_out, want_params, want_t, want_w, terms)
    b = o.mlptex_backward(_jittered(o, t, offset), aabb, min_max, params, lv, weights, d_out_jit, want_params, want_t or want_offset,
                          want_w, terms)
    dp = a[0] + b[0] if want_params else None
    dt = a[1] + b[1] if want_t else None
    dw = [x + y for x, y in zip(a[2], b[2])] if want_w else None
    return dp, dt, b[1] if want_offset else None, dw
