"""CPU oracle of the multiresolution hash-grid encoding -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/hashgrid.c`` (level table, forward, d x, d params; the contract is stated in
nvdiffrecmc_b200/csrc/hashgrid.cu).  Two builds of the same source: fp32 (``HashGridOracle()``, compared bit for bit with the CUDA
forward and d x) and fp64 (``HashGridOracle(f64=True)``, checked by finite differences).  Only ``tests/`` and the developer tools import
it; ``nvdiffrecmc_b200`` never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
_SRC = os.path.join(_HERE, "hashgrid.c")

# the configuration render/mlptexture.py:57-70 hard-codes
REF_CONFIG = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16,
              "per_level_scale": float(np.exp(np.log(4096 / 16) / 15))}


def _lib_path(f64):
    return os.path.join(_BUILD, "libhashgrid_f64.so" if f64 else "libhashgrid_f32.so")


def build(force=False):
    """Compile oracle/hashgrid.c with gcc (fp32 + fp64); -ffp-contract=off is what makes the fp32 build bit-comparable."""
    os.makedirs(_BUILD, exist_ok=True)
    for f64 in (False, True):
        out = _lib_path(f64)
        if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(_SRC):
            continue
        tmp = out + ".%d.tmp" % os.getpid()
        cmd = ["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", tmp, _SRC, "-lm"]
        if f64:
            cmd.insert(1, "-DORACLE_F64")
        subprocess.run(cmd, check=True)
        os.replace(tmp, out)


def init_params(n_params, seed=1337):
    """The contract's initialisation: uniform in [-1e-4, 1e-4] from a CPU torch.Generator seeded with `seed`."""
    import torch
    g = torch.Generator().manual_seed(int(seed))
    return ((torch.rand(n_params, generator=g, dtype=torch.float32) * 2.0 - 1.0) * 1e-4).numpy()


class HashGridOracle:
    def __init__(self, f64=False):
        build()
        self.f64 = f64
        self.dt = np.float64 if f64 else np.float32
        self.lib = C.CDLL(_lib_path(f64))
        assert self.lib.hg_sizeof_real() == (8 if f64 else 4)

    def levels(self, cfg):
        """Level table of an encoding config: dict(n_levels, offset [L+1] uint64, res [L] uint32, scale [L] fp32, dense_mask)."""
        L = int(cfg.get("n_levels", 16))
        off = np.zeros(17, np.uint64); res = np.zeros(16, np.uint32); scale = np.zeros(16, np.float32); mask = C.c_uint32(0)
        rc = self.lib.hg_levels(C.c_int(L), C.c_int(int(cfg.get("log2_hashmap_size", 19))), C.c_double(float(cfg.get("base_resolution", 16))),
                                C.c_double(float(cfg.get("per_level_scale", 2.0))), C.c_void_p(off.ctypes.data), C.c_void_p(res.ctypes.data),
                                C.c_void_p(scale.ctypes.data), C.byref(mask))
        assert rc == 0, cfg
        return {"n_levels": L, "offset": off[:L + 1].copy(), "res": res[:L].copy(), "scale": scale[:L].copy(), "dense_mask": int(mask.value)}

    def _args(self, lv):
        off = np.zeros(17, np.uint64); res = np.zeros(16, np.uint32); scale = np.zeros(16, np.float32)
        L = lv["n_levels"]
        off[:L + 1] = lv["offset"]; res[:L] = lv["res"]; scale[:L] = lv["scale"]
        keep = (off, res, scale)
        return keep, [C.c_int(L), C.c_void_p(off.ctypes.data), C.c_void_p(res.ctypes.data), C.c_void_p(scale.ctypes.data),
                      C.c_uint32(lv["dense_mask"])]

    def _a(self, x):
        return np.ascontiguousarray(np.asarray(x, dtype=self.dt))

    def forward(self, x, params, lv):
        """[N, 2L]"""
        x = self._a(x).reshape(-1, 3); p = self._a(params)
        assert p.size == 2 * int(lv["offset"][-1])
        out = np.zeros((x.shape[0], 2 * lv["n_levels"]), self.dt)
        keep, a = self._args(lv)
        self.lib.hg_fwd(C.c_void_p(x.ctypes.data), C.c_int64(x.shape[0]), C.c_void_p(p.ctypes.data), *a, C.c_void_p(out.ctypes.data))
        return out

    def backward(self, x, params, lv, d_out, want_params=True, want_x=True):
        """-> (d_params or None, d_x or None)"""
        x = self._a(x).reshape(-1, 3); p = self._a(params); g = self._a(d_out)
        assert g.shape == (x.shape[0], 2 * lv["n_levels"])
        dp = np.zeros_like(p) if want_params else None
        dx = np.zeros_like(x) if want_x else None
        keep, a = self._args(lv)
        self.lib.hg_bwd(C.c_void_p(x.ctypes.data), C.c_int64(x.shape[0]), C.c_void_p(p.ctypes.data), *a, C.c_void_p(g.ctypes.data),
                        C.c_void_p(dp.ctypes.data) if want_params else None, C.c_void_p(dx.ctypes.data) if want_x else None)
        return dp, dx


_CACHE = {}


def hashgrid_oracle(f64=False):
    if f64 not in _CACHE:
        _CACHE[f64] = HashGridOracle(f64=f64)
    return _CACHE[f64]
