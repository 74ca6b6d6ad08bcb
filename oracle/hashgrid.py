"""CPU oracle of the multiresolution hash-grid encoding -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrapper around ``oracle/hashgrid.c`` (level table, forward, d x, d params; the contract is stated in
nvdiffrecmc_b200/csrc/hashgrid.cu).  Two builds of the same source: fp32 (``hashgrid_oracle()``, compared bit for bit with the CUDA
forward and d x) and fp64 (``hashgrid_oracle(f64=True)``, checked by finite differences).  Only ``tests/`` and the developer tools import
it; ``nvdiffrecmc_b200`` never does.
"""
import ctypes as C

import numpy as np

from oracle import CLib, _I, _I64, _P

# the configuration render/mlptexture.py:57-70 hard-codes
REF_CONFIG = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16,
              "per_level_scale": float(np.exp(np.log(4096 / 16) / 15))}


def init_params(n_params, seed=1337):
    """The contract's initialisation: uniform in [-1e-4, 1e-4] from a CPU torch.Generator seeded with `seed`."""
    import torch
    g = torch.Generator().manual_seed(int(seed))
    return ((torch.rand(n_params, generator=g, dtype=torch.float32) * 2.0 - 1.0) * 1e-4).numpy()


class HashGridOracle(CLib):
    LIB = "hashgrid"
    SIGS = {
        "hg_sizeof_real": ([], _I),
        "hg_levels": ([_I, _I, C.c_double, C.c_double] + [_P] * 4, _I),
        "hg_fwd": ([_P, _I64, _P, _I, _P, _P, _P, C.c_uint32, _P], None),
        "hg_bwd": ([_P, _I64, _P, _I, _P, _P, _P, C.c_uint32] + [_P] * 3, None),
    }

    def levels(self, cfg):
        """Level table of an encoding config: dict(n_levels, offset [L+1] uint64, res [L] uint32, scale [L] fp32, dense_mask)."""
        L = int(cfg.get("n_levels", 16))
        off = np.zeros(17, np.uint64); res = np.zeros(16, np.uint32); scale = np.zeros(16, np.float32); mask = C.c_uint32(0)
        rc = self.lib.hg_levels(L, int(cfg.get("log2_hashmap_size", 19)), float(cfg.get("base_resolution", 16)), float(cfg.get("per_level_scale", 2.0)),
                                off.ctypes.data, res.ctypes.data, scale.ctypes.data, C.byref(mask))
        assert rc == 0, cfg
        return {"n_levels": L, "offset": off[:L + 1].copy(), "res": res[:L].copy(), "scale": scale[:L].copy(), "dense_mask": int(mask.value)}

    def _args(self, lv):
        off = np.zeros(17, np.uint64); res = np.zeros(16, np.uint32); scale = np.zeros(16, np.float32)
        L = lv["n_levels"]
        off[:L + 1] = lv["offset"]; res[:L] = lv["res"]; scale[:L] = lv["scale"]
        keep = (off, res, scale)
        return keep, [L, off.ctypes.data, res.ctypes.data, scale.ctypes.data, lv["dense_mask"]]

    def forward(self, x, params, lv):
        """[N, 2L]"""
        x = self._a(x).reshape(-1, 3); p = self._a(params)
        assert p.size == 2 * int(lv["offset"][-1])
        out = np.zeros((x.shape[0], 2 * lv["n_levels"]), self.dt)
        keep, a = self._args(lv)
        self.lib.hg_fwd(x.ctypes.data, x.shape[0], p.ctypes.data, *a, out.ctypes.data)
        return out

    def backward(self, x, params, lv, d_out, want_params=True, want_x=True):
        """-> (d_params or None, d_x or None)"""
        x = self._a(x).reshape(-1, 3); p = self._a(params); g = self._a(d_out)
        assert g.shape == (x.shape[0], 2 * lv["n_levels"])
        dp = np.zeros_like(p) if want_params else None
        dx = np.zeros_like(x) if want_x else None
        keep, a = self._args(lv)
        self.lib.hg_bwd(x.ctypes.data, x.shape[0], p.ctypes.data, *a, g.ctypes.data, dp.ctypes.data if want_params else None,
                        dx.ctypes.data if want_x else None)
        return dp, dx


hashgrid_oracle = HashGridOracle.get
