"""CPU oracle for the nvdiffrecmc hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy/ctypes wrappers around the six C restatements in this directory (see each file's header for what it restates and how it is
pinned): ``Oracle`` and ``Scene`` here wrap ``mcoracle.c``; ``oracle.geometry``, ``oracle.hashgrid``, ``oracle.texture``,
``oracle.mlptexture`` and ``oracle.dmtet`` wrap the C file of the same name.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import this package; ``nvdiffrecmc_b200`` never does.

``build()`` compiles every library twice from the same source: fp32 (the oracle proper, compared with the CUDA kernels) and fp64
(``f64=True``), used only to validate derivatives and hand-derived adjoints by finite differences.  ``CLib`` is the wrappers' common base:
it loads one library at one precision with a declared signature for every function the library exports, and ``get(f64)`` returns the one
shared instance of each (library, precision).

``build_ref()`` / ``Reference`` compile and drive the reference's OWN raygen source on the CPU (oracle/ref_shim -> oracle/_ref, only
where /root/reference exists; the built library is git-ignored and travels to the GPU box) -- the check of this restatement
against the reference itself, and the `--impl reference` arm of bench.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
# library: [its source, then the files that source #includes]
LIBS = {"mcoracle": ["mcoracle.c", "detmath.h"], "geometry": ["geometry.c"], "hashgrid": ["hashgrid.c"], "texture": ["texture.c"],
        "mlptexture": ["mlptexture.c", "hashgrid.c"], "dmtet": ["dmtet.c"]}


def _cpu_has_fma():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return " fma " in (line + " ")
    except OSError:
        pass
    return False


# -ffp-contract=off is mandatory: the fp32 builds make the CUDA kernels' discrete decisions with the same roundings and reproduce their
# explicitly rounded operations.  -mfma only turns the explicit fmaf() / fma() calls into one instruction (contraction stays off).
_CFLAGS = ["-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC"] + (["-mfma"] if _cpu_has_fma() else [])


def _lib_path(name, f64):
    return os.path.join(_BUILD, "lib%s_%s.so" % (name, "f64" if f64 else "f32"))


def _compile(cmd, out, inputs, force=False):
    """Run the compiler command `cmd` with `-o out` unless `out` is at least as new as every input.  The compiler writes a per-process
    temporary file that then replaces `out` in one step, so another process (a torchrun rank, a test worker) never loads a half-written
    library."""
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(s) for s in inputs):
        return
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = "%s.%d.tmp" % (out, os.getpid())
    subprocess.run(cmd + ["-o", tmp], check=True)
    os.replace(tmp, out)


def _build_lib(name, f64, force=False):
    srcs = [os.path.join(_HERE, s) for s in LIBS[name]]
    _compile(["gcc"] + _CFLAGS + (["-DORACLE_F64"] if f64 else []) + [srcs[0], "-lm"], _lib_path(name, f64), srcs, force)


def build(force=False):
    """Compile every library of LIBS with gcc, fp32 and fp64 (-DORACLE_F64), into oracle/_build/."""
    for name in LIBS:
        for f64 in (False, True):
            _build_lib(name, f64, force)


# A signature table maps every function a library exports to ([argument types], result type) (tests/test_oracle_signatures.py checks
# the tables against the sources).  REAL is a scalar `real`: c_float in the fp32 build, c_double in the fp64 one.
REAL = "real"
_P, _I, _I64 = C.c_void_p, C.c_int, C.c_int64
# the `terms` mode of the entry points that scatter (test-only): the sum of the terms, the sum of their absolute values, or the number of
# non-zero terms.  With n terms of absolute sum A, summing them in another order changes the sum by at most about 2 (n - 1) 2^-24 A.
TERMS = {"sum": 0, "abs": 1, "count": 2}


class CLib:
    """One oracle library at one precision: ``f64``, ``dt`` and ``real`` (the numpy and ctypes types of `real`), ``lib`` (rebuilt if
    stale, then loaded with every function of ``SIGS`` declared) and ``_a``.  ``get(f64)`` returns the one instance of a class and
    precision that every caller shares."""
    LIB, SIGS = None, {}
    _instances = {}

    def __init__(self, f64=False):
        self.f64 = f64
        self.dt, self.real = (np.float64, C.c_double) if f64 else (np.float32, C.c_float)
        _build_lib(self.LIB, f64)
        self.lib = C.CDLL(_lib_path(self.LIB, f64))
        for name, (args, res) in self.SIGS.items():
            fn = getattr(self.lib, name)          # AttributeError if the library does not export it
            fn.argtypes = [self.real if a is REAL else a for a in args]
            fn.restype = res
        sizeof_real, = [n for n in self.SIGS if n.endswith("_sizeof_real")]      # every library exports one
        assert getattr(self.lib, sizeof_real)() == C.sizeof(self.real)

    @classmethod
    def get(cls, f64=False):
        key = (cls, bool(f64))
        if key not in CLib._instances:
            CLib._instances[key] = cls(f64)
        return CLib._instances[key]

    def _a(self, x, shape=None):
        x = np.ascontiguousarray(np.asarray(x, dtype=self.dt))
        if shape is not None:
            x = np.ascontiguousarray(np.broadcast_to(x, shape))
        return x


# ------------------------------------------------------------------------------------------------
# oracle/_ref: the UNMODIFIED reference raygen program compiled for the host (oracle/ref_shim/), only where /root/reference exists
# ------------------------------------------------------------------------------------------------
REF_KERNEL = "/root/reference/render/optixutils/c_src/envsampling/kernel.cu"
REF_DENOISE = "/root/reference/render/optixutils/c_src/denoising.cu"
REF_RU_BSDF = "/root/reference/render/renderutils/c_src/bsdf.cu"
REF_RU_NORMAL = "/root/reference/render/renderutils/c_src/normal.cu"
REF_RU_LOSS = "/root/reference/render/renderutils/c_src/loss.cu"
REF_RU_MESH = "/root/reference/render/renderutils/c_src/mesh.cu"
_REF_DIR = os.path.join(_HERE, "_ref")
_REF_LIB = os.path.join(_REF_DIR, "libref_envshade.so")
_REF_LIB_DN = os.path.join(_REF_DIR, "libref_denoise.so")
_REF_LIB_RU = os.path.join(_REF_DIR, "libref_renderutils.so")
_SHIM = os.path.join(_HERE, "ref_shim")


def build_ref(force=False):
    """g++ on the reference's own kernel.cu / denoising.cu (and the headers they include) where they lie, through the host shims.  Returns
    the env_shade library path, or None when the reference tree is not present (GPU box) and no prebuilt library travelled with the snapshot."""
    if not os.path.exists(REF_KERNEL):
        return _REF_LIB if all(os.path.exists(l) for l in (_REF_LIB, _REF_LIB_DN, _REF_LIB_RU)) else None
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    jobs = [(_REF_LIB, "ref_env_shade.cpp", {"REF_KERNEL": REF_KERNEL}), (_REF_LIB_DN, "ref_denoise.cpp", {"REF_DENOISE": REF_DENOISE}),
            (_REF_LIB_RU, "ref_renderutils.cpp", {"REF_RU_BSDF": REF_RU_BSDF, "REF_RU_NORMAL": REF_RU_NORMAL, "REF_RU_LOSS": REF_RU_LOSS, "REF_RU_MESH": REF_RU_MESH})]
    for out, shim, macros in jobs:
        srcs = [os.path.join(_SHIM, shim), os.path.join(_SHIM, "optix.h")] + list(macros.values())
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-w", "-I" + cuda_inc, "-I" + _SHIM]
        cmd += ["-I" + d for d in sorted({os.path.dirname(v) for v in macros.values()})] + ['-D%s="%s"' % kv for kv in macros.items()]
        _compile(cmd + [srcs[0]], out, srcs, force)
    return _REF_LIB


class Reference:
    """The reference's own __raygen__rg / process_sample (kernel.cu:403-542) running on the CPU.  Visibility comes from `scene`
    (an fp32 oracle Scene): OptiX itself is closed source.  Raises RuntimeError when oracle/_ref cannot be built or found."""

    def __init__(self, orc):
        path = build_ref()
        if path is None:
            raise RuntimeError("oracle/_ref unavailable: /root/reference is not present and no prebuilt libref_envshade.so was found")
        assert not orc.f64, "the reference kernel is fp32"
        self.orc = orc
        self.lib = C.CDLL(path)
        self.lib.ref_set_visibility.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        self.lib.ref_env_shade.argtypes = [C.c_int] * 7 + [C.c_uint, C.c_uint, C.c_float, C.c_int] + [C.c_void_p] * 21
        self.lib.ref_set_ray_log.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        self.dn = C.CDLL(_REF_LIB_DN)
        self.dn.ref_bilateral_fwd.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float] + [C.c_void_p] * 4
        self.dn.ref_bilateral_bwd.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float] + [C.c_void_p] * 5

        self.ru = C.CDLL(_REF_LIB_RU)

        class _Desc(C.Structure):
            _fields_ = [("val", C.c_void_p), ("d_val", C.c_void_p), ("dims", C.c_int * 4)]
        self._Desc = _Desc
        self.ru.ref_ru_run.argtypes = [C.c_char_p, C.c_int, C.POINTER(_Desc), C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int]

    def image_loss(self, img, target, loss="l1", tonemapper="none", dout=None):
        """imgLossFwdKernel / imgLossBwdKernel (loss.cu:105-227).  Forward -> the mean of the per-pixel loss, as renderutils/ops.py:494 returns
        it; with dout (upstream gradient of that mean) -> (img_grad, target_grad)."""
        li = {"l1": 0, "mse": 1, "relmse": 2, "smape": 3, "n2n": 4}[loss]
        ti = 1 if tonemapper == "log_srgb" else 0
        img = np.ascontiguousarray(img, np.float32); target = np.ascontiguousarray(target, np.float32)
        n = img.shape[0] * img.shape[1] * img.shape[2]
        if dout is None:
            return float(self.renderutils("loss_fwd", [img, target], 1, i0=ti, i1=li).astype(np.float64).sum() / n)
        g = np.full(img.shape[:3] + (1,), np.float32(dout) / np.float32(n), np.float32)
        return self.renderutils("loss_bwd", [img, target], dout=g, i0=ti, i1=li)

    def xfm(self, points, matrix, is_points=True, dout=None):
        """xfmPointsFwdKernel / xfmPointsBwdKernel (mesh.cu:19-90).  points [B|1,V,3], matrix [B,4,4] -> [B,V,4|3]; with dout -> points gradient
        on the full batch [B,V,3] (the Python side sums it for a broadcast input)."""
        pts = np.ascontiguousarray(points, np.float32); mtx = np.ascontiguousarray(matrix, np.float32)
        B, V = mtx.shape[0], pts.shape[1]
        D = self._Desc
        descs = (D * 3)()
        out = np.zeros((B, V, 4 if is_points else 3), np.float32) if dout is None else np.ascontiguousarray(dout, np.float32)
        grad = np.zeros((B, V, 3), np.float32)
        for i, a in enumerate((pts, mtx, out)):
            descs[i].val = a.ctypes.data
            for k, v in enumerate(a.shape + (1,)):
                descs[i].dims[k] = v
        if dout is not None:
            descs[0].d_val = grad.ctypes.data
        rc = self.ru.ref_ru_run(b"xfm_bwd" if dout is not None else b"xfm_fwd", 3, descs, V, 1, B, 0.0, 1 if is_points else 0, 0)
        assert rc == 0
        return grad if dout is not None else out

    def renderutils(self, kernel, ins, out_channels=None, dout=None, f0=0.0, i0=0, i1=0):
        """Run one per-pixel kernel of render/renderutils/c_src/{bsdf,normal}.cu.  `kernel`: lambert|frostbite|fresnel|ndf|lambda|masking|
        specular|bsdf|psn + _fwd / _bwd.  ins: [N|1, H|1, W|1, C] arrays in the order of the kernel's parameter struct.  Forward returns
        out [N,H,W,out_channels]; backward (dout = upstream gradient) returns one full-grid gradient per input, as the plugin does
        before the Python side sums broadcast dimensions (renderutils/ops.py)."""
        ins = [np.ascontiguousarray(a, np.float32) for a in ins]
        grid = np.broadcast_shapes(*[a.shape[:3] for a in ins])
        N, H, W = grid
        bwd = dout is not None
        keep, descs = [], (self._Desc * (len(ins) + 1))()
        grads = []
        for i, a in enumerate(ins):
            descs[i].val = a.ctypes.data
            if bwd:
                g = np.zeros((N, H, W, a.shape[3]), np.float32); grads.append(g); descs[i].d_val = g.ctypes.data
            for k in range(4):
                descs[i].dims[k] = a.shape[k]
        out = np.ascontiguousarray(dout, np.float32) if bwd else np.zeros((N, H, W, out_channels), np.float32)
        descs[len(ins)].val = out.ctypes.data
        for k, v in enumerate(out.shape):
            descs[len(ins)].dims[k] = v
        rc = self.ru.ref_ru_run(kernel.encode(), len(ins) + 1, descs, W, H, N, float(f0), int(i0), int(i1))
        if rc != 0:
            raise ValueError("ref_ru_run(%s): %s" % (kernel, {1: "unknown kernel", 2: "wrong tensor count"}.get(rc, rc)))
        return grads if bwd else out

    def bilateral_fwd(self, col, nrm, zdz, sigma):
        """bilateral_denoiser_fwd_kernel (denoising.cu:14-72): -> [B,H,W,4] (rgb weighted sum, weight)."""
        f = lambda a: np.ascontiguousarray(a, np.float32)
        col, nrm, zdz = f(col), f(nrm), f(zdz)
        B, H, W = col.shape[:3]
        out = np.zeros((B, H, W, 4), np.float32)
        self.dn.ref_bilateral_fwd(B, H, W, float(sigma), col.ctypes.data, nrm.ctypes.data, zdz.ctypes.data, out.ctypes.data)
        return out

    def bilateral_bwd(self, nrm, zdz, sigma, out_grad, col=None):
        """bilateral_denoiser_bwd_kernel (denoising.cu:74-130): out_grad [B,H,W,4] -> col_grad [B,H,W,3]."""
        f = lambda a: np.ascontiguousarray(a, np.float32)
        nrm, zdz, og = f(nrm), f(zdz), f(out_grad)
        B, H, W = nrm.shape[:3]
        col = np.zeros((B, H, W, 3), np.float32) if col is None else f(col)
        cg = np.zeros((B, H, W, 3), np.float32)
        self.dn.ref_bilateral_bwd(B, H, W, float(sigma), col.ctypes.data, nrm.ctypes.data, zdz.ctypes.data, og.ctypes.data, cg.ctypes.data)
        return cg

    def env_shade(self, scene, mask, ro, gb_pos, gb_normal, gb_view_pos, gb_kd, gb_ks, light, pdf, rows, cols, perms, BSDF="pbr", n_samples_x=8,
                  rnd_seed=0, shadow_scale=1.0, grads=None, vis_mode="brute", ray_log=False):
        """Forward -> (diff, spec); with grads=(diff_grad, spec_grad) -> (pos_grad, nrm_grad, kd_grad, ks_grad, light_grad).
        ray_log=True (forward only) appends the directions of the shadow rays the reference traced, [B,H,W,2*n^2,3] in sample-slot
        order (NaN where the pixel is masked)."""
        f = lambda a: np.ascontiguousarray(a, np.float32)
        mask, ro, gb_pos, gb_normal, gb_kd, gb_ks = [f(a) for a in (mask, ro, gb_pos, gb_normal, gb_kd, gb_ks)]
        B, H, W = mask.shape
        view = np.ascontiguousarray(np.broadcast_to(f(gb_view_pos), (B, 1, 1, 3)))
        light, pdf, rows, cols = f(light), f(pdf), f(rows), f(cols)
        perms = np.ascontiguousarray(perms, np.int32)
        assert perms.shape[1] == n_samples_x * n_samples_x
        Hl, Wl = light.shape[:2]
        z4 = lambda: np.zeros((B, H, W, 3), np.float32)
        diff, spec = z4(), z4()
        dg, sg = (f(grads[0]), f(grads[1])) if grads is not None else (z4(), z4())
        pg, ng, kg, sgd, lg = z4(), z4(), z4(), z4(), np.zeros((Hl, Wl, 3), np.float32)
        occ = C.cast(self.orc.lib.orc_occluded1, C.c_void_p)
        self.lib.ref_set_visibility(occ, scene.h, {"brute": 0, "bvh": 1}[vis_mode])
        p = lambda a: a.ctypes.data
        S2 = 2 * n_samples_x * n_samples_x
        if ray_log:
            dirs = np.full((B, H, W, S2, 3), np.nan, np.float32); cnt = np.zeros((B, H, W), np.int32)
            self.lib.ref_set_ray_log(p(dirs), p(cnt), S2)
        self.lib.ref_env_shade(B, H, W, Hl, Wl, perms.shape[0], n_samples_x, BSDF_MODES.index(BSDF), int(rnd_seed) & 0xFFFFFFFF, float(shadow_scale),
                               0 if grads is None else 1, p(mask), p(ro), p(gb_pos), p(gb_normal), p(view), p(gb_kd), p(gb_ks), p(light), p(pdf), p(rows),
                               p(cols), p(perms), p(diff), p(spec), p(dg), p(sg), p(pg), p(ng), p(kg), p(sgd), p(lg))
        if ray_log:
            self.lib.ref_set_ray_log(None, None, 0)
            assert int(cnt.max()) <= S2
            return diff, spec, dirs
        return (diff, spec) if grads is None else (pg, ng, kg, sgd, lg)


def _envshade_struct(real):
    P = C.POINTER
    class S(C.Structure):
        _fields_ = [
            ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Hl", C.c_int32), ("Wl", C.c_int32),
            ("n_perms", C.c_int32), ("N", C.c_int32), ("bsdf", C.c_int32), ("seed", C.c_uint32),
            ("batch_offset", C.c_int32), ("backward", C.c_int32), ("vis_mode", C.c_int32), ("parallel_bwd", C.c_int32), ("shadow_scale", real),
            ("mask", C.c_void_p), ("ro", C.c_void_p), ("pos", C.c_void_p), ("nrm", C.c_void_p), ("view", C.c_void_p),
            ("kd", C.c_void_p), ("ks", C.c_void_p),
            ("light", C.c_void_p), ("pdf", C.c_void_p), ("rows", C.c_void_p), ("cols", C.c_void_p),
            ("perms", C.c_void_p), ("scene", C.c_void_p),
            ("diff", C.c_void_p), ("spec", C.c_void_p), ("diff_grad", C.c_void_p), ("spec_grad", C.c_void_p),
            ("pos_grad", C.c_void_p), ("nrm_grad", C.c_void_p), ("kd_grad", C.c_void_p), ("ks_grad", C.c_void_p),
            ("light_grad", C.c_void_p),
            ("rec_texel", C.c_void_p), ("rec_vis", C.c_void_p), ("counters", C.c_void_p),
            ("s_pos", C.c_void_p), ("s_nrm", C.c_void_p), ("s_kd", C.c_void_p), ("s_ks", C.c_void_p), ("abs_terms", C.c_int32),
        ]
    return S


BSDF_MODES = ["pbr", "diffuse", "white"]     # render/optixutils/ops.py:136

PEEL_SEP = np.float32(1.0 + 2.0 ** -16)


def peel_sep(t):
    """fl32(t * (1 + 2^-16)): the separation between consecutive depth-peel layers along a ray."""
    return (np.asarray(t, np.float32) * PEEL_SEP).astype(np.float32)


class Scene:
    """Triangle soup + canonical LBVH held by the C side."""
    def __init__(self, orc, verts, tris):
        self.orc = orc
        self.verts = np.ascontiguousarray(verts, dtype=orc.dt).reshape(-1, 3)
        self.tris = np.ascontiguousarray(tris, dtype=np.int32).reshape(-1, 3)
        assert self.tris.shape[0] > 0 and self.verts.shape[0] > 0
        self.T = self.tris.shape[0]
        self.h = orc.lib.orc_scene_create(self.verts.ctypes.data, self.verts.shape[0], self.tris.ctypes.data, self.T)
        orc.lib.orc_lbvh_build(self.h, self.verts.ctypes.data, self.tris.ctypes.data)

    def __del__(self):
        try:
            self.orc.lib.orc_scene_destroy(self.h)
        except Exception:
            pass

    def export_lbvh(self):
        T = self.T
        morton = np.zeros(T, np.uint32); prim = np.zeros(T, np.int32)
        left = np.zeros(max(T - 1, 1), np.int32); right = np.zeros(max(T - 1, 1), np.int32)
        lo = np.zeros((2 * T - 1, 3), self.orc.dt); hi = np.zeros((2 * T - 1, 3), self.orc.dt)
        self.orc.lib.orc_lbvh_export(self.h, morton.ctypes.data, prim.ctypes.data, left.ctypes.data, right.ctypes.data,
                                     lo.ctypes.data, hi.ctypes.data)
        return dict(morton=morton, prim=prim, left=left[:T - 1], right=right[:T - 1], lo=lo, hi=hi)

    def visibility(self, ro, rd, mode="brute", return_counters=False):
        ro = np.ascontiguousarray(ro, self.orc.dt).reshape(-1, 3); rd = np.ascontiguousarray(rd, self.orc.dt).reshape(-1, 3)
        vis = np.zeros(ro.shape[0], np.uint8); cnt = np.zeros(2, np.uint64)
        self.orc.lib.orc_visibility(self.h, 0 if mode == "brute" else 1, ro.shape[0], ro.ctypes.data, rd.ctypes.data,
                                    vis.ctypes.data, cnt.ctypes.data)
        return (vis, cnt) if return_counters else vis

    def closest_hit(self, ro, rd, t_after=None):
        """(tri_id [n] (-1 = miss), tuv [n,3] = (t, u, v)) of the closest hit, ties to the lowest id; with t_after [n], the closest
        hit with t > sep(t_after) (depth peeling's query; t_after = +inf: a miss)."""
        ro = np.ascontiguousarray(ro, self.orc.dt).reshape(-1, 3); rd = np.ascontiguousarray(rd, self.orc.dt).reshape(-1, 3)
        tid = np.zeros(ro.shape[0], np.int32); tuv = np.zeros((ro.shape[0], 3), self.orc.dt)
        if t_after is None:
            self.orc.lib.orc_closest_hit(self.h, ro.shape[0], ro.ctypes.data, rd.ctypes.data, tid.ctypes.data, tuv.ctypes.data)
        else:
            ta = np.ascontiguousarray(t_after, self.orc.dt).reshape(-1)
            assert ta.shape[0] == ro.shape[0]
            self.orc.lib.orc_closest_hit_beyond(self.h, ro.shape[0], ro.ctypes.data, rd.ctypes.data, ta.ctypes.data, tid.ctypes.data,
                                               tuv.ctypes.data)
        return tid, tuv

    def peel(self, ro, rd, layers):
        """Per-layer (tri_id, tuv) of `layers` successive closest_hit(t_after=) calls, each after the previous layer's t (+inf once a
        ray has no further hit), as one pixel of raster.DepthPeeler."""
        ta = np.zeros(np.asarray(ro).reshape(-1, 3).shape[0], self.orc.dt)
        out = []
        for _ in range(layers):
            tid, tuv = self.closest_hit(ro, rd, ta)
            out.append((tid, tuv))
            ta = np.where(tid >= 0, tuv[:, 0], np.inf).astype(self.orc.dt)
        return out

    def all_hits(self, ro, rd):
        """Sorted (t [k], tri_id [k]) of every triangle one ray hits."""
        t_all = np.zeros(self.T, self.orc.dt)
        o = np.ascontiguousarray(ro, self.orc.dt).reshape(3); d = np.ascontiguousarray(rd, self.orc.dt).reshape(3)
        self.orc.lib.orc_every_hit(self.h, o.ctypes.data, d.ctypes.data, t_all.ctypes.data)
        ids = np.nonzero(t_all >= 0)[0]
        order = np.lexsort((ids, t_all[ids]))
        return t_all[ids][order], ids[order].astype(np.int32)

    def invert4(self, mtx):
        """k_invert4: [B,4,4] (or [4,4]) -> the inverse of each matrix, Gauss-Jordan in double rounded to `real`."""
        return self.orc.invert4(mtx)

    def rasterize(self, mtx, res, t_state=None, px=None):
        """k_rasterize for the clip matrices mtx [B,4,4] at res = (H, W): (rast [B,H,W,4], t_state [B,H,W]).  t_state (the peel state
        after the previous layer, +inf where exhausted; None: layer 0 / plain rasterize) is not modified; the returned one is the
        state after this layer.  px: flat indices into [B,H,W] -> rast [n,4] and t_state [n] of those pixels only (t_state, when
        given, is then the state of those pixels)."""
        m = np.ascontiguousarray(mtx, self.orc.dt).reshape(-1, 4, 4)
        B, (H, W) = m.shape[0], res
        if px is None:
            n, shape, pp = B * H * W, (B, H, W), None
        else:
            pp = np.ascontiguousarray(px, np.int64).reshape(-1)
            assert pp.size == 0 or (pp.min() >= 0 and pp.max() < B * H * W)
            n, shape = pp.shape[0], (pp.shape[0],)
        ts = np.zeros(n, self.orc.dt) if t_state is None else np.array(t_state, self.orc.dt).reshape(-1)
        assert ts.shape[0] == n
        rast = np.zeros((n, 4), self.orc.dt)
        self.orc.lib.orc_rasterize(self.h, B, H, W, m.ctypes.data, n, None if pp is None else pp.ctypes.data, ts.ctypes.data, rast.ctypes.data)
        return rast.reshape(shape + (4,)), ts.reshape(shape)


class Oracle(CLib):
    LIB = "mcoracle"
    SIGS = {
        "orc_lambert_fwd": ([_I] + [_P] * 3, None),
        "orc_lambert_bwd": ([_I] + [_P] * 5, None),
        "orc_frostbite_fwd": ([_I] + [_P] * 5, None),
        "orc_frostbite_bwd": ([_I] + [_P] * 9, None),
        "orc_fresnel_shlick_fwd": ([_I] + [_P] * 4, None),
        "orc_fresnel_shlick_bwd": ([_I] + [_P] * 7, None),
        "orc_ndf_ggx_fwd": ([_I] + [_P] * 3, None),
        "orc_ndf_ggx_bwd": ([_I] + [_P] * 5, None),
        "orc_lambda_ggx_fwd": ([_I] + [_P] * 3, None),
        "orc_lambda_ggx_bwd": ([_I] + [_P] * 5, None),
        "orc_masking_smith_fwd": ([_I] + [_P] * 4, None),
        "orc_masking_smith_bwd": ([_I] + [_P] * 7, None),
        "orc_pbr_specular_fwd": ([_I] + [_P] * 5 + [REAL, _P], None),
        "orc_pbr_specular_bwd": ([_I] + [_P] * 5 + [REAL] + [_P] * 6, None),
        "orc_pbr_bsdf_fwd": ([_I] + [_P] * 6 + [REAL, _I, _P], None),
        "orc_pbr_bsdf_bwd": ([_I] + [_P] * 6 + [REAL, _I] + [_P] * 7, None),
        "orc_prepare_shading_normal_fwd": ([_I] + [_P] * 6 + [_I, _I, _P], None),
        "orc_prepare_shading_normal_bwd": ([_I] + [_P] * 6 + [_I, _I] + [_P] * 7, None),
        "orc_update_pdf": ([_I, _I] + [_P] * 4, None),
        "orc_rand_pcg": ([_P], C.c_uint32),
        "orc_hash_pcg": ([C.c_uint32, C.c_uint32], C.c_uint32),
        "orc_scene_create": ([_P, _I, _P, _I], _P),
        "orc_scene_destroy": ([_P], None),
        "orc_lbvh_build": ([_P] * 3, None),
        "orc_lbvh_export": ([_P] * 7, None),
        "orc_visibility": ([_P, _I, _I] + [_P] * 4, None),
        "orc_occluded1": ([_P, _I, _P, _P], _I),
        "orc_closest_hit": ([_P, _I] + [_P] * 4, None),
        "orc_closest_hit_beyond": ([_P, _I] + [_P] * 5, None),
        "orc_every_hit": ([_P] * 4, _I),
        "orc_invert4": ([_I, _P, _P], None),
        "orc_rasterize": ([_P, _I, _I, _I, _P, _I64, _P, _P, _P], None),
        "orc_dirs_to_texels": ([_I] * 3 + [_P] * 2, None),
        "orc_env_shade": ([_P], None),
        "orc_bilateral_fwd": ([_I] * 3 + [_P] * 3 + [REAL, _P], None),
        "orc_bilateral_bwd": ([_I] * 3 + [_P] * 2 + [REAL, _P, _P], None),
        "orc_bilateral_tap_weight": ([_I] * 3 + [_P] * 2 + [REAL, _I, _I64] + [_P] * 4, None),
        "orc_det_sincos": ([_I] + [_P] * 3, None),
        "orc_det_atan2": ([_I] + [_P] * 3, None),
        "orc_det_acos": ([_I] + [_P] * 2, None),
        "orc_sizeof_real": ([], _I),
        "orc_sizeof_envshade": ([], _I),
        "orc_image_loss_fwd": ([_I, _P, _P, _I, _I, _P], None),
        "orc_image_loss_bwd": ([_I, _P, _P, _I, _I] + [_P] * 3, None),
        "orc_shade_combine_fwd": ([_I] + [_P] * 4 + [_I, _P], None),
        "orc_shade_combine_bwd": ([_I] + [_P] * 4 + [_I] + [_P] * 5, None),
        "orc_xfm_fwd": ([_I] * 3 + [_P, _P, _I, _P], None),
        "orc_xfm_bwd": ([_I, _I, _P, _P, _I, _P], None),
    }

    def __init__(self, f64=False):
        super().__init__(f64)
        self._ES = _envshade_struct(self.real)
        assert self.lib.orc_sizeof_envshade() == C.sizeof(self._ES), "struct layout mismatch"

    # ------------------------------------------------------------------ helpers
    def set_threads(self, n):
        """OpenMP team size of the oracle's parallel loops.  Called explicitly because OMP_NUM_THREADS is only read when libgomp
        initialises (torch has usually loaded it already) and torchrun exports OMP_NUM_THREADS=1.  Returns the size in effect."""
        self.lib.omp_set_num_threads(int(n))
        return int(self.lib.omp_get_max_threads())

    def _bc(self, *arrs, chans):
        """Broadcast NHWC arrays over their leading dims (size-1 dims broadcast, tensor.h:32)."""
        arrs = [np.asarray(a, dtype=self.dt) for a in arrs]
        lead = np.broadcast_shapes(*[a.shape[:-1] for a in arrs])
        out = [np.ascontiguousarray(np.broadcast_to(a, lead + (c,))) for a, c in zip(arrs, chans)]
        return lead, out

    def scene(self, verts, tris):
        return Scene(self, verts, tris)

    def invert4(self, mtx):
        """k_invert4 (raster.cu): the inverse of each 4x4 matrix of mtx [...,4,4], Gauss-Jordan with partial pivoting in double,
        rounded to `real` (fp32 build: to float, as the kernel).  A singular matrix gives inf / NaN entries."""
        m = np.ascontiguousarray(mtx, self.dt)
        inv = np.zeros_like(m)
        self.lib.orc_invert4(int(m.size // 16), m.ctypes.data, inv.ctypes.data)
        return inv

    # ------------------------------------------------------------------ elementwise ops
    def _run(self, name, ins, chans, extra, outs_ch, extra_after_ins=True, dout=None, dout_ch=None):
        allin = list(ins) + ([dout] if dout is not None else [])
        allch = list(chans) + ([dout_ch] if dout is not None else [])
        lead, arrs = self._bc(*allin, chans=allch)
        n = int(np.prod(lead)) if len(lead) else 1
        outs = [np.zeros(lead + (c,), self.dt) for c in outs_ch]
        ptr = lambda arrays: [a.ctypes.data for a in arrays]
        getattr(self.lib, name)(n, *ptr(arrs[:len(ins)]), *extra, *ptr(arrs[len(ins):] + outs))     # arrs[len(ins):]: dout, if given
        return outs[0] if len(outs) == 1 else tuple(outs)

    def lambert(self, nrm, wi):
        return self._run("orc_lambert_fwd", [nrm, wi], [3, 3], [], [1])

    def lambert_bwd(self, nrm, wi, dout):
        return self._run("orc_lambert_bwd", [nrm, wi], [3, 3], [], [3, 3], dout=dout, dout_ch=1)

    def frostbite_diffuse(self, nrm, wi, wo, lr):
        return self._run("orc_frostbite_fwd", [nrm, wi, wo, lr], [3, 3, 3, 1], [], [1])

    def frostbite_diffuse_bwd(self, nrm, wi, wo, lr, dout):
        return self._run("orc_frostbite_bwd", [nrm, wi, wo, lr], [3, 3, 3, 1], [], [3, 3, 3, 1], dout=dout, dout_ch=1)

    def fresnel_shlick(self, f0, f90, cosT):
        return self._run("orc_fresnel_shlick_fwd", [f0, f90, cosT], [3, 3, 1], [], [3])

    def fresnel_shlick_bwd(self, f0, f90, cosT, dout):
        return self._run("orc_fresnel_shlick_bwd", [f0, f90, cosT], [3, 3, 1], [], [3, 3, 1], dout=dout, dout_ch=3)

    def ndf_ggx(self, a2, c):
        return self._run("orc_ndf_ggx_fwd", [a2, c], [1, 1], [], [1])

    def ndf_ggx_bwd(self, a2, c, dout):
        return self._run("orc_ndf_ggx_bwd", [a2, c], [1, 1], [], [1, 1], dout=dout, dout_ch=1)

    def lambda_ggx(self, a2, c):
        return self._run("orc_lambda_ggx_fwd", [a2, c], [1, 1], [], [1])

    def lambda_ggx_bwd(self, a2, c, dout):
        return self._run("orc_lambda_ggx_bwd", [a2, c], [1, 1], [], [1, 1], dout=dout, dout_ch=1)

    def masking_smith(self, a2, ci, co):
        return self._run("orc_masking_smith_fwd", [a2, ci, co], [1, 1, 1], [], [1])

    def masking_smith_bwd(self, a2, ci, co, dout):
        return self._run("orc_masking_smith_bwd", [a2, ci, co], [1, 1, 1], [], [1, 1, 1], dout=dout, dout_ch=1)

    def pbr_specular(self, col, nrm, wo, wi, alpha, min_roughness=0.08):
        return self._run("orc_pbr_specular_fwd", [col, nrm, wo, wi, alpha], [3, 3, 3, 3, 1], [float(min_roughness)], [3])

    def pbr_specular_bwd(self, col, nrm, wo, wi, alpha, dout, min_roughness=0.08):
        return self._run("orc_pbr_specular_bwd", [col, nrm, wo, wi, alpha], [3, 3, 3, 3, 1], [float(min_roughness)],
                         [3, 3, 3, 3, 1], dout=dout, dout_ch=3)

    def pbr_bsdf(self, kd, arm, pos, nrm, view_pos, light_pos, min_roughness=0.08, bsdf="lambert"):
        return self._run("orc_pbr_bsdf_fwd", [kd, arm, pos, nrm, view_pos, light_pos], [3] * 6,
                         [float(min_roughness), 1 if bsdf == "frostbite" else 0], [3])

    def pbr_bsdf_bwd(self, kd, arm, pos, nrm, view_pos, light_pos, dout, min_roughness=0.08, bsdf="lambert"):
        return self._run("orc_pbr_bsdf_bwd", [kd, arm, pos, nrm, view_pos, light_pos], [3] * 6,
                         [float(min_roughness), 1 if bsdf == "frostbite" else 0], [3] * 6, dout=dout, dout_ch=3)

    def prepare_shading_normal(self, pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm, two_sided_shading=True, opengl=True):
        if perturbed_nrm is None:
            perturbed_nrm = np.array([0, 0, 1], self.dt)[None, None, None, :]   # renderutils/ops.py:217-218
        return self._run("orc_prepare_shading_normal_fwd", [pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm],
                         [3] * 6, [int(two_sided_shading), int(opengl)], [3])

    def prepare_shading_normal_bwd(self, pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm, dout, two_sided_shading=True, opengl=True):
        if perturbed_nrm is None:
            perturbed_nrm = np.array([0, 0, 1], self.dt)[None, None, None, :]
        return self._run("orc_prepare_shading_normal_bwd", [pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm],
                         [3] * 6, [int(two_sided_shading), int(opengl)], [3] * 6, dout=dout, dout_ch=3)

    # ------------------------------------------------------------------ light pdf / cdf
    def dirs_to_texels(self, dirs, Hl, Wl):
        """Env texel ((y << 16) | x) of each direction, computed exactly as env_shade records it."""
        d = np.ascontiguousarray(dirs, self.dt).reshape(-1, 3)
        out = np.zeros(d.shape[0], np.int32)
        self.lib.orc_dirs_to_texels(d.shape[0], Hl, Wl, d.ctypes.data, out.ctypes.data)
        return out.reshape(np.asarray(dirs).shape[:-1])

    def update_pdf(self, base):
        base = self._a(base); H, W = base.shape[:2]
        pdf = np.zeros((H, W), self.dt); rows = np.zeros(H, self.dt); cols = np.zeros((H, W), self.dt)
        self.lib.orc_update_pdf(H, W, base.ctypes.data, pdf.ctypes.data, rows.ctypes.data, cols.ctypes.data)
        return pdf, rows, cols

    # ------------------------------------------------------------------ env shade
    def env_shade(self, scene, mask, ro, gb_pos, gb_normal, gb_view_pos, gb_kd, gb_ks, light, pdf, rows, cols, perms,
                  BSDF="pbr", n_samples_x=8, rnd_seed=0, shadow_scale=1.0, batch_offset=0, vis_mode="brute",
                  grads=None, records=False, counters=False, parallel_bwd=False, sampling_gbuffer=None, abs_terms=False):
        """Forward (grads=None) -> (diff, spec[, records][, counters]);
        backward (grads=(diff_grad, spec_grad)) -> (pos_grad, nrm_grad, kd_grad, ks_grad, light_grad).
        Mirrors env_shade_fwd / env_shade_bwd, render/optixutils/c_src/torch_bindings.cpp:123-272.
        abs_terms (test-only): every output is the sum of the absolute values of its per-ray terms instead (see OrcEnvShade)."""
        assert scene is None or scene.orc is self, "scene was built by a different Oracle instance (fp32 vs fp64 layouts differ)"
        ro = np.asarray(ro, self.dt)
        B, H, W = ro.shape[:3]
        full = (B, H, W, 3)
        mask = self._a(mask, (B, H, W))
        ro = self._a(ro, full); pos = self._a(gb_pos, full); nrm = self._a(gb_normal, full)
        view = self._a(gb_view_pos, full); kd = self._a(gb_kd, full); ks = self._a(gb_ks, full)
        light = self._a(light); pdf = self._a(pdf); rows = self._a(rows); cols = self._a(cols)
        perms = np.ascontiguousarray(perms, np.int32)
        N = int(n_samples_x); S = N * N
        assert perms.shape[1] == S and rows.ndim == 1
        p = self._ES()
        p.B, p.H, p.W = B, H, W
        p.Hl, p.Wl = light.shape[0], light.shape[1]
        p.n_perms = perms.shape[0]; p.N = N
        p.bsdf = BSDF_MODES.index(BSDF) if isinstance(BSDF, str) else int(BSDF)
        p.seed = int(rnd_seed) & 0xFFFFFFFF
        p.batch_offset = int(batch_offset)
        p.vis_mode = 2 if scene is None else {"brute": 0, "bvh": 1, "none": 2}[vis_mode]
        p.shadow_scale = float(shadow_scale)
        p.parallel_bwd = int(parallel_bwd)
        p.abs_terms = int(abs_terms)
        keep = [mask, ro, pos, nrm, view, kd, ks, light, pdf, rows, cols, perms]
        p.mask, p.ro, p.pos, p.nrm, p.view, p.kd, p.ks = [a.ctypes.data for a in (mask, ro, pos, nrm, view, kd, ks)]
        p.light, p.pdf, p.rows, p.cols, p.perms = [a.ctypes.data for a in (light, pdf, rows, cols, perms)]
        p.scene = scene.h if scene is not None else None
        if sampling_gbuffer is not None:       # test-only: (pos, nrm, kd, ks) used for the sampling decisions
            sg_ = [self._a(x, full) for x in sampling_gbuffer]
            keep += sg_
            p.s_pos, p.s_nrm, p.s_kd, p.s_ks = [a.ctypes.data for a in sg_]
        cnt = np.zeros(3, np.uint64); p.counters = cnt.ctypes.data
        rec_t = rec_v = None
        if records:
            rec_t = np.full((B, H, W, 2 * S), -1, np.int32); rec_v = np.full((B, H, W, 2 * S), 255, np.uint8)
            p.rec_texel = rec_t.ctypes.data; p.rec_vis = rec_v.ctypes.data
        if grads is None:
            diff = np.zeros(full, self.dt); spec = np.zeros(full, self.dt)
            p.backward = 0; p.diff = diff.ctypes.data; p.spec = spec.ctypes.data
            self.lib.orc_env_shade(C.byref(p))
            out = [diff, spec]
            if records:
                out.append((rec_t, rec_v))
            if counters:
                out.append(cnt)
            return tuple(out)
        dg = self._a(grads[0], full); sg = self._a(grads[1], full)
        pg, ng, kg, sgr = (np.zeros(full, self.dt) for _ in range(4))
        lg = np.zeros(light.shape, self.dt)
        p.backward = 1
        p.diff_grad, p.spec_grad = dg.ctypes.data, sg.ctypes.data
        p.pos_grad, p.nrm_grad, p.kd_grad, p.ks_grad, p.light_grad = [a.ctypes.data for a in (pg, ng, kg, sgr, lg)]
        self.lib.orc_env_shade(C.byref(p))
        del keep
        return pg, ng, kg, sgr, lg

    # ------------------------------------------------------------------ denoiser
    def bilateral_fwd(self, col, nrm, zdz, sigma):
        """out [B,H,W,4] = (sum w*col, max(sum w, 1e-4)); denoising.cu:14-72."""
        col = self._a(col); nrm = self._a(nrm); zdz = self._a(zdz)
        B, H, W = col.shape[:3]
        out = np.zeros((B, H, W, 4), self.dt)
        self.lib.orc_bilateral_fwd(B, H, W, col.ctypes.data, nrm.ctypes.data, zdz.ctypes.data, sigma, out.ctypes.data)
        return out

    def bilateral_bwd(self, nrm, zdz, sigma, out_grad):
        nrm = self._a(nrm); zdz = self._a(zdz); out_grad = self._a(out_grad)
        B, H, W = nrm.shape[:3]
        cg = np.zeros((B, H, W, 3), self.dt)
        self.lib.orc_bilateral_bwd(B, H, W, nrm.ctypes.data, zdz.ctypes.data, sigma, out_grad.ctypes.data, cg.ctypes.data)
        return cg

    def bilateral_tap_weight(self, nrm, zdz, sigma, pix, dy, dx, transposed=False):
        """Test-only: the weight bilateral_fwd (transposed=False: the centre's depth gradient) or bilateral_bwd (transposed=True: the
        tap's) gives the tap at pixel + (dy, dx) in the output at pixel, a flat index into [B,H,W]; exactly 0 for a tap outside the image
        or the window.  pix, dy, dx broadcast against each other; returns an array of their shape."""
        nrm = self._a(nrm); zdz = self._a(zdz)
        B, H, W = nrm.shape[:3]
        p, y, x = np.broadcast_arrays(np.asarray(pix, np.int64), np.asarray(dy, np.int32), np.asarray(dx, np.int32))
        shape = p.shape
        p, y, x = [np.ascontiguousarray(a).reshape(-1) for a in (p, y, x)]
        out = np.zeros(p.shape[0], self.dt)
        self.lib.orc_bilateral_tap_weight(B, H, W, nrm.ctypes.data, zdz.ctypes.data, sigma, int(transposed), p.shape[0], p.ctypes.data,
                                          y.ctypes.data, x.ctypes.data, out.ctypes.data)
        return out.reshape(shape)

    def bilateral_denoiser(self, col, nrm, zdz, sigma):
        """render/optixutils/ops.py:139-141"""
        o = self.bilateral_fwd(col, nrm, zdz, sigma)
        return o[..., 0:3] / o[..., 3:4]

    # ------------------------------------------------------------------ row f3: image loss, xfm
    _LOSSES = {"l1": 0, "mse": 1, "relmse": 2, "smape": 3, "n2n": 4}

    def image_loss_px(self, img, target, loss="l1", tonemapper="none"):
        """The per-pixel loss mean_c(loss) of loss.cu:105-141 on the broadcast grid of img and target: [N,H,W]."""
        lead, (a, b) = self._bc(img, target, chans=[3, 3])
        n = int(np.prod(lead)); px = np.zeros(n, self.dt)
        self.lib.orc_image_loss_fwd(n, a.ctypes.data, b.ctypes.data, self._LOSSES[loss], 1 if tonemapper == "log_srgb" else 0, px.ctypes.data)
        return px.reshape(lead)

    @staticmethod
    def _img_pixels(img):
        s = np.shape(img)
        return int(s[0] * s[1] * s[2])

    def image_loss(self, img, target, loss="l1", tonemapper="none"):
        """renderutils/ops.py:476-498: the per-pixel losses summed over the broadcast grid, divided by IMG's pixel count N*H*W, as
        renderutils/ops.py:494 divides by img.shape[0:3].  So where img broadcasts against a batched target (img [1,H,W,3], target
        [N,H,W,3]) the result is N times the mean per-pixel loss, as in the reference and the product."""
        return self.image_loss_px(img, target, loss, tonemapper).sum(dtype=np.float64) / self._img_pixels(img)

    def image_loss_bwd(self, img, target, loss="l1", tonemapper="none", dout=1.0):
        """Full-grid [N,H,W,3] gradients (img_grad, target_grad).  dout: a scalar, the upstream gradient of image_loss() (so every pixel
        gets dout / img's pixel count, the divisor rule of image_loss), or an [N,H,W] array, the upstream gradient of each pixel of
        image_loss_px()."""
        lead, (a, b) = self._bc(img, target, chans=[3, 3])
        n = int(np.prod(lead))
        if np.ndim(dout) == 0:
            dpx = np.full(n, dout / self._img_pixels(img), self.dt)
        else:
            dpx = np.ascontiguousarray(np.broadcast_to(np.asarray(dout, self.dt), lead)).reshape(n)
        gi = np.zeros(lead + (3,), self.dt); gt = np.zeros(lead + (3,), self.dt)
        self.lib.orc_image_loss_bwd(n, a.ctypes.data, b.ctypes.data, self._LOSSES[loss], 1 if tonemapper == "log_srgb" else 0, dpx.ctypes.data,
                                    gi.ctypes.data, gt.ctypes.data)
        return gi, gt

    def shade_combine(self, a4, b4, kd, ks, pbr=True):
        """orc_shade_combine_fwd: the tail of render.shade() (render.py:119-127) on the raw denoiser outputs a4 / b4 [...,4] (rgb weighted
        sum, weight) -> [...,3].  pbr=False: 'diffuse' / 'white', b4 and ks unused (None allowed)."""
        b4 = a4 if b4 is None else b4
        ks = kd if ks is None else ks
        return self._run("orc_shade_combine_fwd", [a4, b4, kd, ks], [4, 4, 3, 3], [int(pbr)], [3])

    def shade_combine_bwd(self, a4, b4, kd, ks, dout, pbr=True):
        """-> full-grid (d_a4, d_b4, d_kd, d_ks); d_b4 / d_ks are zero when pbr=False."""
        b4 = a4 if b4 is None else b4
        ks = kd if ks is None else ks
        return self._run("orc_shade_combine_bwd", [a4, b4, kd, ks], [4, 4, 3, 3], [int(pbr)], [4, 4, 3, 3], dout=dout, dout_ch=3)

    def xfm(self, points, matrix, is_points=True):
        pts = self._a(points); m = self._a(matrix)
        B, V = m.shape[0], pts.shape[1]
        out = np.zeros((B, V, 4 if is_points else 3), self.dt)
        self.lib.orc_xfm_fwd(B, pts.shape[0], V, pts.ctypes.data, m.ctypes.data, int(is_points), out.ctypes.data)
        return out

    def xfm_bwd(self, matrix, dout, is_points=True):
        m = self._a(matrix); g = self._a(dout)
        B, V = g.shape[0], g.shape[1]
        out = np.zeros((B, V, 3), self.dt)
        self.lib.orc_xfm_bwd(B, V, m.ctypes.data, g.ctypes.data, int(is_points), out.ctypes.data)
        return out

    # ------------------------------------------------------------------ det math (fp32 only)
    def det_sincos(self, a):
        a = np.ascontiguousarray(a, np.float32); s = np.zeros_like(a); c = np.zeros_like(a)
        self.lib.orc_det_sincos(a.size, a.ctypes.data, s.ctypes.data, c.ctypes.data)
        return s, c

    def det_atan2(self, y, x):
        y = np.ascontiguousarray(y, np.float32); x = np.ascontiguousarray(x, np.float32); o = np.zeros_like(y)
        self.lib.orc_det_atan2(y.size, y.ctypes.data, x.ctypes.data, o.ctypes.data)
        return o

    def det_acos(self, x):
        x = np.ascontiguousarray(x, np.float32); o = np.zeros_like(x)
        self.lib.orc_det_acos(x.size, x.ctypes.data, o.ctypes.data)
        return o
