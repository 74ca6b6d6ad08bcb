"""ctypes binding of libmcshade.so (C ABI declared in include/mcshade.h) + the in-tree build recipe.

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError
is raised (the reference silently drops CUDA/OptiX errors, optixutils/c_src/common.h:37-61).
"""
import collections
import ctypes as C
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

_PKG = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_PKG, "csrc")
_LIBDIR = os.path.join(_PKG, "lib")
LIB_PATH = os.environ.get("MCS_LIB", os.path.join(_LIBDIR, "libmcshade.so"))     # MCS_LIB: developer override (kernel variants)
SOURCES = ["core.cu", "elementwise.cu", "denoise.cu", "bvh.cu", "envshade.cu", "lossmesh.cu", "light.cu", "raster.cu", "hashgrid.cu", "texture.cu",
           "mlptexture.cu"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC"]


def _nvcc():
    for cand in (os.environ.get("CUDA_HOME", "") + "/bin/nvcc", "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand)):
            return cand
    return "nvcc"


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a and link nvdiffrecmc_b200/lib/libmcshade.so (in-tree)."""
    os.makedirs(_LIBDIR, exist_ok=True)
    objdir = os.path.join(_LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(os.path.dirname(_PKG), "include", "mcshade.h"))
    newest_hdr = max(os.path.getmtime(h) for h in hdrs)
    nvcc = _nvcc()

    def compile_one(src):
        s = os.path.join(_CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        if not force and os.path.exists(o) and os.path.getmtime(o) >= max(os.path.getmtime(s), newest_hdr):
            return o, False
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            print("[mcshade] compiled", src)
        return o, True

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 1)) as ex:
        res = list(ex.map(compile_one, SOURCES))
    objs = [o for o, _ in res]
    if force or any(ch for _, ch in res) or not os.path.exists(LIB_PATH):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        if verbose:
            print("[mcshade] linked", LIB_PATH)
    return LIB_PATH


class mcs_hashgrid_levels(C.Structure):
    _fields_ = [("n_levels", C.c_int32), ("offset", C.c_uint32 * 17), ("res", C.c_uint32 * 16), ("scale", C.c_float * 16), ("dense_mask", C.c_uint32)]


class mcs_texture_levels(C.Structure):
    _fields_ = [("n_levels", C.c_int32), ("C", C.c_int32), ("ptr", C.c_void_p * 16), ("h", C.c_int32 * 16), ("w", C.c_int32 * 16),
                ("batch_stride", C.c_int64 * 16)]


class mcs_tensor(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("sizes", C.c_int32 * 4), ("strides", C.c_int32 * 4)]


_lib = None
_T = C.POINTER(mcs_tensor)
_P = C.c_void_p
_SIGS = {
    "mcs_abi_version": ([], C.c_int),
    "mcs_last_error": ([], C.c_char_p),
    "mcs_ctx_create": ([C.POINTER(_P)], C.c_int),
    "mcs_ctx_destroy": ([_P], C.c_int),
    "mcs_bvh_build": ([_P, _P, C.c_int32, _P, C.c_int32, C.c_uint32, _P], C.c_int),
    "mcs_bvh_export": ([_P] * 8, C.c_int),
    "mcs_bvh_export_shadow": ([_P] * 5, C.c_int),
    "mcs_trace_visibility": ([_P, _P, _P, C.c_int64, _P, _P], C.c_int),
    "mcs_trace_closest": ([_P, _P, _P, C.c_int64, _P, _P, _P], C.c_int),
    "mcs_trace_closest_after": ([_P, _P, _P, _P, C.c_int64, _P, _P, _P], C.c_int),
    "mcs_env_shade_fwd": ([_P] + [_T] * 12 + [C.c_uint32, C.c_uint32, C.c_uint32, _P, C.c_float, C.c_int32, _P, _P, _P, _P, _P, C.c_int32, _P], C.c_int),
    "mcs_env_shade_bwd_replay": ([_T] * 6 + [C.c_uint32, C.c_uint32, C.c_float, _T, _T, _P, _P, C.c_int32] + [_P] * 6, C.c_int),
    "mcs_env_shade_records": ([_P] + [_T] * 12 + [C.c_uint32, C.c_uint32, C.c_uint32, _P, C.c_float, C.c_int32, _P, _P, _P, _P, _P], C.c_int),
    "mcs_env_shade_bwd": ([_P] + [_T] * 12 + [C.c_uint32, C.c_uint32, C.c_uint32, _P, C.c_float, C.c_int32, _T, _T] + [_P] * 7, C.c_int),
    "mcs_bilateral_fwd": ([_T, _T, _T, C.c_float, _P, _P], C.c_int),
    "mcs_bilateral_bwd": ([_T, _T, C.c_float, _T, _P, _P], C.c_int),
    "mcs_bilateral_fwd2": ([_T, _T, _T, _T, C.c_float, _P, _P, _P], C.c_int),
    "mcs_bilateral_bwd2": ([_T, _T, C.c_float, _T, _T, _P, _P, _P], C.c_int),
    "mcs_lambert_fwd": ([_T] * 2 + [_P] * 2, C.c_int),
    "mcs_lambert_bwd": ([_T] * 3 + [_P] * 3, C.c_int),
    "mcs_frostbite_fwd": ([_T] * 4 + [_P] * 2, C.c_int),
    "mcs_frostbite_bwd": ([_T] * 5 + [_P] * 5, C.c_int),
    "mcs_fresnel_shlick_fwd": ([_T] * 3 + [_P] * 2, C.c_int),
    "mcs_fresnel_shlick_bwd": ([_T] * 4 + [_P] * 4, C.c_int),
    "mcs_ndf_ggx_fwd": ([_T] * 2 + [_P] * 2, C.c_int),
    "mcs_ndf_ggx_bwd": ([_T] * 3 + [_P] * 3, C.c_int),
    "mcs_lambda_ggx_fwd": ([_T] * 2 + [_P] * 2, C.c_int),
    "mcs_lambda_ggx_bwd": ([_T] * 3 + [_P] * 3, C.c_int),
    "mcs_masking_smith_fwd": ([_T] * 3 + [_P] * 2, C.c_int),
    "mcs_masking_smith_bwd": ([_T] * 4 + [_P] * 4, C.c_int),
    "mcs_pbr_specular_fwd": ([_T] * 5 + [C.c_float, _P, _P], C.c_int),
    "mcs_pbr_specular_bwd": ([_T] * 5 + [C.c_float, _T] + [_P] * 6, C.c_int),
    "mcs_pbr_bsdf_fwd": ([_T] * 6 + [C.c_float, C.c_int32, _P, _P], C.c_int),
    "mcs_pbr_bsdf_bwd": ([_T] * 6 + [C.c_float, C.c_int32, _T] + [_P] * 7, C.c_int),
    "mcs_prepare_shading_normal_fwd": ([_T] * 6 + [C.c_int32, C.c_int32, _P, _P], C.c_int),
    "mcs_prepare_shading_normal_bwd": ([_T] * 6 + [C.c_int32, C.c_int32, _T] + [_P] * 7, C.c_int),
    "mcs_image_loss_num_partials": ([C.c_int32] * 3, C.c_int),
    "mcs_image_loss_fwd": ([_T, _T, C.c_int32, C.c_int32, _P, _P], C.c_int),
    "mcs_image_loss_bwd": ([_T, _T, C.c_int32, C.c_int32, _T, _P, _P, _P], C.c_int),
    "mcs_xfm_fwd": ([_T, _T, C.c_int32, _P, _P], C.c_int),
    "mcs_xfm_bwd": ([_T, _T, _T, C.c_int32, _P, _P], C.c_int),
    "mcs_update_pdf": ([_T, _P, _P, _P, _P, _P], C.c_int),
    "mcs_shade_combine_fwd": ([_T, _T, _T, _T, C.c_int32, _P, _P], C.c_int),
    "mcs_shade_combine_bwd": ([_T, _T, _T, _T, C.c_int32, _T, _P, _P, _P, _P, _P], C.c_int),
    "mcs_texel_fetch_fwd": ([_P, C.c_int64, C.c_int32, _P, C.c_int64, _P, _P], C.c_int),
    "mcs_texel_fetch_bwd": ([C.c_int64, C.c_int32, _P, C.c_int64, _P, _P, _P], C.c_int),
    "mcs_rasterize": ([_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P], C.c_int),
    "mcs_rasterize_peel": ([_P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P], C.c_int),
    "mcs_interpolate_fwd": ([_P, C.c_int64, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P], C.c_int),
    "mcs_interpolate_bwd": ([_P, C.c_int64, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P], C.c_int),
    "mcs_interpolate_bwd_rast": ([_P, C.c_int64, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P], C.c_int),
    "mcs_rasterize_bwd": ([_P, C.c_int64, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P], C.c_int),
    "mcs_rast_db": ([_P, C.c_int64, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P], C.c_int),
    "mcs_rasterize_bwd_db": ([_P, C.c_int64, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P], C.c_int),
    "mcs_interpolate_da_fwd": ([_P, C.c_int64, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P],
                               C.c_int),
    "mcs_interpolate_da_bwd": ([_P, C.c_int64, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P,
                                _P, _P], C.c_int),
    "mcs_aa_topology_workspace_bytes": ([C.c_int32], C.c_int64),
    "mcs_aa_topology": ([_P, C.c_int32, _P, _P, _P], C.c_int),
    "mcs_antialias_fwd": ([_P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int32, _P, _P, _P], C.c_int),
    "mcs_antialias_bwd": ([_P, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int32, _P, _P, _P, _P, _P], C.c_int),
    "mcs_hashgrid_fwd": ([_P, C.c_int64, _P, _P, _P, _P], C.c_int),
    "mcs_hashgrid_bwd": ([_P, C.c_int64, _P, _P, _P, _P, _P, _P], C.c_int),
    "mcs_mlptex_workspace_bytes": ([C.c_int64, C.c_int32, C.c_int32], C.c_int64),
    "mcs_mlptex_fwd": ([_P, C.c_int64] + [_P] * 4 + [C.c_int32, C.c_int32] + [_P] * 4, C.c_int),
    "mcs_mlptex_bwd": ([_P, C.c_int64] + [_P] * 4 + [C.c_int32, C.c_int32] + [_P] * 8, C.c_int),
    "mcs_texture_fwd": ([_P, _P, _P] + [C.c_int32] * 5 + [_P, _P], C.c_int),
    "mcs_texture_bwd": ([_P, _P, _P] + [C.c_int32] * 5 + [_P] * 5, C.c_int),
}
EXPORTED_SYMBOLS = sorted(_SIGS)


def lib():
    """Load libmcshade.so (once). Fails loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libmcshade.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU / PyTorch fallback for the hot path." % LIB_PATH)
    l = C.CDLL(LIB_PATH)
    for name, (args, res) in _SIGS.items():
        fn = getattr(l, name)          # AttributeError if the symbol is missing
        fn.argtypes = args
        fn.restype = res
    if l.mcs_abi_version() != 2:
        raise RuntimeError("libmcshade ABI version mismatch")
    _lib = l
    return l


# Count of OUR kernels launched through the C ABI (bench.py's gpu_launches claim).  optix_build_bvh launches thirteen hand-written
# kernels: bounds init, triangle bounds, Morton codes, radix sort (histogram + 4 passes), Karras topology, leaves + refit, node emission,
# and for meshes of 5 to 16 384 triangles the shadow view's clustering and emission.
LAUNCHES = collections.Counter()
_KERNELS_PER_CALL = {"optix_build_bvh": 13, "bvh_export": 0, "bvh_export_shadow": 0, "update_pdf": 2, "rasterize": 2, "rasterize_peel": 2,
                     "antialias_topology": 2, "hashgrid_bwd_both": 2, "mlptex_bwd_dw": 2,
                     "texture_fwd": 1, "texture_bwd": 1}


def check(status, what):
    LAUNCHES[what] += _KERNELS_PER_CALL.get(what, 1)
    if status != 0:
        msg = lib().mcs_last_error()
        raise RuntimeError("%s failed (status %d): %s" % (what, status, msg.decode() if msg else "?"))


def _desc(ptr, sizes, strides):
    t = mcs_tensor()
    t.ptr = ptr
    for i in range(4):
        t.sizes[i] = int(sizes[i])
        t.strides[i] = int(strides[i])
    return t


def nhwc(t):
    """mcs_tensor view of a torch CUDA fp32/int32 tensor with 1..4 dims interpreted as trailing NHWC dims
    ([B,H,W,C]; [B,H,W] gets C=1 appended -- use the explicit helpers below for other layouts)."""
    assert t.dim() == 4, "expected a 4-D NHWC tensor, got %s" % (tuple(t.shape),)
    return _desc(t.data_ptr(), t.shape, t.stride())


def nhw1(t):
    assert t.dim() == 3
    return _desc(t.data_ptr(), list(t.shape) + [1], list(t.stride()) + [0])


def view_hwc(t):      # [H,W,C] -> (1,H,W,C)
    assert t.dim() == 3
    return _desc(t.data_ptr(), [1] + list(t.shape), [0] + list(t.stride()))


def view_hw(t):       # [H,W] -> (1,H,W,1)
    assert t.dim() == 2
    return _desc(t.data_ptr(), [1, t.shape[0], t.shape[1], 1], [0, t.stride(0), t.stride(1), 0])


def view_h(t):        # [H] -> (1,H,1,1)
    assert t.dim() == 1
    return _desc(t.data_ptr(), [1, t.shape[0], 1, 1], [0, t.stride(0), 0, 0])


def view_perms(t):    # [P,S] -> (1,P,1,S)
    assert t.dim() == 2
    return _desc(t.data_ptr(), [1, t.shape[0], 1, t.shape[1]], [0, t.stride(0), 0, t.stride(1)])


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    import torch
    for t in tensors:
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RuntimeError("libmcshade ops need CUDA tensors (got %s); there is no CPU path" %
                               (t.device if isinstance(t, torch.Tensor) else type(t)))
