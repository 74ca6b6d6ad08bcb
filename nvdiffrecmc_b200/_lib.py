"""ctypes binding of libmcshade.so, read from the C ABI's header include/mcshade.h, + the in-tree build recipe.

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError
is raised (the reference silently drops CUDA/OptiX errors, optixutils/c_src/common.h:37-61).
"""
import collections
import ctypes as C
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

_PKG = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_PKG, "csrc")
_LIBDIR = os.path.join(_PKG, "lib")
HEADER = os.path.join(os.path.dirname(_PKG), "include", "mcshade.h")
LIB_PATH = os.environ.get("MCS_LIB", os.path.join(_LIBDIR, "libmcshade.so"))     # MCS_LIB: developer override (kernel variants)
SOURCES = ["core.cu", "elementwise.cu", "denoise.cu", "bvh.cu", "envshade.cu", "lossmesh.cu", "light.cu", "raster.cu", "hashgrid.cu", "texture.cu",
           "mlptexture.cu", "dmtet.cu", "regularizer.cu", "taps.cu", "composite.cu"]
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
    hdrs.append(HEADER)
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


# The binding is read from include/mcshade.h, the one place the ABI is written down: its structs become ctypes Structures and every
# mcs_* prototype gets declared argument and result types.  The type map is closed, so a header edit it does not cover fails at import.
_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "float": C.c_float, "mcs_stream": C.c_void_p}


def _ctype(decl, where, result=False):
    """ctypes type of the C type `decl` (written without a name, e.g. 'const mcs_tensor *') in the declaration `where`."""
    t = " ".join(decl.replace("*", " * ").split())
    if result and t == "const char *":
        return C.c_char_p
    if t == "const mcs_tensor *":
        return C.POINTER(mcs_tensor)
    if "*" in t:
        return C.c_void_p
    if t not in _SCALARS:
        raise TypeError("include/mcshade.h: %s: no ctypes type for the C type '%s'" % (where, t))
    return _SCALARS[t]


def _structs(src):
    """{name: Structure} of every `typedef struct mcs_X { ... } mcs_X;` in the comment-free header text `src`."""
    out = {}
    for name, body in re.findall(r"typedef struct (mcs_\w+)\s*\{([^}]*)\}\s*\1\s*;", src):
        fields = [(f, _ctype(decl, name) * int(n) if n else _ctype(decl, name))
                  for decl, f, n in re.findall(r"([^;]*?)\b(\w+)\s*(?:\[(\d+)\])?\s*;", body)]
        out[name] = type(name, (C.Structure,), {"_fields_": fields})
    return out


def _prototypes(src):
    """{name: ([argument types], result type)} of every mcs_* prototype in the comment-free header text `src`."""
    sigs = {}
    for res, name, params in re.findall(r"^([A-Za-z_][\w \*]*?)\b(mcs_\w+)\s*\(([^)]*)\)\s*;", src, re.M):
        args = [] if params.strip() == "void" else [_ctype(re.sub(r"\w+\s*$", "", p), name) for p in params.split(",")]
        sigs[name] = (args, _ctype(res, name, result=True))
    return sigs


with open(HEADER) as _f:
    _src = re.sub(r"/\*.*?\*/", " ", _f.read(), flags=re.S)
_STRUCTS = _structs(_src)
mcs_tensor, mcs_hashgrid_levels, mcs_texture_levels = _STRUCTS["mcs_tensor"], _STRUCTS["mcs_hashgrid_levels"], _STRUCTS["mcs_texture_levels"]
_ABI_VERSION = int(re.search(r"#define MCS_ABI_VERSION (\d+)", _src).group(1))
_SIGNATURES = _prototypes(_src)
EXPORTED_SYMBOLS = sorted(_SIGNATURES)
_lib = None


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
    for name, (args, res) in _SIGNATURES.items():
        fn = getattr(l, name)          # AttributeError if the symbol is missing
        fn.argtypes = args
        fn.restype = res
    if l.mcs_abi_version() != _ABI_VERSION:
        raise RuntimeError("libmcshade ABI version mismatch: the library has %d, include/mcshade.h %d" % (l.mcs_abi_version(), _ABI_VERSION))
    _lib = l
    return l


# Count of OUR kernels launched through the C ABI (bench.py's gpu_launches claim).  optix_build_bvh launches thirteen hand-written
# kernels: bounds init, triangle bounds, Morton codes, radix sort (histogram + 4 passes), Karras topology, leaves + refit, node emission,
# and for meshes of 5 to 16 384 triangles the shadow view's clustering and emission.
LAUNCHES = collections.Counter()
_KERNELS_PER_CALL = {"optix_build_bvh": 13, "bvh_export": 0, "bvh_export_shadow": 0, "update_pdf": 2, "rasterize": 2, "rasterize_peel": 2,
                     "antialias_topology": 2, "hashgrid_bwd_both": 2, "mlptex_bwd_dw": 2, "mlptex_pair_bwd_dw": 2,
                     "texture_fwd": 1, "texture_bwd": 1, "dmtet_count": 1, "dmtet_emit": 1, "dmtet_bwd": 1, "sdf_reg_fwd": 2, "sdf_reg_bwd": 1,
                     "shading_loss_fwd": 2, "material_smoothness_grad_fwd": 2, "chroma_loss_fwd": 2, "coverage_loss_fwd": 2,
                     "mip_chain_bwd": 1, "mip_clamp": 1, "mip_normalize": 1, "composite_fwd": 1, "composite_bwd": 1}     # mip_chain_fwd: mcs_mip_chain_fwd_launches(n_levels)


def check(status, what, launches=None):
    """Raise on a failed call; count its launches (`launches` for an entry whose count depends on its arguments)."""
    LAUNCHES[what] += _KERNELS_PER_CALL.get(what, 1) if launches is None else launches
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
