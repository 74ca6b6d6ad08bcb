"""CPU: the C-ABI shared library loads and exports every symbol include/mcshade.h declares, and the binding read from the header
agrees with it (no compute without a GPU)."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

from nvdiffrecmc_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    """{name: parameter count} of every prototype of the header."""
    src = open(os.path.join(ROOT, "include", "mcshade.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {n: 0 if p.strip() == "void" else p.count(",") + 1 for n, p in re.findall(r"\b(mcs_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_library_is_built_in_tree_and_loads():
    assert os.path.exists(_lib.LIB_PATH), "run __graft_entry__.build()"
    assert os.path.commonpath([ROOT, os.path.abspath(_lib.LIB_PATH)]) == ROOT
    l = _lib.lib()
    assert l.mcs_abi_version() == 2


def test_every_declared_symbol_is_exported_and_bound():
    declared = _declared()
    assert len(declared) >= 30
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in declared:
        assert hasattr(raw, n), "missing export: " + n
    assert _lib.EXPORTED_SYMBOLS == sorted(declared)
    l = _lib.lib()
    for n, n_params in declared.items():
        fn = getattr(l, n)
        assert fn.argtypes is not None, "not bound: " + n
        assert len(fn.argtypes) == n_params, n


_T, _P = ctypes.POINTER(_lib.mcs_tensor), ctypes.c_void_p
PINNED = {
    "mcs_env_shade_fwd": ([_P] + [_T] * 12 + [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, _P, ctypes.c_float, ctypes.c_int32, _P, _P, _P, _P, _P,
                                             ctypes.c_int32, _P], ctypes.c_int),
    "mcs_dmtet_emit": ([_P, ctypes.c_int64, ctypes.c_int64, _P, ctypes.c_int64, _P, ctypes.c_int32, _P, _P, ctypes.c_int32] + [_P] * 7, ctypes.c_int),
    "mcs_texture_bwd": ([_P, _P, _P] + [ctypes.c_int32] * 5 + [_P] * 5, ctypes.c_int),
    "mcs_mlptex_bwd": ([_P, ctypes.c_int64] + [_P] * 4 + [ctypes.c_int32, ctypes.c_int32] + [_P] * 8, ctypes.c_int),
    "mcs_last_error": ([], ctypes.c_char_p),
    "mcs_aa_topology_workspace_bytes": ([ctypes.c_int32], ctypes.c_int64),
}


@pytest.mark.parametrize("name", sorted(PINNED))
def test_pinned_signatures(name):
    args, res = PINNED[name]
    fn = getattr(_lib.lib(), name)
    assert list(fn.argtypes) == args and fn.restype is res


def test_struct_layout_matches_the_c_compiler():
    """Each header struct's ctypes layout equals gcc's: its size, and every field's offset and size."""
    structs = [_lib.mcs_tensor, _lib.mcs_hashgrid_levels, _lib.mcs_texture_levels]
    prints, want = [], []
    for s in structs:
        n = s.__name__
        prints.append('printf("%s %%zu\\n", sizeof(%s));' % (n, n))
        want.append("%s %d" % (n, ctypes.sizeof(s)))
        for f, _ in s._fields_:
            prints.append('printf("%s.%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s *)0)->%s));' % (n, f, n, f, n, f))
            want.append("%s.%s %d %d" % (n, f, getattr(s, f).offset, getattr(s, f).size))
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        open(c, "w").write('#include <stddef.h>\n#include <stdio.h>\n#include "mcshade.h"\nint main(void){\n%s\nreturn 0; }\n' % "\n".join(prints))
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split("\n")[:-1]
    assert got == want


@pytest.mark.parametrize("src,where", [("int mcs_x(size_t n);", "mcs_x"), ("size_t mcs_y(int n);", "mcs_y"),
                                       ("typedef struct mcs_z { size_t n; } mcs_z;", "mcs_z")])
def test_unknown_c_type_is_an_error_naming_the_declaration(src, where):
    parse = _lib._structs if src.startswith("typedef") else _lib._prototypes
    with pytest.raises(TypeError, match=r"\b%s\b.*'size_t'" % where):
        parse(src)


def test_header_is_plain_c():
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write('#include "mcshade.h"\nint main(void){ mcs_tensor t; (void)t; return MCS_ABI_VERSION == 2 ? 0 : 1; }\n')
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", c, "-o", os.path.join(d, "t.o")], check=True)


def test_errors_without_gpu_are_reported_not_swallowed():
    """ctx creation needs a device: on a CPU-only box it must FAIL with a message (the reference drops CUDA errors)."""
    import torch
    if torch.cuda.is_available():
        return
    l = _lib.lib()
    h = ctypes.c_void_p()
    rc = l.mcs_ctx_create(ctypes.byref(h))
    assert rc != 0 and b"cudaGetDevice" in l.mcs_last_error()


def test_argument_validation_returns_status_and_message():
    """Every entry point validates its arguments BEFORE touching the device and reports through the status code + mcs_last_error()
    (the reference's CUDA_CHECK / OPTIX_CHECK format a string and drop it, optixutils/c_src/common.h:37-61).  Null arguments never
    reach a kernel launch, so this runs without a GPU."""
    l = _lib.lib()
    N = None
    T = ctypes.POINTER(_lib.mcs_tensor)()
    calls = [
        ("mcs_bvh_build", lambda: l.mcs_bvh_build(N, N, 0, N, 0, 1, N), b"null context"),
        ("mcs_trace_visibility", lambda: l.mcs_trace_visibility(N, N, N, 4, N, N), b"no acceleration structure"),
        ("mcs_rasterize", lambda: l.mcs_rasterize(N, N, 1, 4, 4, N, N), b"no acceleration structure"),
        ("mcs_interpolate_fwd", lambda: l.mcs_interpolate_fwd(N, 0, 3, 3, N, 1, N, 1, 2, 2, N, N), b"bad arguments"),
        ("mcs_texel_fetch_fwd", lambda: l.mcs_texel_fetch_fwd(N, 4, 3, N, 1, N, N), b"bad arguments"),
        ("mcs_texel_fetch_bwd", lambda: l.mcs_texel_fetch_bwd(4, 3, N, 1, N, N, N), b"bad arguments"),
        ("mcs_update_pdf", lambda: l.mcs_update_pdf(T, N, N, N, N, N), b"null / empty"),
        ("mcs_bilateral_fwd", lambda: l.mcs_bilateral_fwd(T, T, T, ctypes.c_float(1.0), N, N), b"null / empty"),
        ("mcs_shade_combine_fwd", lambda: l.mcs_shade_combine_fwd(T, T, T, T, 1, N, N), b"null / empty"),
        ("mcs_pbr_bsdf_fwd", lambda: l.mcs_pbr_bsdf_fwd(T, T, T, T, T, T, ctypes.c_float(0.08), 0, N, N), b"null / empty"),
        ("mcs_image_loss_fwd", lambda: l.mcs_image_loss_fwd(T, T, 0, 0, N, N), b"null"),
        ("mcs_xfm_fwd", lambda: l.mcs_xfm_fwd(T, T, 1, N, N), b"null / empty"),
    ]
    for name, call, frag in calls:
        rc = call()
        msg = l.mcs_last_error() or b""
        assert rc != 0, name
        assert frag in msg, (name, msg)


# The renderutils streaming ops: operands (name, channels), the forward output's channel count and the scalar arguments.
# The backward takes the operands, the scalars and d_out, and writes one gradient per operand.
EW_OPS = {
    "lambert": ([("nrm", 3), ("wi", 3)], 1, []),
    "frostbite": ([("nrm", 3), ("wi", 3), ("wo", 3), ("lin_rough", 1)], 1, []),
    "fresnel_shlick": ([("f0", 3), ("f90", 3), ("cos_theta", 1)], 3, []),
    "ndf_ggx": ([("alpha_sqr", 1), ("cos_theta", 1)], 1, []),
    "lambda_ggx": ([("alpha_sqr", 1), ("cos_theta", 1)], 1, []),
    "masking_smith": ([("alpha_sqr", 1), ("cos_i", 1), ("cos_o", 1)], 1, []),
    "pbr_specular": ([("col", 3), ("nrm", 3), ("wo", 3), ("wi", 3), ("alpha", 1)], 3, [0.08]),
    "pbr_bsdf": ([("kd", 3), ("arm", 3), ("pos", 3), ("nrm", 3), ("view_pos", 3), ("light_pos", 3)], 3, [0.08, 0]),
    "prepare_shading_normal": ([(n, 3) for n in ("pos", "view_pos", "perturbed_nrm", "smooth_nrm", "smooth_tng", "geom_nrm")], 3, [1, 1]),
    "shade_combine": ([("a4", 4), ("b4", 4), ("kd", 3), ("ks", 3)], 3, [1]),
}


def _named(name, msg):
    return re.search(rb"(^|[^a-z_])" + name.encode() + rb"([^a-z_]|$)", msg) is not None


@pytest.mark.parametrize("entry", ["mcs_%s_%s" % (op, way) for op in EW_OPS for way in ("fwd", "bwd")])
def test_streaming_ops_check_every_operand_and_output(entry):
    """Each streaming op entry refuses, before any launch, an operand with the wrong channel count, a dimension that does not
    broadcast, a null or empty descriptor and a null output pointer, and names the operand or output.  The descriptors point
    at fake addresses: a check that went missing would end in the failed launch of a device-less machine, whose message
    names neither."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("the calls would launch on the fake pointers")
    l = _lib.lib()
    op, way = entry[len("mcs_"):].rsplit("_", 1)
    operands, out_c, scalars = EW_OPS[op]
    bwd = way == "bwd"
    tensors = operands + [("d_out", out_c)] if bwd else operands
    outputs = ["d_" + n for n, _ in operands] if bwd else ["out"]

    def desc(C, sizes=(2, 4, 4)):
        N, H, W = sizes
        return _lib._desc(0x10000, (N, H, W, C), (H * W * C, W * C, C, 1))

    def call(ts, outs, pbr=1):
        sc = scalars[:-1] + [pbr] if op == "shade_combine" else scalars
        ts = [ctypes.byref(t) if t is not None else None for t in ts]
        args = ts[:len(operands)] + sc + ts[len(operands):] + list(outs) + [None]
        rc = getattr(l, entry)(*args)
        return rc, l.mcs_last_error() or b""

    good = [desc(C) for _, C in tensors]
    fake_outs = [0x20000 * (i + 1) for i in range(len(outputs))]
    for i, (name, C) in enumerate(tensors):
        for bad, what in ((desc(C + 1), "channels"), (desc(C, (2, 3, 4)), "broadcast")):
            rc, msg = call(good[:i] + [bad] + good[i + 1:], fake_outs)
            assert rc != 0 and _named(name, msg), (entry, name, what, msg)
        for bad in (None, desc(C, (2, 0, 4))):
            rc, msg = call(good[:i] + [bad] + good[i + 1:], fake_outs)
            assert rc != 0 and msg == ("%s: null / empty tensor argument" % entry).encode(), (entry, name, msg)
    for i, name in enumerate(outputs):
        rc, msg = call(good, fake_outs[:i] + [None] + fake_outs[i + 1:])
        assert rc != 0 and msg == ("%s: null output pointer %s" % (entry, name)).encode(), (entry, name, msg)
    if entry == "mcs_shade_combine_bwd":
        # 'diffuse' neither reads b4 / ks nor writes d_b4 / d_ks, so those two may be null: the call gets past every check.
        rc, msg = call(good, [fake_outs[0], None, fake_outs[2], None], pbr=0)
        assert rc != 0 and b"d_b4" not in msg and b"d_ks" not in msg, msg
