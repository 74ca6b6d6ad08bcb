"""CPU: the layer-compositing entry points check their descriptor tables before any launch and report through the status code and
mcs_last_error(); the descriptors point at fake addresses, so a check that went missing would end in a failed launch instead."""
import ctypes

import pytest

from nvdiffrecmc_b200 import _lib


def _table(shapes, ptr=0x10000):
    arr = (_lib.mcs_tensor * len(shapes))()
    for k, s in enumerate(shapes):
        if s is not None:
            B, H, W, C = s
            arr[k] = _lib._desc(ptr + 0x100000 * k, s, (H * W * C, W * C, C, 1))
    return arr


def _fwd(n, bufs, acc_in, acc_out, V=3, T=1):
    l = _lib.lib()
    rc = l.mcs_composite_fwd(n, bufs, acc_in, acc_out, 0x1000, 0x2000, 0, V, 0x3000, T, 0x4000, None)
    return rc, l.mcs_last_error() or b""


def _bwd(n, bufs, acc_in, d_out, d_in, d_bufs):
    l = _lib.lib()
    rc = l.mcs_composite_bwd(n, bufs, acc_in, d_out, d_in, d_bufs, 0x1000, 0x2000, 0, 3, 0x3000, 1, 0x4000, None, None)
    return rc, l.mcs_last_error() or b""


def test_composite_tables_are_checked_before_any_launch():
    import torch
    if torch.cuda.is_available():
        pytest.skip("the calls would launch on the fake pointers")
    sh = [(2, 4, 5, 4), (2, 4, 5, 1)]
    good, none = _table(sh), _table([None, None])
    cases = [
        (_fwd(0, good, none, good), b"0 buffers (1 to 16 allowed)"),
        (_fwd(17, _table(sh * 9), _table([None] * 18), _table(sh * 9)), b"17 buffers (1 to 16 allowed)"),
        (_fwd(2, None, none, good), b"bad arguments"),
        (_fwd(2, good, none, good, T=0), b"bad arguments"),
        (_fwd(2, _table([sh[0], None]), none, good), b"buffers[1] is null"),
        (_fwd(2, _table([sh[0], (2, 4, 6, 1)]), none, good), b"buffers[1] is [2,4,6,1], expected [2,4,5,1]"),
        (_fwd(2, _table([sh[0], (2, 4, 5, 0)]), none, good), b"buffers[1] has no channels"),
        (_fwd(2, good, _table([(2, 4, 5, 3), None]), good), b"accum_in[0] is [2,4,5,3], expected [2,4,5,4]"),
        (_fwd(2, good, none, _table([sh[0], None])), b"accum_out[1] is null"),
        (_fwd(2, good, none, None), b"null accum_out"),
        (_bwd(2, good, none, _table([None, sh[1]]), none, none), b"d_accum_out[0] is null"),
        (_bwd(2, good, none, good, _table([(1, 4, 5, 4), None]), none), b"d_accum_in[0] is [1,4,5,4], expected [2,4,5,4]"),
        (_bwd(2, good, none, good, none, _table([None, (2, 4, 5, 2)])), b"d_buffers[1] is [2,4,5,2], expected [2,4,5,1]"),
        (_bwd(2, good, none, good, None, none), b"null gradient table"),
    ]
    neg = _table(sh)
    neg[0].strides[2] = -4
    cases.append((_fwd(2, neg, none, good), b"buffers[0] has a negative stride"))
    for (rc, msg), want in cases:
        assert rc != 0 and want in msg, (want, msg)


def test_composite_signatures():
    T, P = ctypes.POINTER(_lib.mcs_tensor), ctypes.c_void_p
    l = _lib.lib()
    geom = [P, P, ctypes.c_int64, ctypes.c_int32, P, ctypes.c_int32, P]
    assert list(l.mcs_composite_fwd.argtypes) == [ctypes.c_int32, T, T, T] + geom + [P]
    assert list(l.mcs_composite_bwd.argtypes) == [ctypes.c_int32, T, T, T, T, T] + geom + [P, P]
