"""CPU: supersampled layer compositing (raster.composite with spp > 1) without a device.  The C entry points mcs_composite_ss_fwd / _bwd
check spp, the image size and every table's resolution before any launch (fake pointers, so a missing check would end in a failed
launch); their ctypes signatures are the header's; composite's argument errors raise ValueError naming the argument before any launch;
and render_layer's MSAA glue, rast[:, ::spp, ::spp] and the nearest upscale, is what the reference's scale_img_nhwc computes."""
import ctypes

import pytest
import torch

import nvdiffrecmc_b200._lib as L
from nvdiffrecmc_b200.raster import composite


def _table(shapes, ptr=0x10000):
    arr = (L.mcs_tensor * len(shapes))()
    for k, s in enumerate(shapes):
        if s is not None:
            B, H, W, C = s
            arr[k] = L._desc(ptr + 0x100000 * k, s, (H * W * C, W * C, C, 1))
    return arr


def _fwd(bufs, acc_in, acc_out, B=2, H=8, W=12, spp=2, n=2):
    l = L.lib()
    rc = l.mcs_composite_ss_fwd(n, bufs, acc_in, acc_out, B, H, W, spp, 0x1000, 0x2000, 0, 3, 0x3000, 1, 0x4000, None)
    return rc, l.mcs_last_error() or b""


def _bwd(bufs, acc_in, d_out, d_in, d_bufs, B=2, H=8, W=12, spp=2, n=2):
    l = L.lib()
    rc = l.mcs_composite_ss_bwd(n, bufs, acc_in, d_out, d_in, d_bufs, B, H, W, spp, 0x1000, 0x2000, 0, 3, 0x3000, 1, 0x4000, None, None)
    return rc, l.mcs_last_error() or b""


def test_supersampled_tables_are_checked_before_any_launch():
    if torch.cuda.is_available():
        pytest.skip("the calls would launch on the fake pointers")
    full, outr = [(2, 8, 12, 4), (2, 8, 12, 1)], [(2, 4, 6, 4), (2, 4, 6, 1)]
    F, O, none = _table(full), _table(outr), _table([None, None])
    cases = [
        (_fwd(F, none, O, spp=0), b"spp 0 (1 or more allowed)"),
        (_fwd(F, none, O, spp=-2), b"spp -2 (1 or more allowed)"),
        (_bwd(F, none, O, none, none, spp=0), b"spp 0 (1 or more allowed)"),
        (_fwd(F, none, O, H=9), b"H x W = 9 x 12 is not a multiple of spp 2"),
        (_fwd(F, none, O, W=13), b"H x W = 8 x 13 is not a multiple of spp 2"),
        (_bwd(F, none, O, none, none, spp=3), b"H x W = 8 x 12 is not a multiple of spp 3"),
        (_fwd(F, none, O, B=0), b"empty buffers"),
        (_fwd(_table([(2, 8, 12, 4), (2, 2, 3, 1)]), none, O), b"buffers[1] is [2,2,3,1], expected [2,8,12,1] or [2,4,6,1]"),
        (_fwd(_table([(2, 8, 12, 4), (2, 4, 6, 1)]), none, O), b"buffers[1] is at output resolution, an earlier entry at full resolution"),
        (_fwd(F, _table([(2, 4, 6, 4), (2, 8, 12, 1)]), O), b"accum_in[1] is at full resolution, an earlier entry at output resolution"),
        (_fwd(F, none, _table([(2, 4, 6, 4), (2, 8, 12, 1)])), b"accum_out[1] is at full resolution, an earlier entry at output resolution"),
        (_fwd(F, none, _table([(2, 4, 6, 4), (2, 4, 6, 2)])), b"accum_out[1] is [2,4,6,2], expected [2,8,12,1] or [2,4,6,1]"),
        (_fwd(F, none, O, spp=1), b"accum_out[0] is [2,4,6,4], expected [2,8,12,4]"),
        (_bwd(F, none, _table([(2, 4, 6, 4), (2, 8, 12, 1)]), none, none), b"d_accum_out[1] is at full resolution"),
        (_bwd(F, none, O, none, _table([None, (2, 4, 6, 1)])), b"d_buffers is at output resolution, buffers at full"),
        (_bwd(O, none, O, none, _table([(2, 8, 12, 4), None])), b"d_buffers is at full resolution, buffers at output"),
        (_bwd(F, O, O, _table([(2, 8, 12, 4), None]), none), b"d_accum_in is at full resolution, accum_in at output"),
        (_bwd(F, none, O, none, none, n=0), b"0 buffers (1 to 16 allowed)"),
        (_bwd(F, none, O, None, none), b"null gradient table"),
    ]
    for (rc, msg), want in cases:
        assert rc != 0 and want in msg, (want, msg)


def test_supersampled_signatures():
    T, P, i32 = ctypes.POINTER(L.mcs_tensor), ctypes.c_void_p, ctypes.c_int32
    l = L.lib()
    geom = [P, P, ctypes.c_int64, i32, P, i32, P]
    assert list(l.mcs_composite_ss_fwd.argtypes) == [i32, T, T, T, i32, i32, i32, i32] + geom + [P]
    assert list(l.mcs_composite_ss_bwd.argtypes) == [i32, T, T, T, T, T, i32, i32, i32, i32] + geom + [P, P]
    assert l.mcs_composite_ss_fwd.restype is ctypes.c_int and l.mcs_composite_ss_bwd.restype is ctypes.c_int


class _FakeCuda(torch.Tensor):
    """A CPU tensor that reports itself as a CUDA tensor, so composite's checks run past the device test on a machine without one."""
    @property
    def is_cuda(self):
        return True


def _fake(*shape, dtype=torch.float32):
    return torch.Tensor._make_subclass(_FakeCuda, torch.zeros(*shape, dtype=dtype))


def test_argument_errors_raise_before_any_launch():
    B, H, W = 2, 12, 18
    rast = _fake(B, H, W, 4)
    pos, tri = _fake(5, 4), _fake(3, 3, dtype=torch.int32)
    lo = lambda *c: {"shaded": _fake(B, H // 2, W // 2, 4), "kd": _fake(B, H // 2, W // 2, *c or (4,))}
    hi = lambda: {"shaded": _fake(B, H, W, 4), "kd": _fake(B, H, W, 4)}
    cases = [
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp=0)),
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp=-1)),
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp=2.0)),
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp=True)),
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp="2")),
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp=5)),                                 # H, W not multiples
        ("spp", lambda: composite([(lo(), rast)], pos, tri, spp=4)),                                 # W = 18 not a multiple
        ("layers", lambda: composite([({**lo(), "kd": _fake(B, 4, 6, 4)}, rast)], pos, tri, spp=2)),  # neither resolution
        ("layers", lambda: composite([({**lo(), "kd": _fake(B, H, W, 4)}, rast)], pos, tri, spp=2)),  # mixed within a layer
        ("layers", lambda: composite([(lo(), rast), (hi(), rast)], pos, tri, spp=2)),                # mixed between layers
        ("layers", lambda: composite([(lo(), rast), (lo(3), rast)], pos, tri, spp=2)),               # channel counts differ
        ("background", lambda: composite([(lo(), rast)], pos, tri, background={"shaded": _fake(B, H, W, 4)}, spp=2)),
        ("background", lambda: composite([(hi(), rast)], pos, tri, background={"shaded": _fake(B, H, W, 4)}, spp=3)),
        ("background", lambda: composite([(lo(), rast)], pos, tri, background={"shaded": _fake(B, H // 2, W // 2, 3)}, spp=2)),
    ]
    for name, call in cases:
        before = L.LAUNCHES.copy()
        with pytest.raises(ValueError, match=name):
            call()
        assert L.LAUNCHES == before, name


def _scale_nearest(x, size):
    """The reference's scale_img_nhwc(x, size, mag='nearest', min='nearest'): one F.interpolate in NCHW, back to contiguous NHWC."""
    return torch.nn.functional.interpolate(x.permute(0, 3, 1, 2), size, mode="nearest").permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("spp", range(2, 9))
def test_msaa_glue_is_the_reference_nearest_scaling(spp):
    g = torch.Generator().manual_seed(spp)
    for H, W in ((3, 5), (16, 24), (37, 64)):
        rast = torch.rand(2, H * spp, W * spp, 4, generator=g)
        assert torch.equal(rast[:, ::spp, ::spp], _scale_nearest(rast, (H, W)))
        buf = torch.rand(2, H, W, 3, generator=g)
        up = buf.repeat_interleave(spp, dim=1).repeat_interleave(spp, dim=2)
        assert torch.equal(up, _scale_nearest(buf, (H * spp, W * spp)))
