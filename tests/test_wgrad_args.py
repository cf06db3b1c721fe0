"""Argument checks of dm_conv2d_wgrad / dm_gemm_wgrad.  They return before the library touches the device, so the
pointers here are never dereferenced and no GPU is needed."""
import ctypes as C

DM_EINVAL, DM_EUNSUPPORTED = -1, -2
X, DY, DW, DB = (C.c_void_p(a) for a in (0x10000, 0x20000, 0x30000, 0x40000))


def _conv(bf16=1, x=X, Cin=64, dy=DY, ld_dy=64, ksize=3, dw=DW, Ho=16, Wo=16):
    from dreammat_b200._cabi import lib
    return lib().dm_conv2d_wgrad(bf16, x, 2, 16, 16, Cin, dy, ld_dy, 64, ksize, 1, 1, 1, Ho, Wo, dw, DB, None)


def _gemm(bf16=1, dy=DY, ld_dy=64, x=X, ldx=128, K=128, dw=DW):
    from dreammat_b200._cabi import lib
    return lib().dm_gemm_wgrad(bf16, dy, ld_dy, x, ldx, 100, 64, K, dw, DB, None)


def test_wgrad_rejects_fp32_storage():
    from dreammat_b200._cabi import lib
    assert _conv(bf16=2) == DM_EUNSUPPORTED and b"fp32" in lib().dm_last_error()
    assert _gemm(bf16=2) == DM_EUNSUPPORTED and b"fp32" in lib().dm_last_error()


def test_wgrad_rejects_bad_shapes_strides_and_alignment():
    from dreammat_b200._cabi import lib
    odd = C.c_void_p(0x10002)
    for kw in (dict(bf16=3), dict(Cin=96), dict(ld_dy=60), dict(ld_dy=32), dict(ksize=2), dict(ksize=5), dict(x=odd),
               dict(dy=odd), dict(dw=odd), dict(x=None), dict(Ho=12, Wo=12)):
        assert _conv(**kw) == DM_EINVAL, (kw, lib().dm_last_error())
    for kw in (dict(K=96), dict(ld_dy=60), dict(ldx=100), dict(ldx=64), dict(x=odd), dict(dy=odd), dict(dw=odd)):
        assert _gemm(**kw) == DM_EINVAL, (kw, lib().dm_last_error())
