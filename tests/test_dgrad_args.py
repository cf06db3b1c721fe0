"""Argument checks of dm_conv2d_dgrad / dm_gemm_dgrad / dm_silu_bwd / dm_rowvec_grad.  They return before the library touches
the device, so the pointers here are never dereferenced and no GPU is needed."""
import ctypes as C

DM_EINVAL, DM_EUNSUPPORTED = -1, -2
DY, W, DX, Z = (C.c_void_p(a) for a in (0x10000, 0x20000, 0x30000, 0x40000))
ODD = C.c_void_p(0x10002)


def _ep(**kw):
    from dreammat_b200.dense_ops import Epilogue
    e = Epilogue()
    e.alpha = e.out_scale = 1.0
    for k, v in kw.items():
        setattr(e, k, v)
    return C.byref(e)


def _conv(bf16=1, dy=DY, H=16, Wd=16, Cout=64, w=W, Cin=64, ksize=3, pad=1, dx=DX, ldc=64, ep=None):
    from dreammat_b200._cabi import lib
    return lib().dm_conv2d_dgrad(bf16, dy, 2, H, Wd, Cout, w, Cin, ksize, pad, pad, dx, ldc, ep, 0, None)


def _gemm(bf16=1, dy=DY, ld_dy=128, w=W, ldw=64, dx=DX, ldc=64, M=100, N=128, K=64, ep=None):
    from dreammat_b200._cabi import lib
    return lib().dm_gemm_dgrad(bf16, dy, ld_dy, w, ldw, dx, ldc, M, N, K, ep, 0, None)


def _silu(bf16=1, z=Z, dy=DY, n=64, dx=DX):
    from dreammat_b200._cabi import lib
    return lib().dm_silu_bwd(bf16, z, dy, n, dx, None)


def _rowvec(bf16=1, dy=DY, ld=64, n_img=2, rows=16, N=64, out=DX, ld_out=64):
    from dreammat_b200._cabi import lib
    return lib().dm_rowvec_grad(bf16, dy, ld, n_img, rows, N, out, ld_out, None)


def test_dgrad_entry_points_reject_fp32_storage():
    from dreammat_b200._cabi import lib
    for fn in (_conv, _gemm, _silu, _rowvec):
        assert fn(bf16=2) == DM_EUNSUPPORTED and b"fp32" in lib().dm_last_error(), fn.__name__


def test_dgrad_rejects_bad_shapes_strides_and_alignment():
    from dreammat_b200._cabi import lib
    for kw in (dict(bf16=3), dict(Cout=96), dict(Cout=0), dict(Cin=12), dict(Cin=0), dict(ksize=2), dict(ksize=5), dict(pad=3),
               dict(pad=-1), dict(dy=ODD), dict(w=ODD), dict(dx=ODD), dict(dy=None), dict(w=None), dict(dx=None),
               dict(ldc=32), dict(ldc=68), dict(H=12, Wd=12), dict(H=0), dict(ep=_ep(act=3)), dict(ep=_ep(out_f32=1), ldc=66),
               dict(ep=_ep(residual=0x50000, ld_res=32))):
        assert _conv(**kw) == DM_EINVAL, (kw, lib().dm_last_error())
    for kw in (dict(bf16=-1), dict(N=96), dict(K=60), dict(M=0), dict(ld_dy=64), dict(ld_dy=132), dict(ldw=32), dict(ldw=68),
               dict(ldc=32), dict(ldc=68), dict(dy=ODD), dict(w=ODD), dict(dx=ODD), dict(dy=None), dict(ep=_ep(act=3))):
        assert _gemm(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


def test_streaming_backward_kernels_reject_bad_arguments():
    from dreammat_b200._cabi import lib
    for kw in (dict(bf16=3), dict(n=60), dict(n=-8), dict(z=ODD), dict(dy=ODD), dict(dx=ODD), dict(z=None), dict(dx=None)):
        assert _silu(**kw) == DM_EINVAL, (kw, lib().dm_last_error())
    for kw in (dict(bf16=3), dict(N=60), dict(N=0), dict(ld=60), dict(ld=32), dict(n_img=0), dict(rows=0), dict(dy=ODD),
               dict(dy=None), dict(out=None), dict(ld_out=32)):
        assert _rowvec(**kw) == DM_EINVAL, (kw, lib().dm_last_error())
