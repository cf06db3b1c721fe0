"""Argument checks of dm_mse_loss_grad / dm_upsample2x_bwd, and UNet.forward's refusal of a tape together with the CSD
epilogue.  The library calls return before touching the device, so the pointers here are never dereferenced and no GPU is
needed."""
import ctypes as C

import pytest

DM_EINVAL, DM_EUNSUPPORTED = -1, -2
PRED, TGT, DP, LOSS, DY, DX = (C.c_void_p(a) for a in (0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000))
ODD2, ODD8 = C.c_void_p(0x10002), C.c_void_p(0x10008)


def _mse(bf16=1, pred=PRED, target=TGT, n=2, Cc=4, HW=256, grad_scale=1.0, d_pred=DP, ld=64, loss=LOSS):
    from dreammat_b200._cabi import lib
    return lib().dm_mse_loss_grad(bf16, pred, target, n, Cc, HW, grad_scale, d_pred, ld, loss, None)


def _up(bf16=1, dy=DY, n=2, H=8, W=8, Cc=64, dx=DX):
    from dreammat_b200._cabi import lib
    return lib().dm_upsample2x_bwd(bf16, dy, n, H, W, Cc, dx, None)


def test_loss_and_upsample_backward_reject_fp32_storage():
    from dreammat_b200._cabi import lib
    for fn in (_mse, _up):
        assert fn(bf16=2) == DM_EUNSUPPORTED and b"fp32" in lib().dm_last_error(), fn.__name__


def test_mse_loss_grad_rejects_bad_arguments():
    from dreammat_b200._cabi import lib
    for kw in (dict(bf16=3), dict(bf16=-1), dict(pred=None), dict(target=None), dict(d_pred=None), dict(loss=None),
               dict(n=0), dict(Cc=0), dict(HW=0), dict(n=-1), dict(ld=32), dict(ld=96), dict(ld=0), dict(Cc=65),
               dict(d_pred=ODD8), dict(pred=ODD2), dict(target=ODD2), dict(loss=ODD2)):
        assert _mse(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


def test_upsample2x_bwd_rejects_bad_arguments():
    from dreammat_b200._cabi import lib
    for kw in (dict(bf16=3), dict(bf16=-1), dict(dy=None), dict(dx=None), dict(Cc=60), dict(Cc=0), dict(n=0), dict(H=0),
               dict(W=-2), dict(dy=ODD8), dict(dx=ODD8)):
        assert _up(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


def test_unet_forward_refuses_tape_with_csd():
    from dreammat_b200.nets import UNet
    net = UNet.__new__(UNet)        # the check comes before any weight or device is touched
    with pytest.raises(ValueError, match="tape"):
        net.forward(None, None, None, csd={}, tape={})
