"""Argument checks of dm_attention_lse / dm_attention_bwd.  They return before the library touches the device, so the
pointers here are never dereferenced and no GPU is needed."""
import ctypes as C

DM_EINVAL, DM_EUNSUPPORTED = -1, -2
Q, K, V, O, DO, DQ, DK, DV = (C.c_void_p(0x100000 * (i + 1)) for i in range(8))
LSE, DELTA = C.c_void_p(0x900000), C.c_void_p(0xA00000)


def _bwd(bf16=1, q=Q, ldq=320, k=K, ldkv=640, o=O, ldo=320, do=DO, dq=DQ, lddq=960, dk=DK, dv=DV, lse=LSE, delta=DELTA,
         bs=8 * 1000, qbs=None, head_dim=64, heads=5):
    from dreammat_b200._cabi import lib
    return lib().dm_attention_bwd(bf16, q, ldq, bs * ldq if qbs is None else qbs, k, V, ldkv, bs * ldkv,
                                  o, ldo, bs * ldo, do, ldo, bs * ldo, lse, dq, lddq, bs * lddq, dk, lddq, bs * lddq,
                                  dv, lddq, bs * lddq, delta, 2, heads, 300, 77, head_dim, 0.125, None)


def _lse(bf16=1, q=Q, ldq=320, k=K, v=V, o=O, obs=300 * 320, lse=LSE, head_dim=64):
    from dreammat_b200._cabi import lib
    return lib().dm_attention_lse(bf16, q, ldq, 300 * ldq, k, v, 320, 77 * 320, o, 320, obs, 2, 5, 300, 77, head_dim,
                                  0.125, lse, None)


def test_attention_bwd_rejects_fp32_storage():
    from dreammat_b200._cabi import lib
    assert _bwd(bf16=2) == DM_EUNSUPPORTED and b"fp32" in lib().dm_last_error()
    assert _lse(bf16=2) == DM_EUNSUPPORTED and b"fp32" in lib().dm_last_error()


def test_attention_bwd_rejects_bad_shapes_strides_and_alignment():
    from dreammat_b200._cabi import lib
    odd = C.c_void_p(0x100008)      # 8-byte aligned: not enough for TMA
    for kw in (dict(bf16=3), dict(head_dim=32), dict(head_dim=128), dict(ldq=324), dict(ldkv=644), dict(ldo=316),
               dict(lddq=100), dict(ldq=256), dict(q=odd), dict(k=odd), dict(o=odd), dict(do=odd), dict(dq=odd),
               dict(dk=odd), dict(dv=odd), dict(lse=C.c_void_p(0x900002)), dict(q=None), dict(k=None), dict(do=None),
               dict(dq=None), dict(dv=None), dict(lse=None), dict(delta=None), dict(heads=0), dict(qbs=8 * 1000 * 320 + 4)):
        assert _bwd(**kw) == DM_EINVAL, (kw, lib().dm_last_error())
    for kw in (dict(bf16=3), dict(head_dim=32), dict(ldq=324), dict(ldq=256), dict(q=None), dict(lse=None),
               dict(lse=C.c_void_p(0x900002)), dict(q=odd), dict(k=odd), dict(v=odd), dict(o=odd), dict(obs=300 * 320 + 4)):
        assert _lse(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


def test_norm_and_geglu_backward_reject_fp32_and_bad_args():
    from dreammat_b200._cabi import lib
    L = lib()
    X, DY, G, OUT, DG, DB, ST = (C.c_void_p(0x100000 * (i + 1)) for i in range(7))
    ln = lambda bf16=1, x=X, C_=320: L.dm_layernorm_bwd(bf16, x, DY, 100, C_, G, 1e-5, None, OUT, DG, DB, None)  # noqa: E731
    gn = lambda bf16=1, x=X, C_=320, G_=32: L.dm_groupnorm_affine_grad(bf16, x, DY, 2, 64, C_, G_, G, G, 0, ST, DG, DB, None)  # noqa: E731
    gg = lambda bf16=1, h=X, D_=1280: L.dm_geglu_bwd(bf16, h, DY, 100, D_, OUT, None)  # noqa: E731
    for f in (ln, gn, gg):
        assert f(bf16=2) == DM_EUNSUPPORTED and b"fp32" in L.dm_last_error()
        assert f(bf16=3) == DM_EINVAL
    for kw in (dict(x=None), dict(C_=1288), dict(C_=324)):
        assert ln(**kw) == DM_EINVAL, kw
    for kw in (dict(x=None), dict(C_=324), dict(G_=0), dict(G_=33)):
        assert gn(**kw) == DM_EINVAL, kw
    for kw in (dict(h=None), dict(D_=1288)):
        assert gg(**kw) == DM_EINVAL, kw
