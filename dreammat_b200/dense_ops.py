"""torch-facing wrappers of the dense-path C-ABI entry points (tensor-core GEMM / conv, norms,
attention, elementwise).  Activations are NHWC fp16 (or bf16); accumulation is fp32.

fp32 tensors select the high-precision mode (half_precision_weights=false, dreammat_guidance.py:56,92-94): the
contractions run on the same bf16 tensor-core kernel over 3-way split operands (csrc/dense_hp.cu), everything
else on fp32 storage."""
from __future__ import annotations

import ctypes as C

import torch

from ._cabi import check, lib, ptr, stream_ptr


class Epilogue(C.Structure):
    _fields_ = [("bias", C.c_void_p), ("rowvec", C.c_void_p), ("rows_per_vec", C.c_int32), ("ld_rowvec", C.c_int32),
                ("residual", C.c_void_p), ("ld_res", C.c_int32), ("res_batch_stride", C.c_int64),
                ("alpha", C.c_float), ("out_scale", C.c_float), ("act", C.c_int32), ("out_f32", C.c_int32)]


ACT = {None: 0, "none": 0, "silu": 1, "gelu": 2, "geglu": 3}


def _ep(bias=None, rowvec=None, rows_per_vec=1, residual=None, ld_res=0, res_batch_stride=0, alpha=1.0, out_scale=1.0,
        act=None, out_f32=False):
    e = Epilogue()
    e.bias = bias.data_ptr() if bias is not None else None
    e.rowvec = rowvec.data_ptr() if rowvec is not None else None
    e.rows_per_vec = rows_per_vec
    e.ld_rowvec = (rowvec.stride(-2) if rowvec.dim() > 1 else rowvec.shape[-1]) if rowvec is not None else 0
    e.residual = residual.data_ptr() if residual is not None else None
    e.ld_res = ld_res
    e.res_batch_stride = res_batch_stride
    e.alpha = alpha
    e.out_scale = out_scale
    e.act = ACT[act]
    e.out_f32 = 1 if out_f32 else 0
    return e


def _is_bf16(t):
    """storage selector of the C-ABI: 0 fp16, 1 bf16, 2 fp32 (high-precision mode)."""
    if t.dtype == torch.bfloat16:
        return 1
    if t.dtype == torch.float16:
        return 0
    if t.dtype == torch.float32:
        return 2
    raise TypeError(f"dense path expects fp16/bf16/fp32, got {t.dtype}")


def _dt_code(dtype):
    return {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}[dtype]


def hp_split(x2d, pattern):
    """fp32 [rows, cols] (row stride allowed) -> bf16 [rows, 6*cols]; pattern 0: A operand, 1: B operand."""
    assert x2d.dtype == torch.float32 and x2d.dim() == 2 and x2d.stride(1) == 1
    rows, cols = x2d.shape
    out = torch.empty(rows, 6 * cols, device=x2d.device, dtype=torch.bfloat16)
    check(lib().dm_hp_split(ptr_any(x2d), rows, cols, x2d.stride(0), pattern, ptr_any(out), stream_ptr()), "dm_hp_split")
    return out


def _hp_rows(t):
    """[.., R, C] view with a uniform row stride -> 2-D [rows, C] view (no copy when possible)."""
    if t.dim() == 2:
        return t
    if t.stride(0) == t.shape[1] * t.stride(1):
        return t.as_strided((t.shape[0] * t.shape[1], t.shape[2]), (t.stride(1), 1))
    return t.contiguous().view(-1, t.shape[-1])


def _hp_finish(raw, rows, N, rows_per_batch, e, out, ldc, out_bs):
    check(lib().dm_hp_epilogue(ptr_any(raw), rows, N, rows_per_batch, C.byref(e), ptr_any(out), ldc, out_bs, stream_ptr()),
          "dm_hp_epilogue")
    return out


def _hp_gemm(a, b, bias, rowvec, rows_per_vec, residual, alpha, out_scale, act, out, bn):
    batched = a.dim() == 3
    batch = a.shape[0] if batched else 1
    M, K = a.shape[-2], a.shape[-1]
    N = b.shape[-2]
    a6 = hp_split(_hp_rows(a), 0)
    b6 = hp_split(_hp_rows(b), 1)
    raw = torch.empty(batch * M, N, device=a.device, dtype=torch.float32)
    K6 = 6 * K
    e0 = _ep(out_f32=True)
    bshared = b.dim() == 2
    check(lib().dm_gemm(1, ptr_any(a6), K6, M * K6, ptr_any(b6), K6, 0 if bshared else N * K6, ptr_any(raw), N, M * N, M, N, K6,
                        batch, C.byref(e0), bn, stream_ptr()), "dm_gemm")
    n_out = N // 2 if act == "geglu" else N
    if out is None:
        out = torch.empty((batch, M, n_out) if batched else (M, n_out), device=a.device, dtype=torch.float32)
    assert out.dtype == torch.float32 and out.stride(-1) == 1
    ld_res = residual.stride(-2) if residual is not None else 0
    r_bs = residual.stride(0) if (residual is not None and residual.dim() == 3) else 0
    e = _ep(bias, rowvec, rows_per_vec, residual, ld_res, r_bs, alpha, out_scale, act, True)
    return _hp_finish(raw, batch * M, N, M, e, out, out.stride(-2), out.stride(0) if batched else 0)


def _hp_conv2d(x, w, ksize, stride, pad, Ho, Wo, bias, rowvec, residual, out_scale, act, out, bn):
    n, H, W, Cin = x.shape
    Cout = w.shape[0]
    taps = ksize * ksize
    x6 = hp_split(x.view(-1, Cin), 0).view(n, H, W, 6 * Cin)
    w6 = hp_split(w.view(Cout * taps, Cin), 1).view(Cout, taps * 6 * Cin)
    raw = torch.empty(n * Ho * Wo, Cout, device=x.device, dtype=torch.float32)
    e0 = _ep(out_f32=True)
    check(lib().dm_conv2d(1, ptr_any(x6), n, H, W, 6 * Cin, ptr_any(w6), Cout, ksize, stride, pad[0], pad[1], Ho, Wo,
                          ptr_any(raw), Cout, C.byref(e0), bn, stream_ptr()), "dm_conv2d")
    if out is None:
        out = torch.empty(n, Ho, Wo, Cout, device=x.device, dtype=torch.float32)
    assert out.dtype == torch.float32
    ld_res = residual.stride(2) if residual is not None else 0
    e = _ep(bias, rowvec, Ho * Wo, residual, ld_res, 0, 1.0, out_scale, act, True)
    return _hp_finish(raw, n * Ho * Wo, Cout, n * Ho * Wo, e, out, out.stride(2), 0)


_WORKSPACE = {}


def _ensure_workspace():
    """Hand the library its split-K scratch (a zero-filled torch buffer, owned here) once per process; skipped while a
    CUDA graph is being captured -- the eager warm-up that precedes every capture has already done it."""
    dev = torch.cuda.current_device()
    if dev in _WORKSPACE or torch.cuda.is_current_stream_capturing():
        return
    n = int(lib().dm_gemm_workspace_bytes())
    buf = torch.zeros(n // 4, device=f"cuda:{dev}", dtype=torch.float32)
    check(lib().dm_gemm_set_workspace(ptr_any(buf), n), "dm_gemm_set_workspace")
    _WORKSPACE[dev] = buf


def gemm(a, b, bias=None, rowvec=None, rows_per_vec=1, residual=None, alpha=1.0, out_scale=1.0, act=None,
         out=None, out_f32=False, bn=0):
    """a [.., M, K] @ b [.., N, K]^T -> [.., M, N].  Leading dim (if any) is a batch; b may be 2-D (shared)."""
    _ensure_workspace()
    bf = _is_bf16(a)
    assert b.dtype == a.dtype
    if bf == 2:
        assert a.stride(-1) == 1 and b.stride(-1) == 1 and b.shape[-1] == a.shape[-1]
        return _hp_gemm(a, b, bias, rowvec, rows_per_vec, residual, alpha, out_scale, act, out, bn)
    batched = a.dim() == 3
    batch = a.shape[0] if batched else 1
    M, K = a.shape[-2], a.shape[-1]
    N = b.shape[-2]
    assert b.shape[-1] == K
    assert a.stride(-1) == 1 and b.stride(-1) == 1
    lda, ldb = a.stride(-2), b.stride(-2)
    a_bs = a.stride(0) if batched else 0
    b_bs = b.stride(0) if b.dim() == 3 else 0
    if out is None:
        n_out = N // 2 if act == "geglu" else N      # GEGLU epilogue: value * gelu(gate), see geglu_interleave
        shape = (batch, M, n_out) if batched else (M, n_out)
        out = torch.empty(shape, device=a.device, dtype=torch.float32 if out_f32 else a.dtype)
    assert out.stride(-1) == 1
    ldc = out.stride(-2)
    c_bs = out.stride(0) if batched else 0
    ld_res = residual.stride(-2) if residual is not None else 0
    r_bs = residual.stride(0) if (residual is not None and residual.dim() == 3) else 0
    e = _ep(bias, rowvec, rows_per_vec, residual, ld_res, r_bs, alpha, out_scale, act, out.dtype == torch.float32)
    check(lib().dm_gemm(bf, ptr_any(a), lda, a_bs, ptr_any(b), ldb, b_bs, ptr_any(out), ldc, c_bs, M, N, K, batch,
                        C.byref(e), bn, stream_ptr()), "dm_gemm")
    return out


def ptr_any(t):
    return C.c_void_p(t.data_ptr())


def _conv_out_hw(H, W, ksize, stride, pad, out_hw):
    """output extent of conv2d: symmetric padding pad = (top, left) unless out_hw fixes it (then the bottom / right
    padding is whatever out_hw implies)"""
    if out_hw is not None:
        return tuple(out_hw)
    pt, pl = pad
    return (H + 2 * pt - ksize) // stride + 1, (W + 2 * pl - ksize) // stride + 1


def conv2d(x, w, ksize, stride=1, pad=(1, 1), out_hw=None, bias=None, rowvec=None, residual=None, out_scale=1.0,
           act=None, out=None, out_f32=False, bn=0):
    """x [n,H,W,Cin] NHWC (contiguous), w [Cout, k*k*Cin] -> y [n,Ho,Wo,Cout] (or into `out`, whose last-dim
    stride must be 1; its pixel stride gives ldc so it can be a channel slice of a wider buffer)."""
    _ensure_workspace()
    bf = _is_bf16(x)
    assert x.is_contiguous() and w.is_contiguous()
    n, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert w.shape[1] == ksize * ksize * Cin
    Ho, Wo = _conv_out_hw(H, W, ksize, stride, pad, out_hw)
    if out is None:
        out = torch.empty(n, Ho, Wo, Cout, device=x.device, dtype=torch.float32 if out_f32 else x.dtype)
    assert out.stride(-1) == 1 and out.shape[:3] == (n, Ho, Wo)
    ldc = out.stride(2)
    assert out.stride(1) == Wo * ldc and out.stride(0) == Ho * Wo * ldc
    ld_res = 0
    if residual is not None:
        ld_res = residual.stride(2)
        assert residual.stride(-1) == 1 and residual.stride(1) == Wo * ld_res and residual.stride(0) == Ho * Wo * ld_res
    if bf == 2:
        return _hp_conv2d(x, w, ksize, stride, pad, Ho, Wo, bias, rowvec, residual, out_scale, act, out, bn)
    e = _ep(bias, rowvec, Ho * Wo, residual, ld_res, 0, 1.0, out_scale, act, out.dtype == torch.float32)
    check(lib().dm_conv2d(bf, ptr_any(x), n, H, W, Cin, ptr_any(w), Cout, ksize, stride, pad[0], pad[1], Ho, Wo,
                          ptr_any(out), ldc, C.byref(e), bn, stream_ptr()), "dm_conv2d")
    return out


def _wgrad_storage(t):
    bf = _is_bf16(t)
    if bf == 2:
        raise TypeError("weight gradients need fp16 / bf16 storage (the fp32 high-precision mode has none)")
    return bf


def conv2d_wgrad(x, dy, ksize, stride=1, pad=(1, 1), out_hw=None, bias=False):
    """Weight (and bias) gradient of conv2d(x, w, ksize, stride, pad, out_hw) for the output gradient dy [n,Ho,Wo,Cout],
    which may be a channel slice of a wider buffer (its pixel stride is passed on).  Returns (dw, db): dw [Cout, k*k*Cin]
    fp32 in conv2d's weight layout (tap-major, channel-minor, padded channels included), db [Cout] fp32 or None."""
    _ensure_workspace()
    bf = _wgrad_storage(x)
    assert dy.dtype == x.dtype and x.is_contiguous()
    n, H, W, Cin = x.shape
    Ho, Wo = _conv_out_hw(H, W, ksize, stride, pad, out_hw)
    assert dy.shape[:3] == (n, Ho, Wo) and dy.stride(-1) == 1
    ld = dy.stride(2)
    assert dy.stride(1) == Wo * ld and dy.stride(0) == Ho * Wo * ld
    Cout = dy.shape[3]
    dw = torch.empty(Cout, ksize * ksize * Cin, device=x.device, dtype=torch.float32)
    db = torch.empty(Cout, device=x.device, dtype=torch.float32) if bias else None
    check(lib().dm_conv2d_wgrad(bf, ptr_any(x), n, H, W, Cin, ptr_any(dy), ld, Cout, ksize, stride, pad[0], pad[1], Ho, Wo,
                                ptr_any(dw), ptr_any(db) if bias else None, stream_ptr()), "dm_conv2d_wgrad")
    return dw, db


def gemm_wgrad(dy, x, bias=False):
    """Weight (and bias) gradient of gemm(x, w) = x w^T for the output gradient dy: dy [.., M, N], x [.., M, K] (leading
    dims fold into M; row strides allowed, e.g. a column slice of a fused projection).  Returns (dw, db): dw [N, K] fp32 in
    the layout and row order of w, db [N] fp32 or None."""
    _ensure_workspace()
    bf = _wgrad_storage(x)
    assert dy.dtype == x.dtype and dy.stride(-1) == 1 and x.stride(-1) == 1
    dy2, x2 = _hp_rows(dy), _hp_rows(x)
    M, N = dy2.shape
    K = x2.shape[1]
    assert x2.shape[0] == M
    dw = torch.empty(N, K, device=x.device, dtype=torch.float32)
    db = torch.empty(N, device=x.device, dtype=torch.float32) if bias else None
    check(lib().dm_gemm_wgrad(bf, ptr_any(dy2), dy2.stride(0), ptr_any(x2), x2.stride(0), M, N, K, ptr_any(dw),
                              ptr_any(db) if bias else None, stream_ptr()), "dm_gemm_wgrad")
    return dw, db


def conv2d_dgrad(dy, w, ksize, pad=(1, 1), cin=None, residual=None, alpha=1.0, out_scale=1.0, out=None, out_f32=False, bn=0):
    """Input gradient of the stride-1 conv2d(x, w, ksize, pad=pad) for the output gradient dy [n,H,W,Cout] (contiguous),
    read from the forward weight w [Cout, k*k*Cin] itself: dx [n,H,W,Cin] (+ residual, a second gradient branch), or into
    `out`, which may be a channel slice of a wider buffer.  cin defaults to w's.  A stride-2 forward is differentiated by
    upsample2x(dy, zero_insert=True) followed by this.  16-bit storage only."""
    _ensure_workspace()
    bf = _wgrad_storage(dy)
    assert w.dtype == dy.dtype and dy.is_contiguous() and w.is_contiguous()
    n, H, W, Cout = dy.shape
    taps = ksize * ksize
    assert w.shape[0] == Cout and w.shape[1] % taps == 0
    Cin = w.shape[1] // taps
    assert cin is None or cin == Cin, "cin must be the channel count of the weight's layout"
    if out is None:
        out = torch.empty(n, H, W, Cin, device=dy.device, dtype=torch.float32 if out_f32 else dy.dtype)
    assert out.stride(-1) == 1 and tuple(out.shape) == (n, H, W, Cin)
    ldc = out.stride(2)
    assert out.stride(1) == W * ldc and out.stride(0) == H * W * ldc
    ld_res = 0
    if residual is not None:
        ld_res = residual.stride(2)
        assert residual.stride(-1) == 1 and residual.stride(1) == W * ld_res and residual.stride(0) == H * W * ld_res
    e = _ep(None, None, H * W, residual, ld_res, 0, alpha, out_scale, None, out.dtype == torch.float32)
    check(lib().dm_conv2d_dgrad(bf, ptr_any(dy), n, H, W, Cout, ptr_any(w), Cin, ksize, pad[0], pad[1], ptr_any(out), ldc,
                                C.byref(e), bn, stream_ptr()), "dm_conv2d_dgrad")
    return out


def gemm_dgrad(dy, w, residual=None, alpha=1.0, out_scale=1.0, out=None, out_f32=False, bn=0):
    """Input gradient of gemm(x, w) = x w^T for the output gradient dy [.., M, N] (leading dims fold into M; row stride
    allowed), read from the forward weight w [N, K] itself: dx [M, K] (+ residual [M, K]).  16-bit storage only."""
    _ensure_workspace()
    bf = _wgrad_storage(dy)
    assert w.dtype == dy.dtype and dy.stride(-1) == 1 and w.dim() == 2 and w.stride(1) == 1
    dy2 = _hp_rows(dy)
    M, N = dy2.shape
    K = w.shape[1]
    assert w.shape[0] == N
    if out is None:
        out = torch.empty(M, K, device=dy.device, dtype=torch.float32 if out_f32 else dy.dtype)
    assert out.dim() == 2 and tuple(out.shape) == (M, K) and out.stride(1) == 1
    ld_res = 0
    if residual is not None:
        assert residual.dim() == 2 and residual.stride(1) == 1 and tuple(residual.shape) == (M, K)
        ld_res = residual.stride(0)
    e = _ep(None, None, 1, residual, ld_res, 0, alpha, out_scale, None, out.dtype == torch.float32)
    check(lib().dm_gemm_dgrad(bf, ptr_any(dy2), dy2.stride(0), ptr_any(w), w.stride(0), ptr_any(out), out.stride(0), M, N, K,
                              C.byref(e), bn, stream_ptr()), "dm_gemm_dgrad")
    return out


class Csd(C.Structure):
    _fields_ = [("noise", C.c_void_p), ("w", C.c_void_p), ("coef", C.c_void_p), ("grad", C.c_void_p),
                ("dlatents", C.c_void_p), ("norms", C.c_void_p), ("eps_out", C.c_void_p)]


def csd_supported(x_dtype, B, h, w):
    """the fused conv_out + CSD epilogue needs 16-bit storage and whole 128-row tiles inside one CFG branch"""
    if x_dtype == torch.float32 or (B * h * w) % 128 != 0:
        return False
    tw = min(w, 128)
    th = min(128 // tw, h)
    tn = 128 // (tw * th)
    return tw * th * tn == 128 and w % tw == 0 and h % th == 0 and (tn == 1 or B % tn == 0)


def conv2d_csd(x, w, bias, noise, w1mac, coef, grad=None, dlat=None, norms=None, eps_out=None):
    """conv_out + CSD combine in one kernel (dm_conv2d_csd).  x [3B,h,w,Cin] ordered [branch][view]; noise / grad / dlat
    [B,4,h,w] fp32; coef = device tensor (c_text, c_uncond, c_null, c_noise, dlat_scale); norms[10] is accumulated into."""
    bf = _is_bf16(x)
    assert x.is_contiguous() and w.is_contiguous() and noise.is_contiguous() and coef.dtype == torch.float32
    n3, h, ww, Cin = x.shape
    B = n3 // 3
    assert n3 == 3 * B and w.shape == (4, 9 * Cin) and noise.shape == (B, 4, h, ww) and norms is not None
    c = Csd(noise.data_ptr(), w1mac.data_ptr(), coef.data_ptr(), grad.data_ptr() if grad is not None else None,
            dlat.data_ptr() if dlat is not None else None, norms.data_ptr(), eps_out.data_ptr() if eps_out is not None else None)
    check(lib().dm_conv2d_csd(bf, ptr_any(x), B, h, ww, Cin, ptr_any(w), ptr_any(bias), C.byref(c), stream_ptr()), "dm_conv2d_csd")


def conv_weight_to_gemm(w_oihw: torch.Tensor, cin_pad: int = 0, cout_pad: int = 0, dtype=torch.float16):
    """[Cout,Cin,kh,kw] (diffusers layout) -> [Cout_pad, kh*kw*Cin_pad], tap-major / channel-minor."""
    Cout, Cin, kh, kw = w_oihw.shape
    cin_p = max(cin_pad, Cin)
    cout_p = max(cout_pad, Cout)
    w = torch.zeros(cout_p, kh, kw, cin_p, dtype=torch.float32, device=w_oihw.device)
    w[:Cout, :, :, :Cin] = w_oihw.float().permute(0, 2, 3, 1)
    return w.reshape(cout_p, kh * kw * cin_p).to(dtype).contiguous()


# ----------------------------------------------------------------------------- streaming kernels


def groupnorm(x, gamma, beta, groups=32, eps=1e-5, silu=False, out=None, stats=None):
    """x [n, H, W, C] (channel slice allowed: stride(-2) = ld) -> same shape; returns (y, stats)."""
    bf = _is_bf16(x)
    n, Hh, W, Cc = x.shape
    ld = x.stride(2)
    assert x.stride(3) == 1 and x.stride(1) == W * ld and x.stride(0) == Hh * W * ld
    if out is None:
        out = torch.empty(n, Hh, W, Cc, device=x.device, dtype=x.dtype)
    if stats is None:
        stats = torch.empty(n * groups * 2, device=x.device, dtype=torch.float32)
    check(lib().dm_groupnorm(bf, ptr_any(x), n, Hh * W, Cc, ld, groups, ptr_any(gamma), ptr_any(beta), eps,
                             1 if silu else 0, ptr_any(out), out.stride(2), ptr_any(stats), stream_ptr()), "dm_groupnorm")
    return out, stats


def groupnorm_bwd(x, dz, gamma, beta, stats, groups=32, eps=1e-5, silu=False, dx_add=None):
    bf = _is_bf16(x)
    n, Hh, W, Cc = x.shape
    assert x.is_contiguous() and dz.is_contiguous()
    dx = torch.empty_like(x)
    bstats = torch.empty(n * groups * 2, device=x.device, dtype=torch.float32)
    check(lib().dm_groupnorm_bwd(bf, ptr_any(x), ptr_any(dz), n, Hh * W, Cc, groups, ptr_any(gamma), ptr_any(beta), eps,
                                 1 if silu else 0, ptr_any(stats), ptr_any(bstats),
                                 ptr_any(dx_add) if dx_add is not None else None, ptr_any(dx), stream_ptr()),
          "dm_groupnorm_bwd")
    return dx


def layernorm(x, gamma, beta, eps=1e-5):
    bf = _is_bf16(x)
    assert x.is_contiguous()
    Cc = x.shape[-1]
    M = x.numel() // Cc
    y = torch.empty_like(x)
    check(lib().dm_layernorm(bf, ptr_any(x), M, Cc, ptr_any(gamma), ptr_any(beta), eps, ptr_any(y), stream_ptr()),
          "dm_layernorm")
    return y


def layernorm_bwd(x, dy, gamma, eps=1e-5, dx_add=None):
    """Backward of layernorm(x, gamma, beta, eps): returns (dx [storage dtype] (+ dx_add), dgamma, dbeta [C] fp32).
    16-bit storage only; deterministic."""
    bf = _is_bf16(x)
    assert x.is_contiguous() and dy.is_contiguous() and dy.shape == x.shape
    assert dx_add is None or (dx_add.is_contiguous() and dx_add.shape == x.shape)
    Cc = x.shape[-1]
    dx = torch.empty_like(x)
    dg = torch.empty(Cc, device=x.device, dtype=torch.float32)
    db = torch.empty(Cc, device=x.device, dtype=torch.float32)
    check(lib().dm_layernorm_bwd(bf, ptr_any(x), ptr_any(dy), x.numel() // Cc, Cc, ptr_any(gamma), eps,
                                 ptr_any(dx_add) if dx_add is not None else None, ptr_any(dx), ptr_any(dg), ptr_any(db),
                                 stream_ptr()), "dm_layernorm_bwd")
    return dx, dg, db


def groupnorm_affine_grad(x, dz, gamma, beta, stats, groups=32, silu=False):
    """(dgamma, dbeta) [C] fp32 of groupnorm(x, gamma, beta, groups, silu=silu) for the output gradient dz (x, dz dense
    [n, H, W, C]; stats from groupnorm).  16-bit storage only; deterministic."""
    bf = _is_bf16(x)
    n, Hh, W, Cc = x.shape
    assert x.is_contiguous() and dz.is_contiguous() and dz.shape == x.shape
    dg = torch.empty(Cc, device=x.device, dtype=torch.float32)
    db = torch.empty(Cc, device=x.device, dtype=torch.float32)
    check(lib().dm_groupnorm_affine_grad(bf, ptr_any(x), ptr_any(dz), n, Hh * W, Cc, groups, ptr_any(gamma), ptr_any(beta),
                                         1 if silu else 0, ptr_any(stats), ptr_any(dg), ptr_any(db), stream_ptr()),
          "dm_groupnorm_affine_grad")
    return dg, db


def geglu_interleave(w):
    """Row order the fused GEGLU epilogue of dm_gemm expects: [value | gate] halves (diffusers GEGLU.proj,
    attention.py chunk(2, dim=-1)) -> alternating blocks of 32 value rows and their 32 gate rows."""
    D = w.shape[0] // 2
    assert D % 32 == 0
    v, g = w[:D].reshape(D // 32, 1, 32, *w.shape[1:]), w[D:].reshape(D // 32, 1, 32, *w.shape[1:])
    return torch.cat([v, g], 1).reshape(w.shape).contiguous()


def geglu(h):
    bf = _is_bf16(h)
    assert h.is_contiguous()
    D = h.shape[-1] // 2
    M = h.numel() // (2 * D)
    out = torch.empty(*h.shape[:-1], D, device=h.device, dtype=h.dtype)
    check(lib().dm_geglu(bf, ptr_any(h), M, D, ptr_any(out), stream_ptr()), "dm_geglu")
    return out


def geglu_bwd(h, dout):
    """Gradient of the fused GEGLU epilogue (gemm(..., act="geglu")) with respect to its interleaved pre-activation h
    [.., 2D] (geglu_interleave's row order) for dout [.., D]: dh in h's layout.  16-bit storage only."""
    bf = _is_bf16(h)
    assert h.is_contiguous() and dout.is_contiguous()
    D2 = h.shape[-1]
    M = h.numel() // D2
    assert dout.numel() == M * (D2 // 2)
    dh = torch.empty_like(h)
    check(lib().dm_geglu_bwd(bf, ptr_any(h), ptr_any(dout), M, D2 // 2, ptr_any(dh), stream_ptr()), "dm_geglu_bwd")
    return dh


def upsample2x(x, zero_insert=False):
    bf = _is_bf16(x)
    assert x.is_contiguous()
    n, Hh, W, Cc = x.shape
    y = torch.empty(n, 2 * Hh, 2 * W, Cc, device=x.device, dtype=x.dtype)
    check(lib().dm_upsample2x(bf, ptr_any(x), n, Hh, W, Cc, 1 if zero_insert else 0, ptr_any(y), stream_ptr()),
          "dm_upsample2x")
    return y


def axpby(s1, a=1.0, s2=None, b=1.0, out=None):
    """out[..., :] = a*s1 + b*s2 over 2-D views [rows, cols] with arbitrary row strides (last dim contiguous)."""
    bf = _is_bf16(s1)
    cols = s1.shape[-1]
    rows = s1.numel() // cols

    def ld(t):
        assert t.stride(-1) == 1
        return t.stride(-2) if t.dim() > 1 else cols
    if out is None:
        out = torch.empty(s1.shape, device=s1.device, dtype=s1.dtype)
    check(lib().dm_axpby2d(bf, ptr_any(s1), ld(s1), a, ptr_any(s2) if s2 is not None else None,
                           ld(s2) if s2 is not None else 0, b, rows, cols, ptr_any(out), ld(out), stream_ptr()),
          "dm_axpby2d")
    return out


def transpose(x):
    """[B, R, C] -> [B, C, R] (or 2-D)."""
    bf = _is_bf16(x)
    squeeze = x.dim() == 2
    if squeeze:
        x = x.unsqueeze(0)
    assert x.stride(2) == 1
    B, R, Cc = x.shape
    y = torch.empty(B, Cc, R, device=x.device, dtype=x.dtype)
    check(lib().dm_transpose(bf, ptr_any(x), B, R, Cc, x.stride(1), x.stride(0), ptr_any(y), R, Cc * R, stream_ptr()),
          "dm_transpose")
    return y[0] if squeeze else y


def softmax_rows(x, scale=1.0):
    bf = _is_bf16(x)
    assert x.is_contiguous()
    cols = x.shape[-1]
    y = torch.empty_like(x)
    check(lib().dm_softmax_rows(bf, ptr_any(x), x.numel() // cols, cols, cols, scale, ptr_any(y), stream_ptr()),
          "dm_softmax_rows")
    return y


def softmax_bwd(P, dP, scale=1.0):
    bf = _is_bf16(P)
    cols = P.shape[-1]
    dS = torch.empty_like(P)
    check(lib().dm_softmax_bwd(bf, ptr_any(P), ptr_any(dP), P.numel() // cols, cols, cols, scale, ptr_any(dS),
                               stream_ptr()), "dm_softmax_bwd")
    return dS


def pad_convert(x_f32, cpad, scale=1.0, shift=0.0, dtype=torch.float16):
    x_f32 = x_f32.contiguous()
    cin = x_f32.shape[-1]
    rows = x_f32.numel() // cin
    y = torch.empty(*x_f32.shape[:-1], cpad, device=x_f32.device, dtype=dtype)
    check(lib().dm_pad_convert(_dt_code(dtype), ptr_any(x_f32), rows, cin, cpad, scale, shift,
                               ptr_any(y), stream_ptr()), "dm_pad_convert")
    return y


def cond_gather(depth, normal_u8, light_u8, view_ids_i32, env_ids_i32, cpad=64, dtype=torch.float16, out=None):
    """Resident pre-rendered maps -> ControlNet condition [B,H,W,cpad] (N1).  depth [V,H,W,1] fp32, normal [V,H,W,3] u8,
    light [V,E,H,W,18] u8 on the device; ids int32 device tensors [B]."""
    V, Hh, W = depth.shape[0], depth.shape[1], depth.shape[2]
    B = view_ids_i32.shape[0]
    assert depth.is_contiguous() and normal_u8.is_contiguous() and light_u8.is_contiguous()
    assert normal_u8.dtype == torch.uint8 and light_u8.dtype == torch.uint8 and view_ids_i32.dtype == torch.int32
    if out is None:
        out = torch.empty(B, Hh, W, cpad, device=depth.device, dtype=dtype)
    check(lib().dm_cond_gather(_dt_code(dtype), ptr_any(depth), ptr_any(normal_u8), ptr_any(light_u8), light_u8.shape[1], Hh * W,
                               ptr_any(view_ids_i32), ptr_any(env_ids_i32), B, cpad, ptr_any(out), stream_ptr()), "dm_cond_gather")
    return out


def unpad_convert(x, cout, scale=1.0):
    bf = _is_bf16(x)
    assert x.is_contiguous()
    ld = x.shape[-1]
    rows = x.numel() // ld
    y = torch.empty(*x.shape[:-1], cout, device=x.device, dtype=torch.float32)
    check(lib().dm_unpad_convert(bf, ptr_any(x), rows, ld, cout, scale, ptr_any(y), stream_ptr()), "dm_unpad_convert")
    return y


def nhwc_to_nchw_f32(x, Cc):
    bf = _is_bf16(x)
    assert x.is_contiguous()
    n, Hh, W, ld = x.shape
    y = torch.empty(n, Cc, Hh, W, device=x.device, dtype=torch.float32)
    check(lib().dm_nhwc_to_nchw_f32(bf, ptr_any(x), n, Hh * W, ld, Cc, ptr_any(y), stream_ptr()), "dm_nhwc_to_nchw_f32")
    return y


def vae_sample(moments, eps, scaling=0.18215):
    bf = _is_bf16(moments)
    n, Hh, W, ld = moments.shape
    z = torch.empty(n, 4, Hh, W, device=moments.device, dtype=torch.float32)
    check(lib().dm_vae_sample(bf, ptr_any(moments), n, Hh * W, ld, ptr_any(eps.contiguous()), scaling, ptr_any(z),
                              stream_ptr()), "dm_vae_sample")
    return z


def vae_sample_bwd(moments, eps, dz, scaling=0.18215):
    bf = _is_bf16(moments)
    n, Hh, W, ld = moments.shape
    dm = torch.empty_like(moments)
    check(lib().dm_vae_sample_bwd(bf, ptr_any(moments), n, Hh * W, ld, ptr_any(eps.contiguous()), scaling,
                                  ptr_any(dz.contiguous()), ptr_any(dm), stream_ptr()), "dm_vae_sample_bwd")
    return dm


def add_noise(z, noise, sqrt_ac, sqrt_1mac, rep=3, cpad=64, dtype=torch.float16):
    B, _, Hh, W = z.shape
    out = torch.empty(rep * B, Hh, W, cpad, device=z.device, dtype=dtype)
    check(lib().dm_add_noise(_dt_code(dtype), ptr_any(z.contiguous()), ptr_any(noise.contiguous()),
                             ptr_any(sqrt_ac.contiguous()), ptr_any(sqrt_1mac.contiguous()), B, Hh * W, cpad, rep,
                             ptr_any(out), stream_ptr()), "dm_add_noise")
    return out


def timestep_embedding(t_f32, dim=320, dtype=torch.float16):
    n = t_f32.shape[0]
    out = torch.empty(n, dim, device=t_f32.device, dtype=dtype)
    check(lib().dm_timestep_embedding(_dt_code(dtype), ptr_any(t_f32.contiguous()), n, dim,
                                      ptr_any(out), stream_ptr()), "dm_timestep_embedding")
    return out


def silu(x):
    bf = _is_bf16(x)
    assert x.is_contiguous()
    y = torch.empty_like(x)
    check(lib().dm_silu(bf, ptr_any(x), x.numel(), ptr_any(y), stream_ptr()), "dm_silu")
    return y


def silu_bwd(z, dy):
    """dy * silu'(z) on the pre-activation z.  16-bit storage only."""
    bf = _is_bf16(z)    # fp32 storage: the library returns DM_EUNSUPPORTED
    assert z.is_contiguous() and dy.is_contiguous() and dy.shape == z.shape and dy.dtype == z.dtype
    dx = torch.empty_like(z)
    check(lib().dm_silu_bwd(bf, ptr_any(z), ptr_any(dy), z.numel(), ptr_any(dx), stream_ptr()), "dm_silu_bwd")
    return dx


def rowvec_grad(dy, n_img, out=None):
    """Gradient of the GEMM / conv epilogue's per-image `rowvec`: per-image column sums of dy [n_img * rows, N] (any leading
    shape; a uniform row stride is allowed) -> [n_img, N] in the storage dtype, or into `out` (a column slice of a wider
    buffer is fine).  16-bit storage only; deterministic."""
    bf = _is_bf16(dy)
    N = dy.shape[-1]
    dy2 = dy.reshape(-1, N) if dy.is_contiguous() else _hp_rows(dy)
    assert dy2.stride(1) == 1 and dy2.shape[0] % n_img == 0
    if out is None:
        out = torch.empty(n_img, N, device=dy.device, dtype=dy.dtype)
    assert tuple(out.shape) == (n_img, N) and out.stride(1) == 1 and out.dtype == dy.dtype
    check(lib().dm_rowvec_grad(bf, ptr_any(dy2), dy2.stride(0), n_img, dy2.shape[0] // n_img, N, ptr_any(out), out.stride(0),
                               stream_ptr()), "dm_rowvec_grad")
    return out


def attention(q, k, v, heads, scale=None, out=None):
    """q [B,Nq,*], k/v [B,Nk,*] token-major views (last dim contiguous, heads*64 wide) -> [B,Nq,heads*64]."""
    bf = _is_bf16(q)
    B, Nq, Cq = q.shape
    Nk = k.shape[1]
    assert Cq == heads * 64 and k.shape[2] == Cq and v.shape[2] == Cq
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1
    assert k.stride(1) == v.stride(1) and k.stride(0) == v.stride(0)
    if out is None:
        out = torch.empty(B, Nq, Cq, device=q.device, dtype=q.dtype)
    if scale is None:
        scale = 1.0 / 8.0
    check(lib().dm_attention(bf, ptr_any(q), q.stride(1), q.stride(0), ptr_any(k), ptr_any(v), k.stride(1), k.stride(0),
                             ptr_any(out), out.stride(1), out.stride(0), B, heads, Nq, Nk, 64, scale, stream_ptr()),
          "dm_attention")
    return out


def _attn_views(q, k, v, heads):
    B, Nq, Cq = q.shape
    assert Cq == heads * 64 and k.shape[2] == Cq and v.shape[2] == Cq and k.shape[:2] == v.shape[:2] and k.shape[0] == B
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride(2) == 1
    assert k.stride(1) == v.stride(1) and k.stride(0) == v.stride(0)
    return B, Nq, k.shape[1], Cq


def attention_lse(q, k, v, heads, scale=None, out=None):
    """attention() that also returns lse [B, heads, Nq] fp32 = logsumexp_k(scale q.k) per query row, which attention_bwd
    needs; the output is bit-identical to attention()'s.  16-bit storage only."""
    bf = _is_bf16(q)    # fp32 storage: the library returns DM_EUNSUPPORTED
    B, Nq, Nk, Cq = _attn_views(q, k, v, heads)
    if out is None:
        out = torch.empty(B, Nq, Cq, device=q.device, dtype=q.dtype)
    lse = torch.empty(B, heads, Nq, device=q.device, dtype=torch.float32)
    check(lib().dm_attention_lse(bf, ptr_any(q), q.stride(1), q.stride(0), ptr_any(k), ptr_any(v), k.stride(1), k.stride(0),
                                 ptr_any(out), out.stride(1), out.stride(0), B, heads, Nq, Nk, 64,
                                 1.0 / 8.0 if scale is None else scale, ptr_any(lse), stream_ptr()), "dm_attention_lse")
    return out, lse


def attention_bwd(q, k, v, o, do, lse, heads, scale=None, dq=None, dk=None, dv=None):
    """Gradients (dq, dk, dv) of attention(q, k, v, heads, scale) = o for the output gradient do, from the lse of
    attention_lse.  Every operand may be a token-major view with its own row / batch strides (last dim contiguous), as
    attention() takes; dq / dk / dv given as column slices of one gradient buffer are written in place, its other columns
    untouched.  16-bit storage only; deterministic."""
    bf = _is_bf16(q)    # fp32 storage: the library returns DM_EUNSUPPORTED
    B, Nq, Nk, Cq = _attn_views(q, k, v, heads)
    assert o.shape == (B, Nq, Cq) and do.shape == (B, Nq, Cq) and lse.shape == (B, heads, Nq)
    assert lse.dtype == torch.float32 and lse.is_contiguous()
    if dq is None:
        dq = torch.empty(B, Nq, Cq, device=q.device, dtype=q.dtype)
    if dk is None:
        dk = torch.empty(B, Nk, Cq, device=q.device, dtype=q.dtype)
    if dv is None:
        dv = torch.empty(B, Nk, Cq, device=q.device, dtype=q.dtype)
    for t, shape in ((o, (B, Nq)), (do, (B, Nq)), (dq, (B, Nq)), (dk, (B, Nk)), (dv, (B, Nk))):
        assert t.dtype == q.dtype and t.stride(2) == 1 and tuple(t.shape) == (*shape, Cq)
    delta = torch.empty(B, heads, Nq, device=q.device, dtype=torch.float32)
    check(lib().dm_attention_bwd(bf, ptr_any(q), q.stride(1), q.stride(0), ptr_any(k), ptr_any(v), k.stride(1), k.stride(0),
                                 ptr_any(o), o.stride(1), o.stride(0), ptr_any(do), do.stride(1), do.stride(0), ptr_any(lse),
                                 ptr_any(dq), dq.stride(1), dq.stride(0), ptr_any(dk), dk.stride(1), dk.stride(0),
                                 ptr_any(dv), dv.stride(1), dv.stride(0), ptr_any(delta), B, heads, Nq, Nk, 64,
                                 1.0 / 8.0 if scale is None else scale, stream_ptr()), "dm_attention_bwd")
    return dq, dk, dv
