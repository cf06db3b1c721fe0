"""The TMA epilogue of tc_gemm_kernel against its per-thread path.

A 16-bit output whose base and row pitch are multiples of 16 bytes leaves the kernel as whole 128 x 32 boxes: the
residual tile comes into shared memory by TMA, the epilogue threads combine it in place, and one thread stores the boxes
(clipped to [M, N] by the tensor map).  An output whose row pitch is not a multiple of 8 elements cannot be addressed by
TMA, so the same call then runs the per-thread path, which loads the residual and stores the output from each thread.
Both apply the same per-element expression in the same order, so every case here must be bit-identical between them.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

BM = 128
DTYPES = pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
BNS = pytest.mark.parametrize("bn", [64, 128])


def _r(g, *shape, dt, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dt)


def _pair(shape, dt, pad_tma=0):
    """(TMA-addressable output, output with an odd row pitch): same logical shape, both prefilled with 5."""
    *lead, n = shape
    tma = torch.full((*lead, n + pad_tma), 5.0, device="cuda", dtype=dt)[..., :n]
    slow = torch.full((*lead, n + 1), 5.0, device="cuda", dtype=dt)[..., :n]
    return tma, slow


def _assert_same(name, tma, slow):
    assert tma.shape == slow.shape, name
    if not torch.equal(tma, slow):
        bad = int((tma.view(torch.int16) != slow.view(torch.int16)).sum())
        raise AssertionError(f"{name}: {bad} of {tma.numel()} elements differ")


def _variants(g, M, N, dt, bias_n):
    bias, rv, res = _r(g, bias_n, dt=dt), _r(g, -(-M // 96), N, dt=dt), _r(g, M, N, dt=dt)
    return {
        "plain": {}, "bias": dict(bias=bias), "rowvec": dict(rowvec=rv, rows_per_vec=96),
        "residual": dict(residual=res), "silu": dict(bias=bias, act="silu"), "gelu": dict(bias=bias, act="gelu"),
        "scale": dict(bias=bias, alpha=0.8, out_scale=1.25),
        "all_silu": dict(bias=bias, rowvec=rv, rows_per_vec=96, act="silu", residual=res, alpha=0.8, out_scale=1.25),
        "all_gelu": dict(bias=bias, rowvec=rv, rows_per_vec=96, act="gelu", residual=res, alpha=1.1, out_scale=0.5),
    }


@DTYPES
@BNS
@pytest.mark.parametrize("M,N,K", [(8 * 132 * BM, 256, 64), (3000, 200, 320), (777, 40, 128)],
                         ids=["many_tiles", "ragged", "narrow"])
def test_gemm_epilogues_tma_matches_per_thread(dt, bn, M, N, K):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(M + N + K + bn)
    a, b = _r(g, M, K, dt=dt), _r(g, N, K, dt=dt, scale=K ** -0.5)
    for name, kw in _variants(g, M, N, dt, N).items():
        tma, slow = _pair((M, N), dt)
        D.gemm(a, b, bn=bn, out=tma, **kw)
        D.gemm(a, b, bn=bn, out=slow, **kw)
        _assert_same(f"{name} {M}x{N}x{K} bn{bn}", tma, slow)


@DTYPES
@BNS
@pytest.mark.parametrize("M,N", [(4 * 132 * BM, 512), (1000, 192)], ids=["many_tiles", "ragged"])
def test_geglu_tma_matches_per_thread(dt, bn, M, N):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(5 + M + bn)
    K = 320
    a, w, bias = _r(g, M, K, dt=dt), _r(g, N, K, dt=dt, scale=K ** -0.5), _r(g, N, dt=dt)
    wi, bi = D.geglu_interleave(w), D.geglu_interleave(bias)
    for name, kw in {"geglu": dict(bias=bi), "geglu_scale": dict(bias=bi, alpha=0.9, out_scale=1.5),
                     "geglu_nobias": {}}.items():
        tma, slow = _pair((M, N // 2), dt)
        D.gemm(a, wi, bn=bn, out=tma, act="geglu", **kw)
        D.gemm(a, wi, bn=bn, out=slow, act="geglu", **kw)
        _assert_same(f"{name} {M}x{N} bn{bn}", tma, slow)


@DTYPES
@BNS
def test_batched_tma_matches_per_thread(dt, bn):
    """Per-batch B: the output and residual maps are 3-D, and ragged M must not spill into the next batch."""
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(17 + bn)
    Z, M, N, K = 3, 1000, 200, 192
    a, b = _r(g, Z, M, K, dt=dt), _r(g, Z, N, K, dt=dt, scale=K ** -0.5)
    bias, res = _r(g, N, dt=dt), _r(g, Z, M, N, dt=dt)
    for name, kw in {"plain": {}, "bias_residual_gelu": dict(bias=bias, residual=res, act="gelu", out_scale=0.75)}.items():
        tma, slow = _pair((Z, M, N), dt)
        D.gemm(a, b, bn=bn, out=tma, **kw)
        D.gemm(a, b, bn=bn, out=slow, **kw)
        _assert_same(f"batched {name} bn{bn}", tma, slow)


@DTYPES
@BNS
def test_channel_slice_tma_matches_per_thread(dt, bn):
    """Output into channels [16, 16 + N) of a wider buffer: the box stores clip at N and leave the other channels."""
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(23 + bn)
    M, N, K = 2000, 136, 128
    a, b = _r(g, M, K, dt=dt), _r(g, N, K, dt=dt, scale=K ** -0.5)
    bias, res = _r(g, N, dt=dt), _r(g, M, N, dt=dt)
    buf_tma = torch.full((M, N + 64), 5.0, device="cuda", dtype=dt)
    buf_slow = torch.full((M, N + 63), 5.0, device="cuda", dtype=dt)
    D.gemm(a, b, bn=bn, out=buf_tma[:, 16:16 + N], bias=bias, residual=res)
    D.gemm(a, b, bn=bn, out=buf_slow[:, 16:16 + N], bias=bias, residual=res)
    _assert_same(f"channel slice bn{bn}", buf_tma[:, 16:16 + N], buf_slow[:, 16:16 + N])
    assert bool((buf_tma[:, :16] == 5.0).all()) and bool((buf_tma[:, 16 + N:] == 5.0).all()), "stores left the slice"


@DTYPES
@BNS
def test_conv_tma_matches_per_thread(dt, bn):
    """3x3 convolution with bias, per-image vector, SiLU and residual: the tile's 128 pixels are 128 consecutive rows."""
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(29 + bn)
    n, H, C, Co = 4, 32, 128, 192
    x, w = _r(g, n, H, H, C, dt=dt), _r(g, Co, 9 * C, dt=dt, scale=(9 * C) ** -0.5)
    kw = dict(bias=_r(g, Co, dt=dt), rowvec=_r(g, n, Co, dt=dt), act="silu", residual=_r(g, n, H, H, Co, dt=dt),
              out_scale=0.5)
    tma, slow = _pair((n, H, H, Co), dt)
    D.conv2d(x, w, 3, bn=bn, out=tma, **kw)
    D.conv2d(x, w, 3, bn=bn, out=slow, **kw)
    _assert_same(f"conv3x3 {n}x{H}x{H} {C}->{Co} bn{bn}", tma, slow)
