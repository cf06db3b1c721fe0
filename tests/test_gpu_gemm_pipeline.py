"""The hand-off of accumulator tiles from the MMA warpgroups to the epilogue warpgroup of tc_gemm_kernel.

The kernel is persistent: one CTA per SM walks many output tiles, and its epilogue warpgroup stores tile i while the MMA
warpgroups already compute tile i + 1.  Both sides share one staging tile, guarded by two mbarriers.  A CTA that
overwrote the staging tile before its epilogue had read it would corrupt outputs only when a CTA owns several tiles.

So every call here is compared with the same computation cut into slices small enough that no CTA gets more than one
tile (at most DM_NUM_SMS = 132 tiles per call), where no hand-off can race.  Each output element gets the same MMA
sequence and the same epilogue either way, so the two must be bit-identical.  The whole calls are sized so that every
CTA walks at least 8 tiles, and short K (one K-block) makes the epilogue the slow side of the hand-off.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

SMS = 132          # DM_NUM_SMS: the persistent grid is min(#tiles, SMS) CTAs
BM = 128
DTYPES = pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
BNS = pytest.mark.parametrize("bn", [64, 128])


def _r(g, *shape, dt, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dt)


def _diff(a, b):
    return int((a.view(torch.int16) != b.view(torch.int16)).sum()) if a.dtype != torch.float32 else int((a != b).sum())


def _assert_same(name, whole, sliced):
    assert whole.shape == sliced.shape, name
    assert torch.equal(whole, sliced), f"{name}: {_diff(whole, sliced)} of {whole.numel()} elements differ"


@DTYPES
@BNS
@pytest.mark.parametrize("K", [64, 320, 1152])
def test_gemm_whole_matches_row_slices(dt, bn, K):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(7 + K + bn)
    N = 192                                         # ragged against the 128-wide tile, three 64-wide tiles
    n_tiles = -(-N // bn)
    m_tiles = 8 * SMS // n_tiles + 1                # >= 8 tiles for every CTA
    M = m_tiles * BM - 45                           # the last row tile is partial
    rows = BM * (SMS // n_tiles)                    # slice: at most SMS tiles, one per CTA
    a, b = _r(g, M, K, dt=dt), _r(g, N, K, dt=dt, scale=K ** -0.5)
    bias, res, rv = _r(g, N, dt=dt), _r(g, M, N, dt=dt), _r(g, m_tiles, N, dt=dt)
    bg = D.geglu_interleave(b)
    variants = {
        "plain": {}, "bias": dict(bias=bias), "rowvec": dict(rowvec=rv, rows_per_vec=BM),
        "silu": dict(bias=bias, act="silu"), "gelu": dict(bias=bias, act="gelu"), "residual": dict(residual=res),
        "geglu": dict(bias=D.geglu_interleave(bias), act="geglu"), "out_f32": dict(bias=bias, out_f32=True),
        "all": dict(bias=bias, rowvec=rv, rows_per_vec=BM, act="silu", residual=res, alpha=0.8, out_scale=1.25),
        "ldc": dict(bias=bias, residual=res),
    }
    for name, kw in variants.items():
        bb = bg if name == "geglu" else b
        n_out = N // 2 if name == "geglu" else N
        odt = torch.float32 if kw.get("out_f32") else dt

        def run(lo, hi, out):
            k = dict(kw)
            if "residual" in k:
                k["residual"] = res[lo:hi]
            if "rowvec" in k:
                k["rowvec"] = rv[lo // BM:]
            D.gemm(a[lo:hi], bb, bn=bn, out=out, **k)

        if name == "ldc":       # output into a channel slice of a wider buffer (skip concatenation)
            whole_buf = torch.full((M, N + 64), 5.0, device="cuda", dtype=dt)
            sliced_buf = whole_buf.clone()
            whole, sliced = whole_buf[:, 16:16 + N], sliced_buf[:, 16:16 + N]
        else:
            whole = torch.empty(M, n_out, device="cuda", dtype=odt)
            sliced = torch.empty(M, n_out, device="cuda", dtype=odt)
            whole_buf, sliced_buf = whole, sliced
        run(0, M, whole)
        for lo in range(0, M, rows):
            run(lo, min(M, lo + rows), sliced[lo:lo + rows])
        _assert_same(f"{name} {tuple(a.shape)}x{N} bn{bn}", whole_buf, sliced_buf)


def _conv_case(dt, bn, stride, ep, g):
    """(whole, sliced) outputs of a 3x3 conv, pad 1, at a VAE-level shape: 8 images of 128x128 output pixels, 128 -> 128
    channels.  Slices are 64 output rows of one image (a zero-padded band of input rows), 64 or 128 tiles each."""
    from dreammat_b200 import dense_ops as D
    n, Ho, Wo, C = 8, 128, 128, 128
    H = Ho * stride
    x = _r(g, n, H, H, C, dt=dt)
    w = _r(g, C, 9 * C, dt=dt, scale=(9 * C) ** -0.5)
    kw = {}
    if ep in ("bias_residual", "all"):
        kw["bias"], kw["residual"] = _r(g, C, dt=dt), _r(g, n, Ho, Wo, C, dt=dt)
    if ep == "all":
        kw.update(rowvec=_r(g, n, C, dt=dt), act="silu", out_scale=0.5)
    whole = D.conv2d(x, w, 3, stride=stride, pad=(1, 1), bn=bn, **kw)
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, 1, 1))     # the top / bottom zero rows, explicit
    band = 64
    sliced = torch.empty_like(whole)
    for i in range(n):
        for r0 in range(0, Ho, band):
            k = dict(kw)
            if "residual" in k:
                k["residual"] = kw["residual"][i, r0:r0 + band].unsqueeze(0)
            if "rowvec" in k:
                k["rowvec"] = kw["rowvec"][i:i + 1]
            xs = xp[i:i + 1, stride * r0:stride * (r0 + band) + 3 - stride]
            sliced[i:i + 1, r0:r0 + band] = D.conv2d(xs, w, 3, stride=stride, pad=(0, 1), out_hw=(band, Wo), bn=bn, **k)
    return whole, sliced


@DTYPES
@BNS
@pytest.mark.parametrize("stride", [1, 2])
def test_conv_whole_matches_row_slices(dt, bn, stride):
    g = torch.Generator(device="cuda").manual_seed(11 + stride + bn)
    for ep in ("plain", "bias_residual", "all"):
        whole, sliced = _conv_case(dt, bn, stride, ep, g)
        _assert_same(f"conv3x3 s{stride} {ep} bn{bn}", whole, sliced)


@DTYPES
@BNS
def test_consecutive_calls_identical(dt, bn):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(3)
    M, N, K = 8 * SMS * BM, 256, 64
    a, b = _r(g, M, K, dt=dt), _r(g, N, K, dt=dt, scale=K ** -0.5)
    bias, res = _r(g, N, dt=dt), _r(g, M, N, dt=dt)
    one, two = (D.gemm(a, b, bias=bias, residual=res, act="gelu", bn=bn) for _ in range(2))
    _assert_same(f"gemm {M}x{N}x{K} twice bn{bn}", one, two)
    x, w = _r(g, 8, 128, 128, 128, dt=dt), _r(g, 128, 9 * 128, dt=dt, scale=(9 * 128) ** -0.5)
    one, two = (D.conv2d(x, w, 3, bias=bias[:128], act="silu", bn=bn) for _ in range(2))
    _assert_same(f"conv3x3 8x128x128 128->128 twice bn{bn}", one, two)
