"""Input gradients from the forward weight (dm_conv2d_dgrad / dm_gemm_dgrad via dense_ops.conv2d_dgrad / gemm_dgrad).

The strongest check is bit-identity: the kernel runs the K order and the products of the forward kernel on a flipped,
transposed weight copy (conv) or on W^T (linear), so the results must be torch.equal to those.  Beside it: fp32 output
against float64 on the same rounded inputs (2e-5 of max|ref|, the bound of the weight gradients), and the adjoint identity
<conv2d(x, W), dy> = <x, conv2d_dgrad(dy, W)>, which pins the tap flip and the padding convention without the re-laid-out
weight."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
BOUND = 2e-5

# (name, n, H, W, Cin, Cout, ksize, forward pad).  H, W are dy's (= dx's) extents.
CONV_CASES = [
    ("320-level 3x3", 4, 32, 32, 320, 320, 3, 1),
    ("1280->640 at 8x8", 4, 8, 8, 1280, 640, 3, 1),      # dy has 640 channels, dx 1280
    ("640->1280 at 4x4 split-K", 4, 4, 4, 640, 1280, 3, 1),
    ("thin 64-padded at 256x256", 1, 256, 256, 64, 64, 3, 1),
    ("1x1 shortcut 960->640", 2, 16, 16, 960, 640, 1, 0),
    ("Cin 40", 2, 16, 16, 40, 128, 3, 1),
]
CONV_IDS = [c[0].replace(" ", "_") for c in CONV_CASES]
# (M, N_out, K_in)
LINEAR_CASES = [(4, 1280, 320), (308, 640, 1024), (1000, 320, 320), (4096, 320, 320), (2048, 10240, 1280), (77, 2560, 1024)]


def _rnd(g, *shape, dt, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dt)


def _flipped(w, Cout, Cin, k, dt):
    """the weight of the input-gradient convolution as a copy: Wd[ci, tap, co] = W[co, taps-1-tap, ci]"""
    from dreammat_b200 import dense_ops as D
    w4 = w.view(Cout, k, k, Cin).permute(0, 3, 1, 2)                     # [Cout, Cin, kh, kw]
    return D.conv_weight_to_gemm(w4.flip(2, 3).permute(1, 0, 2, 3), Cout, 0, dt).cuda()


def _conv_inputs(case, dt, seed):
    _, n, H, W, Cin, Cout, k, _ = case
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = _rnd(g, n, H, W, Cout, dt=dt)
    w = _rnd(g, Cout, k * k * Cin, dt=dt, scale=(k * k * Cout) ** -0.5)
    res = _rnd(g, n, H, W, Cin, dt=dt)
    return dy, w, res


def _plan(M, N, K):
    from dreammat_b200._cabi import check, lib
    kern, bn, split = C.c_int(), C.c_int(), C.c_int()
    check(lib().dm_gemm_plan(M, N, K, 0, 0, C.byref(kern), C.byref(bn), C.byref(split)), "dm_gemm_plan")
    return bn.value, split.value


@DTYPES
@pytest.mark.parametrize("case", CONV_CASES, ids=CONV_IDS)
def test_conv_dgrad_bit_identical_to_conv_on_flipped_weight(dt, case):
    from dreammat_b200 import dense_ops as D
    name, n, H, W, Cin, Cout, k, pad = case
    dy, w, res = _conv_inputs(case, dt, 1 + CONV_CASES.index(case))
    wd = _flipped(w, Cout, Cin, k, dt)
    pd = k - 1 - pad
    for kw_ref, kw in ((dict(), dict()), (dict(residual=res, out_scale=0.5), dict(residual=res, out_scale=0.5)),
                       (dict(out_f32=True), dict(out_f32=True))):
        ref = D.conv2d(dy, wd, k, pad=(pd, pd), out_hw=(H, W), **kw_ref)
        got = D.conv2d_dgrad(dy, w, k, pad=(pad, pad), cin=Cin, **kw)
        assert got.shape == (n, H, W, Cin) and got.dtype == ref.dtype
        assert torch.equal(got, ref), f"{name} {kw.keys()}: max|d| {(got.float() - ref.float()).abs().max().item():.3e}"
    # dx as a channel slice of a wider buffer
    wide = torch.full((n, H, W, Cin + 64), 7.0, device="cuda", dtype=dt)
    D.conv2d_dgrad(dy, w, k, pad=(pad, pad), out=wide[..., :Cin])
    assert torch.equal(wide[..., :Cin], D.conv2d(dy, wd, k, pad=(pd, pd), out_hw=(H, W))) and bool((wide[..., Cin:] == 7.0).all())
    if "split-K" in name:
        bn, split = _plan(n * H * W, Cin, k * k * Cout)
        print(f"{name}: plan BN {bn}, split {split}")
        assert split > 1


@DTYPES
@pytest.mark.parametrize("pad", [0, 1], ids=["vae_pad0", "unet_pad1"])
def test_zero_inserted_stride2_dgrad(dt, pad):
    """a stride-2 forward: zero insertion of dy, then the stride-1 input gradient; bit-identical to the copy-based path and
    equal to autograd's conv input gradient"""
    from dreammat_b200 import dense_ops as D
    n, Ho, Cin, Cout, k = 2, 16, 128, 192, 3
    g = torch.Generator(device="cuda").manual_seed(40 + pad)
    dy = _rnd(g, n, Ho, Ho, Cout, dt=dt)
    w = _rnd(g, Cout, k * k * Cin, dt=dt, scale=(k * k * Cout) ** -0.5)
    up = D.upsample2x(dy, zero_insert=True)
    pd = k - 1 - pad
    ref = D.conv2d(up, _flipped(w, Cout, Cin, k, dt), k, pad=(pd, pd), out_hw=(2 * Ho, 2 * Ho), out_f32=True)
    got = D.conv2d_dgrad(up, w, k, pad=(pad, pad), out_f32=True)
    assert torch.equal(got, ref)
    w4 = w.double().view(Cout, k, k, Cin).permute(0, 3, 1, 2)
    x = torch.zeros(n, Cin, 2 * Ho, 2 * Ho, device="cuda", dtype=torch.float64, requires_grad=True)
    xp = F.pad(x, (pad, 2, pad, 2))                                      # bottom / right: more than the conv reads
    y = F.conv2d(xp, w4, stride=2)[:, :, :Ho, :Ho]
    y.backward(dy.double().permute(0, 3, 1, 2))
    r = ((got.double() - x.grad.permute(0, 2, 3, 1)).abs().max() / x.grad.abs().max()).item()
    print(f"stride-2 pad {pad} {dt}: max|d| / max|ref| = {r:.2e}")
    assert r <= BOUND


@DTYPES
@pytest.mark.parametrize("M,N,K", LINEAR_CASES, ids=[f"M{m}_{n}to{k}" for m, n, k in LINEAR_CASES])
def test_gemm_dgrad_bit_identical_to_gemm_on_transpose(dt, M, N, K):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    dy = _rnd(g, M, N, dt=dt)
    w = _rnd(g, N, K, dt=dt, scale=N ** -0.5)
    res = _rnd(g, M, K, dt=dt)
    wt = D.transpose(w)
    for kw in (dict(), dict(residual=res), dict(out_f32=True), dict(residual=res, out_f32=True, alpha=0.5)):
        assert torch.equal(D.gemm_dgrad(dy, w, **kw), D.gemm(dy, wt, **kw)), kw
    r = ((D.gemm_dgrad(dy, w, out_f32=True).double() - dy.double() @ w.double()).abs().max() / (dy.double() @ w.double()).abs().max()).item()
    print(f"linear M{M} {N}->{K} {dt}: max|d| / max|ref| = {r:.2e}")
    assert r <= BOUND
    # dy a column slice of a fused gradient buffer with the matching rows of the fused weight; dx a column slice
    fused = _rnd(g, M, 2 * N, dt=dt)
    wide = torch.zeros(M, K + 64, device="cuda", dtype=dt)
    D.gemm_dgrad(fused[:, N:], w, out=wide[:, :K])
    assert torch.equal(wide[:, :K], D.gemm(fused[:, N:], wt)) and not wide[:, K:].any()


@DTYPES
@pytest.mark.parametrize("case", CONV_CASES, ids=CONV_IDS)
def test_conv_dgrad_fp32_output_matches_float64(dt, case):
    from dreammat_b200 import dense_ops as D
    name, n, H, W, Cin, Cout, k, pad = case
    dy, w, _ = _conv_inputs(case, dt, 50 + CONV_CASES.index(case))
    got = D.conv2d_dgrad(dy, w, k, pad=(pad, pad), out_f32=True)
    w4 = w.double().view(Cout, k, k, Cin).permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_input((n, Cin, H, W), w4, dy.double().permute(0, 3, 1, 2), padding=pad).permute(0, 2, 3, 1)
    r = ((got.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"{name} {dt}: max|d| / max|ref| = {r:.2e}")
    assert r <= BOUND


@DTYPES
@pytest.mark.parametrize("case", [CONV_CASES[0], CONV_CASES[4], CONV_CASES[5]], ids=[CONV_IDS[0], CONV_IDS[4], CONV_IDS[5]])
def test_conv_dgrad_is_adjoint_of_forward(dt, case):
    from dreammat_b200 import dense_ops as D
    name, n, H, W, Cin, Cout, k, pad = case
    dy, w, _ = _conv_inputs(case, dt, 70 + CONV_CASES.index(case))
    g = torch.Generator(device="cuda").manual_seed(99)
    cin_f = (Cin + 63) // 64 * 64                          # the forward needs 64-padded input channels
    x = torch.zeros(n, H, W, cin_f, device="cuda", dtype=dt)
    x[..., :Cin] = _rnd(g, n, H, W, Cin, dt=dt)
    wf = torch.zeros(Cout, k * k, cin_f, device="cuda", dtype=dt)
    wf[..., :Cin] = w.view(Cout, k * k, Cin)
    y = D.conv2d(x, wf.view(Cout, -1), k, pad=(pad, pad), out_f32=True)
    dx = D.conv2d_dgrad(dy, w, k, pad=(pad, pad), out_f32=True)
    lhs = (y.double() * dy.double()).sum().item()
    rhs = (x[..., :Cin].double() * dx.double()).sum().item()
    rel = abs(lhs - rhs) / abs(lhs)
    print(f"{name} {dt}: <conv(x, W), dy> = {lhs:.6e}, <x, dgrad(dy, W)> = {rhs:.6e}, rel {rel:.2e}")
    assert rel <= 1e-4


@DTYPES
def test_dgrad_deterministic_graph_replay_and_plan(dt):
    from dreammat_b200 import dense_ops as D
    case = CONV_CASES[2]
    _, n, H, W, Cin, Cout, k, pad = case
    dy, w, res = _conv_inputs(case, dt, 7)
    g = torch.Generator(device="cuda").manual_seed(8)
    ldy, lw = _rnd(g, 308, 640, dt=dt), _rnd(g, 640, 1024, dt=dt, scale=0.04)

    def run():
        return D.conv2d_dgrad(dy, w, k, pad=(pad, pad), residual=res), D.gemm_dgrad(ldy, lw)

    one, two = run(), run()
    for a, b in zip(one, two):
        assert torch.equal(a, b)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(one, captured):
        assert torch.equal(a, b)
    # the plan reported for [M, N = Cin, K = taps*Cout] is the split the call takes: with split-K switched off the result
    # of a split shape changes in the last bits, that of an unsplit shape does not
    from dreammat_b200._cabi import lib
    big = CONV_CASES[0]
    bdy, bw, _ = _conv_inputs(big, dt, 9)
    assert _plan(n * H * W, Cin, k * k * Cout)[1] > 1 and _plan(big[1] * big[2] * big[3], big[4], 9 * big[5])[1] == 1
    on = D.conv2d_dgrad(dy, w, k, out_f32=True), D.conv2d_dgrad(bdy, bw, 3, out_f32=True)
    try:
        assert lib().dm_tune_gemm(20) == 0
        off = D.conv2d_dgrad(dy, w, k, out_f32=True), D.conv2d_dgrad(bdy, bw, 3, out_f32=True)
    finally:
        lib().dm_tune_gemm(21)
    assert not torch.equal(on[0], off[0]) and torch.allclose(on[0], off[0], rtol=0, atol=BOUND * on[0].abs().max().item())
    assert torch.equal(on[1], off[1])
