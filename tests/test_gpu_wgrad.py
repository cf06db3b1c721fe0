"""Weight gradients of the tensor-core kernel (dm_conv2d_wgrad / dm_gemm_wgrad via dense_ops.conv2d_wgrad / gemm_wgrad).

Inputs are random values rounded to fp16 / bf16, and the references are float64 on those same rounded values, so what is
left is the kernel's fp32 accumulation.  Bound: max|dW - ref| <= 2e-5 * max|ref| (and the same for db), the bound the
fp32-mode GEMM is held to, since both are the same wgmma fp32 accumulation.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
BOUND = 2e-5

# (name, n, H, W, Cin, Cout, ksize, stride, pad, out_hw, dy channel width)
CONV_CASES = [
    ("320-level 3x3", 4, 32, 32, 320, 320, 3, 1, (1, 1), None, 320),
    ("long reduction 3x3", 1, 128, 128, 64, 64, 3, 1, (1, 1), None, 64),
    ("downsampler s2 p1", 2, 32, 32, 128, 192, 3, 2, (1, 1), None, 192),
    ("vae downsampler s2 p0", 1, 64, 64, 128, 128, 3, 2, (0, 0), (32, 32), 128),
    ("1x1", 2, 16, 16, 640, 1280, 1, 1, (0, 0), None, 1280),
    ("lowest level 4x4", 4, 4, 4, 1280, 1280, 3, 1, (1, 1), None, 1280),
    ("Cout 40 of a 64-wide dy", 2, 16, 16, 64, 40, 3, 1, (1, 1), None, 64),
]
CONV_IDS = [c[0].replace(" ", "_") for c in CONV_CASES]
ADJOINT = ["downsampler s2 p1", "vae downsampler s2 p0", "Cout 40 of a 64-wide dy"]


def _rnd(g, *shape, dt):
    return torch.randn(*shape, device="cuda", generator=g).to(dt)


def _ratio(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def _check(name, got, ref):
    r = _ratio(got, ref)
    print(f"{name}: max|d| / max|ref| = {r:.2e}")
    assert r <= BOUND, f"{name}: {r:.2e} > {BOUND:.0e}"


def _conv_inputs(case, dt, seed):
    _, n, H, W, Cin, Cout, k, s, pad, out_hw, ld = case
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = _rnd(g, n, H, W, Cin, dt=dt)
    if Cout == 40:
        x[..., 48:] = 0                     # zero-padded input channels, as a padded first layer has them
    Ho, Wo = D._conv_out_hw(H, W, k, s, pad, out_hw)
    dy = _rnd(g, n, Ho, Wo, ld, dt=dt)[..., :Cout]
    return x, dy, (Ho, Wo)


def _conv_ref(x, dy, k, s, pad, Ho, Wo):
    """float64 dW [Cout, k*k*Cin] (tap-major, channel-minor) and db [Cout]"""
    n, H, W, Cin = x.shape
    pt, pl = pad
    pb, pr = (Ho - 1) * s + k - pt - H, (Wo - 1) * s + k - pl - W        # negative: rows / cols the conv never reads
    xp = F.pad(x.double().permute(0, 3, 1, 2), (pl, pr, pt, pb))
    g = dy.double().permute(0, 3, 1, 2)
    dw = torch.nn.grad.conv2d_weight(xp, (dy.shape[3], Cin, k, k), g, stride=s)
    return dw.permute(0, 2, 3, 1).reshape(dy.shape[3], k * k * Cin), g.sum((0, 2, 3))


def _plan(M, N, K):
    from dreammat_b200._cabi import check, lib
    kern, bn, split = C.c_int(), C.c_int(), C.c_int()
    check(lib().dm_gemm_plan(M, N, K, 0, 0, C.byref(kern), C.byref(bn), C.byref(split)), "dm_gemm_plan")
    return bn.value, split.value


@DTYPES
@pytest.mark.parametrize("case", CONV_CASES, ids=CONV_IDS)
def test_conv_wgrad_matches_float64(dt, case):
    from dreammat_b200 import dense_ops as D
    name, n, H, W, Cin, Cout, k, s, pad, out_hw, _ = case
    x, dy, (Ho, Wo) = _conv_inputs(case, dt, 1 + CONV_CASES.index(case))
    dw, db = D.conv2d_wgrad(x, dy, k, stride=s, pad=pad, out_hw=out_hw, bias=True)
    ref_w, ref_b = _conv_ref(x, dy, k, s, pad, Ho, Wo)
    assert dw.shape == (Cout, k * k * Cin) and dw.dtype == torch.float32 and db.shape == (Cout,)
    _check(f"{name} {dt} dW", dw, ref_w)
    _check(f"{name} {dt} db", db, ref_b)
    if name == "long reduction 3x3":
        bn, split = _plan(Cout, k * k * Cin, -(-n * Ho * Wo // 64) * 64)
        print(f"{name}: plan BN {bn}, split {split}")
        assert split > 1


@DTYPES
@pytest.mark.parametrize("case", [c for c in CONV_CASES if c[0] in ADJOINT], ids=[c.replace(" ", "_") for c in ADJOINT])
def test_conv_wgrad_is_adjoint_of_forward(dt, case):
    """<dW, W'> = <dY, conv2d(x, W')> with W' = dW itself rounded to the storage dtype: pins dW's layout to the one
    dm_conv2d consumes (a permuted tap or channel order keeps the left side and moves the right side by O(1))."""
    from dreammat_b200 import dense_ops as D
    name, n, H, W, Cin, Cout, k, s, pad, out_hw, _ = case
    x, dy, _ = _conv_inputs(case, dt, 100 + CONV_CASES.index(case))
    dw, _ = D.conv2d_wgrad(x, dy, k, stride=s, pad=pad, out_hw=out_hw)
    w2 = dw.to(dt).contiguous()
    y = D.conv2d(x, w2, k, stride=s, pad=pad, out_hw=out_hw, out_f32=True)
    lhs = (dw.double() * w2.double()).sum().item()
    rhs = (dy.double() * y.double()).sum().item()
    rel = abs(lhs - rhs) / abs(lhs)
    print(f"{name} {dt}: <dW, W'> = {lhs:.6e}, <dY, conv(x, W')> = {rhs:.6e}, rel {rel:.2e}")
    assert rel <= 1e-4


@DTYPES
@pytest.mark.parametrize("M", [4, 308, 1000, 4096])
@pytest.mark.parametrize("N,K,ld", [(320, 1280, 320), (640, 1024, 640), (2560, 320, 2560), (40, 320, 64)],
                         ids=["ff.net.2", "fused_kv", "geglu_proj", "N40_of_64"])
def test_gemm_wgrad_matches_float64(dt, M, N, K, ld):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    x = _rnd(g, M, K, dt=dt)
    dy = _rnd(g, M, ld, dt=dt)[:, :N]
    dw, db = D.gemm_wgrad(dy, x, bias=True)
    assert dw.shape == (N, K) and db.shape == (N,)
    _check(f"linear M{M} {N}x{K} {dt} dW", dw, dy.double().T @ x.double())
    _check(f"linear M{M} {N}x{K} {dt} db", db, dy.double().sum(0))


@DTYPES
def test_wgrad_deterministic_and_graph_replay(dt):
    from dreammat_b200 import dense_ops as D
    case = CONV_CASES[2]
    _, n, H, W, Cin, Cout, k, s, pad, out_hw, _ = case
    x, dy, _ = _conv_inputs(case, dt, 7)
    g = torch.Generator(device="cuda").manual_seed(8)
    lx, ldy = _rnd(g, 308, 1024, dt=dt), _rnd(g, 308, 640, dt=dt)

    def run():
        return (*D.conv2d_wgrad(x, dy, k, stride=s, pad=pad, bias=True), *D.gemm_wgrad(ldy, lx, bias=True))

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


@DTYPES
def test_wgrad_split_k_off_matches_on(dt):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200._cabi import lib
    g = torch.Generator(device="cuda").manual_seed(21)
    x, dy = _rnd(g, 1, 64, 64, 64, dt=dt), _rnd(g, 1, 64, 64, 64, dt=dt)
    lx, ldy = _rnd(g, 8192, 64, dt=dt), _rnd(g, 8192, 64, dt=dt)
    D._ensure_workspace()
    assert _plan(64, 576, 4096)[1] > 1 and _plan(64, 64, 8192)[1] > 1
    on = (*D.conv2d_wgrad(x, dy, 3, bias=True), *D.gemm_wgrad(ldy, lx, bias=True))
    try:
        assert lib().dm_tune_gemm(20) == 0
        off = (*D.conv2d_wgrad(x, dy, 3, bias=True), *D.gemm_wgrad(ldy, lx, bias=True))
    finally:
        lib().dm_tune_gemm(21)
    for name, a, b in zip(("conv dW", "conv db", "linear dW", "linear db"), on, off):
        _check(f"split on vs off {name} {dt}", a, b.double())
