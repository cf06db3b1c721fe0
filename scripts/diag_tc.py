"""GPU diagnostic for the wgmma GEMM / conv kernel: prints one line per case, never aborts early."""
import sys, os, traceback
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from dreammat_b200 import dense_ops as D

torch.manual_seed(0)
dev = "cuda"


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def case(name, fn):
    try:
        r = fn()
        torch.cuda.synchronize()
        print(f"{name:60s} rel_err={r:.3e} {'OK' if r < 2e-3 else 'BAD'}", flush=True)
    except Exception as e:
        print(f"{name:60s} EXC {type(e).__name__}: {e}", flush=True)
        traceback.print_exc()


def gemm_case(M, N, K, dtype=torch.float16, batch=0, bn=0, **ep):
    def f():
        sh = (batch,) if batch else ()
        a = (torch.randn(*sh, M, K, device=dev) * 0.5).to(dtype)
        b = (torch.randn(*(sh if ep.pop("b_batched", batch > 0) else ()), N, K, device=dev) * 0.5).to(dtype)
        kw = {}
        ref = a.float() @ b.float().transpose(-1, -2)
        if ep.get("bias"):
            kw["bias"] = torch.randn(N, device=dev).to(dtype); ref = ref + kw["bias"].float()
        if ep.get("act"):
            kw["act"] = ep["act"]; ref = F.silu(ref) if ep["act"] == "silu" else F.gelu(ref)
        if ep.get("residual"):
            kw["residual"] = torch.randn(*sh, M, N, device=dev).to(dtype); ref = ref + kw["residual"].float()
        if ep.get("out_f32"):
            kw["out_f32"] = True
        out = D.gemm(a, b, bn=bn, **kw)
        return rel(out.float(), ref)
    return f


def identity_probe():
    """A = I (128x64 block), B = random: exposes swizzle / descriptor mistakes as structured errors."""
    M, N, K = 128, 128, 64
    a = torch.zeros(M, K, device=dev, dtype=torch.float16)
    a[torch.arange(64), torch.arange(64)] = 1
    b = torch.randn(N, K, device=dev).half()
    out = D.gemm(a, b)
    ref = a.float() @ b.float().t()
    bad = (out.float() - ref).abs() > 1e-2
    print("   identity probe: bad rows", bad.any(1).nonzero().flatten()[:16].tolist(), "bad cols",
          bad.any(0).nonzero().flatten()[:16].tolist())
    return rel(out.float(), ref)


def conv_case(n, H, W, Cin, Cout, k=3, stride=1, pad=(1, 1), dtype=torch.float16, bn=0, bias=True, res=False, act=None,
              temb=False):
    def f():
        x = (torch.randn(n, H, W, Cin, device=dev) * 0.5).to(dtype)
        w = (torch.randn(Cout, Cin, k, k, device=dev) * (1.0 / (Cin * k * k) ** 0.5)).to(dtype)
        wg = D.conv_weight_to_gemm(w, dtype=dtype)
        xn = x.float().permute(0, 3, 1, 2)
        if pad == "vae":   # (0,1,0,1) asymmetric pad, stride 2
            xp = F.pad(xn, (0, 1, 0, 1)); ref = F.conv2d(xp, w.float(), stride=2); pt = (0, 0)
            Ho, Wo = ref.shape[2], ref.shape[3]
        else:
            ref = F.conv2d(xn, w.float(), stride=stride, padding=pad); pt = pad
            Ho, Wo = ref.shape[2], ref.shape[3]
        kw = {}
        if bias:
            kw["bias"] = torch.randn(Cout, device=dev).to(dtype); ref = ref + kw["bias"].float().view(1, -1, 1, 1)
        if temb:
            kw["rowvec"] = torch.randn(n, Cout, device=dev).to(dtype); ref = ref + kw["rowvec"].float().view(n, -1, 1, 1)
        if act:
            kw["act"] = act; ref = F.silu(ref)
        if res:
            kw["residual"] = torch.randn(n, Ho, Wo, Cout, device=dev).to(dtype)
            ref = ref + kw["residual"].float().permute(0, 3, 1, 2)
        out = D.conv2d(x, wg, k, stride=stride, pad=pt, out_hw=(Ho, Wo), bn=bn, **kw)
        return rel(out.float().permute(0, 3, 1, 2), ref)
    return f


case("gemm 128x128x64 identity probe", identity_probe)
case("gemm 128x128x64", gemm_case(128, 128, 64))
case("gemm 128x128x256", gemm_case(128, 128, 256))
case("gemm 256x256x512", gemm_case(256, 256, 512))
case("gemm 300x200x128 (ragged M,N)", gemm_case(300, 200, 128))
case("gemm 4096x320x320 bn=64", gemm_case(4096, 320, 320, bn=64))
case("gemm 4096x1280x320 bias+gelu", gemm_case(4096, 1280, 320, bias=True, act="gelu"))
case("gemm 1024x640x2560 bias+res", gemm_case(1024, 640, 2560, bias=True, residual=True))
case("gemm 24x1280x320 (tiny M) silu", gemm_case(24, 1280, 320, bias=True, act="silu"))
case("gemm 512x256x128 bn=256", gemm_case(512, 256, 128, bn=256))
case("gemm bf16 256x128x128", gemm_case(256, 128, 128, dtype=torch.bfloat16))
case("gemm batched 4x(256x128x64)", gemm_case(256, 128, 64, batch=4))
case("gemm batched shared-B 3x(128x64x64)", gemm_case(128, 64, 64, batch=3, b_batched=False))
case("gemm f32 out 128x4x320 (N=4)", gemm_case(128, 4, 320, out_f32=True))
case("conv3x3 s1 2x64x64 64->128", conv_case(2, 64, 64, 64, 128))
case("conv3x3 s1 1x128x128 64->64 (row segments)", conv_case(1, 128, 128, 64, 64))
case("conv3x3 s1 1x256x256 64->64 (tile_w<Wo)", conv_case(1, 256, 256, 64, 64))
case("conv3x3 s1 3x32x32 128->320 res+temb", conv_case(3, 32, 32, 128, 320, res=True, temb=True))
case("conv3x3 s1 4x8x8 128->128 (tile_n=2)", conv_case(4, 8, 8, 128, 128))
case("conv3x3 s1 3x8x8 64->64 (ragged batch)", conv_case(3, 8, 8, 64, 64))
case("conv3x3 s1 2x16x16 192->64", conv_case(2, 16, 16, 192, 64))
case("conv1x1 2x32x32 128->256", conv_case(2, 32, 32, 128, 256, k=1, pad=(0, 0)))
case("conv3x3 s2 p1 2x64x64 64->64 (unet down)", conv_case(2, 64, 64, 64, 64, stride=2))
case("conv3x3 s2 vae pad 1x128x128 64->64", conv_case(1, 128, 128, 64, 64, stride=2, pad="vae"))
case("conv3x3 s2 vae pad 1x512x512 128->128", conv_case(1, 512, 512, 128, 128, stride=2, pad="vae"))
case("conv3x3 pad(2,2) dgrad-style 1x64x64 64->64", conv_case(1, 64, 64, 64, 64, pad=(2, 2)))
case("conv3x3 bf16 1x64x64 128->128 silu", conv_case(1, 64, 64, 128, 128, dtype=torch.bfloat16, act="silu"))

# timing of a big conv and a big GEMM
def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n

try:
    x = torch.randn(8, 64, 64, 1280, device=dev).half(); w = torch.randn(1280, 9 * 1280, device=dev).half() * 0.01
    ms = timeit(lambda: D.conv2d(x, w, 3))
    print(f"conv3x3 8x64x64 1280->1280: {ms:.3f} ms  {2*8*4096*1280*1280*9/ms/1e9:.1f} TFLOP/s")
    x = torch.randn(2, 512, 512, 128, device=dev).half(); w = torch.randn(128, 9 * 128, device=dev).half() * 0.01
    ms = timeit(lambda: D.conv2d(x, w, 3))
    print(f"conv3x3 2x512x512 128->128: {ms:.3f} ms  {2*2*262144*128*128*9/ms/1e9:.1f} TFLOP/s")
    a = torch.randn(8192, 4096, device=dev).half(); b = torch.randn(4096, 4096, device=dev).half()
    ms = timeit(lambda: D.gemm(a, b))
    print(f"gemm 8192x4096x4096: {ms:.3f} ms  {2*8192*4096*4096/ms/1e9:.1f} TFLOP/s")
    ms = timeit(lambda: D.gemm(a, b, bn=256))
    print(f"gemm 8192x4096x4096 bn=256: {ms:.3f} ms  {2*8192*4096*4096/ms/1e9:.1f} TFLOP/s")
except Exception as e:
    print("timing EXC", e)
