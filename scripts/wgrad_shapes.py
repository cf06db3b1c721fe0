"""Per-shape time of the weight gradients (dm_conv2d_wgrad / dm_gemm_wgrad) of the ControlNet training step, against
torch's own weight gradient of the same layers.

Builds nets.ControlNet from weights.random_controlnet at the per-GPU shape of the ControlNet training step
(diffusers_train_controlnet.py, global batch 32 on 8 GPUs): bf16, 4 images, 32^2 latents, 256^2 condition, context
4 x 77 x 1024, one branch.  One forward runs with dense_ops.conv2d and dense_ops.gemm wrapped, recording every weight
layer: each conv2d, and each gemm whose B is a 2-D weight (batched-B products have no weight).  Identical layers are
merged.  For each, the weight (and bias) gradient that layer needs in the backward is computed from a random output
gradient:

    ours   dense_ops.conv2d_wgrad / gemm_wgrad on the NHWC / token-major buffers
    torch  autograd of F.conv2d (bf16, channels_last) / F.linear restricted to the weight and bias, on the same
           (channel-padded) shapes

Each side is replayed alone as a CUDA graph of --iters calls and timed with CUDA events after a warm-up.  One row per
shape: time, TFLOP/s, the fraction of the H100 SXM data-sheet bf16 roof (989 TFLOP/s dense, 3.35 TB/s HBM3; whichever
bounds the shape), the ratio torch / ours (> 1: ours is faster) and our plan (dm_gemm_plan: tile width BN, split-K).
The per-step totals follow, with the card's name and power limit.

    python scripts/wgrad_shapes.py [--iters 20] [--json OUT.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from gemm_shapes import PEAK_GBS, PEAK_TFLOPS, _key, card, plan  # noqa: E402

IMAGES, LATENT, COND, CTX_TOKENS = 4, 32, 256, 77


class Recorder:
    """wraps dense_ops.conv2d / gemm: every weight layer of the forward, merged by shape"""

    def __init__(self):
        self.rows = {}

    def wrap(self, D):
        orig = {"gemm": D.gemm, "conv2d": D.conv2d}

        def conv2d(x, w, ksize, **kw):
            stride, pad, out_hw = kw.get("stride", 1), kw.get("pad", (1, 1)), kw.get("out_hw")
            self._add(("conv", _key((x, w, ksize), dict(stride=stride, pad=pad, out_hw=out_hw))),
                      lambda: dict(kind="conv", x=x, Cout=w.shape[0], ksize=ksize, stride=stride, pad=pad, out_hw=out_hw))
            return orig["conv2d"](x, w, ksize, **kw)

        def gemm(a, b, **kw):
            if b.dim() == 2:
                self._add(("gemm", _key((a, b), {})), lambda: dict(kind="gemm", x=a.reshape(-1, a.shape[-1]), N=b.shape[0]))
            return orig["gemm"](a, b, **kw)

        D.conv2d, D.gemm = conv2d, gemm
        return orig

    def _add(self, key, make):
        r = self.rows.get(key)
        if r is None:
            r = self.rows[key] = dict(make(), calls=0)
            r["x"] = r["x"].clone()       # the forward may reuse the buffer
        r["calls"] += 1


def controlnet_forward(dev, dtype):
    from dreammat_b200 import nets, weights
    cfg = weights.UNetConfig()
    net = nets.ControlNet(weights.random_controlnet(cfg, dev), cfg, dev, dtype)
    g = torch.Generator(device=dev).manual_seed(0)
    sample = torch.zeros(IMAGES, LATENT, LATENT, 64, device=dev, dtype=dtype)
    sample[..., :cfg.in_channels] = torch.randn(IMAGES, LATENT, LATENT, cfg.in_channels, device=dev, generator=g).to(dtype)
    cond = torch.zeros(IMAGES, COND, COND, 64, device=dev, dtype=dtype)
    cond[..., :cfg.cond_channels] = torch.rand(IMAGES, COND, COND, cfg.cond_channels, device=dev, generator=g).to(dtype)
    ctx = torch.randn(IMAGES, CTX_TOKENS, cfg.cross_attention_dim, device=dev, generator=g).to(dtype)
    t = torch.full((IMAGES,), 500.0, device=dev)
    net.forward(sample, t, ctx, cond)
    torch.cuda.synchronize()


def describe(r, g):
    """our call, torch's call and the shape's work for one recorded layer"""
    from dreammat_b200 import dense_ops as D
    x, dev = r["x"], r["x"].device
    if r["kind"] == "conv":
        n, H, W, Cin = x.shape
        k, s, pad, Cout = r["ksize"], r["stride"], r["pad"], r["Cout"]
        Ho, Wo = D._conv_out_hw(H, W, k, s, pad, r["out_hw"])
        dy = torch.randn(n, Ho, Wo, Cout, device=dev, generator=g).to(x.dtype)
        P, Nw = n * Ho * Wo, k * k * Cin
        ours = lambda: D.conv2d_wgrad(x, dy, k, stride=s, pad=pad, out_hw=r["out_hw"], bias=True)  # noqa: E731
        pt, pl = pad
        pb, pr = (Ho - 1) * s + k - pt - H, (Wo - 1) * s + k - pl - W
        xt = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb)).contiguous(memory_format=torch.channels_last)
        wt = torch.randn(Cout, Cin, k, k, device=dev, generator=g).to(x.dtype).contiguous(memory_format=torch.channels_last)
        dyt = dy.permute(0, 3, 1, 2)                                  # NHWC storage = channels_last NCHW
        fwd = lambda w, b: F.conv2d(xt, w, b, stride=s)               # noqa: E731
        shape = f"conv{k}x{k}s{s} {n}x{H}x{W} {Cin}->{Cout}"
    else:
        M, Nw = x.shape
        K, Cout = Nw, r["N"]
        dy = torch.randn(M, Cout, device=dev, generator=g).to(x.dtype)
        P = M
        ours = lambda: D.gemm_wgrad(dy, x, bias=True)                 # noqa: E731
        wt = torch.randn(Cout, K, device=dev, generator=g).to(x.dtype)
        dyt = dy
        fwd = lambda w, b: F.linear(x, w, b)                          # noqa: E731
        shape = f"linear {M}x{K} -> {Cout}"
    bn, split = plan(Cout, Nw, -(-P // 64) * 64, 0, 0)
    flops = 2.0 * Cout * Nw * P
    byts = (x.numel() + dy.numel()) * x.element_size() + (Cout * Nw + Cout) * 4
    return dict(shape=shape, calls=r["calls"], flops=flops, bytes=byts, bn=bn, split=split, ours=ours,
                torch=(fwd, wt, torch.zeros(Cout, device=dev, dtype=x.dtype), dyt))


def time_graph(fn, iters, stream, warmup=3):
    stream.wait_stream(torch.cuda.current_stream())     # inputs were made on the default stream
    with torch.cuda.stream(stream):
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        for _ in range(iters):
            fn()
    g.replay()                       # first replay uploads the graph
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters      # us per call


def torch_wgrad(fwd, w, b, dy, stream):
    """autograd of the layer restricted to its weight and bias: the forward runs once (on the capture stream, where
    autograd then runs the backward) and each call is torch.autograd.grad of it"""
    w, b = w.requires_grad_(True), b.requires_grad_(True)
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        y = fwd(w, b)
    return lambda: torch.autograd.grad(y, (w, b), dy, retain_graph=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", help="also write the rows to this file")
    args = ap.parse_args()
    assert args.iters >= 20, "at least 20 launches per shape"
    if not torch.cuda.is_available():
        sys.exit("wgrad_shapes.py times kernels on the GPU; no CUDA device found")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    from dreammat_b200 import dense_ops as D
    dtype = torch.bfloat16
    rec = Recorder()
    orig = rec.wrap(D)
    try:
        controlnet_forward(dev, dtype)
    finally:
        D.gemm, D.conv2d = orig["gemm"], orig["conv2d"]
    g = torch.Generator(device=dev).manual_seed(1)
    stream = torch.cuda.Stream()
    rows = []
    for r in rec.rows.values():
        d = describe(r, g)
        d["us"] = time_graph(d.pop("ours"), args.iters, stream)
        d["us_torch"] = time_graph(torch_wgrad(*d.pop("torch"), stream), args.iters, stream)
        d["tflops"] = d["flops"] / (d["us"] * 1e-6) / 1e12
        t_mma, t_hbm = d["flops"] / (PEAK_TFLOPS * 1e12), d["bytes"] / (PEAK_GBS * 1e9)
        d["bound"] = "mma" if t_mma >= t_hbm else "hbm"
        d["roof_frac"] = max(t_mma, t_hbm) / (d["us"] * 1e-6)
        d["vs_torch"] = d["us_torch"] / d["us"]
        rows.append(d)
    rows.sort(key=lambda d: -d["us"] * d["calls"])
    total = sum(d["us"] * d["calls"] for d in rows) / 1e3
    total_torch = sum(d["us_torch"] * d["calls"] for d in rows) / 1e3
    info = card()
    print(f"# {info}")
    print(f"# ControlNet weight gradients, bf16, {IMAGES} images, {LATENT}^2 latents, {COND}^2 condition, context "
          f"{IMAGES}x{CTX_TOKENS}x1024; {len(rows)} shapes, {sum(d['calls'] for d in rows)} layers; CUDA-graph replay of "
          f"{args.iters} calls per shape")
    print(f"{'shape':34s} {'calls':>5s} {'us/call':>8s} {'TFLOP/s':>8s} {'bound':>5s} {'roof':>6s} {'torch us':>9s} "
          f"{'torch/ours':>10s} {'BN':>3s} {'spl':>3s}")
    for d in rows:
        print(f"{d['shape']:34s} {d['calls']:5d} {d['us']:8.1f} {d['tflops']:8.1f} {d['bound']:>5s} "
              f"{100 * d['roof_frac']:5.1f}% {d['us_torch']:9.1f} {d['vs_torch']:10.2f} {d['bn']:3d} {d['split']:3d}")
    print(f"# per step: ours {total:.3f} ms, torch {total_torch:.3f} ms (torch / ours = {total_torch / total:.2f})")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "iters": args.iters, "total_ms": total, "total_ms_torch": total_torch, "rows": rows},
                      f, indent=1)


if __name__ == "__main__":
    main()
