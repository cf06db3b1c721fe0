"""Time of the ControlNet forward-with-tape + backward (nets.ControlNet.forward / backward) against torch autograd of
oracle.sd.controlnet_forward, and where the time goes.

Shape: the per-GPU shape of the ControlNet training step (as scripts/wgrad_shapes.py): bf16, 4 images, 32^2 latents, 256^2
condition, context 4 x 77 x 1024, conditioning_scale 1.

  1. whole step: each side (ours; torch in bf16 on the same card: cuDNN / cuBLAS / SDPA) is captured as one CUDA graph of
     forward + backward for every parameter, warmed up, and replayed in windows of --window seconds; the two alternate for
     --rounds rounds and the median and the spread over rounds are printed.  The oracle's sinusoidal timestep embedding is
     built on the host, so it is replaced by its (constant) value for the capture; everything after it is timed.
  2. per-kind breakdown of ours (forward GEMM / conv, dgrad, wgrad, attention forward, attention backward, streaming) from
     a separate torch.profiler run of one eager step.
  3. the input gradient alone, per distinct convolution shape of the backward: dense_ops.conv2d_dgrad (forward weight)
     against dense_ops.conv2d on a pre-flipped weight copy, with achieved TFLOP/s from 2 * pixels * taps * Cin * Cout.

The card's name and power limit are printed with the numbers.  There is no fallback: without a GPU the script fails.

    python scripts/controlnet_bwd.py [--window 1.0] [--rounds 5] [--json OUT.json]
"""
import argparse
import json
import os
import re
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from gemm_shapes import PEAK_TFLOPS, card  # noqa: E402
from wgrad_shapes import COND, CTX_TOKENS, IMAGES, LATENT, time_graph  # noqa: E402


def build(dev, dtype):
    from dreammat_b200 import nets, weights
    from oracle import sd as O
    cfg = weights.UNetConfig()
    w = {k: v.to(dtype) for k, v in weights.random_controlnet(cfg, dev).items()}
    net = nets.ControlNet(w, cfg, dev, dtype)
    g = torch.Generator(device=dev).manual_seed(0)
    sample = torch.zeros(IMAGES, LATENT, LATENT, 64, device=dev, dtype=dtype)
    sample[..., :cfg.in_channels] = torch.randn(IMAGES, LATENT, LATENT, cfg.in_channels, device=dev, generator=g).to(dtype)
    cond = torch.zeros(IMAGES, COND, COND, 64, device=dev, dtype=dtype)
    cond[..., :cfg.cond_channels] = torch.rand(IMAGES, COND, COND, cfg.cond_channels, device=dev, generator=g).to(dtype)
    ctx = torch.randn(IMAGES, CTX_TOKENS, cfg.cross_attention_dim, device=dev, generator=g).to(dtype)
    t = torch.full((IMAGES,), 500.0, device=dev)
    down, mid = net.forward(sample, t, ctx, cond)
    d_down = [torch.randn(d.shape, device=dev, generator=g).to(dtype) for d in down]
    d_mid = torch.randn(mid.shape, device=dev, generator=g).to(dtype)

    def ours():
        tape = {}
        net.forward(sample, t, ctx, cond, tape=tape)
        return net.backward(tape, d_down, d_mid)

    wt = {k: v.to(dev, dtype).requires_grad_() for k, v in w.items()}
    emb = O.timestep_embedding(t.cpu(), cfg.block_out_channels[0]).to(dev, dtype)
    nchw = lambda x: x.permute(0, 3, 1, 2)      # noqa: E731   NHWC storage = channels_last NCHW
    s_t, c_t = nchw(sample[..., :cfg.in_channels]), nchw(cond[..., :cfg.cond_channels])
    gt = [nchw(d) for d in d_down] + [nchw(d_mid)]

    def theirs():
        host_embedding = O.timestep_embedding
        O.timestep_embedding = lambda *_: emb
        try:
            down_t, mid_t = O.controlnet_forward(wt, cfg, s_t, t, ctx, c_t, 1.0)
        finally:
            O.timestep_embedding = host_embedding
        return torch.autograd.grad(down_t + [mid_t], list(wt.values()), gt)

    return ours, theirs


class Replay:
    """one captured call, replayed in windows of about `window` seconds"""

    def __init__(self, fn, stream, window):
        self.us1 = time_graph(fn, 1, stream)                 # also warms up and sizes the library scratch
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=stream):
            fn()
        self.n = max(3, int(window * 1e6 / self.us1))

    def ms(self):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(self.n):
            self.graph.replay()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / self.n


KINDS = [("attention backward", r"attn_(delta|dkdv|dq)_kernel"), ("attention forward", r"attention_kernel"),
         ("dgrad", r"tc_gemm_kernel<.*, *2>"), ("wgrad", r"tc_gemm_kernel<.*, *1>|bias_grad_"),
         ("forward GEMM / conv", r"tc_gemm_kernel<"), ("split-K finish (all modes)", r"splitk_finish_kernel")]


def breakdown(ours):
    from torch.profiler import ProfilerActivity, profile
    ours()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ours()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if us <= 0:
            continue
        kind = next((k for k, pat in KINDS if re.search(pat, ev.key)), "streaming (norms, SiLU, adds, zero insertion, ...)")
        o = out.setdefault(kind, [0.0, 0])
        o[0] += us / 1e3
        o[1] += ev.count
    return out


def dgrad_shapes(ours, stream, iters=20):
    from dreammat_b200 import dense_ops as D
    seen, orig = {}, D.conv2d_dgrad

    def rec(dy, w, ksize, **kw):
        seen.setdefault((tuple(dy.shape), tuple(w.shape), ksize), [dy.clone(), w, 0])[2] += 1
        return orig(dy, w, ksize, **kw)

    D.conv2d_dgrad = rec
    try:
        ours()
    finally:
        D.conv2d_dgrad = orig
    rows = []
    for (shape, wshape, k), (dy, w, calls) in seen.items():
        n, H, W, Cout = shape
        Cin = wshape[1] // (k * k)
        wd = D.conv_weight_to_gemm(w.view(Cout, k, k, Cin).permute(0, 3, 1, 2).flip(2, 3).permute(1, 0, 2, 3), Cout, 0, dy.dtype).to(dy.device)
        pd = k - 2      # forward padding 1 (3x3): the flipped convolution pads k - 1 - 1
        us = time_graph(lambda: D.conv2d_dgrad(dy, w, k), iters, stream)
        us_copy = time_graph(lambda: D.conv2d(dy, wd, k, pad=(pd, pd), out_hw=(H, W)), iters, stream)
        flops = 2.0 * n * H * W * k * k * Cin * Cout
        rows.append(dict(shape=f"dgrad{k}x{k} {n}x{H}x{W} {Cout}->{Cin}", calls=calls, us=us, us_copy=us_copy,
                         tflops=flops / us / 1e6, roof_frac=flops / us / 1e6 / PEAK_TFLOPS))
    rows.sort(key=lambda r: -r["us"] * r["calls"])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of replays per timing window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", help="also write the numbers to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("controlnet_bwd.py times kernels on the GPU; no CUDA device found")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    ours, theirs = build(dev, torch.bfloat16)
    stream = torch.cuda.Stream()
    a, b = Replay(ours, stream, args.window), Replay(theirs, stream, args.window)
    ms_a, ms_b = [], []
    for _ in range(args.rounds):
        ms_a.append(a.ms())
        ms_b.append(b.ms())
    info = card()
    print(f"# {info}")
    print(f"# ControlNet forward + backward (every parameter), bf16, {IMAGES} images, {LATENT}^2 latents, {COND}^2 condition; "
          f"CUDA-graph replay, {args.rounds} alternating rounds of {a.n} / {b.n} replays")
    med_a, med_b = statistics.median(ms_a), statistics.median(ms_b)
    print(f"ours : median {med_a:.2f} ms  (min {min(ms_a):.2f}, max {max(ms_a):.2f})")
    print(f"torch: median {med_b:.2f} ms  (min {min(ms_b):.2f}, max {max(ms_b):.2f})")
    print(f"torch / ours = {med_b / med_a:.2f}  (< 1: torch autograd is faster)")
    kinds = breakdown(ours)
    total = sum(v[0] for v in kinds.values())
    print(f"# kernel time of one eager step of ours by kind (torch.profiler, separate run): {total:.2f} ms")
    for k, (ms, cnt) in sorted(kinds.items(), key=lambda kv: -kv[1][0]):
        print(f"{k:52s} {ms:8.2f} ms {100 * ms / total:5.1f}%  {cnt:5d} launches")
    rows = dgrad_shapes(ours, stream)
    print("# conv input gradient alone: from the forward weight (ours) vs dm_conv2d on a pre-flipped copy")
    print(f"{'shape':34s} {'calls':>5s} {'us/call':>8s} {'copy us':>8s} {'copy/ours':>9s} {'TFLOP/s':>8s} {'roof':>6s}")
    for r in rows:
        print(f"{r['shape']:34s} {r['calls']:5d} {r['us']:8.1f} {r['us_copy']:8.1f} {r['us_copy'] / r['us']:9.2f} "
              f"{r['tflops']:8.1f} {100 * r['roof_frac']:5.1f}%")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, ours_ms=ms_a, torch_ms=ms_b, kinds=kinds, dgrad=rows), f, indent=1)


if __name__ == "__main__":
    main()
