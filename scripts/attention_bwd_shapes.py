"""Per-shape time of the fused attention backward (dm_attention_bwd) and of the lse forward (dm_attention_lse, against
dm_attention) at the attention shapes of the ControlNet training step, against torch's SDPA backward.

Per-GPU shapes of the training step (diffusers_train_controlnet.py, global batch 32 on 8 GPUs): bf16, 4 images, 32^2
latents, context 4 x 77 x 1024.  Self-attention runs over 1024 tokens x 5 heads, 256 x 10, 64 x 20 and 16 x 20;
cross-attention over the same query counts x 77 text tokens.  The 4096-token level (64^2 latents, 5 heads) is timed too.
q / k / v / O / dO are token-major [B, N, heads*64]; self-attention's q / k / v are column slices of one [B, N, 3C]
buffer and its gradients are written into one [B, N, 3C] buffer, as the transformer block holds them.

    ours        dense_ops.attention_bwd (delta, dK/dV and dQ kernels), and attention_lse vs attention
    torch       autograd of F.scaled_dot_product_attention on [B, heads, N, 64] views of the same buffers; the backend
                torch picked is named from the kernels a profiled call launched

Each side is replayed alone as a CUDA graph of --iters calls and timed with CUDA events after a warm-up.  TFLOP/s counts
the four algorithmic products of the backward, 8 * Nq * Nk * 64 flops per (batch, head) (dV, dP, dQ, dK; the S that the
backward recomputes is not counted, nor our second S and dP), and the forward's two, 4 * Nq * Nk * 64.  The roof share
is against the H100 SXM data-sheet bf16 rate (989 TFLOP/s dense); the card's name and power limit are printed with it.

    python scripts/attention_bwd_shapes.py [--iters 20] [--json OUT.json]
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

from gemm_shapes import PEAK_TFLOPS, card  # noqa: E402
from wgrad_shapes import time_graph  # noqa: E402

IMAGES, CTX_TOKENS = 4, 77
SHAPES = [  # (kind, tokens, heads); the 4096-token level last
    ("self", 1024, 5), ("self", 256, 10), ("self", 64, 20), ("self", 16, 20),
    ("cross", 1024, 5), ("cross", 256, 10), ("cross", 64, 20), ("cross", 16, 20),
    ("self", 4096, 5), ("cross", 4096, 5),
]


def make(kind, N, heads, g, dt=torch.bfloat16):
    Cc = heads * 64
    r = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)  # noqa: E731
    if kind == "self":
        qkv = r(IMAGES, N, 3 * Cc)
        q, k, v = qkv[..., :Cc], qkv[..., Cc:2 * Cc], qkv[..., 2 * Cc:]
        d_qkv = torch.empty_like(qkv)
        grads = dict(dq=d_qkv[..., :Cc], dk=d_qkv[..., Cc:2 * Cc], dv=d_qkv[..., 2 * Cc:])
        Nk = N
    else:
        kv = r(IMAGES, CTX_TOKENS, 2 * Cc)
        q, k, v = r(IMAGES, N, Cc), kv[..., :Cc], kv[..., Cc:]
        d_kv = torch.empty_like(kv)
        grads = dict(dk=d_kv[..., :Cc], dv=d_kv[..., Cc:])
        Nk = CTX_TOKENS
    return q, k, v, r(IMAGES, N, Cc), grads, Nk


def torch_bwd(q, k, v, do, heads, stream):
    sp = lambda t: t.unflatten(-1, (heads, 64)).transpose(1, 2)  # noqa: E731
    qt, kt, vt = (sp(t.detach()).requires_grad_(True) for t in (q, k, v))
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        o = F.scaled_dot_product_attention(qt, kt, vt)
    dot = sp(do)
    return lambda: torch.autograd.grad(o, (qt, kt, vt), dot, retain_graph=True)


def backend_of(fn):
    """names the SDPA backward backend from the CUDA kernels one call launches"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = " ".join(e.name.lower() for e in prof.events())
    for tag, label in (("cudnn", "cudnn"), ("flash", "flash"), ("fmha", "mem-efficient"), ("efficient", "mem-efficient")):
        if tag in names:
            return label
    return "math"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", help="also write the rows to this file")
    args = ap.parse_args()
    assert args.iters >= 20, "at least 20 launches per shape"
    if not torch.cuda.is_available():
        sys.exit("attention_bwd_shapes.py times kernels on the GPU; no CUDA device found")
    torch.cuda.set_device(0)
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(0)
    stream = torch.cuda.Stream()
    rows = []
    for kind, N, heads in SHAPES:
        q, k, v, do, grads, Nk = make(kind, N, heads, g)
        o, lse = D.attention_lse(q, k, v, heads)
        flops_bwd = 8.0 * IMAGES * heads * N * Nk * 64
        flops_fwd = 4.0 * IMAGES * heads * N * Nk * 64
        d = dict(shape=f"{kind} {N}x{Nk} h{heads}", flops_bwd=flops_bwd, flops_fwd=flops_fwd)
        d["us_bwd"] = time_graph(lambda: D.attention_bwd(q, k, v, o, do, lse, heads, **grads), args.iters, stream)
        d["us_fwd_lse"] = time_graph(lambda: D.attention_lse(q, k, v, heads), args.iters, stream)
        d["us_fwd"] = time_graph(lambda: D.attention(q, k, v, heads), args.iters, stream)
        tb = torch_bwd(q, k, v, do, heads, stream)
        d["torch_backend"] = backend_of(tb)
        d["us_torch_bwd"] = time_graph(tb, args.iters, stream)
        d["tflops_bwd"] = flops_bwd / (d["us_bwd"] * 1e-6) / 1e12
        d["roof_bwd"] = d["tflops_bwd"] / PEAK_TFLOPS
        d["tflops_fwd_lse"] = flops_fwd / (d["us_fwd_lse"] * 1e-6) / 1e12
        d["vs_torch"] = d["us_torch_bwd"] / d["us_bwd"]
        rows.append(d)
    info = card()
    print(f"# {info}")
    print(f"# attention backward, bf16, {IMAGES} images, context {CTX_TOKENS} tokens; CUDA-graph replay of {args.iters} "
          f"calls per shape; TFLOP/s of the backward counts 8*Nq*Nk*64 per head, roof = {PEAK_TFLOPS:.0f} TFLOP/s bf16")
    print(f"{'shape':22s} {'bwd us':>8s} {'TFLOP/s':>8s} {'roof':>6s} {'torch us':>9s} {'backend':>13s} {'torch/ours':>10s} "
          f"{'fwd+lse us':>10s} {'fwd us':>8s}")
    for d in rows:
        print(f"{d['shape']:22s} {d['us_bwd']:8.1f} {d['tflops_bwd']:8.1f} {100 * d['roof_bwd']:5.1f}% "
              f"{d['us_torch_bwd']:9.1f} {d['torch_backend']:>13s} {d['vs_torch']:10.2f} {d['us_fwd_lse']:10.1f} "
              f"{d['us_fwd']:8.1f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "iters": args.iters, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
