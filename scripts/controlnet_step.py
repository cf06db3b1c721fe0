"""Time of the ControlNet training step's loss and gradients (nets.controlnet_loss_and_grads: taped ControlNet forward,
taped frozen-UNet forward, mse_loss_grad, UNet.backward_residuals, ControlNet.backward) against torch autograd of
F.mse_loss(oracle.sd.unet_forward(wu, ..., *oracle.sd.controlnet_forward(wc, ...)), target) in bf16, the UNet weights not
requiring grad, and where the time goes.

Shape: the per-GPU shape of scripts/controlnet_bwd.py (bf16, 4 images, 32^2 latents, 256^2 condition, context 4 x 77 x
1024, conditioning_scale 1, grad_scale 1), whose Replay, breakdown and timestep-embedding workaround are reused.

  1. whole step: each side captured as one CUDA graph, warmed up, replayed in windows of --window seconds, alternating for
     --rounds rounds; median and spread over rounds.
  2. kernel time of one eager step of ours by kind (torch.profiler, separate run), and on its own line the kernel time of
     the UNet decoder's input gradient (backward_residuals, profiled alone) as a share of the step.

The card's name and power limit are printed with the numbers.  There is no fallback: without a GPU the script fails.

    python scripts/controlnet_step.py [--window 1.0] [--rounds 5] [--json OUT.json]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from controlnet_bwd import Replay, breakdown  # noqa: E402
from gemm_shapes import card  # noqa: E402
from wgrad_shapes import COND, CTX_TOKENS, IMAGES, LATENT  # noqa: E402


def build(dev, dtype):
    from dreammat_b200 import dense_ops as D, nets, weights
    from oracle import sd as O
    cfg = weights.UNetConfig()
    wc = {k: v.to(dtype) for k, v in weights.random_controlnet(cfg, dev).items()}
    wu = {k: v.to(dtype) for k, v in weights.random_unet(cfg, dev).items()}
    cnet, unet = nets.ControlNet(wc, cfg, dev, dtype), nets.UNet(wu, cfg, dev, dtype)
    g = torch.Generator(device=dev).manual_seed(0)
    sample = torch.zeros(IMAGES, LATENT, LATENT, 64, device=dev, dtype=dtype)
    sample[..., :cfg.in_channels] = torch.randn(IMAGES, LATENT, LATENT, cfg.in_channels, device=dev, generator=g).to(dtype)
    cond = torch.zeros(IMAGES, COND, COND, 64, device=dev, dtype=dtype)
    cond[..., :cfg.cond_channels] = torch.rand(IMAGES, COND, COND, cfg.cond_channels, device=dev, generator=g).to(dtype)
    ctx = torch.randn(IMAGES, CTX_TOKENS, cfg.cross_attention_dim, device=dev, generator=g).to(dtype)
    t = torch.full((IMAGES,), 500.0, device=dev)
    target = torch.randn(IMAGES, cfg.out_channels, LATENT, LATENT, device=dev, generator=g)

    def ours():
        return nets.controlnet_loss_and_grads(unet, cnet, sample, t, ctx, cond, target)

    # the decoder's input gradient alone, on a tape of the same step
    utape = {}
    down, mid = cnet.forward(sample, t, ctx, cond)
    eps = unet.forward(sample, t, ctx, down, mid, tape=utape)
    _, d_eps = D.mse_loss_grad(eps, target, dtype)

    def decoder():
        return unet.backward_residuals(utape, d_eps)

    wct = {k: v.to(dev, dtype).requires_grad_() for k, v in wc.items()}
    wut = {k: v.to(dev, dtype) for k, v in wu.items()}                     # frozen
    emb = O.timestep_embedding(t.cpu(), cfg.block_out_channels[0]).to(dev, dtype)
    nchw = lambda x: x.permute(0, 3, 1, 2)      # noqa: E731   NHWC storage = channels_last NCHW
    s_t, c_t = nchw(sample[..., :cfg.in_channels]), nchw(cond[..., :cfg.cond_channels])

    def theirs():
        host_embedding = O.timestep_embedding
        O.timestep_embedding = lambda *_: emb
        try:
            down_t, mid_t = O.controlnet_forward(wct, cfg, s_t, t, ctx, c_t, 1.0)
            eps_t = O.unet_forward(wut, cfg, s_t, t, ctx, down_t, mid_t)
        finally:
            O.timestep_embedding = host_embedding
        loss = F.mse_loss(eps_t.float(), target)
        return (loss,) + torch.autograd.grad(loss, list(wct.values()))

    return ours, theirs, decoder


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of replays per timing window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", help="also write the numbers to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("controlnet_step.py times kernels on the GPU; no CUDA device found")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    ours, theirs, decoder = build(dev, torch.bfloat16)
    loss_ours, loss_theirs = float(ours()[0]), float(theirs()[0])
    stream = torch.cuda.Stream()
    a, b = Replay(ours, stream, args.window), Replay(theirs, stream, args.window)
    ms_a, ms_b = [], []
    for _ in range(args.rounds):
        ms_a.append(a.ms())
        ms_b.append(b.ms())
    info = card()
    print(f"# {info}")
    print(f"# ControlNet training step, loss + every ControlNet gradient through the frozen UNet, bf16, {IMAGES} images, "
          f"{LATENT}^2 latents, {COND}^2 condition; CUDA-graph replay, {args.rounds} alternating rounds of {a.n} / {b.n} replays")
    print(f"loss: ours {loss_ours:.6f}, torch {loss_theirs:.6f}")
    med_a, med_b = statistics.median(ms_a), statistics.median(ms_b)
    print(f"ours : median {med_a:.2f} ms  (min {min(ms_a):.2f}, max {max(ms_a):.2f})")
    print(f"torch: median {med_b:.2f} ms  (min {min(ms_b):.2f}, max {max(ms_b):.2f})")
    print(f"torch / ours = {med_b / med_a:.2f}  (< 1: torch autograd is faster)")
    kinds = breakdown(ours)
    total = sum(v[0] for v in kinds.values())
    dec = sum(v[0] for v in breakdown(decoder).values())
    print(f"# kernel time of one eager step of ours by kind (torch.profiler, separate run): {total:.2f} ms")
    for k, (ms, cnt) in sorted(kinds.items(), key=lambda kv: -kv[1][0]):
        print(f"{k:52s} {ms:8.2f} ms {100 * ms / total:5.1f}%  {cnt:5d} launches")
    print(f"{'UNet decoder input gradient (profiled alone)':52s} {dec:8.2f} ms {100 * dec / total:5.1f}%  of the step")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=info, ours_ms=ms_a, torch_ms=ms_b, loss=[loss_ours, loss_theirs], kinds=kinds,
                           decoder_ms=dec), f, indent=1)


if __name__ == "__main__":
    main()
