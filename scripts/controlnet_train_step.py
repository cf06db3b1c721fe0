"""Time of the whole ControlNet training step (controlnet_train.ControlNetTrainer.step: add_noise, loss and gradients
through the frozen UNet written into the flat gradient arena, gradient norm, clip, AdamW on fp32 master weights with the
16-bit copy refreshed) against the same step in torch, and where the time goes.

Shape: the per-GPU shape of scripts/controlnet_step.py (bf16, 4 images, 32^2 latents, 256^2 condition, context 4 x 77 x
1024), whose build / Replay / breakdown / card are reused.  Fixed noise and timesteps on both sides.

  1. whole step, CUDA-graph replay of each side, alternating for --rounds rounds of --window seconds; median and spread.
     torch: the autograd step of controlnet_step.py, gradients cast to fp32, clip_grad_norm_, torch.optim.AdamW(fused=True,
     capturable=True) on fp32 master copies, _foreach_copy_ back into the bf16 weights.
  2. the optimizer section alone (dm_grad_sumsq + dm_adamw_prepare + dm_adamw_step) against torch's three calls
     (clip_grad_norm_, AdamW.step, _foreach_copy_): time, bytes from the arena size (34 B per parameter: the norm pass
     reads 4, the update reads 16 and writes 12 + 2), GB/s, and that as a share of the 3.35 TB/s data-sheet figure and of
     the copy rate in BASELINE.md.
  3. loss + gradients with the gradients allocated per call against written in place (`into`).
  4. kernel time of one eager step of ours by kind (torch.profiler, separate run), the optimizer kernels their own kind.

The card's name and power limit are printed with the numbers.  There is no fallback: without a GPU the script fails.

    python scripts/controlnet_train_step.py [--window 1.0] [--rounds 5] [--json OUT.json]
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

import controlnet_bwd  # noqa: E402
from controlnet_bwd import Replay, breakdown  # noqa: E402
from gemm_shapes import PEAK_GBS, card  # noqa: E402
from wgrad_shapes import COND, IMAGES, LATENT  # noqa: E402

COPY_GBS = 3014.6          # device-to-device copy rate of this card class, BASELINE.md
BYTES_PER_PARAM = 34
OPT_KIND = ("optimizer (sumsq, prepare, AdamW)", r"grad_sumsq|adamw_")


def build(dev, dtype):
    """(trainer, its batch, closures)"""
    from dreammat_b200 import dense_ops as D, nets, weights
    from dreammat_b200.controlnet_train import ControlNetTrainer
    from oracle import sd as O
    import torch.nn.functional as F
    cfg = weights.UNetConfig()
    wc = {k: v.to(dtype) for k, v in weights.random_controlnet(cfg, dev).items()}
    wu = {k: v.to(dtype) for k, v in weights.random_unet(cfg, dev).items()}
    cnet, unet = nets.ControlNet(wc, cfg, dev, dtype), nets.UNet(wu, cfg, dev, dtype)
    g = torch.Generator(device=dev).manual_seed(0)
    latents = torch.randn(IMAGES, cfg.in_channels, LATENT, LATENT, device=dev, generator=g)
    noise = torch.randn(IMAGES, cfg.in_channels, LATENT, LATENT, device=dev, generator=g)
    cond = torch.zeros(IMAGES, COND, COND, 64, device=dev, dtype=dtype)
    cond[..., :cfg.cond_channels] = torch.rand(IMAGES, COND, COND, cfg.cond_channels, device=dev, generator=g).to(dtype)
    ctx = torch.randn(IMAGES, 77, cfg.cross_attention_dim, device=dev, generator=g).to(dtype)
    steps = torch.full((IMAGES,), 500, device=dev)
    tr = ControlNetTrainer(unet, cnet)

    def ours():
        return tr._core(latents, cond, ctx, noise, steps)

    def ours_optimizer():
        D.grad_sumsq(tr.grad, out=tr._sumsq)
        D.adamw_prepare(tr._sumsq, tr.state, tr.betas, tr.max_grad_norm, 1.0)
        D.adamw_step(tr.master, tr.m, tr.v, tr.grad, tr.w16, tr.state, tr.betas, tr.eps, tr.weight_decay)

    t_f = steps.float()
    noisy = D.add_noise(latents, noise, tr.sqrt_ac[steps], tr.sqrt_1mac[steps], rep=1, cpad=64, dtype=dtype)

    def grads_alloc():
        return nets.controlnet_loss_and_grads(unet, cnet, noisy, t_f, ctx, cond, noise)

    def grads_inplace():
        return nets.controlnet_loss_and_grads(unet, cnet, noisy, t_f, ctx, cond, noise, into=tr.grad_views)

    # ---- torch: bf16 weights with autograd, fp32 masters under a fused AdamW
    w16 = [v.to(dev, dtype).requires_grad_() for v in wc.values()]
    wct = dict(zip(wc, w16))
    wut = {k: v.to(dev, dtype) for k, v in wu.items()}
    masters = [w.detach().float().requires_grad_() for w in w16]
    for p in masters:
        p.grad = torch.zeros_like(p)
    opt = torch.optim.AdamW(masters, lr=1e-5, betas=tr.betas, eps=tr.eps, weight_decay=tr.weight_decay, fused=True, capturable=True)
    emb = O.timestep_embedding(t_f.cpu(), cfg.block_out_channels[0]).to(dev, dtype)
    s_t = noisy[..., :cfg.in_channels].permute(0, 3, 1, 2)
    c_t = cond[..., :cfg.cond_channels].permute(0, 3, 1, 2)

    def theirs_optimizer():
        torch.nn.utils.clip_grad_norm_(masters, tr.max_grad_norm)
        opt.step()
        torch._foreach_copy_([w.detach() for w in w16], masters)

    def theirs():
        host_embedding = O.timestep_embedding
        O.timestep_embedding = lambda *_: emb
        try:
            down_t, mid_t = O.controlnet_forward(wct, cfg, s_t, t_f, ctx, c_t, 1.0)
            eps_t = O.unet_forward(wut, cfg, s_t, t_f, ctx, down_t, mid_t)
        finally:
            O.timestep_embedding = host_embedding
        loss = F.mse_loss(eps_t.float(), noise)
        grads = torch.autograd.grad(loss, w16)
        torch._foreach_copy_([p.grad for p in masters], list(grads))
        theirs_optimizer()
        return loss

    n_real = sum(v.numel() for v in wc.values())
    return tr, n_real, dict(ours=ours, theirs=theirs, ours_optimizer=ours_optimizer, theirs_optimizer=theirs_optimizer,
                            grads_alloc=grads_alloc, grads_inplace=grads_inplace)


def alternate(a, b, rounds):
    ms_a, ms_b = [], []
    for _ in range(rounds):
        ms_a.append(a.ms())
        ms_b.append(b.ms())
    return ms_a, ms_b


def line(name, ms):
    print(f"{name:28s} median {statistics.median(ms):8.3f} ms  (min {min(ms):.3f}, max {max(ms):.3f})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0, help="seconds of replays per timing window")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", help="also write the numbers to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("controlnet_train_step.py times kernels on the GPU; no CUDA device found")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    tr, n_real, fn = build(dev, torch.bfloat16)
    stream = torch.cuda.Stream()
    info = card()
    out = dict(card=info, arena_elements=tr.n, parameters=n_real)
    print(f"# {info}")
    print(f"# ControlNet training step, bf16, {IMAGES} images, {LATENT}^2 latents, {COND}^2 condition; {n_real} parameters in "
          f"arenas of {tr.n} elements (channel padding and alignment included); CUDA-graph replay, {args.rounds} alternating rounds")

    print("# 1. whole step")
    a, b = alternate(Replay(fn["ours"], stream, args.window), Replay(fn["theirs"], stream, args.window), args.rounds)
    line("ours", a); line("torch", b)
    print(f"torch / ours = {statistics.median(b) / statistics.median(a):.2f}  (< 1: torch is faster)")
    out.update(step_ours_ms=a, step_torch_ms=b)

    print("# 2. optimizer section alone")
    a, b = alternate(Replay(fn["ours_optimizer"], stream, args.window), Replay(fn["theirs_optimizer"], stream, args.window), args.rounds)
    line("ours (3 entry points)", a); line("torch (clip, AdamW, copy)", b)
    gb = BYTES_PER_PARAM * tr.n / 1e9
    gbs = gb / (statistics.median(a) / 1e3)
    print(f"ours: {gb:.2f} GB moved -> {gbs:.0f} GB/s = {100 * gbs / PEAK_GBS:.1f}% of the {PEAK_GBS:.0f} GB/s data-sheet HBM3 figure, "
          f"{100 * gbs / COPY_GBS:.1f}% of the {COPY_GBS} GB/s copy rate (BASELINE.md); HBM-bound")
    out.update(opt_ours_ms=a, opt_torch_ms=b, opt_gb=gb, opt_gbs=gbs)

    print("# 3. loss + gradients: gradients allocated per call vs written into the arena")
    a, b = alternate(Replay(fn["grads_alloc"], stream, args.window), Replay(fn["grads_inplace"], stream, args.window), args.rounds)
    line("allocated per call", a); line("in place (into=)", b)
    out.update(grads_alloc_ms=a, grads_inplace_ms=b)

    controlnet_bwd.KINDS.insert(0, OPT_KIND)
    kinds = breakdown(fn["ours"])
    total = sum(v[0] for v in kinds.values())
    print(f"# 4. kernel time of one eager step of ours by kind (torch.profiler, separate run): {total:.2f} ms")
    for k, (ms, cnt) in sorted(kinds.items(), key=lambda kv: -kv[1][0]):
        print(f"{k:52s} {ms:8.2f} ms {100 * ms / total:5.1f}%  {cnt:5d} launches")
    out.update(kinds=kinds)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
