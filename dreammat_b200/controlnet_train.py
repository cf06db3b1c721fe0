"""The ControlNet training step (controlnet_train/diffusers_train_controlnet.py:856-918, SURVEY.md section 3.4):

    noise, timesteps -> scheduler.add_noise -> controlnet -> frozen unet -> F.mse_loss(pred, noise) -> backward
    -> clip_grad_norm_(max_grad_norm) -> torch.optim.AdamW.step()

on fp32 master weights with a 16-bit copy for the kernels.  The parameters live in five flat arenas with one element order
(16-bit weights, fp32 master, Adam m and v, fp32 gradient), so the optimizer is three streaming launches over flat buffers
(dm_grad_sumsq, dm_adamw_prepare, dm_adamw_step) and the backward writes every gradient straight into its slice of the
gradient arena.  Nothing in the step synchronises with the host: lr, the step counter and the gradient norm live in device
memory, so the step can be captured once and replayed as a CUDA graph for a whole run.

Defaults are those of diffusers' train_controlnet.py (adam_beta1 0.9, adam_beta2 0.999, adam_weight_decay 1e-2,
adam_epsilon 1e-8, max_grad_norm 1.0) with the reference's learning rate 1e-5.  The text encoder is outside (ctx is an
input), as everywhere in this package.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import dense_ops as D
from . import nets
from .guidance import alphas_cumprod
from .parallel import allreduce_mean_buckets

ARENA_ALIGN = 8      # elements: 16 bytes of the 16-bit arena (a TMA base address), 32 of the fp32 ones


def arena_layout(shapes: Dict[str, Tuple[int, ...]]) -> Tuple[Dict[str, int], int]:
    """Element offset of every tensor in the flat arenas, in the dict's order, each a multiple of ARENA_ALIGN; and the
    arenas' length.  The gaps this leaves (at most 7 elements after a tensor) are zero weights with zero gradients."""
    off, n = {}, 0
    for k, shape in shapes.items():
        off[k] = n
        numel = 1
        for d in shape:
            numel *= int(d)
        n += (numel + ARENA_ALIGN - 1) // ARENA_ALIGN * ARENA_ALIGN
    return off, n


def arena_views(flat: torch.Tensor, shapes: Dict[str, Tuple[int, ...]], offsets: Dict[str, int]) -> Dict[str, torch.Tensor]:
    out = {}
    for k, shape in shapes.items():
        numel = 1
        for d in shape:
            numel *= int(d)
        out[k] = flat[offsets[k]:offsets[k] + numel].view(tuple(shape))
    return out


class ControlNetTrainer:
    """Owns the optimizer state of `controlnet` (a nets.ControlNet) and runs training steps against the frozen `unet`.

    Construction moves controlnet.p into one flat 16-bit arena: every controlnet.p[k] becomes a view of it with the same
    bits and shape, so the existing forward / backward run unchanged and see each update as soon as dm_adamw_step has
    written it.  master_weights (optional): the fp32 checkpoint under diffusers names the ControlNet was built from; the
    master copy then starts from those instead of from the rounded 16-bit values.  The UNet is not touched.

    grad_scale: the loss scale (fp16 storage needs one: the loss gradient 2 / numel underflows; bf16 uses 1).  A step whose
    gradient norm is not finite is dropped and counted in skipped_steps, as torch's GradScaler drops an overflowed step; the
    scale itself is fixed.  world > 1: the gradient arena is all-reduced (SUM, parallel.allreduce_mean_buckets) before the
    norm, the mean folded into the optimizer's gradient multiplier; every rank then clips and updates identically.
    max_grad_norm None disables clipping."""

    def __init__(self, unet: nets.UNet, controlnet: nets.ControlNet, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8,
                 max_grad_norm=1.0, conditioning_scale=1.0, grad_scale=1.0, world=1, vae: Optional[nets.VAEEncoder] = None,
                 master_weights: Optional[Dict[str, torch.Tensor]] = None):
        if unet.dt != controlnet.dt or controlnet.dt not in (torch.float16, torch.bfloat16):
            raise ValueError("ControlNetTrainer needs fp16 or bf16 storage, the same for the UNet and the ControlNet")
        self.unet, self.cnet, self.vae = unet, controlnet, vae
        self.betas, self.weight_decay, self.eps, self.max_grad_norm = (float(betas[0]), float(betas[1])), weight_decay, eps, max_grad_norm
        self.conditioning_scale, self.grad_scale, self.world = conditioning_scale, float(grad_scale), int(world)
        dev, dt = controlnet.dev, controlnet.dt
        self.shapes = {k: tuple(v.shape) for k, v in controlnet.p.items()}
        self.offsets, self.n = arena_layout(self.shapes)
        self.w16 = torch.zeros(self.n, device=dev, dtype=dt)
        views = arena_views(self.w16, self.shapes, self.offsets)
        for k in list(controlnet.p):
            views[k].copy_(controlnet.p[k])
            controlnet.p[k] = views[k]
        self.master = self.w16.float()
        self.m, self.v, self.grad = (torch.zeros(self.n, device=dev, dtype=torch.float32) for _ in range(3))
        self.grad_views = arena_views(self.grad, self.shapes, self.offsets)
        self.state = D.adamw_state(lr, dev)
        self._sumsq = torch.zeros((), device=dev, dtype=torch.float32)
        ac = alphas_cumprod().to(dev)
        self.sqrt_ac, self.sqrt_1mac = ac.sqrt(), (1.0 - ac).sqrt()
        self._graph = None
        if master_weights is not None:
            self._scatter(self.master, master_weights)
            self.w16.copy_(self.master)

    # ---- the step
    def _core(self, latents, cond_nhwc, ctx, noise, timesteps):
        sa, s1 = self.sqrt_ac.index_select(0, timesteps), self.sqrt_1mac.index_select(0, timesteps)
        noisy = D.add_noise(latents, noise, sa, s1, rep=1, cpad=64, dtype=self.cnet.dt)
        loss, _ = nets.controlnet_loss_and_grads(self.unet, self.cnet, noisy, timesteps.float(), ctx, cond_nhwc, noise,
                                                 self.conditioning_scale, self.grad_scale, into=self.grad_views)
        inv = 1.0 / self.grad_scale
        if self.world > 1:
            inv *= allreduce_mean_buckets(self.grad, self.world)
        D.grad_sumsq(self.grad, out=self._sumsq)
        D.adamw_prepare(self._sumsq, self.state, self.betas, self.max_grad_norm, inv)
        D.adamw_step(self.master, self.m, self.v, self.grad, self.w16, self.state, self.betas, self.eps, self.weight_decay)
        return loss

    def step(self, latents, cond_nhwc, ctx, noise=None, timesteps=None):
        """One optimizer step on a batch: latents fp32 NCHW [B, 4, h, w] (encode()'s output), cond_nhwc [B, 8h, 8w, 64] in
        the storage type (22 real channels), ctx [B, 77, D].  noise (fp32, latents' shape) and timesteps (int64 [B]) are
        drawn on the device unless given.  Returns the loss, a 0-dim fp32 device tensor (after capture(): the graph's
        output buffer, overwritten by the next step).  No host synchronisation."""
        if self._graph is None:
            noise = torch.randn_like(latents) if noise is None else noise
            timesteps = torch.randint(0, self.sqrt_ac.numel(), (latents.shape[0],), device=latents.device) if timesteps is None else timesteps
            return self._core(latents, cond_nhwc, ctx, noise, timesteps)
        s = self._static
        s["latents"].copy_(latents); s["cond"].copy_(cond_nhwc); s["ctx"].copy_(ctx)
        if noise is None:
            s["noise"].normal_()
        else:
            s["noise"].copy_(noise)
        if timesteps is None:
            s["timesteps"].random_(0, self.sqrt_ac.numel())
        else:
            s["timesteps"].copy_(timesteps)
        self._graph.replay()
        return self._loss

    def capture(self, latents, cond_nhwc, ctx):
        """Record the step as one CUDA graph over static input buffers shaped like the arguments (which are only read for
        their shapes and types); step() then copies its inputs in, draws noise / timesteps into their buffers when they
        are not given, and replays.  The recording itself applies no update: two warm-up steps that size the library's
        scratch run and are undone."""
        if self.world > 1:
            raise ValueError("the captured step is the single-GPU one; with world > 1 the all-reduce runs eagerly")
        B = latents.shape[0]
        self._static = dict(latents=torch.zeros_like(latents), cond=torch.zeros_like(cond_nhwc), ctx=torch.zeros_like(ctx),
                            noise=torch.zeros_like(latents), timesteps=torch.zeros(B, device=latents.device, dtype=torch.int64))
        keep = [t.clone() for t in (self.w16, self.master, self.m, self.v, self.state)]
        s = self._static
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._core(s["latents"], s["cond"], s["ctx"], s["noise"], s["timesteps"])
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._loss = self._core(s["latents"], s["cond"], s["ctx"], s["noise"], s["timesteps"])
        for dst, src in zip((self.w16, self.master, self.m, self.v, self.state), keep):
            dst.copy_(src)
        self._graph = graph

    def encode(self, images_nhwc, eps):
        """Latents of a batch of images [B, H, W, 64] (3 real channels, 2 * rgb - 1) with the posterior noise eps [B, 4,
        H/8, W/8]: AutoencoderKL.encode(...).latent_dist.sample() * scaling_factor, no tape (nothing upstream trains)."""
        if self.vae is None:
            raise ValueError("ControlNetTrainer was built without a VAEEncoder")
        return D.vae_sample(self.vae.encode_moments(images_nhwc), eps, self.vae.cfg.scaling_factor)

    # ---- optimizer state (these read device memory: host synchronisation, not for the step loop)
    def _ints(self):
        return self.state.view(torch.int32)

    @property
    def grad_norm(self) -> float:
        """L2 norm of the last step's unscaled gradient, before clipping"""
        return float(self.state[4])

    @property
    def steps(self) -> int:
        return int(self._ints()[1])

    @property
    def skipped_steps(self) -> int:
        return int(self._ints()[2])

    def set_lr(self, lr: float):
        """a 4-byte H2D copy; takes effect at the next step, also of a captured graph"""
        self.state[:1].copy_(torch.tensor([lr], dtype=torch.float32), non_blocking=True)

    # ---- checkpoint
    def _index_map(self, key):
        """diffusers name -> flat arena indices of that tensor's elements, for the prepared tensor `key`: the layout map
        grads_to_state_dict run over the element indices themselves"""
        numel = 1
        for d in self.shapes[key]:
            numel *= d
        idx = torch.arange(self.offsets[key], self.offsets[key] + numel, device=self.w16.device).view(self.shapes[key])
        return self.cnet.grads_to_state_dict({key: idx})

    def _gather(self, flat):
        return self.cnet.grads_to_state_dict(arena_views(flat, self.shapes, self.offsets))

    def _scatter(self, flat, sd):
        seen = set()
        for key in self.shapes:
            for name, idx in self._index_map(key).items():
                src = sd[name]
                if tuple(src.shape) != tuple(idx.shape):
                    raise ValueError(f"{name}: shape {tuple(src.shape)}, expected {tuple(idx.shape)}")
                flat[idx.reshape(-1)] = src.to(flat.device, torch.float32).reshape(-1)
                seen.add(name)
        if seen != set(sd):
            raise ValueError(f"unexpected keys: {sorted(set(sd) - seen)[:5]}")

    def state_dict(self):
        """fp32 master weights, Adam moments (all under diffusers names and shapes), step counters and lr."""
        clone = lambda d: {k: v.clone() for k, v in d.items()}    # noqa: E731
        return dict(weights=clone(self._gather(self.master)), exp_avg=clone(self._gather(self.m)),
                    exp_avg_sq=clone(self._gather(self.v)), step=self.steps, skipped_steps=self.skipped_steps,
                    lr=float(self.state[0]))

    def load_state_dict(self, sd):
        self._scatter(self.master, sd["weights"])
        self._scatter(self.m, sd["exp_avg"])
        self._scatter(self.v, sd["exp_avg_sq"])
        self.w16.copy_(self.master)
        self.state.zero_()
        self.set_lr(sd["lr"])
        self._ints()[1:3] = torch.tensor([sd["step"], sd["skipped_steps"]], dtype=torch.int32)
