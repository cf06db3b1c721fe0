"""Host-side mirror of the reference's guidance plugin on top of the H100 kernels.

    StableDiffusionLightGuidance  <->  threestudio `stable-diffusion-dreammat-guidance`
                                       (models/guidance/dreammat_guidance.py:44-626)
    PromptProcessorOutput         <->  models/prompt_processors/base.py:36-85 (tensor provider only)

Same Config field names / defaults, same `__call__` signature and returned keys, same `update_step`
schedules, so the reference's system (`systems/dreammat.py:57-86`) can drive it unchanged.  The text
encoder is not on the per-iteration path (embeddings are computed once and cached by the reference's
prompt processor); this mirror takes the cached tensors.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import torch

from . import dense_ops as D
from . import render_ops as R
from .nets import ControlNet, UNet, VAEEncoder


def C(value: Any, epoch: int, global_step: int) -> float:
    """utils/misc.py:65-86 (piecewise-linear schedule [start_step, v0, v1, end_step])."""
    if isinstance(value, (int, float)):
        return value
    value = list(value)
    if len(value) == 3:
        value = [0] + value
    assert len(value) == 4
    s0, v0, v1, s1 = value
    cur = global_step if isinstance(s1, int) else epoch
    return v0 + (v1 - v0) * max(min(1.0, (cur - s0) / (s1 - s0)), 0.0)


def shift_azimuth_deg(azimuth):
    """models/prompt_processors/base.py `shift_azimuth_deg`: to [-180, 180)."""
    return (azimuth + 180) % 360 - 180


@dataclass
class PromptProcessorOutput:
    """models/prompt_processors/base.py:36-85; direction order: side, front, back, overhead."""
    text_embeddings: torch.Tensor             # [1, 77, D]
    uncond_text_embeddings: torch.Tensor      # [1, 77, D]
    null_text_embeddings: torch.Tensor        # [1, 77, D]
    text_embeddings_vd: torch.Tensor          # [4, 77, D]
    uncond_text_embeddings_vd: torch.Tensor   # [4, 77, D]
    use_perp_neg: bool = False
    front_threshold: float = 45.0
    back_threshold: float = 45.0
    overhead_threshold: float = 60.0

    def direction_index(self, elevation, azimuth, camera_distances):
        idx = torch.zeros_like(elevation, dtype=torch.long)            # side
        az = shift_azimuth_deg(azimuth)
        idx[(az > -self.front_threshold) & (az < self.front_threshold)] = 1
        idx[(az > 180 - self.back_threshold) | (az < -180 + self.back_threshold)] = 2
        idx[elevation > self.overhead_threshold] = 3
        return idx

    def get_text_embeddings(self, elevation, azimuth, camera_distances, view_dependent_prompting=True,
                            return_null_text_embeddings=False):
        B = elevation.shape[0]
        if view_dependent_prompting:
            idx = self.direction_index(elevation, azimuth, camera_distances).to(self.text_embeddings_vd.device)
            te, ue = self.text_embeddings_vd[idx], self.uncond_text_embeddings_vd[idx]
        else:
            te, ue = self.text_embeddings.expand(B, -1, -1), self.uncond_text_embeddings.expand(B, -1, -1)
        if return_null_text_embeddings:
            return torch.cat([te, ue, self.null_text_embeddings.expand(B, -1, -1)], dim=0)
        return torch.cat([te, ue], dim=0)


def alphas_cumprod(n=1000, b0=0.00085, b1=0.012):
    """DDIMScheduler(scaled_linear) of stable-diffusion-2-1-base (dreammat_guidance.py:160-172)."""
    betas = torch.linspace(b0 ** 0.5, b1 ** 0.5, n, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class _VAEEncode(torch.autograd.Function):
    """encode_images (dreammat_guidance.py:285-292) with its input gradient."""

    @staticmethod
    def forward(ctx, rgb_bhwc, vae: VAEEncoder, vae_eps, dtype):
        x = D.pad_convert(rgb_bhwc, 64, 2.0, -1.0, dtype)            # imgs * 2 - 1, NHWC, channel-padded
        tape: list = []
        mom = vae.encode_moments(x, tape)
        z = D.vae_sample(mom, vae_eps, vae.cfg.scaling_factor)
        ctx.vae, ctx.tape, ctx.mom, ctx.eps = vae, tape, mom, vae_eps
        return z

    @staticmethod
    def backward(ctx, dz):
        vae = ctx.vae
        dmom = D.vae_sample_bwd(ctx.mom, ctx.eps, dz.float().contiguous(), vae.cfg.scaling_factor)
        dx = vae.backward_input(ctx.tape, dmom)
        drgb = D.unpad_convert(dx, 3, 2.0)
        ctx.tape = None
        return drgb, None, None, None


class _SDSLoss(torch.autograd.Function):
    """0.5 * mse_sum(latents, (latents - grad).detach()) / B  (dreammat_guidance.py:590-594)."""

    @staticmethod
    def forward(ctx, latents, dlat, loss_value):
        ctx.save_for_backward(dlat)
        return loss_value.clone()

    @staticmethod
    def backward(ctx, g):
        (dlat,) = ctx.saved_tensors
        return dlat * g, None, None


class _DenseGraphs:
    """Static buffers + three captured CUDA graphs for the dense section (shapes fixed by B, H, W)."""

    def __init__(self, guid, B, H, W, maps=None):
        self.guid, self.B = guid, B
        # N1: condition maps resident on the device as uint8 (scene.FixViewMaps); gathered + de-quantised inside the graph
        self.maps = maps if (maps is not None and tuple(maps.depths.shape[1:3]) == (H, W) and guid.weights_dtype != torch.float32) else None
        self.vid = torch.zeros(B, device=guid.device, dtype=torch.int32)
        self.eid = torch.zeros(B, device=guid.device, dtype=torch.int32)
        dev, dt = guid.device, guid.weights_dtype
        h, w = H // 8, W // 8
        Dm = guid.unet.cfg.cross_attention_dim
        self.rgb = torch.ones(B, H, W, 3, device=dev)
        self.vae_eps = torch.zeros(B, 4, h, w, device=dev)
        self.noise = torch.zeros(B, 4, h, w, device=dev)
        self.sqrt_ac, self.sqrt_1mac = torch.ones(B, device=dev), torch.zeros(B, device=dev)
        self.t3 = torch.full((3 * B,), 500.0, device=dev)
        self.ctx = torch.zeros(3 * B, 77, Dm, device=dev, dtype=dt)
        self.cond = torch.zeros(B, H, W, 22, device=dev)
        self.dz = torch.zeros(B, 4, h, w, device=dev)
        # fused conv_out + CSD epilogue (D.conv2d_csd): its schedule scalars live on the device so replays see new values
        self.fused_csd = guid.fuse_csd and D.csd_supported(dt, B, h, w)
        self.w1mac = torch.zeros(B, device=dev)
        self.coef = torch.zeros(5, device=dev)
        self.sums = torch.zeros(10, device=dev)
        self.grad = torch.zeros(B, 4, h, w, device=dev)
        self.pool = torch.cuda.graph_pool_handle()
        self.cond_scale = None
        # eager warm-up on a side stream (first-launch attribute setup must not happen under capture)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._vae_fwd(); self._unet(1.0); self._vae_bwd()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        from ._cabi import lib
        self.replayed_launches = 0          # kernels launched through graph replays (for bench.py's gpu_launches)
        n0 = lib().dm_launch_count()
        self.g_vae = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_vae, pool=self.pool):
            self._vae_fwd()
        self.n_vae = lib().dm_launch_count() - n0
        self.capture_unet(float(guid.cfg.condition_scales[0]) if guid.use_controlnet else 0.0)
        n0 = lib().dm_launch_count()
        self.g_bwd = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_bwd, pool=self.pool):
            self._vae_bwd()
        self.n_bwd = lib().dm_launch_count() - n0

    def _vae_fwd(self):
        g = self.guid
        x = D.pad_convert(self.rgb, 64, 2.0, -1.0, g.weights_dtype)
        self.tape = []
        self.mom = g.vae.encode_moments(x, self.tape)
        self.z = D.vae_sample(self.mom, self.vae_eps, g.vae.cfg.scaling_factor)

    def _unet(self, scale):
        g = self.guid
        zt = D.add_noise(self.z, self.noise, self.sqrt_ac, self.sqrt_1mac, rep=3, cpad=64, dtype=g.weights_dtype)
        down = mid = None
        if g.use_controlnet and scale != 0:
            if self.maps is not None:
                cond = D.cond_gather(self.maps.depths, self.maps.normals, self.maps.lightmaps, self.vid, self.eid, 64, g.weights_dtype)
            else:
                cond = D.pad_convert(self.cond, 64, 1.0, 0.0, g.weights_dtype)
            down, mid = g.controlnet.forward(zt, self.t3, self.ctx, cond, scale)
        if self.fused_csd:
            R.fill_(self.sums, 0.0)
            g.unet.forward(zt, self.t3, self.ctx, down, mid,
                           csd=dict(noise=self.noise, w1mac=self.w1mac, coef=self.coef, grad=self.grad, dlat=self.dz, norms=self.sums))
            self.eps = None
        else:
            self.eps = g.unet.forward(zt, self.t3, self.ctx, down, mid)

    def _vae_bwd(self):
        g = self.guid
        dmom = D.vae_sample_bwd(self.mom, self.vae_eps, self.dz, g.vae.cfg.scaling_factor)
        dx = g.vae.backward_input(list(self.tape), dmom)
        self.drgb = D.unpad_convert(dx, 3, 2.0)

    def capture_unet(self, scale):
        from ._cabi import lib
        self.cond_scale = scale
        n0 = lib().dm_launch_count()
        self.g_unet = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.g_unet, pool=self.pool):
            self._unet(scale)
        self.n_unet = lib().dm_launch_count() - n0


class StableDiffusionLightGuidance:
    @dataclass
    class Config:
        # field names and defaults of dreammat_guidance.py:45-84
        width: int = 512
        height: int = 512
        cache_dir: Optional[str] = None
        pretrained_model_name_or_path: str = "stabilityai/stable-diffusion-2-1-base"
        controlnet_path: Optional[str] = None
        enable_memory_efficient_attention: bool = False
        enable_sequential_cpu_offload: bool = False
        enable_attention_slicing: bool = False
        enable_channels_last_format: bool = False
        half_precision_weights: bool = True
        use_controlnet: bool = False
        condition_scale: float = 1.5
        control_anneal_start_step: Optional[int] = None
        control_anneal_end_scale: Optional[float] = None
        control_types: List = field(default_factory=lambda: ["depth", "canny"])
        condition_scales: List = field(default_factory=lambda: [1.0, 1.0])
        condition_scales_anneal: List = field(default_factory=lambda: [1.0, 1.0])
        p2p_condition_type: str = "p2p"
        canny_lower_bound: int = 50
        canny_upper_bound: int = 100
        min_step_percent: Any = 0.02
        max_step_percent: Any = 0.98
        cond_scale: Any = 1
        uncond_scale: Any = 0
        null_scale: Any = -1
        noise_scale: Any = 0
        perpneg_scale: Any = 0.0
        view_dependent_prompting: bool = True
        grad_clip_val: Optional[float] = None
        grad_normalize: Optional[bool] = False

    def __init__(self, cfg: Optional[dict] = None, unet_cfg=None, vae_cfg=None, unet_weights=None, controlnet_weights=None,
                 vae_weights=None, device="cuda", dtype=None):
        self.cfg = self.Config(**(cfg or {}))
        self.device = torch.device(device)
        # dreammat_guidance.py:92-94: fp16 weights unless half_precision_weights=false (then fp32 = the high-precision
        # mode of the kernels, csrc/dense_hp.cu); an explicit dtype (bf16: BASELINE config 3) overrides
        self.weights_dtype = dtype if dtype is not None else (torch.float16 if self.cfg.half_precision_weights else torch.float32)
        self.maps = None              # optional device-resident scene.FixViewMaps (N1); set by the host / enable_graphs
        self.fuse_csd = True          # conv_out + CSD combination in one kernel where the shape allows (D.csd_supported)
        self.keep_debug = False       # parity tests: keep latents / eps / grad of the last evaluation in self.debug
        self.debug: Dict[str, torch.Tensor] = {}
        self.use_controlnet = self.cfg.use_controlnet
        if self.use_controlnet and list(self.cfg.control_types) != ["light"]:
            # dreammat.yaml:62 selects ['light']; the annotator-based types need controlnet_aux (out of scope)
            raise ValueError(f"control_types {self.cfg.control_types}: only ['light'] is supported on this path")
        self.unet = UNet(unet_weights, unet_cfg, device, self.weights_dtype)
        self.controlnet = ControlNet(controlnet_weights, unet_cfg, device, self.weights_dtype) if self.use_controlnet else None
        self.vae = VAEEncoder(vae_weights, vae_cfg, device, self.weights_dtype)
        self.num_train_timesteps = 1000
        self.alphas = alphas_cumprod().to(self.device)
        self.set_min_max_steps()
        self.update_step(0, 0)
        self.graphs = None

    # ---- schedules (dreammat_guidance.py:604-626)
    def set_min_max_steps(self, min_step_percent=0.02, max_step_percent=0.98):
        self.min_step = int(self.num_train_timesteps * min_step_percent)
        self.max_step = int(self.num_train_timesteps * max_step_percent)

    def update_step(self, epoch: int, global_step: int, on_load_weights: bool = False):
        c = self.cfg
        self.noise_scale = C(c.noise_scale, epoch, global_step)
        self.cond_scale = C(c.cond_scale, epoch, global_step)
        self.uncond_scale = C(c.uncond_scale, epoch, global_step)
        self.null_scale = C(c.null_scale, epoch, global_step)
        self.perpneg_scale = C(c.perpneg_scale, epoch, global_step)
        self.set_min_max_steps(C(c.min_step_percent, epoch, global_step), C(c.max_step_percent, epoch, global_step))
        if (self.use_controlnet and c.control_anneal_start_step is not None
                and global_step > c.control_anneal_start_step):
            c.condition_scales = c.condition_scales_anneal

    # ---- pieces
    def encode_images(self, rgb_bhwc, vae_eps=None):
        """rgb [B,512,512,3] fp32 in [0,1] -> latents [B,4,64,64] fp32 (differentiable w.r.t. rgb)."""
        B, H, W, _ = rgb_bhwc.shape
        if vae_eps is None:
            vae_eps = torch.randn(B, 4, H // 8, W // 8, device=self.device)     # posterior.sample() (appendix B #7)
        return _VAEEncode.apply(rgb_bhwc.contiguous(), self.vae, vae_eps, self.weights_dtype)

    @staticmethod
    def _cond_to_latent_grid(cond_bhwc, h, w):
        """prepare_image_cond (dreammat_guidance.py:518-534): a condition map that is not at the VAE input size (8 x the
        latent grid, 512^2 for SD) is resized with F.interpolate(..., mode="bilinear", align_corners=False)."""
        if cond_bhwc.shape[1] != 8 * h or cond_bhwc.shape[2] != 8 * w:
            return R.resize_bilinear(cond_bhwc, 8 * h, 8 * w)
        return cond_bhwc

    @torch.no_grad()
    def predict_noise(self, latents, t, noise, ctx3, cond_bhwc, condition_scale, csd=None):
        """compute_without_perpneg (:388-438): 3-branch batch [text | uncond | null] -> eps [3,B,4,h,w] fp32
        (or, with `csd`, straight into the fused CSD epilogue of conv_out: nothing returned)."""
        B = latents.shape[0]
        ac = self.alphas[t]
        zt = D.add_noise(latents, noise, ac.sqrt(), (1 - ac).sqrt(), rep=3, cpad=64, dtype=self.weights_dtype)
        t3 = torch.cat([t] * 3).float()
        ctx = ctx3.to(self.device, self.weights_dtype).contiguous()
        down = mid = None
        if self.use_controlnet and condition_scale != 0:
            cond = D.pad_convert(self._cond_to_latent_grid(cond_bhwc, latents.shape[-2], latents.shape[-1]), 64, 1.0, 0.0,
                                 self.weights_dtype)
            down, mid = self.controlnet.forward(zt, t3, ctx, cond, float(condition_scale))
        eps = self.unet.forward(zt, t3, ctx, down, mid, csd=csd)
        return eps.view(3, B, *eps.shape[1:]) if csd is None else None

    def compute_grad_sds(self, latents, cond_bhwc, ctx3, t=None, noise=None):
        """:440-497.  Returns (grad, dlatents, sums) with sums = the 10 squared diagnostic norms."""
        B = latents.shape[0]
        if t is None:
            t = torch.randint(self.min_step, self.max_step + 1, [B], dtype=torch.long, device=self.device)
        if noise is None:
            noise = torch.randn_like(latents)
        scale = self.cfg.condition_scales[0] if self.use_controlnet else 0.0
        w = (1 - self.alphas[t]).float()
        if self.fuse_csd and D.csd_supported(self.weights_dtype, B, latents.shape[-2], latents.shape[-1]):
            noise = noise.float().contiguous()
            grad, dlat, sums = torch.empty_like(noise), torch.empty_like(noise), torch.zeros(10, device=self.device)
            eps = torch.empty(3, *noise.shape, device=self.device) if self.keep_debug else None
            coef = torch.tensor([float(self.cond_scale), float(self.uncond_scale), float(self.null_scale),
                                 float(self.noise_scale), 1.0 / B], dtype=torch.float32).to(self.device)
            self.predict_noise(latents.detach(), t, noise, ctx3, cond_bhwc, scale,
                               csd=dict(noise=noise, w1mac=w.contiguous(), coef=coef, grad=grad, dlat=dlat, norms=sums, eps_out=eps))
            out = (grad, dlat, sums)
        else:
            eps = self.predict_noise(latents.detach(), t, noise, ctx3, cond_bhwc, scale)
            out = R.sds_grad(eps, noise, w, float(self.cond_scale), float(self.uncond_scale), float(self.null_scale),
                             float(self.noise_scale))
        if self.keep_debug:
            self.debug = {"latents": latents.detach().clone(), "eps": eps.clone(), "grad": out[0].clone()}
        return out

    # ---- CUDA-graph path: the dense section has static shapes, so its ~900 launches are captured once
    def enable_graphs(self, B: int, H: int, W: int, maps=None):
        """Capture (1) VAE encode, (2) add_noise + ControlNet + UNet, (3) the VAE input-gradient as three CUDA graphs
        over static buffers.  Schedules that change kernel arguments (the ControlNet scale) trigger a re-capture.
        maps: a device-resident scene.FixViewMaps at the VAE input size -> the condition is gathered from it by (view, env) id."""
        if maps is not None:
            self.maps = maps
        self.graphs = _DenseGraphs(self, B, H, W, maps)
        return self.graphs

    def graph_step(self, cond_bhwc, ctx3, grad_scale: float, t=None, noise=None, vae_eps=None, mark=None, view_id=None,
                   env_id=None):
        """One guidance evaluation through the captured graphs.  `graphs.rgb` must hold the rendered batch.
        Returns (d loss / d rgb [B,H,W,3], sums[10]) with d loss_sds / d latents = grad / B * grad_scale."""
        g = self.graphs
        B = g.B
        scale = float(self.cfg.condition_scales[0]) if self.use_controlnet else 0.0
        if scale != g.cond_scale:
            g.capture_unet(scale)
        if vae_eps is None:
            g.vae_eps.normal_()
        else:
            g.vae_eps.copy_(vae_eps)
        g.g_vae.replay()
        if mark:
            mark("vae_fwd")
        if t is None:
            t = torch.randint(self.min_step, self.max_step + 1, [B], dtype=torch.long, device=self.device)
        if noise is None:
            g.noise.normal_()
        else:
            g.noise.copy_(noise)
        ac = self.alphas[t]
        g.sqrt_ac.copy_(ac.sqrt()); g.sqrt_1mac.copy_((1 - ac).sqrt()); g.t3.copy_(torch.cat([t] * 3).float())
        g.ctx.copy_(ctx3)
        if g.maps is not None:
            g.vid.copy_(view_id.to(torch.int32)); g.eid.copy_(env_id.to(torch.int32))       # a few integers per step
        else:
            g.cond.copy_(self._cond_to_latent_grid(cond_bhwc, g.noise.shape[-2], g.noise.shape[-1]))
        if g.fused_csd:
            # the CSD combination, nan_to_num, d loss / d latents and the logged norms come out of conv_out's epilogue
            g.w1mac.copy_(1 - ac)
            g.coef.copy_(torch.tensor([float(self.cond_scale), float(self.uncond_scale), float(self.null_scale),
                                       float(self.noise_scale), grad_scale / B], dtype=torch.float32))
            g.g_unet.replay()
            sums = g.sums
        else:
            g.g_unet.replay()
            grad, dlat, sums = R.sds_grad(g.eps.view(3, B, *g.eps.shape[1:]), g.noise, (1 - ac).float(), float(self.cond_scale),
                                          float(self.uncond_scale), float(self.null_scale), float(self.noise_scale))
            g.dz.copy_(dlat)
            g.dz.mul_(grad_scale)
        if mark:
            mark("unet_cn")
        g.g_bwd.replay()
        g.replayed_launches += g.n_vae + g.n_unet + g.n_bwd
        if mark:
            mark("vae_bwd")
        return g.drgb, sums

    def __call__(self, rgb, prompt_utils: PromptProcessorOutput, elevation, azimuth, camera_distances, env_id=None,
                 rgb_as_latents=False, **kwargs) -> Dict[str, torch.Tensor]:
        """dreammat_guidance.py:536-602.  kwargs: condition_map [B,H,W,22]; optional explicit randomness
        `t`, `noise`, `vae_eps` (appendix B #7-#9) for parity tests."""
        assert not prompt_utils.use_perp_neg, "perp-neg is off on this path (prompt_processors/base.py:214)"
        B = rgb.shape[0]
        if rgb_as_latents:
            latents = rgb.permute(0, 3, 1, 2).contiguous()
        else:
            if rgb.shape[1] != 512 or rgb.shape[2] != 512:
                # :507-513 bilinear resize to 512^2 before the VAE (512^2 renders skip it)
                rgb = R.resize_bilinear(rgb, 512, 512)
            latents = self.encode_images(rgb, kwargs.get("vae_eps"))
        cond = kwargs.get("condition_map")
        ctx3 = prompt_utils.get_text_embeddings(elevation, azimuth, camera_distances, self.cfg.view_dependent_prompting,
                                                return_null_text_embeddings=True)
        grad, dlat, sums = self.compute_grad_sds(latents, cond, ctx3, kwargs.get("t"), kwargs.get("noise"))
        if self.cfg.grad_clip_val is not None or self.cfg.grad_normalize:
            raise NotImplementedError("grad_clip_val / grad_normalize are off in dreammat.yaml")
        loss_sds = _SDSLoss.apply(latents, dlat, sums[0] / B)
        n = sums.sqrt()
        return {"loss_sds": loss_sds, "grad_norm": n[1], "uncond_m_noise_norm": n[2], "text_m_noise_norm": n[3],
                "text_m_uncond_norm": n[4], "text_m_null_norm": n[5], "null_m_uncond_norm": n[6], "noise_norm": n[7],
                "uncond_norm": n[8], "text_norm": n[9], "_grad": grad, "_latents": latents}
