"""Dense half of `__graft_entry__.smoke()`: one tiny guidance evaluation (VAE encode with grad, ControlNet + UNet x3,
CSD gradient, VAE backward) on cuda:0, checked against the CPU oracle (the oracle is only the checker here)."""
import torch


def run():
    from oracle import sd as O
    from dreammat_b200 import weights as Wt
    from dreammat_b200.guidance import PromptProcessorOutput, StableDiffusionLightGuidance, _SDSLoss
    Q = lambda x: x.half().float()  # noqa: E731
    ucfg = O.UNetConfig(block_out_channels=(64, 128, 128, 128), heads=(1, 2, 2, 2), cross_attention_dim=64)
    vcfg = O.VAEConfig(block_out_channels=(64, 64, 64, 64))
    wu, wc, wv = (O.round_weights(O.random_unet_weights(ucfg, 0)), O.round_weights(O.random_controlnet_weights(ucfg, 1)),
                  O.round_weights(O.random_vae_weights(vcfg, 2)))
    dev = "cuda:0"
    g = torch.Generator().manual_seed(0)
    B, R = 1, 64
    rgb, cond = torch.rand(B, R, R, 3, generator=g), torch.rand(B, R, R, 22, generator=g)
    vd, uvd, null = torch.randn(4, 77, 64, generator=g), torch.randn(4, 77, 64, generator=g), torch.randn(1, 77, 64, generator=g)
    pu = PromptProcessorOutput(vd[:1], uvd[:1], null, vd, uvd)
    el, az, dist = torch.tensor([10.0]), torch.tensor([20.0]), torch.tensor([3.5])
    t, noise, veps = torch.tensor([400]), torch.randn(B, 4, 8, 8, generator=g), torch.randn(B, 4, 8, 8, generator=g)
    guid = StableDiffusionLightGuidance(dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05,
                                             uncond_scale=-0.7, null_scale=-0.2), Wt.UNetConfig(**ucfg.__dict__),
                                        Wt.VAEConfig(**vcfg.__dict__), wu, wc, wv, dev)
    x = rgb.to(dev).requires_grad_(True)
    lat = guid.encode_images(x, veps.to(dev))
    ctx3 = pu.get_text_embeddings(el, az, dist, True, return_null_text_embeddings=True)
    grad, dlat, sums = guid.compute_grad_sds(lat, cond.to(dev), ctx3, t.to(dev), noise.to(dev))
    _SDSLoss.apply(lat, dlat, sums[0] / B).backward()
    torch.cuda.synchronize()
    xo = rgb.clone().requires_grad_(True)
    loss_o, grad_o, z_o = O.guidance_step(wv, wc, wu, ucfg, vcfg, xo, cond, Q(ctx3), t, noise, veps, scales=(1.05, -0.7, -0.2, 0.0), q=Q)
    loss_o.backward()
    rel = lambda a, b: float((a.double().cpu() - b.double()).norm() / b.double().norm())  # noqa: E731
    e_z, e_g, e_r = rel(lat.detach(), z_o.detach()), rel(grad, grad_o), rel(x.grad, xo.grad)
    # the fp16 floor of the same chain, measured by the oracle itself (fp16 emulation vs pure fp32)
    w32 = (O.random_unet_weights(ucfg, 0), O.random_controlnet_weights(ucfg, 1), O.random_vae_weights(vcfg, 2))
    x32 = rgb.clone().requires_grad_(True)
    loss32, grad32, z32 = O.guidance_step(w32[2], w32[1], w32[0], ucfg, vcfg, x32, cond, ctx3, t, noise, veps, scales=(1.05, -0.7, -0.2, 0.0))
    loss32.backward()
    f_g, f_r = rel(grad_o, grad32), rel(xo.grad, x32.grad)
    print(f"smoke (dense, fp16 mode): latents rel err {e_z:.2e}, sds-grad {e_g:.2e} (oracle fp16 floor {f_g:.2e}), d-rgb {e_r:.2e} (floor {f_r:.2e})")
    assert e_z < 5e-3 and e_g < max(2 * f_g, 5e-3) and e_r < max(2 * f_r, 5e-3), (e_z, e_g, e_r, f_g, f_r)
    # the same slice in the high-precision mode (half_precision_weights=false): north_star's 1e-3 on the SDS gradient
    guid32 = StableDiffusionLightGuidance(dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05,
                                               uncond_scale=-0.7, null_scale=-0.2, half_precision_weights=False),
                                          Wt.UNetConfig(**ucfg.__dict__), Wt.VAEConfig(**vcfg.__dict__), *w32, dev)
    xh = rgb.to(dev).requires_grad_(True)
    lat_h = guid32.encode_images(xh, veps.to(dev))
    grad_h, dlat_h, sums_h = guid32.compute_grad_sds(lat_h, cond.to(dev), ctx3, t.to(dev), noise.to(dev))
    _SDSLoss.apply(lat_h, dlat_h, sums_h[0] / B).backward()
    h_z, h_g, h_r = rel(lat_h.detach(), z32.detach()), rel(grad_h, grad32), rel(xh.grad, x32.grad)
    print(f"smoke (dense, fp32 mode on the bf16x3 wgmma path): latents {h_z:.2e}, sds-grad {h_g:.2e}, d-rgb {h_r:.2e} vs the pure fp32 oracle")
    assert h_z < 1e-3 and h_g < 1e-3 and h_r < 1e-3, (h_z, h_g, h_r)
