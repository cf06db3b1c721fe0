"""GPU parity: dense path (VAE encoder fwd+bwd, ControlNet, UNet, CSD gradient) vs the CPU oracle.

The product computes in fp16 storage / fp32 accumulation, exactly the reference's default
(`half_precision_weights=True`).  The oracle therefore runs with fp16-rounded weights and the
storage-rounding hook `q = half().float()`; the residual difference is accumulation order and
fusion boundaries.  Tolerance: relative L2 error <= 5e-3 on network outputs at this precision
(measured values are printed; the fp32 drift is reported alongside), 1e-3 on the pure fp32 pieces.
"""
import math

import pytest
import torch

from oracle import sd as O

pytestmark = pytest.mark.gpu

Q = lambda x: x.half().float()  # noqa: E731
TOL16 = 5e-3


def rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def nchw(x_nhwc, c=None):
    x = x_nhwc.float().permute(0, 3, 1, 2)
    return x if c is None else x[:, :c]


@pytest.fixture(scope="module")
def small():
    ucfg = O.UNetConfig(block_out_channels=(64, 128, 256, 256), heads=(1, 2, 4, 4), cross_attention_dim=128)
    vcfg = O.VAEConfig(block_out_channels=(64, 64, 128, 128))
    wu = O.round_weights(O.random_unet_weights(ucfg, 0))
    wc = O.round_weights(O.random_controlnet_weights(ucfg, 1))
    wv = O.round_weights(O.random_vae_weights(vcfg, 2))
    return ucfg, vcfg, wu, wc, wv


def test_gemm_conv_match_torch_fp32():
    """Numerics of the tensor-core kernel against a plain fp32 reference of the same op (on the GPU)."""
    import torch.nn.functional as F
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(300, 192, device="cuda", generator=g).half()
    b = torch.randn(200, 192, device="cuda", generator=g).half()
    bias = torch.randn(200, device="cuda", generator=g).half()
    out = D.gemm(a, b, bias=bias, act="silu")
    ref = F.silu(a.float() @ b.float().t() + bias.float())
    assert rel(out, ref) < 1e-3
    x = torch.randn(2, 32, 32, 128, device="cuda", generator=g).half()
    w = (torch.randn(192, 128, 3, 3, device="cuda", generator=g) / 34).half()
    y = D.conv2d(x, D.conv_weight_to_gemm(w), 3)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=1)
    assert rel(nchw(y), ref) < 1e-3
    y = D.conv2d(x, D.conv_weight_to_gemm(w), 3, stride=2, pad=(0, 0), out_hw=(16, 16))
    ref = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), w.float(), stride=2)
    assert rel(nchw(y), ref) < 1e-3
    with pytest.raises(Exception):
        D.gemm(a[:, :100].contiguous(), b[:, :100].contiguous())  # K % 64 != 0 must fail loudly
    # fused GEGLU epilogue (diffusers attention.py GEGLU: hidden, gate = proj(x).chunk(2); hidden * gelu(gate))
    for M, Dh in ((300, 256), (4096, 1280), (150, 64)):
        for bn in (0, 64, 128, 256):
            if bn > 2 * Dh:
                continue
            a = torch.randn(M, 192, device="cuda", generator=g).half()
            w = (torch.randn(2 * Dh, 192, device="cuda", generator=g) / 14).half()
            bias = torch.randn(2 * Dh, device="cuda", generator=g).half()
            out = D.gemm(a, D.geglu_interleave(w), bias=D.geglu_interleave(bias), act="geglu", bn=bn)
            pr = a.float() @ w.float().t() + bias.float()
            ref = pr[:, :Dh] * F.gelu(pr[:, Dh:])
            assert out.shape == (M, Dh) and rel(out, ref) < 1e-3, (M, Dh, bn, rel(out, ref))


def test_tile_widths_and_splitk_match_torch_fp32():
    """Both tile widths, a ragged last 128-row tile, ragged N, stride-2 conv, and split-K (run twice: the workspace slices
    are rewritten by every call, so the second call must be as exact as the first)."""
    import torch.nn.functional as F
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(1)
    for (M, N, K, bn) in ((256, 128, 64, 128), (300, 200, 192, 128), (1000, 320, 320, 64), (513, 768, 1024, 128), (4096, 640, 640, 64)):
        a = torch.randn(M, K, device="cuda", generator=g).half(); b = (torch.randn(N, K, device="cuda", generator=g) * 0.05).half()
        bias = torch.randn(N, device="cuda", generator=g).half(); res = torch.randn(M, N, device="cuda", generator=g).half()
        out = D.gemm(a, b, bias=bias, residual=res, bn=bn)
        ref = a.float() @ b.float().t() + bias.float() + res.float()
        assert rel(out, ref) < 1e-3, (M, N, K, bn, rel(out, ref))
    x = torch.randn(2, 64, 64, 64, device="cuda", generator=g).half()
    w = (torch.randn(128, 64, 3, 3, device="cuda", generator=g) / 24).half()
    y = D.conv2d(x, D.conv_weight_to_gemm(w), 3, stride=2, pad=(0, 0), out_hw=(32, 32), bn=128)
    ref = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), w.float(), stride=2)
    assert rel(nchw(y), ref) < 1e-3
    # split-K: few tiles, long K (auto heuristics); 8x8 latents of a one-view batch
    for (n, hw, ci, co) in ((3, 8, 1280, 1280), (3, 8, 2560, 1280), (3, 16, 1280, 1280)):
        x = torch.randn(n, hw, hw, ci, device="cuda", generator=g).half()
        w = (torch.randn(co, ci, 3, 3, device="cuda", generator=g) / 100).half()
        tp = torch.randn(n, co, device="cuda", generator=g).half()
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), padding=1) + tp.float()[:, :, None, None]
        for _ in range(2):
            y = D.conv2d(x, D.conv_weight_to_gemm(w), 3, rowvec=tp)
            assert rel(nchw(y), ref) < 1e-3, (n, hw, ci, co, rel(nchw(y), ref))
    a = torch.randn(192, 5120, device="cuda", generator=g).half(); b = (torch.randn(1280, 5120, device="cuda", generator=g) * 0.02).half()
    ref = F.silu(a.float() @ b.float().t())
    for _ in range(2):
        assert rel(D.gemm(a, b, act="silu"), ref) < 1e-3


def test_attention_matches_torch_fp32():
    import torch.nn.functional as F
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(1)
    for (B, heads, Nq, Nk) in ((2, 5, 1024, 1024), (2, 20, 64, 77), (1, 2, 4096, 4096)):
        q = torch.randn(B, Nq, heads * 64, device="cuda", generator=g).half()
        k = torch.randn(B, Nk, heads * 64, device="cuda", generator=g).half()
        v = torch.randn(B, Nk, heads * 64, device="cuda", generator=g).half()
        o = D.attention(q, k, v, heads)
        sp = lambda t, n: t.float().view(B, n, heads, 64).transpose(1, 2)  # noqa: E731
        ref = F.scaled_dot_product_attention(sp(q, Nq), sp(k, Nk), sp(v, Nk)).transpose(1, 2).reshape(B, Nq, -1)
        assert rel(o, ref) < 1e-3, (B, heads, Nq, Nk)


def test_unet_matches_oracle(small):
    from dreammat_b200.nets import UNet
    from dreammat_b200 import dense_ops as D
    ucfg, _, wu, _, _ = small
    g = torch.Generator().manual_seed(3)
    N, hw = 3, 32
    z = torch.randn(N, 4, hw, hw, generator=g)
    t = torch.tensor([37, 500, 940])
    ctx = torch.randn(N, 77, ucfg.cross_attention_dim, generator=g)
    ref16 = O.unet_forward(wu, ucfg, Q(z), t, Q(ctx), q=Q)
    ref32 = O.unet_forward(wu, ucfg, Q(z), t, Q(ctx))
    net = UNet(wu, ucfg)
    zp = D.pad_convert(z.permute(0, 2, 3, 1).contiguous().cuda(), 64)
    out = net.forward(zp, t.float().cuda(), ctx.half().cuda())
    e16, e32 = rel(out, ref16), rel(out, ref32)
    print(f"\nunet small: rel err vs fp16-emulating oracle {e16:.2e}, vs fp32 oracle {e32:.2e}, "
          f"oracle16 vs oracle32 {rel(ref16, ref32):.2e}")
    assert e16 < TOL16


def test_controlnet_matches_oracle(small):
    from dreammat_b200.nets import ControlNet
    from dreammat_b200 import dense_ops as D
    ucfg, _, _, wc, _ = small
    g = torch.Generator().manual_seed(4)
    B, hw = 2, 16
    z = torch.randn(3 * B, 4, hw, hw, generator=g)
    t = torch.tensor([100, 700] * 3)
    ctx = torch.randn(3 * B, 77, ucfg.cross_attention_dim, generator=g)
    cond = torch.rand(B, 22, 8 * hw, 8 * hw, generator=g)
    down_r, mid_r = O.controlnet_forward(wc, ucfg, Q(z), t, Q(ctx), Q(cond), 0.8, q=Q)
    net = ControlNet(wc, ucfg)
    zp = D.pad_convert(z.permute(0, 2, 3, 1).contiguous().cuda(), 64)
    cp = D.pad_convert(cond.permute(0, 2, 3, 1).contiguous().cuda(), 64)
    down, mid = net.forward(zp, t.float().cuda(), ctx.half().cuda(), cp, 0.8)
    errs = [rel(nchw(a), b) for a, b in zip(down, down_r)] + [rel(nchw(mid), mid_r)]
    print("\ncontrolnet small: rel errs", " ".join(f"{e:.1e}" for e in errs))
    assert len(down) == 12 and max(errs) < TOL16


def test_vae_encoder_forward_backward_match_oracle(small):
    from dreammat_b200.nets import VAEEncoder
    from dreammat_b200 import dense_ops as D
    _, vcfg, _, _, wv = small
    g = torch.Generator().manual_seed(5)
    B, R = 2, 128
    rgb = torch.rand(B, R, R, 3, generator=g)
    eps = torch.randn(B, 4, R // 8, R // 8, generator=g)
    x = (rgb * 2 - 1).permute(0, 3, 1, 2).clone().requires_grad_(True)
    mom_r = O.vae_encode_moments(wv, vcfg, Q(x), q=Q)
    z_r = O.vae_sample(mom_r, eps, vcfg.scaling_factor, Q)
    dz = torch.randn(z_r.shape, generator=g)
    # torch casts are differentiable: gradients are rounded to fp16 at the same points as the activations
    z_r.backward(dz)
    vae = VAEEncoder(wv, vcfg)
    xp = D.pad_convert(rgb.cuda(), 64, 2.0, -1.0)
    tape = []
    mom = vae.encode_moments(xp, tape)
    z = D.vae_sample(mom, eps.cuda(), vcfg.scaling_factor)
    e_m, e_z = rel(nchw(mom, 8), mom_r), rel(z, z_r)
    dmom = D.vae_sample_bwd(mom, eps.cuda(), dz.cuda(), vcfg.scaling_factor)
    dx = vae.backward_input(tape, dmom)
    e_g = rel(nchw(dx, 3), x.grad)
    print(f"\nvae small: moments {e_m:.2e} latents {e_z:.2e} input-grad {e_g:.2e}")
    assert e_m < TOL16 and e_z < TOL16 and e_g < 2 * TOL16


def test_guidance_step_matches_oracle(small):
    """Full a7-a9 slice: rgb -> VAE -> add_noise -> ControlNet + UNet x3 -> CSD grad -> loss -> d rgb."""
    from dreammat_b200.guidance import PromptProcessorOutput, StableDiffusionLightGuidance
    ucfg, vcfg, wu, wc, wv = small
    g = torch.Generator().manual_seed(6)
    B, R = 2, 128
    Dm = ucfg.cross_attention_dim
    rgb = torch.rand(B, R, R, 3, generator=g)
    cond = torch.rand(B, R, R, 22, generator=g)
    vd = torch.randn(4, 77, Dm, generator=g)
    uvd = torch.randn(4, 77, Dm, generator=g)
    null = torch.randn(1, 77, Dm, generator=g)
    pu = PromptProcessorOutput(vd[:1], uvd[:1], null, vd, uvd)
    el, az, dist = torch.tensor([10.0, 70.0]), torch.tensor([20.0, -170.0]), torch.tensor([3.5, 3.5])
    t = torch.tensor([321, 777])
    noise = torch.randn(B, 4, R // 8, R // 8, generator=g)
    veps = torch.randn(B, 4, R // 8, R // 8, generator=g)
    cfg = dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05, uncond_scale=-0.7,
               null_scale=-0.2, noise_scale=0.0)
    guid = StableDiffusionLightGuidance(cfg, ucfg, vcfg, wu, wc, wv)
    # the 512-resize branch is exercised separately; feed latents-sized inputs through encode_images directly
    rgb_c = rgb.cuda().requires_grad_(True)
    lat = guid.encode_images(rgb_c, veps.cuda())
    ctx3 = pu.get_text_embeddings(el, az, dist, True, return_null_text_embeddings=True)
    grad, dlat, sums = guid.compute_grad_sds(lat, cond.cuda(), ctx3, t.cuda(), noise.cuda())
    from dreammat_b200.guidance import _SDSLoss
    loss = _SDSLoss.apply(lat, dlat, sums[0] / B)
    loss.backward()
    # oracle
    rgb_o = rgb.clone().requires_grad_(True)
    assert pu.direction_index(el, az, dist).tolist() == [1, 3]
    ctx3_o = Q(ctx3)
    loss_o, grad_o, z_o = O.guidance_step(wv, wc, wu, ucfg, vcfg, rgb_o, cond, ctx3_o, t, noise, veps,
                                          scales=(1.05, -0.7, -0.2, 0.0), cond_scale=1.0, q=Q)
    loss_o.backward()
    e_z, e_g, e_l, e_r = rel(lat, z_o), rel(grad, grad_o), abs(float(loss) - float(loss_o)) / abs(float(loss_o)), rel(rgb_c.grad, rgb_o.grad)
    # fp16 noise floor of the CSD combination: the three CFG branches are strongly correlated and their
    # coefficients nearly cancel (1.05 - 0.7 - 0.2), which amplifies the ~1e-3 storage-rounding error of
    # each eps by ~|c|+|u|+|n| / |c+u+n| ~ 13x.  Measure that floor with the oracle itself (fp16 emulation
    # vs pure fp32) and require the kernels to sit within 2x of it.
    _, grad_32, _ = O.guidance_step(wv, wc, wu, ucfg, vcfg, rgb.clone(), cond, ctx3_o, t, noise, veps,
                                    scales=(1.05, -0.7, -0.2, 0.0), cond_scale=1.0)
    floor = rel(grad_o, grad_32)
    print(f"\nguidance small: latents {e_z:.2e} sds-grad {e_g:.2e} (fp16 floor {floor:.2e}) loss {e_l:.2e} d-rgb {e_r:.2e}")
    assert e_z < TOL16 and e_l < 2 * TOL16
    assert e_g < max(2 * floor, TOL16) and e_r < max(3 * floor, 3 * TOL16)


def test_cond_gather_bit_exact_vs_float_condition_map():
    """N1: gathering + de-quantising the resident uint8 maps inside the kernel gives the SAME fp16 condition tensor as the
    reference's float condition_map (uncond.py:799-802) followed by the channel-padding cast."""
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.scene import FixViewMaps
    maps = FixViewMaps.synthetic(6, 3, 64, 64, device="cuda", seed=3)
    v, e = torch.tensor([4, 0, 5, 4]), torch.tensor([2, 1, 0, 0])
    ref = D.pad_convert(maps.condition_map(v, e), 64, 1.0, 0.0, torch.float16)
    got = D.cond_gather(maps.depths, maps.normals, maps.lightmaps, v.int().cuda(), e.int().cuda(), 64, torch.float16)
    assert got.shape == (4, 64, 64, 64) and torch.equal(got, ref)
    assert float(got[..., 22:].abs().max()) == 0.0 and float(got[..., :22].float().abs().sum()) > 0
    refb = D.pad_convert(maps.condition_map(v, e), 64, 1.0, 0.0, torch.bfloat16)
    assert torch.equal(D.cond_gather(maps.depths, maps.normals, maps.lightmaps, v.int().cuda(), e.int().cuda(), 64, torch.bfloat16), refb)


def test_fused_csd_epilogue_matches_unfused(small):
    """J1: conv_out with the CSD combination fused into its epilogue (dm_conv2d_csd).
    (1) op level, same input activation: the noise predictions it emits equal conv_out + layout change (D.conv2d +
        nhwc_to_nchw) up to fp32 summation order before the fp16 rounding, and grad / dlatents / the ten logged sums equal
        the closed form of dreammat_guidance.py:475-495,584-594 applied to those predictions (fp32 reduction order);
    (2) through the guidance object: fused and unfused evaluation agree within the fp16 noise of the network (two unfused
        runs are compared too and printed; the network is deterministic, so that figure is 0)."""
    import torch.nn.functional as F
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.guidance import StableDiffusionLightGuidance
    g = torch.Generator(device="cuda").manual_seed(9)
    rn = lambda *s_: torch.randn(*s_, device="cuda", generator=g)  # noqa: E731
    for (B, hw, Cin) in ((2, 16, 64), (4, 8, 128), (1, 32, 320), (8, 64, 320)):
        assert D.csd_supported(torch.float16, B, hw, hw)
        x = rn(3 * B, hw, hw, Cin).half()
        w4 = (rn(4, Cin, 3, 3) / (3 * Cin ** 0.5)).half()
        wg = D.conv_weight_to_gemm(w4)
        bias = (rn(4) * 0.1).half()
        noise, w1mac = rn(B, 4, hw, hw), torch.rand(B, device="cuda", generator=g)
        coef = torch.tensor([1.05, -0.7, -0.2, 0.1, 0.37], device="cuda")
        grad, dlat, sums = torch.empty_like(noise), torch.empty_like(noise), torch.zeros(10, device="cuda")
        eps = torch.empty(3, B, 4, hw, hw, device="cuda")
        D.conv2d_csd(x, wg, bias, noise, w1mac, coef, grad, dlat, sums, eps)
        out = torch.empty(3 * B, hw, hw, 8, device="cuda", dtype=torch.float16)
        D.conv2d(x, wg, 3, bias=bias, out=out[..., :4])
        eps_ref = D.nhwc_to_nchw_f32(out, 4).view(3, B, 4, hw, hw)
        et, eu, en = eps[0], eps[1], eps[2]
        gref = torch.nan_to_num(w1mac.view(-1, 1, 1, 1) * (1.05 * et - 0.7 * eu - 0.2 * en + 0.1 * noise))
        sref = torch.stack([0.5 * (gref ** 2).sum(), (gref ** 2).sum(), ((eu - noise) ** 2).sum(), ((et - noise) ** 2).sum(),
                            ((et - eu) ** 2).sum(), ((et - en) ** 2).sum(), ((en - eu) ** 2).sum(), (noise ** 2).sum(), (eu ** 2).sum(),
                            (et ** 2).sum()])
        errs = dict(eps=rel(eps, eps_ref), grad=rel(grad, gref), dlat=rel(dlat, gref * 0.37),
                    sums=float(((sums - sref).abs() / sref.abs().clamp_min(1e-20)).max()))
        print(f"\nfused CSD epilogue op B={B} {hw}x{hw} Cin={Cin}: " + " ".join(f"{k}={v:.1e}" for k, v in errs.items()))
        assert errs["eps"] < 1e-4 and errs["grad"] < 1e-6 and errs["dlat"] < 1e-6 and errs["sums"] < 1e-5, errs
    ucfg, vcfg, wu, wc, wv = small
    gc = torch.Generator().manual_seed(9)
    B, hw, Dm = 2, 16, ucfg.cross_attention_dim
    lat, noise = torch.randn(B, 4, hw, hw, generator=gc).cuda(), torch.randn(B, 4, hw, hw, generator=gc).cuda()
    cond, ctx3 = torch.rand(B, 8 * hw, 8 * hw, 22, generator=gc).cuda(), torch.randn(3 * B, 77, Dm, generator=gc)
    t = torch.randint(20, 981, (B,), generator=gc).cuda()
    guid = StableDiffusionLightGuidance(dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05,
                                             uncond_scale=-0.7, null_scale=-0.2, noise_scale=0.1), ucfg, vcfg, wu, wc, wv)
    guid.keep_debug = True
    runs = []
    for fuse in (True, False, False):
        guid.fuse_csd = fuse
        g_, d_, s_ = guid.compute_grad_sds(lat, cond, ctx3, t, noise)
        runs.append((guid.debug["eps"].clone(), g_.clone(), s_.clone()))
    noise_floor = rel(runs[1][1], runs[2][1])          # unfused vs unfused: the network's own run-to-run difference
    e_fused = rel(runs[0][1], runs[1][1])
    print(f"fused vs unfused through the guidance: sds-grad {e_fused:.1e}, eps {rel(runs[0][0], runs[1][0]):.1e}; "
          f"unfused run-to-run {noise_floor:.1e}")
    assert e_fused < max(3 * noise_floor, 2e-2)


@pytest.mark.slow
def test_vae_and_controlnet_full_size_match_oracle():
    """Full-size SD-2.1-base VAE encoder (128,256,512,512) forward + input gradient at 512^2 and full-size ControlNet
    (22-channel condition at 512^2, 64^2 latents) in the default fp16 mode vs the fp16-emulating oracle.  The bound is the
    measured fp16 floor (oracle fp16-emulation vs oracle fp32, printed), x2."""
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import ControlNet, VAEEncoder
    vcfg, ucfg = O.VAEConfig(), O.UNetConfig()
    wv = O.round_weights(O.random_vae_weights(vcfg, 2))
    g = torch.Generator().manual_seed(5)
    rgb = torch.rand(1, 512, 512, 3, generator=g)
    eps = torch.randn(1, 4, 64, 64, generator=g)
    dz = torch.randn(1, 4, 64, 64, generator=g)
    ref = {}
    for name, q in (("16", Q), ("32", O.Ident)):
        x = (rgb * 2 - 1).permute(0, 3, 1, 2).clone().requires_grad_(True)
        mom_r = O.vae_encode_moments(wv, vcfg, q(x), q=q)
        z_r = O.vae_sample(mom_r, eps, vcfg.scaling_factor, q)
        z_r.backward(dz)
        ref[name] = (mom_r.detach(), z_r.detach(), x.grad.clone())
    vae = VAEEncoder(wv, vcfg)
    tape = []
    mom = vae.encode_moments(D.pad_convert(rgb.cuda(), 64, 2.0, -1.0), tape)
    z = D.vae_sample(mom, eps.cuda(), vcfg.scaling_factor)
    dx = vae.backward_input(tape, D.vae_sample_bwd(mom, eps.cuda(), dz.cuda(), vcfg.scaling_factor))
    got = (nchw(mom, 8), z, nchw(dx, 3))
    names = ("moments", "latents", "input-grad")
    e = [rel(a, b) for a, b in zip(got, ref["16"])]
    floor = [rel(a, b) for a, b in zip(ref["16"], ref["32"])]
    print("\nvae full-size 512^2: " + " ".join(f"{n} {x:.2e} (fp16 floor {f:.2e})" for n, x, f in zip(names, e, floor)))
    for x, f in zip(e, floor):
        assert x < max(2 * f, 2e-3)
    del vae, tape, mom, dx
    torch.cuda.empty_cache()
    wc = O.round_weights(O.random_controlnet_weights(ucfg, 1))
    zz = torch.randn(3, 4, 64, 64, generator=g)
    t = torch.tensor([400, 400, 400])
    ctx = torch.randn(3, 77, 1024, generator=g)
    cond = torch.rand(1, 22, 512, 512, generator=g)
    with torch.no_grad():
        d16, m16 = O.controlnet_forward(wc, ucfg, Q(zz), t, Q(ctx), Q(cond), 0.8, q=Q)
        d32, m32 = O.controlnet_forward(wc, ucfg, Q(zz), t, Q(ctx), Q(cond), 0.8)
    net = ControlNet(wc, ucfg)
    down, mid = net.forward(D.pad_convert(zz.permute(0, 2, 3, 1).contiguous().cuda(), 64), t.float().cuda(), ctx.half().cuda(),
                            D.pad_convert(cond.permute(0, 2, 3, 1).contiguous().cuda(), 64), 0.8)
    errs = [rel(nchw(a), b) for a, b in zip(down, d16)] + [rel(nchw(mid), m16)]
    floors = [rel(a, b) for a, b in zip(d16, d32)] + [rel(m16, m32)]
    print("controlnet full-size: max rel err %.2e (fp16 floor max %.2e)" % (max(errs), max(floors)))
    assert len(down) == 12
    for x, f in zip(errs, floors):
        assert x < max(2 * f, 2e-3)


@pytest.mark.slow
def test_unet_full_size_matches_oracle():
    """SD-2.1-base topology (865.9 M parameters, random init), one view = 3 CFG samples at 64x64 latents."""
    from dreammat_b200.nets import UNet
    from dreammat_b200 import dense_ops as D
    ucfg = O.UNetConfig()
    wu = O.round_weights(O.random_unet_weights(ucfg, 7))
    assert sum(v.numel() for v in wu.values()) == 865910724
    g = torch.Generator().manual_seed(8)
    z = torch.randn(3, 4, 64, 64, generator=g)
    t = torch.tensor([250, 250, 250])
    ctx = torch.randn(3, 77, 1024, generator=g)
    with torch.no_grad():
        ref16 = O.unet_forward(wu, ucfg, Q(z), t, Q(ctx), q=Q)
    net = UNet(wu, ucfg)
    zp = D.pad_convert(z.permute(0, 2, 3, 1).contiguous().cuda(), 64)
    out = net.forward(zp, t.float().cuda(), ctx.half().cuda())
    e = rel(out, ref16)
    print(f"\nunet full-size: rel err vs fp16-emulating oracle {e:.2e}")
    assert e < TOL16
