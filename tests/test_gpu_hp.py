"""GPU parity of the high-precision dense mode (fp32 storage, `half_precision_weights=false`,
dreammat_guidance.py:56,92-94) against the PURE fp32 oracle.

north_star asks for 1e-3 relative on the SDS gradient.  In the reference's default fp16 mode the CSD
combination amplifies the fp16 storage noise ~10x (see test_gpu_dense.py), so that bound is tested where
it is meaningful: with rounding taken away.  The contractions still run on the wgmma kernel (bf16
operands split 3-way, csrc/dense_hp.cu), so these tests also show that the kernels themselves -- tiling,
implicit-GEMM tap walk, split-K, epilogues -- are exact to fp32 accumulation order.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import sd as O

pytestmark = pytest.mark.gpu
TOL = 1e-3          # north_star tolerance
TIGHT = 2e-5        # what fp32 re-association actually gives on single ops


def rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def nchw(x_nhwc, c=None):
    x = x_nhwc.float().permute(0, 3, 1, 2)
    return x if c is None else x[:, :c]


def test_hp_gemm_conv_attention_match_fp64():
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    errs = {}
    for (M, N, K) in ((300, 200, 192), (4096, 640, 640), (192, 1280, 5120), (513, 768, 1024)):
        a, b, bias, res = rn(M, K), rn(N, K) * 0.05, rn(N), rn(M, N)
        out = D.gemm(a, b, bias=bias, residual=res, act="silu")
        ref = F.silu(a.double() @ b.double().t() + bias.double()) + res.double()
        errs[f"gemm{M}x{N}x{K}"] = rel(out, ref)
    # wide dynamic range: the 3-way split must not lose small operands next to large ones
    a = rn(256, 256) * torch.logspace(-4, 4, 256, device="cuda")[None]
    b = rn(128, 256) * torch.logspace(3, -3, 256, device="cuda")[None]
    errs["gemm_range"] = rel(D.gemm(a, b), a.double() @ b.double().t())
    # batched with strided operands (the VAE attention's q k^T and P V)
    qkv = rn(2, 256, 3 * 128)
    S = D.gemm(qkv[..., :128], qkv[..., 128:256])
    errs["bgemm"] = rel(S, qkv[..., :128].double() @ qkv[..., 128:256].double().transpose(1, 2))
    # GEGLU epilogue
    a, w, bias = rn(300, 192), rn(512, 192) / 14, rn(512)
    out = D.gemm(a, D.geglu_interleave(w), bias=D.geglu_interleave(bias), act="geglu")
    pr = a.double() @ w.double().t() + bias.double()
    errs["geglu"] = rel(out, pr[:, :256] * F.gelu(pr[:, 256:]))
    # convolutions: 3x3 stride 1 / stride 2 with the VAE's (0,1,0,1) padding / few-tile long-K (split-K) / rowvec
    x, w = rn(2, 32, 32, 128), rn(192, 128, 3, 3) / 34
    errs["conv3"] = rel(nchw(D.conv2d(x, D.conv_weight_to_gemm(w, dtype=torch.float32), 3)),
                        F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), padding=1))
    y = D.conv2d(x, D.conv_weight_to_gemm(w, dtype=torch.float32), 3, stride=2, pad=(0, 0), out_hw=(16, 16))
    errs["conv3s2"] = rel(nchw(y), F.conv2d(F.pad(x.double().permute(0, 3, 1, 2), (0, 1, 0, 1)), w.double(), stride=2))
    x, w, tp = rn(3, 8, 8, 1280), rn(1280, 1280, 3, 3) / 100, rn(3, 1280)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), padding=1) + tp.double()[:, :, None, None]
    for _ in range(2):
        errs["conv_splitk"] = rel(nchw(D.conv2d(x, D.conv_weight_to_gemm(w, dtype=torch.float32), 3, rowvec=tp)), ref)
    for (B, heads, Nq, Nk) in ((2, 5, 1024, 1024), (2, 20, 64, 77), (1, 2, 300, 4096)):
        q, k, v = rn(B, Nq, heads * 64), rn(B, Nk, heads * 64), rn(B, Nk, heads * 64)
        sp = lambda t, n: t.double().view(B, n, heads, 64).transpose(1, 2)  # noqa: E731
        ref = F.scaled_dot_product_attention(sp(q, Nq), sp(k, Nk), sp(v, Nk)).transpose(1, 2).reshape(B, Nq, -1)
        errs[f"attn{Nq}x{Nk}"] = rel(D.attention(q, k, v, heads), ref)
    print("\nhp ops rel err vs fp64:", " ".join(f"{k}={v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < TIGHT, errs


def test_hp_streaming_kernels_match_torch():
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(1)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    errs = {}
    x = (rn(2, 16, 16, 128) * 3 + 1).requires_grad_(True)
    gm, bt = 1 + 0.1 * rn(128), 0.1 * rn(128)
    for silu in (False, True):
        y, st = D.groupnorm(x.detach(), gm, bt, 32, 1e-6, silu=silu)
        r = F.group_norm(x.permute(0, 3, 1, 2), 32, gm, bt, 1e-6)
        r = (F.silu(r) if silu else r).permute(0, 2, 3, 1)
        errs[f"gn{int(silu)}"] = rel(y, r)
        dz, add = rn(2, 16, 16, 128), rn(2, 16, 16, 128)
        (gx,) = torch.autograd.grad(r, x, dz)
        errs[f"gnbwd{int(silu)}"] = rel(D.groupnorm_bwd(x.detach(), dz, gm, bt, st, 32, 1e-6, silu=silu, dx_add=add), gx + add)
    h = rn(300, 320)
    errs["ln"] = rel(D.layernorm(h, gm.repeat(3)[:320].contiguous(), bt.repeat(3)[:320].contiguous()),
                     F.layer_norm(h, (320,), gm.repeat(3)[:320], bt.repeat(3)[:320], 1e-5))
    hh = rn(100, 512)
    errs["geglu"] = rel(D.geglu(hh), hh[:, :256] * F.gelu(hh[:, 256:]))
    xs = rn(2, 8, 8, 64)
    errs["up"] = rel(nchw(D.upsample2x(xs)), F.interpolate(xs.permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest"))
    zi = D.upsample2x(xs, zero_insert=True)
    errs["zins"] = rel(zi[:, ::2, ::2], xs) + float(zi[:, 1::2].abs().max()) + float(zi[:, :, 1::2].abs().max())
    cat = torch.zeros(64, 192, device="cuda")
    D.axpby(xs.view(-1, 64)[:64], 1.0, xs.view(-1, 64)[64:128], 0.5, out=cat[:, 64:128])
    errs["axpby"] = rel(cat[:, 64:128], xs.view(-1, 64)[:64] + 0.5 * xs.view(-1, 64)[64:128]) + float(cat[:, :64].abs().max())
    t3 = rn(2, 70, 50)
    errs["transpose"] = rel(D.transpose(t3), t3.transpose(1, 2))
    sm = rn(64, 333)
    P = D.softmax_rows(sm, 0.3)
    errs["softmax"] = rel(P, torch.softmax(sm * 0.3, -1))
    dP = rn(64, 333)
    errs["softmax_bwd"] = rel(D.softmax_bwd(P, dP, 0.3), 0.3 * P * (dP - (P * dP).sum(-1, keepdim=True)))
    rgb = torch.rand(2, 8, 8, 3, device="cuda", generator=g)
    pc = D.pad_convert(rgb, 64, 2.0, -1.0, torch.float32)
    errs["pad"] = rel(pc[..., :3], rgb * 2 - 1) + float(pc[..., 3:].abs().max())
    errs["unpad"] = rel(D.unpad_convert(pc, 3, 0.5), (rgb * 2 - 1) * 0.5)
    print("\nhp streaming rel err:", " ".join(f"{k}={v:.1e}" for k, v in errs.items()))
    assert max(errs.values()) < TIGHT, errs


@pytest.fixture(scope="module")
def small32():
    ucfg = O.UNetConfig(block_out_channels=(64, 128, 256, 256), heads=(1, 2, 4, 4), cross_attention_dim=128)
    vcfg = O.VAEConfig(block_out_channels=(64, 64, 128, 128))
    return ucfg, vcfg, O.random_unet_weights(ucfg, 0), O.random_controlnet_weights(ucfg, 1), O.random_vae_weights(vcfg, 2)


def test_hp_guidance_step_matches_fp32_oracle(small32):
    """a7-a9 at fp32: latents, the three eps branches, SDS gradient, loss and d loss / d rgb each <= 1e-3."""
    from dreammat_b200.guidance import PromptProcessorOutput, StableDiffusionLightGuidance, _SDSLoss
    ucfg, vcfg, wu, wc, wv = small32
    g = torch.Generator().manual_seed(6)
    B, R = 2, 128
    Dm = ucfg.cross_attention_dim
    rgb, cond = torch.rand(B, R, R, 3, generator=g), torch.rand(B, R, R, 22, generator=g)
    vd, uvd, null = torch.randn(4, 77, Dm, generator=g), torch.randn(4, 77, Dm, generator=g), torch.randn(1, 77, Dm, generator=g)
    pu = PromptProcessorOutput(vd[:1], uvd[:1], null, vd, uvd)
    el, az, dist = torch.tensor([10.0, 70.0]), torch.tensor([20.0, -170.0]), torch.tensor([3.5, 3.5])
    t = torch.tensor([321, 777])
    noise, veps = torch.randn(B, 4, R // 8, R // 8, generator=g), torch.randn(B, 4, R // 8, R // 8, generator=g)
    cfg = dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05, uncond_scale=-0.7,
               null_scale=-0.2, noise_scale=0.0, half_precision_weights=False)
    guid = StableDiffusionLightGuidance(cfg, ucfg, vcfg, wu, wc, wv, dtype=torch.float32)
    assert guid.weights_dtype == torch.float32
    rgb_c = rgb.cuda().requires_grad_(True)
    lat = guid.encode_images(rgb_c, veps.cuda())
    ctx3 = pu.get_text_embeddings(el, az, dist, True, return_null_text_embeddings=True)
    eps = guid.predict_noise(lat.detach(), t.cuda(), noise.cuda(), ctx3, cond.cuda(), 1.0)
    grad, dlat, sums = guid.compute_grad_sds(lat, cond.cuda(), ctx3, t.cuda(), noise.cuda())
    _SDSLoss.apply(lat, dlat, sums[0] / B).backward()
    rgb_o = rgb.clone().requires_grad_(True)
    loss_o, grad_o, z_o, eps_o = O.guidance_step(wv, wc, wu, ucfg, vcfg, rgb_o, cond, ctx3, t, noise, veps,
                                                 scales=(1.05, -0.7, -0.2, 0.0), cond_scale=1.0, return_eps=True)
    loss_o.backward()
    e = {"latents": rel(lat, z_o), "eps_text": rel(eps[0], eps_o[0]), "eps_uncond": rel(eps[1], eps_o[1]),
         "eps_null": rel(eps[2], eps_o[2]), "sds_grad": rel(grad, grad_o),
         "loss": abs(float(sums[0] / B) - float(loss_o)) / abs(float(loss_o)), "d_rgb": rel(rgb_c.grad, rgb_o.grad)}
    print("\nhp guidance small (fp32 oracle):", " ".join(f"{k}={v:.2e}" for k, v in e.items()))
    assert max(e.values()) < TOL, e


@pytest.mark.slow
def test_hp_full_size_vae_512_and_controlnet_64():
    """Full-size SD-2.1-base VAE encoder fwd + input gradient at 512^2 and full-size ControlNet (22-channel condition)
    at 64^2 latents, fp32 mode vs the pure fp32 oracle: <= 1e-3 (measured values printed)."""
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import ControlNet, VAEEncoder
    vcfg, ucfg = O.VAEConfig(), O.UNetConfig()
    wv = O.random_vae_weights(vcfg, 2)
    g = torch.Generator().manual_seed(5)
    rgb = torch.rand(1, 512, 512, 3, generator=g)
    eps = torch.randn(1, 4, 64, 64, generator=g)
    x = (rgb * 2 - 1).permute(0, 3, 1, 2).clone().requires_grad_(True)
    mom_r = O.vae_encode_moments(wv, vcfg, x)
    z_r = O.vae_sample(mom_r, eps, vcfg.scaling_factor)
    dz = torch.randn(z_r.shape, generator=g)
    z_r.backward(dz)
    vae = VAEEncoder(wv, vcfg, dtype=torch.float32)
    tape = []
    mom = vae.encode_moments(D.pad_convert(rgb.cuda(), 64, 2.0, -1.0, torch.float32), tape)
    z = D.vae_sample(mom, eps.cuda(), vcfg.scaling_factor)
    dx = vae.backward_input(tape, D.vae_sample_bwd(mom, eps.cuda(), dz.cuda(), vcfg.scaling_factor))
    e = {"vae_moments": rel(nchw(mom, 8), mom_r), "vae_latents": rel(z, z_r), "vae_input_grad": rel(nchw(dx, 3), x.grad)}
    del vae, tape, mom, dx
    torch.cuda.empty_cache()
    wc = O.random_controlnet_weights(ucfg, 1)
    zz = torch.randn(3, 4, 64, 64, generator=g)
    t = torch.tensor([400, 400, 400])
    ctx = torch.randn(3, 77, 1024, generator=g)
    cond = torch.rand(1, 22, 512, 512, generator=g)
    with torch.no_grad():
        down_r, mid_r = O.controlnet_forward(wc, ucfg, zz, t, ctx, cond, 0.8)
    net = ControlNet(wc, ucfg, dtype=torch.float32)
    down, mid = net.forward(D.pad_convert(zz.permute(0, 2, 3, 1).contiguous().cuda(), 64, dtype=torch.float32), t.float().cuda(),
                            ctx.cuda(), D.pad_convert(cond.permute(0, 2, 3, 1).contiguous().cuda(), 64, dtype=torch.float32), 0.8)
    errs = [rel(nchw(a), b) for a, b in zip(down, down_r)] + [rel(nchw(mid), mid_r)]
    e["controlnet_max"] = max(errs)
    print("\nhp full-size (fp32 oracle):", " ".join(f"{k}={v:.2e}" for k, v in e.items()))
    assert max(e.values()) < TOL, e
