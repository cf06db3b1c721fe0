"""GPU parity of one whole SDS iteration (rows a3-a9): hash grid -> MC shading -> canvas -> VAE ->
ControlNet + UNet -> CSD -> backward -> Adam, against the CPU oracle on identical inputs and randomness.

Run at a reduced configuration (64x64 render, 2 views, narrow networks) that the oracle finishes in
seconds; the 512x512 / 8-view configuration is exercised by bench.py.
"""
import pytest
import torch

from oracle import render as OR
from oracle import sd as OS
from tests._fixtures import make_scene, rel_err

pytestmark = pytest.mark.gpu
Q = lambda x: x.half().float()  # noqa: E731


def _small_nets():
    ucfg = OS.UNetConfig(block_out_channels=(64, 128, 128, 128), heads=(1, 2, 2, 2), cross_attention_dim=64)
    vcfg = OS.VAEConfig(block_out_channels=(64, 64, 64, 64))
    return (ucfg, vcfg, OS.round_weights(OS.random_unet_weights(ucfg, 0)), OS.round_weights(OS.random_controlnet_weights(ucfg, 1)),
            OS.round_weights(OS.random_vae_weights(vcfg, 2)))


def test_fused_step_matches_oracle():
    from dreammat_b200 import weights as Wt
    from dreammat_b200.guidance import PromptProcessorOutput, StableDiffusionLightGuidance
    from dreammat_b200.system import DreamMat, DreamMatMaterial, DreamMatMesh, RaytraceRender
    dev = "cuda"
    res, B = 64, 2
    sc = make_scene(res=res, subdiv=3, bump=0.12, seed=3, n_views=B)
    ucfg, vcfg, wu, wc, wv = _small_nets()
    g = torch.Generator().manual_seed(11)
    envs = [OR.synthetic_envmap(64, 128, seed=i) for i in range(5)]
    env_id = torch.tensor([1, 3])
    geo = DreamMatMesh({"shape_init": "x"}, dev, mesh=(sc["v"], sc["f"]), seed=5)
    # a livelier starting point than U(-1e-4, 1e-4) so that every factor of the chain rule is exercised
    geo.params[:geo.n_grid] = ((torch.rand(geo.n_grid, generator=g) * 2 - 1) * 0.5).to(dev)
    p0 = geo.params.detach().cpu().clone()
    mat = DreamMatMaterial({"diffuse_sample_num": 200, "specular_sample_num": 128, "use_bump": False}, dev, envs)
    ren = RaytraceRender({}, geo, mat, None, dev)
    gcfg = dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05, uncond_scale=-0.7,
                null_scale=-0.2, noise_scale=0.0)
    guid = StableDiffusionLightGuidance(gcfg, Wt.UNetConfig(**ucfg.__dict__), Wt.VAEConfig(**vcfg.__dict__), wu, wc, wv, dev)
    Dm = ucfg.cross_attention_dim
    vd, uvd, null = torch.randn(4, 77, Dm, generator=g), torch.randn(4, 77, Dm, generator=g), torch.randn(1, 77, Dm, generator=g)
    pu = PromptProcessorOutput(vd[:1], uvd[:1], null, vd, uvd)
    sysm = DreamMat(None, geo, mat, ren, guid, pu, dev)
    sysm.resize_to_vae = False   # reduced-size parity run: the oracle's guidance_step encodes the 64x64 render as is
    # per-view G-buffers from the oracle (the G-buffer kernel has its own parity test)
    gb = sc["gb"]
    views, rng = [], {"rand_ang": [], "normal_eps": [], "rand_d": [], "rand_s": []}
    for b in range(B):
        sel = gb["selector"][b]
        pix = torch.nonzero(sel).view(-1).int()
        v = dict(pix=pix, pts=gb["gb_pos"][b][sel], nrm=gb["gb_normal"][b][sel], vd=gb["gb_viewdirs"][b][sel])
        n = pix.shape[0]
        v.update(rand_ang=torch.rand(n, 1, generator=g), normal_eps=torch.randn(n, 1, generator=g) * 0.05,
                 rand_d=torch.rand(n, 1, 1, generator=g), rand_s=torch.rand(n, 1, 1, generator=g))
        views.append(v)
        # antialias pair list: the product's host precompute on the oracle's rasteriser output; the oracle applies
        # its own scalar restatement below
        from dreammat_b200 import antialias as AA
        import numpy as np
        d_, s_, a_ = AA.build_pairs(gb["rast"][b].numpy(), sc["v"].numpy(), sc["f"].numpy().astype(np.int64), ren._nbr_opp,
                                    sc["cam"]["mvp_mtx"][b].numpy())
        v["aa_oracle"] = OR.antialias_pairs(gb["rast"][b], sc["v"], sc["f"], sc["cam"]["mvp_mtx"][b])
        assert len(v["aa_oracle"]) == len(d_) > 10
        ren._cache[100 + b] = {"pix": pix.to(dev), "pn": n, "pts": v["pts"].to(dev).contiguous(), "nrm": v["nrm"].to(dev).contiguous(),
                               "vd": v["vd"].to(dev).contiguous(),
                               "aa": (torch.from_numpy(d_).to(dev), torch.from_numpy(s_).to(dev), torch.from_numpy(a_).to(dev))}
        for k in rng:
            rng[k].append(v[k])
    el, az, dist = torch.tensor([15.0, -10.0]), torch.tensor([30.0, 160.0]), torch.tensor([3.2, 3.6])
    t = torch.tensor([300, 650])
    noise, veps = torch.randn(B, 4, res // 8, res // 8, generator=g), torch.randn(B, 4, res // 8, res // 8, generator=g)
    cond = torch.rand(B, res, res, 22, generator=g)
    rng.update(t=t, noise=noise, vae_eps=veps)

    class _N:
        def __getitem__(self, i):
            return None
    batch = {"view_id": torch.tensor([100, 101]), "env_id": env_id, "height": res, "width": res, "rays_o": _N(), "rays_d": _N(),
             "mvp_mtx": sc["cam"]["mvp_mtx"].to(dev), "w2c": sc["cam"]["w2c"].to(dev), "elevation": el, "azimuth": az,
             "camera_distances": dist, "condition_map": cond.to(dev)}
    out = sysm.training_step_fused(batch, rng=rng)
    g_dev = geo.grads.detach().cpu().clone()
    p1 = geo.params.detach().cpu().clone()

    # ---------------- oracle (q = the storage-rounding hook: fp16 emulation like the product, or identity = pure fp32)
    meta, _ = OR.hashgrid_meta()

    def oracle_step(q):
        P = p0.clone().requires_grad_(True)
        grid, W1, W2 = P[:geo.n_grid], P[geo.n_grid:geo.n_grid + geo.n_w1].view(64, 32), P[geo.n_grid + geo.n_w1:].view(5, 64)
        canv, ms, mjs = [], [], []
        for b, v in enumerate(views):
            f = OR.geometry_forward(v["pts"], grid, W1, W2, meta)
            fj = OR.geometry_forward(OR.jitter_positions(v["pts"], v["nrm"], v["rand_ang"], v["normal_eps"]), grid, W1, W2, meta)
            al, me, ro, _ = OR.material_params(f, fj)
            ms.append(torch.sigmoid(f)); mjs.append(torch.sigmoid(fj))
            o = OR.shade_raytracing(v["pts"], v["nrm"], v["vd"], envs[int(env_id[b])], me, ro, al, v["rand_d"], v["rand_s"],
                                    lambda oo, dd: sc["tracer"].trace(oo, dd)[1])
            c = torch.ones(res * res, 3)
            c = c.index_put((v["pix"].long(),), o["color"])
            c = OR.antialias_apply(c, v["aa_oracle"])
            canv.append(c.view(1, res, res, 3))
        comp = torch.cat(canv, 0)
        reg = OR.material_smoothness_grad(torch.cat(ms), torch.cat(mjs))
        ctx3 = q(pu.get_text_embeddings(el, az, dist, True, return_null_text_embeddings=True))
        loss_sds, grad_o, _ = OS.guidance_step(wv, wc, wu, ucfg, vcfg, comp, cond, ctx3, t, noise, veps,
                                               scales=(1.05, -0.7, -0.2, 0.0), cond_scale=1.0, q=q)
        (loss_sds + reg).backward()
        return P, comp, reg, loss_sds
    P, comp, reg, loss_sds = oracle_step(Q)
    P32, _, _, loss32 = oracle_step(OS.Ident)
    # what fp16 storage itself costs on this chain, measured by the oracle: fp16-emulating vs pure fp32
    floor_g = rel_err(P.grad, P32.grad)
    floor_l = abs(float(loss_sds) - float(loss32)) / abs(float(loss32))
    opt = torch.optim.Adam([P], lr=0.01, betas=(0.9, 0.99), eps=1e-15)
    opt.step()
    e_rgb = rel_err(out["comp_rgb"].cpu(), comp.detach())
    e_ls = abs(float(out["loss_sds"]) - float(loss_sds)) / abs(float(loss_sds))
    e_lr = abs(float(out["loss_mat_reg"]) - float(reg)) / abs(float(reg))
    e_g = rel_err(g_dev, P.grad)
    e_p = rel_err(p1 - p0, P.detach() - p0)
    big = P.grad.abs() > 1e-3 * P.grad.abs().max()
    e_pb = rel_err((p1 - p0)[big], (P.detach() - p0)[big])
    print(f"\nfused step small (fp16 mode): rgb {e_rgb:.2e} loss_sds {e_ls:.2e} (fp16 floor {floor_l:.2e}) mat_reg {e_lr:.2e} "
          f"param-grad {e_g:.2e} (fp16 floor {floor_g:.2e}) adam-update {e_p:.2e}, {e_pb:.2e} where |g| > 1e-3 max")
    assert e_rgb < 1e-3           # north_star: 1e-3 relative on rendered RGB (fp32 path)
    assert e_lr < 1e-4
    # loss_sds = 0.5 |grad|^2 / B: its relative error is at most 2x that of the SDS gradient, which in fp16 mode sits at ~1e-2
    # (fp16 floor).  Measured: 7e-4, 1.4e-3 and once more than 2e-3; the oracle's own fp16-vs-fp32 figure (floor_l) is a single noisy draw.
    assert e_ls < max(4 * floor_l, 1e-2), (e_ls, floor_l)
    # fp16 mode: the parameter gradient inherits the fp16 noise of the CSD combination (the three branches nearly cancel);
    # the bound is 2x the floor the oracle itself measures between fp16 emulation and fp32.  The fp32 mode of the same
    # step is held to 1e-3 in test_gpu_config1.py.
    assert e_g < 2 * floor_g, (e_g, floor_g)
    # Adam's first step with eps=1e-15 is sign-like (|update| = lr whatever |g|): a coordinate whose fp16-noisy gradient
    # changes sign moves by 2 lr.  Compared where the oracle's gradient is not ~0; bound = the sign-flip rate fp16 noise allows
    assert e_pb < max(4 * floor_g, 5e-2)


def test_training_step_runs_through_autograd_wrappers():
    """API parity path: renderer(**batch) -> guidance(...) -> loss.backward() like systems/dreammat.py:57-86."""
    from dreammat_b200 import weights as Wt
    from dreammat_b200.guidance import PromptProcessorOutput, StableDiffusionLightGuidance
    from dreammat_b200.scene import DataConfig, FixCameraSet
    from dreammat_b200.system import DreamMatMaterial, DreamMatMesh, RaytraceRender
    dev = "cuda"
    res = 64
    v, f = OR.icosphere(3, 0.8, 0.1)
    geo = DreamMatMesh({"shape_init": "x"}, dev, mesh=(v, f))
    mat = DreamMatMaterial({"diffuse_sample_num": 200, "specular_sample_num": 128}, dev, [OR.synthetic_envmap(64, 128, i) for i in range(5)])
    ren = RaytraceRender({}, geo, mat, None, dev)
    ucfg, vcfg, wu, wc, wv = _small_nets()
    guid = StableDiffusionLightGuidance(dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0]),
                                        Wt.UNetConfig(**ucfg.__dict__), Wt.VAEConfig(**vcfg.__dict__), wu, wc, wv, dev)
    cams = FixCameraSet(DataConfig(width=res, height=res), torch.Generator().manual_seed(0))
    vid, eid = cams.collate(torch.Generator().manual_seed(1), 2)
    batch = {k: (x.to(dev) if torch.is_tensor(x) else x) for k, x in cams.cameras(vid).items()}
    out = ren(env_id=eid, view_id=vid, **batch)
    assert set(out) >= {"comp_rgb", "opacity", "comp_depth", "comp_normal", "albedo", "metalness", "roughness",
                        "specular_light", "diffuse_light", "specular_color", "diffuse_color", "loss_mat_reg"}
    assert out["comp_rgb"].shape == (2, res, res, 3)
    D = ucfg.cross_attention_dim
    pu = PromptProcessorOutput(torch.randn(1, 77, D), torch.randn(1, 77, D), torch.randn(1, 77, D), torch.randn(4, 77, D), torch.randn(4, 77, D))
    # the reference resizes non-512 renders to 512 before the VAE; feed latents-sized path via encode_images directly
    lat = guid.encode_images(out["comp_rgb"])
    ctx3 = pu.get_text_embeddings(batch["elevation"].cpu(), batch["azimuth"].cpu(), batch["camera_distances"].cpu(), True, True)
    grad, dlat, sums = guid.compute_grad_sds(lat, torch.rand(2, res, res, 22, device=dev), ctx3)
    from dreammat_b200.guidance import _SDSLoss
    loss = _SDSLoss.apply(lat, dlat, sums[0] / 2) + out["loss_mat_reg"]
    loss.backward()
    # the gradients land on the autograd leaves that alias the flat parameter buffer -- hash grid AND both MLP matrices --
    # and optimizer_step(from_autograd=True) consumes them (fused Adam on the flat buffer)
    leaves = geo.autograd_leaves()
    for leaf in leaves:
        assert leaf.grad is not None and torch.isfinite(leaf.grad).all() and float(leaf.grad.abs().sum()) > 0
    from dreammat_b200.system import DreamMat
    sysm = DreamMat(None, geo, mat, ren, guid, pu, dev)
    p_before = geo.params.clone()
    g_w2 = leaves[2].grad.clone()
    sysm.optimizer_step(from_autograd=True)
    assert torch.equal(geo.dW2, g_w2) and all(leaf.grad is None for leaf in leaves)
    moved = (geo.params != p_before)
    assert bool(moved[:geo.n_grid].any()) and bool(moved[geo.n_grid:].all())     # every MLP weight gets a gradient
