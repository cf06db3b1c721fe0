"""GPU parity: render-side kernels (C-ABI, through ctypes) vs the CPU oracle on seeded inputs.

Tolerances (fp32 path): 1e-3 relative (L2 over the tensor) on rendered RGB and on gradients,
as BASELINE.json's north_star states; integer / index outputs must match exactly.
"""
import numpy as np
import pytest
import torch

from oracle import render as O
from tests._fixtures import make_scene, rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(scope="module")
def ops():
    from dreammat_b200 import render_ops
    from dreammat_b200._cabi import lib, check
    check(lib().dm_device_check(0), "dm_device_check")
    return render_ops


@pytest.fixture(scope="module")
def scene():
    return make_scene(res=48, subdiv=3, bump=0.12, seed=0)


def cu(t):
    return t.cuda().contiguous()


def test_bvh_closest_hit_matches_oracle(ops):
    v, f = O.icosphere(3, radius=0.8, bump=0.15)
    g = torch.Generator().manual_seed(3)
    ro = torch.randn(20000, 3, generator=g) * 0.7
    rd = torch.nn.functional.normalize(torch.randn(20000, 3, generator=g), dim=-1)
    t0, i0, uv0 = O.RayTracer(v.numpy(), f.numpy()).trace_raw(ro.numpy(), rd.numpy())
    bvh = ops.Bvh(v, f)
    t1, i1, uv1 = bvh.trace(cu(ro), cu(rd))
    i1 = i1.cpu().numpy()
    mism = (i0 != i1)
    # FMA contraction on the device can flip rays that graze an edge; they must be rare
    assert mism.mean() < 2e-3, mism.mean()
    ok = ~mism & (i0 >= 0)
    assert np.abs(t0[ok] - t1.cpu().numpy()[ok]).max() < 1e-4
    assert np.abs(uv0[ok] - uv1.cpu().numpy()[ok]).max() < 1e-3
    assert np.all(t1.cpu().numpy()[i1 < 0] == 10.0)


def test_gbuffer_matches_oracle(ops, scene):
    sc = scene
    bvh = ops.Bvh(sc["v"], sc["f"])
    cam = sc["cam"]
    rast, gb_pos, gb_nrm, mask, comp_normal = ops.raster_gbuffer(bvh, cu(sc["v"]), cu(sc["vn"]), cu(sc["f"]),
                                                                 cu(cam["rays_o"]), cu(cam["rays_d"]),
                                                                 cu(cam["mvp_mtx"]), cu(cam["w2c"]))
    gb = sc["gb"]
    m0 = gb["selector"].numpy().astype(bool)
    m1 = mask.cpu().numpy().astype(bool)
    assert (m0 != m1).mean() < 1e-3
    both = torch.from_numpy(m0 & m1)
    assert (rast.cpu()[..., 3].reshape(1, -1)[both] == gb["rast"][..., 3].reshape(1, -1)[both]).float().mean() > 0.999
    assert rel_err(gb_pos.cpu()[both], gb["gb_pos"][both]) < 1e-4
    assert rel_err(gb_nrm.cpu()[both], gb["gb_normal"][both]) < 1e-3
    assert rel_err(comp_normal.cpu().reshape(1, -1, 3)[both], gb["comp_normal"].reshape(1, -1, 3)[both]) < 1e-3
    idx = ops.compact_mask(mask)
    assert torch.equal(idx.cpu().long(), torch.nonzero(mask.cpu().view(-1)).view(-1))
    d = ops.depth_normalize(rast, mask).cpu().view(-1)
    d0 = gb["comp_depth"].reshape(-1)
    assert float((d - d0)[both.view(-1)].abs().max()) < 2e-3


def test_hashgrid_encode_and_mlp_match_oracle(ops):
    cfg = ops.default_hashgrid_cfg()
    n_params, offs = ops.hashgrid_num_params(cfg)
    assert n_params == 12599920
    meta, total = O.hashgrid_meta()
    assert offs[:-1] == [m["offset"] for m in meta] and offs[-1] == total
    g = torch.Generator().manual_seed(0)
    grid = (torch.rand(n_params, generator=g) * 2 - 1) * 0.1
    W1 = (torch.rand(64, 32, generator=g) * 2 - 1) / 32 ** 0.5
    W2 = (torch.rand(5, 64, generator=g) * 2 - 1) / 8
    pts = torch.rand(777, 3, generator=g) * 1.9 - 0.95
    pts[:5] = torch.tensor([[-1.03, 0.2, 0.3], [1.02, -1.01, 0.5], [0.0, 0.0, 0.0], [1.0, 1.0, 1.0], [-1.0, -1.0, -1.0]])
    enc_o = O.hashgrid_encode((pts + 1) / 2, grid, meta)
    enc_c = ops.hashgrid_encode(cu(pts), cu(grid), cfg).cpu()
    assert rel_err(enc_c, enc_o) < 2e-4  # fine levels (scale 4096) amplify the fp32 rounding of pos = x*scale+0.5
    gp = grid.clone().requires_grad_(True)
    w1, w2 = W1.clone().requires_grad_(True), W2.clone().requires_grad_(True)
    fo = O.geometry_forward(pts, gp, w1, w2, meta)
    dout = torch.randn(fo.shape, generator=g)
    fo.backward(dout)
    gc, w1c, w2c = cu(grid).requires_grad_(True), cu(W1).requires_grad_(True), cu(W2).requires_grad_(True)
    fc = ops.hashgrid_mlp(cu(pts), gc, w1c, w2c, cfg)
    assert rel_err(fc.detach().cpu(), fo.detach()) < 2e-4
    fc.backward(cu(dout))
    assert rel_err(gc.grad.cpu(), gp.grad) < 1e-4
    assert rel_err(w1c.grad.cpu(), w1.grad) < 1e-4
    assert rel_err(w2c.grad.cpu(), w2.grad) < 1e-4


def test_hashgrid_empty_and_ragged(ops):
    cfg = ops.default_hashgrid_cfg()
    n_params, _ = ops.hashgrid_num_params(cfg)
    grid = torch.zeros(n_params, device="cuda")
    W1 = torch.zeros(64, 32, device="cuda")
    W2 = torch.zeros(5, 64, device="cuda")
    for n in (0, 1, 63, 65):
        out = ops.hashgrid_mlp(torch.zeros(n, 3, device="cuda"), grid, W1, W2, cfg)
        assert out.shape == (n, 5) and float(out.abs().sum()) == 0.0


def test_jitter_matches_oracle(ops, scene):
    sc = scene
    pj = O.jitter_positions(sc["pts"], sc["nrm"], sc["rand_ang"], sc["normal_eps"])
    pc = ops.jitter_positions(cu(sc["pts"]), cu(sc["nrm"]), cu(sc["rand_ang"]), cu(sc["normal_eps"])).cpu()
    assert float((pc - pj).abs().max()) < 1e-6


def _oracle_mc(sc, f, fj):
    albedo, metallic, rough, reg = O.material_params(f, fj, use_raytracing=True)
    out = O.shade_raytracing(sc["pts"], sc["nrm"], sc["vd"], sc["env"], metallic, rough, albedo, sc["rand_d"],
                             sc["rand_s"], lambda o, d: sc["tracer"].trace(o, d)[1])
    return out, reg


def test_shade_mc_forward_backward_match_oracle(ops, scene):
    from dreammat_b200._cabi import MaterialCfg
    sc = scene
    f = sc["features"].clone().requires_grad_(True)
    fj = sc["features_jitter"].clone().requires_grad_(True)
    out, reg = _oracle_mc(sc, f, fj)
    g = torch.Generator().manual_seed(5)
    dcol = torch.randn(out["color"].shape, generator=g)
    ((out["color"] * dcol).sum() + 3.0 * reg).backward()

    cfg = MaterialCfg(0.0, 0.9, 0.01, 0.9, 200, 128)
    bvh = ops.Bvh(sc["v"], sc["f"])
    env = ops.envmap_pack(cu(sc["env"]))
    tab_d, tab_s = cu(ops.direction_tables(200)), cu(ops.direction_tables(128))
    assert torch.equal(tab_d.cpu(), O.direction_tables(200)) and torch.equal(tab_s.cpu(), O.direction_tables(128))
    fc, fjc = cu(sc["features"]).requires_grad_(True), cu(sc["features_jitter"]).requires_grad_(True)
    color, regc, aux = ops.shade_mc(fc, fjc, cu(sc["pts"]), cu(sc["nrm"]), cu(sc["vd"]), cu(sc["rand_d"]),
                                    cu(sc["rand_s"]), cfg, bvh, env, tab_d, tab_s)
    assert rel_err(color.detach().cpu(), out["color"].detach()) < TOL
    assert abs(float(regc) - float(reg)) < 1e-6 + 1e-4 * abs(float(reg))
    for k in ("albedo", "roughness", "metalness", "specular_lights", "diffuse_lights", "specular_colors",
              "diffuse_colors"):
        assert rel_err(aux[k].cpu(), out[k].detach()) < TOL, k
    ((color * cu(dcol)).sum() + 3.0 * regc).backward()
    assert rel_err(fc.grad.cpu(), f.grad) < 5 * TOL
    assert rel_err(fjc.grad.cpu(), fj.grad) < TOL


def test_shade_mc_occlusion_bits_match_oracle(ops, scene):
    """The any-hit result per sample (integer work) must agree with the oracle's closest-hit mask."""
    import ctypes as C
    from dreammat_b200._cabi import MaterialCfg, lib, check, ptr, stream_ptr
    sc = scene
    out, _ = _oracle_mc(sc, sc["features"], sc["features_jitter"])
    hit_o = out["_hit"].numpy()
    cfg = MaterialCfg(0.0, 0.9, 0.01, 0.9, 200, 128)
    bvh = ops.Bvh(sc["v"], sc["f"])
    env = ops.envmap_pack(cu(sc["env"]))
    n = sc["pn"]
    color = torch.empty(n, 3, device="cuda")
    jac = torch.empty(n, 9, device="cuda")
    bits = torch.zeros(n, 11, device="cuda", dtype=torch.int32)
    args = [cu(sc[k]) for k in ("pts", "nrm", "vd", "features", "features_jitter")]
    rd, rs = cu(sc["rand_d"]).view(-1), cu(sc["rand_s"]).view(-1)
    tab_d, tab_s = cu(ops.direction_tables(200)), cu(ops.direction_tables(128))
    check(lib().dm_shade_mc_fwd(C.byref(cfg), bvh.h, ptr(env), env.shape[0], env.shape[1], ptr(tab_d), ptr(tab_s),
                                *[ptr(a) for a in args], ptr(rd), ptr(rs), n, ptr(color), ptr(jac), None,
                                *([None] * 7), ptr(bits), stream_ptr()), "dm_shade_mc_fwd")
    b = bits.cpu().numpy().astype(np.uint32)
    hit_c = ((b[:, :, None] >> np.arange(32, dtype=np.uint32)[None, None, :]) & 1).reshape(n, -1)[:, :328].astype(bool)
    assert (hit_c != hit_o).mean() < 2e-3


def test_shade_splitsum_forward_backward_match_oracle(ops, scene):
    from dreammat_b200._cabi import MaterialCfg
    sc = scene
    g = torch.Generator().manual_seed(9)
    diffuse, spec = O.build_envlight(sc["env"], scale=2.0, max_res=32, min_res=8)
    lut = torch.rand(64, 64, 2, generator=g)
    f = sc["features"].clone().requires_grad_(True)
    fj = sc["features_jitter"].clone().requires_grad_(True)
    albedo, metallic, rough, reg = O.material_params(f, fj, use_raytracing=False)
    out = O.shade_splitsum(sc["nrm"], sc["vd"], diffuse, spec, lut, metallic, rough, albedo)
    dcol = torch.randn(out["color"].shape, generator=g)
    ((out["color"] * dcol).sum() + 2.0 * reg).backward()
    cfg = MaterialCfg(0.0, 0.9, 0.1, 0.95, 200, 128)
    fc, fjc = cu(sc["features"]).requires_grad_(True), cu(sc["features_jitter"]).requires_grad_(True)
    color, regc, aux = ops.shade_splitsum(fc, fjc, cu(sc["nrm"]), cu(sc["vd"]), cfg, cu(lut), cu(diffuse),
                                          [cu(m) for m in spec])
    assert rel_err(color.detach().cpu(), out["color"].detach()) < TOL
    for k in ("albedo", "roughness", "metalness", "specular_lights", "diffuse_lights", "specular_colors",
              "diffuse_colors"):
        assert rel_err(aux[k].cpu(), out[k].detach()) < TOL, k
    ((color * cu(dcol)).sum() + 2.0 * regc).backward()
    assert rel_err(fc.grad.cpu(), f.grad) < 5 * TOL
    assert rel_err(fjc.grad.cpu(), fj.grad) < TOL


def test_scatter_canvas_roundtrip(ops):
    g = torch.Generator().manual_seed(0)
    n_pix = 1000
    pix = torch.randperm(n_pix, generator=g)[:300].sort().values.int()
    vals = torch.rand(300, 3, generator=g)
    v = cu(vals).requires_grad_(True)
    canvas = ops.scatter_canvas(v, cu(pix), n_pix)
    ref = torch.ones(n_pix, 3)
    ref[pix.long()] = vals
    assert torch.equal(canvas.detach().cpu(), ref)
    dc = torch.rand(n_pix, 3, generator=g)
    canvas.backward(cu(dc))
    assert torch.equal(v.grad.cpu(), dc[pix.long()])


def test_adam_matches_torch(ops):
    g = torch.Generator().manual_seed(0)
    n = 10007
    p0 = torch.randn(n, generator=g)
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=0.01, betas=(0.9, 0.99), eps=1e-15)
    p = cu(p0)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for step in range(1, 6):
        grad = torch.randn(n, generator=g) * (1.0 if step != 3 else 0.0)
        ref.grad = grad.clone()
        opt.step()
        ops.adam_step(p, cu(grad), m, v, 0.01, 0.9, 0.99, 1e-15, step)
    assert rel_err(p.cpu(), ref.detach()) < 1e-6


def test_sds_combine_matches_formula(ops):
    g = torch.Generator().manual_seed(0)
    B = 3
    e = torch.randn(3, B, 4, 8, 8, generator=g)
    e[0, 0, 0, 0, 0] = float("nan")
    noise = torch.randn(B, 4, 8, 8, generator=g)
    w = torch.rand(B, generator=g)
    grad, dlat, sums = ops.sds_grad(cu(e), cu(noise), cu(w), 1.05, -0.7, -0.3, 0.1)
    ref = torch.nan_to_num(w.view(-1, 1, 1, 1) * (1.05 * e[0] - 0.7 * e[1] - 0.3 * e[2] + 0.1 * noise))
    assert rel_err(grad.cpu(), ref) < 1e-6
    assert rel_err(dlat.cpu(), ref / B) < 1e-6
    assert abs(float(sums[1]) ** 0.5 - float(ref.norm())) < 1e-3
    assert abs(float(sums[7]) ** 0.5 - float(noise.norm())) < 1e-3


def test_resize_bilinear_matches_torch(ops):
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(0)
    for (Hi, Wi, Ho, Wo) in ((64, 64, 32, 32), (24, 40, 32, 32), (32, 32, 32, 32), (100, 60, 37, 41)):
        x = torch.rand(2, Hi, Wi, 3, generator=g)
        xc = cu(x).requires_grad_(True)
        y = ops.resize_bilinear(xc, Ho, Wo)
        xr = x.clone().requires_grad_(True)
        ref = F.interpolate(xr.permute(0, 3, 1, 2), (Ho, Wo), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
        assert rel_err(y.detach().cpu(), ref.detach()) < 1e-6
        dy = torch.rand(ref.shape, generator=g)
        ref.backward(dy); y.backward(cu(dy))
        assert rel_err(xc.grad.cpu(), xr.grad) < 1e-5


def test_frontier_traversal_is_bit_identical_to_root_traversal():
    """The shared-origin frontier traversal (shade.cu: origin_frontier / anyhit_subtrees) visits exactly the boxes and
    triangles a root traversal would: occlusion bits, colours and Jacobians must be IDENTICAL."""
    import ctypes as C
    from dreammat_b200 import render_ops as R
    from dreammat_b200._cabi import MaterialCfg, check, lib, ptr, stream_ptr
    sc = make_scene(res=64, subdiv=4, bump=0.25, seed=7)
    dev = "cuda"
    bvh = R.Bvh(sc["v"], sc["f"])
    env = R.envmap_pack(sc["env"].to(dev))
    cfg = MaterialCfg(0.0, 0.9, 0.01, 0.9, 200, 128)
    tab_d, tab_s = R.direction_tables(200).to(dev), R.direction_tables(128).to(dev)
    n = sc["pn"]
    t = lambda x: x.to(dev).reshape(n, -1).contiguous()  # noqa: E731
    pts, nrm, vd, f, fj = t(sc["pts"]), t(sc["nrm"]), t(sc["vd"]), t(sc["features"]), t(sc["features_jitter"])
    rd, rs = t(sc["rand_d"]).view(-1), t(sc["rand_s"]).view(-1)
    outs = []
    try:
        for fr in (0, 1):
            check(lib().dm_tune(b"mc_frontier", fr), "dm_tune")
            color, jac, reg = torch.empty(n, 3, device=dev), torch.empty(n, 9, device=dev), torch.zeros(2, device=dev)
            bits = torch.zeros(n, (328 + 31) // 32, device=dev, dtype=torch.int32)
            check(lib().dm_shade_mc_fwd(C.byref(cfg), bvh.h, ptr(env), env.shape[0], env.shape[1], ptr(tab_d), ptr(tab_s), ptr(pts),
                                        ptr(nrm), ptr(vd), ptr(f), ptr(fj), ptr(rd), ptr(rs), n, ptr(color), ptr(jac), ptr(reg),
                                        *([None] * 7), ptr(bits), stream_ptr()), "dm_shade_mc_fwd")
            outs.append((color, jac, bits, reg))
    finally:
        lib().dm_tune(b"mc_frontier", 1)    # the library default
    (color0, jac0, bits0, reg0), (color1, jac1, bits1, reg1) = outs
    occ = int(sum(bin(int(x) & 0xffffffff).count("1") for x in bits0.flatten()[:4096].tolist()))
    assert occ > 0                      # the bumpy mesh self-occludes: the comparison is not vacuous
    assert torch.equal(bits1, bits0)    # every ray: the same any-hit result
    assert torch.equal(color1, color0) and torch.equal(jac1, jac0)   # same visiting order: the sums are bit-identical too
    assert torch.allclose(reg1, reg0, rtol=1e-5)
