"""Run the dominant kernels once each at north-star sizes (for `ncu --set full -k regex:...`)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.chdir(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dreammat_b200 import dense_ops as D, render_ops as R
from dreammat_b200._cabi import MaterialCfg
from dreammat_b200.scene import DataConfig, FixCameraSet, procedural_mesh, synthetic_envmap
from dreammat_b200.system import DreamMatMaterial, DreamMatMesh, RaytraceRender

dev = "cuda"
which = sys.argv[1] if len(sys.argv) > 1 else "all"
if which in ("all", "shade"):
    mesh = procedural_mesh(100000, 0.8, 0)
    geo = DreamMatMesh({"shape_init": "p"}, dev, mesh=mesh)
    mat = DreamMatMaterial({"diffuse_sample_num": 200, "specular_sample_num": 128}, dev, [synthetic_envmap(2048, 4096, 0)])
    ren = RaytraceRender({}, geo, mat, None, dev)
    cams = FixCameraSet(DataConfig(width=512, height=512), torch.Generator().manual_seed(0))
    c = cams.cameras(torch.tensor([3]))
    g = ren.gbuffer(c["rays_o"].to(dev), c["rays_d"].to(dev), c["mvp_mtx"].to(dev), c["w2c"].to(dev), 3)
    n = g["pn"]
    print("pn", n)
    f = torch.randn(n, 5, device=dev); fj = torch.randn(n, 5, device=dev)
    for _ in range(2):
        color, reg, _ = R.shade_mc(f, fj, g["pts"], g["nrm"], g["vd"], torch.rand(n, device=dev), torch.rand(n, device=dev),
                                   mat.mc_cfg, ren.ray_tracer, mat.light[0], mat.tab_d, mat.tab_s, want_aux=False)
        ff = R.hashgrid_mlp(g["pts"], geo.grid.detach().requires_grad_(True), geo.W1, geo.W2, geo.hg)
        ff.sum().backward()
    torch.cuda.synchronize()
if which in ("splitsum",):
    import bench
    sysm, cams = bench.build_system(dev, 512, 100000, (256, 512), 0, torch.float16, "splitsum")
    c = cams.cameras(torch.tensor([3]))
    g = sysm.renderer.gbuffer(c["rays_o"].to(dev), c["rays_d"].to(dev), c["mvp_mtx"].to(dev), c["w2c"].to(dev), 3)
    print("splitsum", bench.splitsum_kernel_roofline(sysm, bench.peaks()[0]))
if which in ("all", "dense"):
    x = torch.randn(8, 512, 512, 128, device=dev).half(); w = (torch.randn(128, 9 * 128, device=dev) * 0.03).half()
    gm = torch.ones(128, device=dev).half(); bt = torch.zeros(128, device=dev).half()
    for _ in range(2):
        y = D.conv2d(x, w, 3)
        D.groupnorm(x, gm, bt, silu=True)
    x2 = torch.randn(24, 16, 16, 1280, device=dev).half(); w2 = (torch.randn(1280, 9 * 1280, device=dev) * 0.01).half()
    x3 = torch.randn(24, 8, 8, 2560, device=dev).half(); w3 = (torch.randn(1280, 9 * 2560, device=dev) * 0.01).half()
    q = torch.randn(24, 4096, 960, device=dev).half()
    for _ in range(2):
        D.conv2d(x2, w2, 3); D.conv2d(x3, w3, 3)
        D.attention(q[..., :320], q[..., 320:640], q[..., 640:], 5)
    torch.cuda.synchronize()
print("done")
