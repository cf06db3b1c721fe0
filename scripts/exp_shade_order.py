"""Sample visiting orders for the MC shader, applied by permuting the direction TABLES on the host (no per-sample
indirection in the kernel): identity (Fibonacci: elevation-sorted, azimuth golden-angle spread), azimuth-sorted,
Morton on the projected disk, azimuth-sector-major."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from dreammat_b200 import render_ops as R
from dreammat_b200.scene import DataConfig, FixCameraSet, procedural_mesh, synthetic_envmap
from dreammat_b200.system import DreamMatMaterial, DreamMatMesh, RaytraceRender
dev = "cuda"
mesh = procedural_mesh(100000, 0.8, 0)
geo = DreamMatMesh({"shape_init": "p"}, dev, mesh=mesh)
mat = DreamMatMaterial({"diffuse_sample_num": 200, "specular_sample_num": 128}, dev, [synthetic_envmap(2048, 4096, 0)])
ren = RaytraceRender({}, geo, mat, None, dev)
cams = FixCameraSet(DataConfig(width=512, height=512), torch.Generator().manual_seed(0))
def orders(tab):
    ua, ue = tab[:, 0].double().numpy(), tab[:, 1].double().numpy()
    n = len(ua)
    out = {"identity": np.arange(n), "azimuth": np.argsort(ua, kind="stable")}
    r = np.sqrt(np.clip(ue, 0, 1)); x, y = r * np.cos(2 * np.pi * ua), r * np.sin(2 * np.pi * ua)
    qx = np.clip(((x + 1) * 0.5 * 255).astype(np.int64), 0, 255); qy = np.clip(((y + 1) * 0.5 * 255).astype(np.int64), 0, 255)
    code = np.zeros_like(qx)
    for b in range(8):
        code |= ((qx >> b) & 1) << (2 * b) | ((qy >> b) & 1) << (2 * b + 1)
    out["morton"] = np.argsort(code, kind="stable")
    sector = np.floor(ua * 8).astype(np.int64)
    out["sector8"] = np.lexsort((ue, sector))
    out["reverse"] = np.arange(n)[::-1].copy()
    return out
od, os_ = orders(mat.tab_d.cpu()), orders(mat.tab_s.cpu())
for vid in (3, 40):
    c = cams.cameras(torch.tensor([vid]))
    g = ren.gbuffer(c["rays_o"].to(dev), c["rays_d"].to(dev), c["mvp_mtx"].to(dev), c["w2c"].to(dev), vid)
    n = g["pn"]
    gen = torch.Generator(device=dev).manual_seed(1)
    f = torch.randn(n, 5, device=dev, generator=gen); fj = torch.randn(n, 5, device=dev, generator=gen)
    rd, rs = torch.rand(n, device=dev, generator=gen), torch.rand(n, device=dev, generator=gen)
    for name in od:
        td = mat.tab_d[torch.from_numpy(od[name]).to(dev)].contiguous(); ts = mat.tab_s[torch.from_numpy(os_[name]).to(dev)].contiguous()
        def run():
            return R.shade_mc(f, fj, g["pts"], g["nrm"], g["vd"], rd, rs, mat.mc_cfg, ren.ray_tracer, mat.light[0], td, ts,
                              want_aux=False)[0]
        for _ in range(2): col = run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5): col = run()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        print(f"view {vid} pn={n} order={name:10s}: {ms:.3f} ms  {n*328/ms/1e6:.2f} Grays/s  checksum {float(col.double().sum()):.4f}", flush=True)
