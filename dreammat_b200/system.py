"""Host-side mirrors of the reference's geometry / material / renderer / system plugins.

    DreamMatMesh       <-> `dreammat-mesh`        models/geometry/dreammat_mesh.py:89-274
    DreamMatMaterial   <-> `dreammat-material`    models/materials/dreammat_material.py:346-797
    RaytraceRender     <-> `raytracing-renderer`  models/renderers/raytracing_renderer.py:86-222
    DreamMat           <-> `dreammat-system`      systems/dreammat.py:19-86 (+ systems/utils.py:34-53 Adam)

Same Config field names / defaults and the same call signatures and output keys; every tensor op on the
per-iteration path is a C-ABI kernel launch.  GPU-first departures (all result-preserving):
  * the mesh and the 128 training cameras are fixed, so each view's G-buffer (covered-pixel indices,
    positions, normals, view directions) is produced once and kept in HBM instead of re-rasterising it
    every iteration (128 views x ~105 k px x 40 B = 0.5 GB of 80 GB);
  * `DreamMat.training_step_fused` runs the iteration as an explicit forward/backward kernel sequence with
    one flat gradient buffer (what the multi-GPU all-reduce and the fused Adam operate on) instead of a
    torch autograd graph; `forward()` + autograd wrappers remain for API parity.
  * the silhouette antialias pass (dr.antialias, raytracing_renderer.py:127,147,199) depends only on the fixed
    G-buffer, so its (dst, src, weight) pair list is built once per view and applied as a sparse blend.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from . import antialias as AA
from . import render_ops as R
from ._cabi import MaterialCfg, check, lib, ptr, stream_ptr
from .scene import normalize_mesh, load_obj, vertex_normals


class DreamMatMesh:
    @dataclass
    class Config:
        # models/geometry/dreammat_mesh.py:93-121 (+ BaseGeometry radius)
        radius: float = 1.0
        n_input_dims: int = 3
        n_feature_dims: int = 5
        pos_encoding_config: dict = field(default_factory=lambda: {
            "otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19,
            "base_resolution": 16, "per_level_scale": 1.447269237440378})
        mlp_network_config: dict = field(default_factory=lambda: {
            "otype": "VanillaMLP", "activation": "ReLU", "output_activation": "none", "n_neurons": 64,
            "n_hidden_layers": 1})
        shape_init: str = ""
        shape_init_params: Optional[Any] = None
        shape_init_mesh_up: str = "+z"
        shape_init_mesh_front: str = "+x"

    def __init__(self, cfg: Optional[dict] = None, device="cuda", mesh=None, seed: int = 0):
        self.cfg = self.Config(**(cfg or {}))
        self.device = torch.device(device)
        if self.cfg.n_input_dims != 3:
            raise NotImplementedError("n_input_dims=2 (uv) is not selected by configs/dreammat.yaml")
        pe = self.cfg.pos_encoding_config
        self.hg = R.default_hashgrid_cfg(self.cfg.radius, pe["n_levels"], pe["log2_hashmap_size"], pe["base_resolution"],
                                         pe["per_level_scale"], self.cfg.mlp_network_config["n_neurons"],
                                         self.cfg.n_feature_dims)
        n_grid, _ = R.hashgrid_num_params(self.hg)
        self.n_grid = n_grid
        enc_dim = pe["n_levels"] * pe["n_features_per_level"]
        nh = self.cfg.mlp_network_config["n_neurons"]
        self.n_w1, self.n_w2 = nh * enc_dim, self.cfg.n_feature_dims * nh
        # ONE flat parameter / gradient / Adam-state buffer: [grid | W1 | W2] (16-byte aligned sub-buffers)
        self.n_params = n_grid + self.n_w1 + self.n_w2
        g = torch.Generator().manual_seed(seed)
        flat = torch.empty(self.n_params)
        flat[:n_grid] = torch.rand(n_grid, generator=g) * 2e-4 - 1e-4            # tcnn init U(-1e-4, 1e-4)
        b1, b2 = 1.0 / enc_dim ** 0.5, 1.0 / nh ** 0.5                             # nn.Linear default (kaiming a=sqrt 5)
        flat[n_grid:n_grid + self.n_w1] = (torch.rand(self.n_w1, generator=g) * 2 - 1) * b1
        flat[n_grid + self.n_w1:] = (torch.rand(self.n_w2, generator=g) * 2 - 1) * b2
        self.params = flat.to(self.device)
        self.grads = torch.zeros_like(self.params)
        self.grid, self.W1, self.W2 = self._views(self.params)
        self.dgrid, self.dW1, self.dW2 = self._views(self.grads)
        if mesh is not None:
            v, f = mesh
        elif self.cfg.shape_init.startswith("mesh:"):
            assert isinstance(self.cfg.shape_init_params, float)
            import os
            if not os.path.exists(self.cfg.shape_init[5:]):
                raise ValueError(f"Mesh file {self.cfg.shape_init[5:]} does not exist.")
            vv, ff = load_obj(self.cfg.shape_init[5:])
            v = torch.from_numpy(normalize_mesh(vv, self.cfg.shape_init_params, self.cfg.shape_init_mesh_up,
                                                self.cfg.shape_init_mesh_front).astype(np.float32))
            f = torch.from_numpy(ff.astype(np.int32))
        else:
            raise ValueError(f"Unknown shape initialization type: {self.cfg.shape_init}")
        self.v_pos, self.t_pos_idx = v.float().contiguous(), f.int().contiguous()
        self.v_nrm = vertex_normals(self.v_pos, self.t_pos_idx)
        # the reference unwraps UVs with xatlas for its (hot-path-unused) vtex_buffer; kept as zeros for checkpoint shape parity
        self.v_tex = torch.zeros(self.v_pos.shape[0], 2)
        self._bound = None      # (grid, W1, W2) nn.Parameters of the plugin layer, sharing this object's flat storage

    def _views(self, flat):
        g = flat[:self.n_grid]
        w1 = flat[self.n_grid:self.n_grid + self.n_w1].view(-1, self.hg.n_levels * 2)
        w2 = flat[self.n_grid + self.n_w1:].view(self.cfg.n_feature_dims, -1)
        return g, w1, w2

    def isosurface(self):
        return self

    def bind_parameters(self, grid_p, W1_p, W2_p):
        """The plugin layer's nn.Parameters (views of self.params): the autograd path differentiates w.r.t. THEM, so
        `loss.backward()` leaves the gradients where the optimizer looks (threestudio_plugin.DreamMatMesh)."""
        assert grid_p.data_ptr() == self.grid.data_ptr() and W1_p.data_ptr() == self.W1.data_ptr() and W2_p.data_ptr() == self.W2.data_ptr()
        self._bound = (grid_p, W1_p, W2_p)

    def autograd_leaves(self):
        """(grid, W1, W2) to differentiate with respect to on the autograd path: the bound nn.Parameters, else leaf
        tensors aliasing the flat buffer created once (their .grad is what `grads_from_autograd` collects)."""
        if self._bound is None:
            self._bound = tuple(t.detach().requires_grad_(True) for t in (self.grid, self.W1, self.W2))
        return self._bound

    def grads_from_autograd(self):
        """Copy the .grad of the autograd leaves into the flat gradient buffer (what optimizer_step consumes)."""
        for leaf, dst in zip(self.autograd_leaves(), (self.dgrid, self.dW1, self.dW2)):
            if leaf.grad is None:
                dst.zero_()
            else:
                dst.copy_(leaf.grad)
                leaf.grad = None

    def forward(self, points: torch.Tensor, output_normal: bool = False) -> Dict[str, torch.Tensor]:
        """dreammat_mesh.py:239-254 (autograd path; the fused step calls the kernels directly)."""
        assert output_normal is False, "Normal output is not supported for DreamMatMesh"
        g, w1, w2 = self.autograd_leaves()
        return {"features": R.hashgrid_mlp(points.view(-1, 3), g, w1, w2, self.hg).view(*points.shape[:-1], -1)}

    __call__ = forward

    def export(self, points: torch.Tensor, **kwargs) -> Dict[str, Any]:
        """dreammat_mesh.py:256-274: features at the (unscaled) query points for the texture bake; no graph."""
        if self.cfg.n_feature_dims == 0:
            return {}
        pts = points.reshape(-1, 3).to(self.device, torch.float32).contiguous()
        with torch.no_grad():
            f = R.hashgrid_mlp(pts, self.grid, self.W1, self.W2, self.hg)
        return {"features": f.view(*points.shape[:-1], self.cfg.n_feature_dims)}

    # ---- checkpoint compatibility (SURVEY.md section 5 / 8f N2): same keys, shapes and tcnn parameter order as the
    # reference's `geometry.*` entries, so a Lightning .ckpt written by either side loads into the other
    def state_dict(self, prefix: str = ""):
        return {prefix + "encoding.encoding.encoding.params": self.grid, prefix + "feature_network.layers.0.weight": self.W1,
                prefix + "feature_network.layers.2.weight": self.W2}

    def load_state_dict(self, sd: Dict[str, torch.Tensor], prefix: str = "", strict: bool = False):
        """Accepts the reference's keys (optionally with the `geometry.` prefix of the system checkpoint).  The dead
        predictors / mesh buffers of the reference checkpoint (dreammat_mesh.py:136-139,207-222) are ignored unless
        strict."""
        want = self.state_dict(prefix)
        used = set()
        for k, dst in want.items():
            src = sd.get(k, sd.get("geometry." + k))
            if src is None:
                raise KeyError(f"missing key {k} in checkpoint")
            if tuple(src.shape) != tuple(dst.shape):
                raise ValueError(f"{k}: shape {tuple(src.shape)} in checkpoint, expected {tuple(dst.shape)}")
            dst.copy_(src.to(dst.device, torch.float32))
            used.add(k)
        if strict:
            extra = [k for k in sd if k not in used and k.replace("geometry.", "", 1) not in used]
            if extra:
                raise KeyError(f"unexpected keys: {extra[:5]}")
        return self


class DreamMatMaterial:
    @dataclass
    class Config:
        # models/materials/dreammat_material.py:348-366
        material_activation: str = "sigmoid"
        environment_texture: str = "load/lights/mud_road_puresky_1k.hdr"
        environment_scale: float = 1.0
        min_metallic: float = 0.0
        max_metallic: float = 0.9
        min_roughness_squre: float = 0.01
        max_roughness_squre: float = 0.9
        min_roughness: float = 0.1
        max_roughness: float = 0.95
        use_bump: bool = True
        diffuse_sample_num: int = 512
        specular_sample_num: int = 256
        geometry_type: str = "schlick"
        random_azimuth: bool = True
        use_raytracing: bool = True

    def __init__(self, cfg: Optional[dict] = None, device="cuda", env_maps: Optional[List[torch.Tensor]] = None,
                 fg_lut: Optional[torch.Tensor] = None, envlight: Optional[list] = None, envlight_cache_dir: Optional[str] = None):
        self.cfg = self.Config(**(cfg or {}))
        self.device = torch.device(device)
        c = self.cfg
        if c.material_activation != "sigmoid" or c.geometry_type != "schlick" or not c.random_azimuth:
            raise NotImplementedError("only the dreammat.yaml material settings are on this path")
        # self.light[i]: lat-long radiance maps (dreammat_material.py:379-386), stored float4-padded
        self.light = [R.envmap_pack(m.to(self.device)) for m in (env_maps or [])]
        self.tab_d = R.direction_tables(c.diffuse_sample_num).to(self.device)
        self.tab_s = R.direction_tables(c.specular_sample_num).to(self.device)
        # visiting order of the samples: identity = the Fibonacci tables' own order, sorted by elevation, so the 32 rays of a
        # lock-step pass have similar traversal lengths.  Direction-coherent orders (R.sample_order, azimuth sectors) measured
        # ~10 % slower (scripts/exp_shade_order.py).
        self.perm = None
        self.mc_cfg = MaterialCfg(c.min_metallic, c.max_metallic, c.min_roughness_squre, c.max_roughness_squre,
                                  c.diffuse_sample_num, c.specular_sample_num)
        self.ss_cfg = MaterialCfg(c.min_metallic, c.max_metallic, c.min_roughness, c.max_roughness,
                                  c.diffuse_sample_num, c.specular_sample_num)
        self.FG_LUT = fg_lut.to(self.device).reshape(fg_lut.shape[-3], fg_lut.shape[-2], 2).contiguous() if fg_lut is not None else None
        self.envlight = envlight  # [(diffuse_cube, [spec mips])] per env (split-sum branch)
        if not c.use_raytracing:
            # split-sum branch (dreammat_material.py:679-711,747-762): needs the FG LUT (:405-410) and one prefiltered
            # EnvLight per map (:383, scale = environment_scale) -- built on the device, cached on disk (envlight.py)
            if self.FG_LUT is None:
                raise ValueError("use_raytracing=false needs the FG LUT (load/lights/bsdf_256_256.bin, scene.load_fg_lut)")
            if self.envlight is None:
                from .envlight import build_envlight
                self.envlight = [build_envlight(m.to(self.device), scale=c.environment_scale, cache_dir=envlight_cache_dir)
                                 for m in (env_maps or [])]
            self._mip_ptrs = [(C.c_void_p * len(mips))(*[m.data_ptr() for m in mips]) for (_, mips) in self.envlight]
        self.bvh = None

    def export(self, features: torch.Tensor, **kwargs) -> Dict[str, Any]:
        """dreammat_material.py:765-797: baked maps use the *squared*-roughness range and sqrt(. + 1e-7); the bump
        slot reads channels 5:8, which exist only when the geometry is configured with n_feature_dims >= 8."""
        c = self.cfg
        m = torch.sigmoid(features)
        out = {"albedo": m[..., :3],
               "metallic": m[..., 3:4] * (c.max_metallic - c.min_metallic) + c.min_metallic,
               "roughness": torch.sqrt(m[..., 4:5] * (c.max_roughness_squre - c.min_roughness_squre) + c.min_roughness_squre + 1e-7)}
        if c.use_bump and m.shape[-1] >= 8:
            pn = (m[..., 5:8] * 2 - 1) + torch.tensor([0.0, 0.0, 1.0], dtype=m.dtype, device=m.device)
            out["bump"] = (torch.nn.functional.normalize(pn.clamp(-1, 1), dim=-1) + 1) / 2
        return out

    def set_raytracer(self, bvh):
        """dreammat_material.py:426-427; here the tracer is the device BVH handle."""
        self.bvh = bvh

    def forward(self, pts, features, features_jitter, viewdirs, normals, env_id, rand_d=None, rand_s=None,
                want_aux=True, reg_weight_n=None, **kwargs):
        """dreammat_material.py:713-763 -> (outputs dict, mat_reg)."""
        n = features.shape[0]
        e = int(env_id)
        if self.cfg.use_raytracing:
            if rand_d is None:
                rand_d = torch.rand(n, device=self.device)           # appendix B #5
            if rand_s is None:
                rand_s = torch.rand(n, device=self.device)           # appendix B #6
            color, reg, aux = R.shade_mc(features, features_jitter, pts, normals, viewdirs, rand_d, rand_s, self.mc_cfg,
                                         self.bvh, self.light[e], self.tab_d, self.tab_s, want_aux, reg_weight_n, self.perm)
        else:
            dcube, mips = self.envlight[e]
            color, reg, aux = R.shade_splitsum(features, features_jitter, normals, viewdirs, self.ss_cfg, self.FG_LUT,
                                               dcube, mips, want_aux, reg_weight_n)
        out = {"color": color}
        out.update(aux)
        return out, reg

    __call__ = forward


class RaytraceRender:
    @dataclass
    class Config:
        context_type: str = "gl"   # raytracing_renderer.py:88-90 (kept for config compatibility; unused)
        radius: float = 1.0

    def __init__(self, cfg: Optional[dict] = None, geometry: DreamMatMesh = None, material: DreamMatMaterial = None,
                 background=None, device="cuda"):
        self.cfg = self.Config(**(cfg or {}))
        self.device = torch.device(device)
        self.geometry, self.material = geometry, material
        self.mesh = geometry.isosurface()
        self.ray_tracer = R.Bvh(self.mesh.v_pos, self.mesh.t_pos_idx)
        self.material.set_raytracer(self.ray_tracer)
        self.v_pos_d = self.mesh.v_pos.to(self.device)
        self.v_nrm_d = self.mesh.v_nrm.to(self.device)
        self.tris_d = self.mesh.t_pos_idx.to(self.device)
        self.change_eps = 0.05
        self._cache: Dict[int, dict] = {}
        self._faces_np = self.mesh.t_pos_idx.numpy().astype(np.int64)
        self._vpos_np = self.mesh.v_pos.numpy()
        self._nbr_opp = AA.edge_neighbours(self._faces_np, self._vpos_np.shape[0])

    def gbuffer(self, rays_o, rays_d, mvp_mtx, w2c, key: Optional[int] = None):
        """raytracing_renderer.py:122-159 for ONE view; cached under `key` (fixed view id)."""
        if key is not None and key in self._cache:
            return self._cache[key]
        dev = self.device
        rast, gb_pos, gb_nrm, mask, comp_normal = R.raster_gbuffer(
            self.ray_tracer, self.v_pos_d, self.v_nrm_d, self.tris_d, rays_o.to(dev), rays_d.to(dev), mvp_mtx.to(dev),
            w2c.to(dev))
        pix = R.compact_mask(mask)
        vd = (-rays_d.to(dev)).reshape(-1, 3).contiguous()
        # antialias pair list of this view (host, once): raytracing_renderer.py:127,147,199
        d_, s_, a_ = AA.build_pairs(rast[0].cpu().numpy(), self._vpos_np, self._faces_np, self._nbr_opp,
                                    mvp_mtx[0].detach().cpu().numpy())
        aa = (torch.from_numpy(d_).to(dev), torch.from_numpy(s_).to(dev), torch.from_numpy(a_).to(dev))
        Hh, Ww = rast.shape[1], rast.shape[2]
        g = {"pix": pix, "pn": int(pix.shape[0]), "pts": R.gather_rows(gb_pos.view(-1, 3), pix),
             "nrm": R.gather_rows(gb_nrm.view(-1, 3), pix), "vd": R.gather_rows(vd, pix), "aa": aa,
             "comp_depth": R.depth_normalize(rast, mask).view(1, Hh, Ww, 1),
             "comp_normal": AA.antialias(comp_normal.view(-1, 3), aa).view(1, Hh, Ww, 3),
             "opacity": AA.antialias(mask.view(-1, 1).float(), aa).view(1, Hh, Ww, 1)}
        if key is not None:
            self._cache[key] = g
        return g

    def forward(self, env_id, rays_o, rays_d, w2c, mvp_mtx, camera_positions=None, light_positions=None, height=None,
                width=None, view_id=None, **kwargs) -> Dict[str, Any]:
        """raytracing_renderer.py:109-222 (per-view loop so that B > 1 is well defined, SURVEY.md a0)."""
        B = mvp_mtx.shape[0]
        H, W = rays_d.shape[1], rays_d.shape[2]
        outs: Dict[str, list] = {}
        regs = []
        gbs = [self.gbuffer(rays_o[b:b + 1], rays_d[b:b + 1], mvp_mtx[b:b + 1], w2c[b:b + 1],
                            int(view_id[b]) if view_id is not None else None) for b in range(B)]
        total = sum(g["pn"] for g in gbs)
        for b, g in enumerate(gbs):
            n = g["pn"]
            ang = torch.rand(n, 1, device=self.device)                               # appendix B #3 (device draw)
            eps = torch.randn(n, 1, device=self.device) * self.change_eps            # appendix B #4
            pj = R.jitter_positions(g["pts"], g["nrm"], ang, eps)
            geo = self.geometry
            grid, w1, w2 = geo.autograd_leaves()
            f = R.hashgrid_mlp(g["pts"], grid, w1, w2, geo.hg)
            fj = R.hashgrid_mlp(pj, grid, w1, w2, geo.hg)
            so, reg = self.material(g["pts"], f, fj, g["vd"], g["nrm"], env_id[b], reg_weight_n=total)
            regs.append(reg)
            canv = {"comp_rgb": AA.antialias(R.scatter_canvas(so["color"], g["pix"], H * W), g["aa"]).view(1, H, W, 3)}
            for k_out, k_in, c in (("albedo", "albedo", 3), ("metalness", "metalness", 1), ("roughness", "roughness", 1),
                                   ("specular_light", "specular_lights", 3), ("diffuse_light", "diffuse_lights", 3),
                                   ("specular_color", "specular_colors", 3), ("diffuse_color", "diffuse_colors", 3)):
                canv[k_out] = R.scatter_canvas(so[k_in].detach().view(n, c), g["pix"], H * W).view(1, H, W, c)
            canv.update(opacity=g["opacity"], comp_depth=g["comp_depth"], comp_normal=g["comp_normal"])
            for k, v in canv.items():
                outs.setdefault(k, []).append(v)
        out = {k: torch.cat(v, 0) for k, v in outs.items()}
        out["loss_mat_reg"] = torch.stack(regs).sum()
        return out

    __call__ = forward


class DreamMat:
    """systems/dreammat.py:19-86 + Adam of systems/utils.py:34-53 (lr .01, betas (.9,.99), eps 1e-15)."""

    @dataclass
    class Config:
        loss: dict = field(default_factory=lambda: {"lambda_sds": 1.0, "lambda_mat_reg": 1.0})
        optimizer: dict = field(default_factory=lambda: {"name": "Adam", "args": {"betas": [0.9, 0.99], "eps": 1e-15, "lr": 0.01}})

    def __init__(self, cfg: Optional[dict], geometry: DreamMatMesh, material: DreamMatMaterial, renderer: RaytraceRender,
                 guidance, prompt_utils, device="cuda"):
        self.cfg = self.Config(**(cfg or {}))
        self.geometry, self.material, self.renderer = geometry, material, renderer
        self.guidance, self.prompt_utils = guidance, prompt_utils
        self.device = torch.device(device)
        self.m = torch.zeros_like(geometry.params)
        self.v = torch.zeros_like(geometry.params)
        self.global_step = 0
        self.world_size, self.rank = 1, 0
        self.balance_pixels = True     # multi-GPU: shade equal pixel intervals of the global batch (parallel.pixel_partition)
        self._steps_fused = 0
        self._balance_ok = False       # set by prepare_balanced(): EVERY rank holds every fixed view's G-buffer
        # dreammat_guidance.py:507-513: renders that are not 512x512 are resized (bilinear) to 512x512 before the VAE
        self.resize_to_vae = True

    def C(self, v):
        from .guidance import C
        return C(v, 0, self.global_step)

    def prepare_balanced(self, view_ids) -> bool:
        """Decide ONCE, identically on every rank, whether pixel-balanced shading may be used: it needs every view of
        `view_ids` in every rank's G-buffer cache.  The local answer is MIN-reduced over the ranks, so no rank can take
        the all-to-all branch while another goes straight to the gradient all-reduce (mismatched collectives)."""
        ok = all(int(v) in self.renderer._cache for v in view_ids)
        if self.world_size > 1:
            import torch.distributed as dist
            flag = torch.tensor([1 if ok else 0], device=self.device, dtype=torch.int32)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
            ok = bool(int(flag.item()))
            if ok:
                from .parallel import warm_exchange
                warm_exchange(max(int(c["pn"]) for c in self.renderer._cache.values()), self.world_size, self.device)
        self._balance_ok = ok
        return ok

    def reserve_step_scratch(self, factor: float = 1.5) -> int:
        """Called at the end of the second step: put one block of `factor` x that step's transient peak into the caching
        allocator's pool.  The per-step scratch (features, colours, Jacobians per covered pixel) changes size with the sampled
        views; without headroom the allocator eventually answers a new maximum with a cudaMalloc inside the loop -- one
        host-blocking call that, with peer mappings (NCCL), stalled a step by ~50 ms on 2 GPUs (bench `slowest_step`:
        host 71 ms, 1 cudaMalloc in 300 steps) while the step itself is 24 ms.  Returns the bytes reserved."""
        dev = self.device
        st = torch.cuda.memory_stats(dev)
        transient = int(st["allocated_bytes.all.peak"]) - int(st["allocated_bytes.all.current"])
        free, _ = torch.cuda.mem_get_info(dev)
        need = min(int(factor * max(transient, 0)) + (256 << 20), free // 4)
        if need > 0:
            block = torch.empty(need, dtype=torch.uint8, device=dev)
            del block                   # stays cached: later requests split it instead of growing the pool
        return need

    def forward(self, batch: Dict[str, Any]) -> Dict[str, Any]:
        return self.renderer(**batch)

    @staticmethod
    def _event():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def _mark(self, name):
        self._events.append((name, self._event()))

    def section_times(self) -> Dict[str, float]:
        """CUDA-event split of the LAST training_step_fused (ms): render fwd | VAE fwd | ControlNet+UNet | VAE bwd |
        shader + hash-grid backward + all-reduce + Adam."""
        torch.cuda.synchronize()
        ev = self._events
        out = {ev[i][0] + "_ms": ev[i - 1][1].elapsed_time(ev[i][1]) for i in range(1, len(ev))}
        out["dense_ms"] = out.get("vae_fwd_ms", 0) + out.get("unet_cn_ms", 0) + out.get("vae_bwd_ms", 0) + out.get("dense_graphs_ms", 0)
        out["total_ms"] = ev[0][1].elapsed_time(ev[-1][1])
        out["pn_local"] = getattr(self, "_last_pn", 0)
        return out

    def profile_step(self, make_batch, V):
        b, tot = make_batch()

        class _N:
            def __getitem__(self, i):
                return None
        b["rays_o"] = b["rays_d"] = _N()
        self.training_step_fused(b, global_views=V, total_pn_global=tot)
        return self.section_times()

    def optimizer_step(self, grad_scale: float = 1.0, from_autograd: bool = False):
        """Fused Adam on the flat buffer.  from_autograd: the gradients were produced by `loss.backward()` through the
        autograd wrappers (forward() path) and are first collected from the leaves."""
        if from_autograd:
            self.geometry.grads_from_autograd()
        a = self.cfg.optimizer["args"]
        self.global_step += 1
        R.adam_step(self.geometry.params, self.geometry.grads, self.m, self.v, a["lr"], a["betas"][0], a["betas"][1],
                    a["eps"], self.global_step, grad_scale)

    def training_step_fused(self, batch: Dict[str, Any], global_views: Optional[int] = None,
                            total_pn_global: Optional[int] = None, rng: Optional[dict] = None,
                            apply_optimizer: bool = True) -> Dict[str, torch.Tensor]:
        """One SDS iteration (systems/dreammat.py:57-86 + backward + Adam) as an explicit kernel sequence.

        batch: output of the data mirror, already on the device (condition_map [B,H,W,22] fp32, cameras, env_id,
        view_id).  `global_views` / `total_pn_global`: batch-wide normalisers when the views are sharded over
        ranks (loss_sds is a mean over views, loss_mat_reg a mean over covered pixels of the whole batch).
        Multi-GPU: the GRADIENT is global (all-reduced); the returned scalars (`loss`, `loss_sds`, `grad_norm`) are this
        rank's share of the global batch -- logging-only values, left un-reduced to keep the step at one large collective.
        `comp_depth` (logging only: `control_types=['light']` never feeds it to the guidance) is normalised per view, the
        B > 1 semantics of SURVEY.md row a0; the reference's single min/max over the batch only exists for B = 1."""
        geo, mat, ren, guid = self.geometry, self.material, self.renderer, self.guidance
        guid.update_step(0, self.global_step)
        lam_sds, lam_reg = self.C(self.cfg.loss["lambda_sds"]), self.C(self.cfg.loss["lambda_mat_reg"])
        B = batch["mvp_mtx"].shape[0]
        Bg = global_views or B
        H, W = batch["height"], batch["width"]
        dev = self.device
        st = stream_ptr()
        if self._steps_fused == 1 and dev.type == "cuda":
            torch.cuda.reset_peak_memory_stats(dev)
        self._events = [("start", self._event())]
        gbs = [ren.gbuffer(batch["rays_o"][b:b + 1], batch["rays_d"][b:b + 1], batch["mvp_mtx"][b:b + 1],
                           batch["w2c"][b:b + 1], int(batch["view_id"][b])) for b in range(B)]
        total_pn = total_pn_global or sum(g["pn"] for g in gbs)
        own_px = sum(g["pn"] for g in gbs)
        # ---- who shades what.  Default: this rank's own views.  With the global batch known (`global_view_id` /
        # `global_env_id`, every view in the G-buffer cache) the covered pixels of ALL views are cut into equal intervals
        # (parallel.pixel_partition) so the ray-tracing load does not depend on which views a rank drew.
        balanced = (self.world_size > 1 and self.balance_pixels and "global_view_id" in batch and
                    self._balance_ok)      # rank-invariant: fixed by prepare_balanced(), never by local cache state
        # explicit randomness (parity tests / bench --check): per-view lists indexed by the LOCAL view, or -- with
        # rng["indexed_by"] == "global_view" -- by the view's position in the global batch (needed when pixels are balanced)
        rng_global = rng is not None and rng.get("indexed_by") == "global_view"
        if rng is not None and balanced and not rng_global:
            raise ValueError("explicit randomness with pixel-balanced shading must be indexed by global view")
        if balanced:
            from .parallel import exchange_rows, pixel_partition
            gvid = [int(v) for v in batch["global_view_id"]]
            missing = [v for v in gvid if v not in ren._cache]
            if missing:
                raise RuntimeError(f"balanced shading was agreed on by all ranks but views {missing[:4]} are not cached here")
            geid = [int(e) for e in batch["global_env_id"]]
            pn_global = [ren._cache[v]["pn"] for v in gvid]
            if total_pn_global is None:
                total_pn = sum(pn_global)          # the global pixel count is known locally: every rank caches every view
            segments, counts = pixel_partition(pn_global, self.world_size)
            my_segs = [(ren._cache[gvid[g]], geid[g], a, bb, g) for (g, a, bb) in segments[self.rank]]
            send_counts = counts[self.rank]
            recv_counts = [counts[r][self.rank] for r in range(self.world_size)]
        else:
            my_segs = [(g, int(batch["env_id"][b]), 0, g["pn"], (self.rank * B + b) if rng_global else b) for b, g in enumerate(gbs)]
        n_sh = sum(bb - a for (_, _, a, bb, _) in my_segs)
        self._last_pn = n_sh
        g_ = getattr(guid, "graphs", None)
        resize = self.resize_to_vae and (H != 512 or W != 512)
        use_graphs = g_ is not None and g_.B == B and rng is None
        if use_graphs:
            want_hw = (512, 512) if resize else (H, W)      # the graphs are captured at the VAE input size
            if tuple(g_.rgb.shape[1:3]) != want_hw:
                raise RuntimeError(f"dense graphs were captured at {tuple(g_.rgb.shape[1:3])}, this step feeds the VAE {want_hw}: "
                                   "call guidance.enable_graphs(B, 512, 512) for renders that are resized")
        canvas = g_.rgb.view(B, H * W, 3) if (use_graphs and not resize) else torch.empty(B, H * W, 3, device=dev)
        raw = torch.empty(B, H * W, 3, device=dev)            # canvas before the antialias blend
        check(lib().dm_fill(ptr(raw), raw.numel(), 1.0, st), "dm_fill")
        reg_sums = torch.zeros(2, device=dev)
        color_sh = torch.empty(max(n_sh, 1), 3, device=dev)   # colours of the pixels this rank shades, segment order
        jac_sh = torch.empty(max(n_sh, 1), 9, device=dev)
        saved = []
        o = 0
        for (ge, env_id, a, bb, gi) in my_segs:
            n = bb - a
            pts, nrm, vd = ge["pts"][a:bb], ge["nrm"][a:bb], ge["vd"][a:bb]
            if rng is not None:   # explicit randomness (SURVEY.md appendix B #3-#6) for parity tests
                ang, eps, rd, rs = (rng[k][gi].to(dev).reshape(-1)[a:bb].contiguous() for k in ("rand_ang", "normal_eps", "rand_d", "rand_s"))
            else:
                ang, eps = torch.rand(n, device=dev), torch.randn(n, device=dev) * ren.change_eps
                rd, rs = torch.rand(n, device=dev), torch.rand(n, device=dev)
            pj = R.jitter_positions(pts, nrm, ang, eps)
            f = torch.empty(n, 5, device=dev); fj = torch.empty(n, 5, device=dev)
            check(lib().dm_hashgrid_mlp_fwd(C.byref(geo.hg), ptr(pts), n, ptr(geo.grid), ptr(geo.W1), ptr(geo.W2), ptr(f), st), "hashgrid fwd")
            check(lib().dm_hashgrid_mlp_fwd(C.byref(geo.hg), ptr(pj), n, ptr(geo.grid), ptr(geo.W1), ptr(geo.W2), ptr(fj), st), "hashgrid fwd")
            color, jac = color_sh[o:o + n], jac_sh[o:o + n]
            if mat.cfg.use_raytracing:
                env = mat.light[env_id]
                check(lib().dm_shade_mc_fwd(C.byref(mat.mc_cfg), ren.ray_tracer.h, ptr(env), env.shape[0], env.shape[1],
                                            ptr(mat.tab_d), ptr(mat.tab_s), ptr(pts), ptr(nrm), ptr(vd), ptr(f),
                                            ptr(fj), ptr(rd), ptr(rs), n, ptr(color), ptr(jac), ptr(reg_sums), *([None] * 7),
                                            None, ptr(mat.perm), st), "dm_shade_mc_fwd")
            else:   # use_raytracing=false: split-sum shading (dreammat_material.py:679-711), three texture lookups per pixel
                dcube, mips = mat.envlight[env_id]
                check(lib().dm_shade_splitsum_fwd(C.byref(mat.ss_cfg), ptr(mat.FG_LUT), mat.FG_LUT.shape[0], ptr(dcube), dcube.shape[1],
                                                  mat._mip_ptrs[env_id], len(mips), mips[0].shape[1], ptr(nrm), ptr(vd), ptr(f), ptr(fj),
                                                  n, ptr(color), ptr(jac), ptr(reg_sums), *([None] * 7), st), "dm_shade_splitsum_fwd")
            saved.append((pts, pj, f, fj, jac, n, o))
            o += n
        # colours travel to the ranks that own the views (one all-to-all); without balancing they are already home
        color_own = exchange_rows(color_sh[:n_sh], send_counts, recv_counts, self.world_size) if balanced else color_sh
        o = 0
        for b, g in enumerate(gbs):
            n = g["pn"]
            check(lib().dm_scatter_canvas(ptr(color_own[o:o + n]), ptr(g["pix"]), n, 3, ptr(raw[b]), st), "dm_scatter_canvas")
            aa = g.get("aa")
            k_aa = int(aa[0].shape[0]) if aa is not None else 0
            check(lib().dm_antialias_fwd(ptr(raw[b]), ptr(aa[0]) if k_aa else None, ptr(aa[1]) if k_aa else None,
                                         ptr(aa[2]) if k_aa else None, k_aa, H * W, 3, ptr(canvas[b]), st), "dm_antialias_fwd")
            o += n
        comp_rgb = canvas.view(B, H, W, 3)
        vae_in = comp_rgb
        if resize:
            vae_in = g_.rgb if use_graphs else torch.empty(B, 512, 512, 3, device=dev)
            check(lib().dm_resize_bilinear(ptr(comp_rgb), B, H, W, 512, 512, 3, ptr(vae_in), 0, st), "dm_resize_bilinear")
        self._mark("render_fwd")
        ctx3 = self.prompt_utils.get_text_embeddings(batch["elevation"], batch["azimuth"], batch["camera_distances"],
                                                     guid.cfg.view_dependent_prompting, return_null_text_embeddings=True)
        if use_graphs:
            # dense section replayed from three captured CUDA graphs (VAE fwd | ControlNet+UNet | VAE bwd)
            drgb, sums = guid.graph_step(batch.get("condition_map"), ctx3, lam_sds * B / Bg, mark=self._mark,
                                         view_id=batch["view_id"], env_id=batch["env_id"])
            loss_sds = sums[0] / Bg
            dvae = drgb
        else:
            # guidance (dreammat_guidance.py:536-602): VAE encode with grad, ControlNet + UNet x3 under no_grad, CSD gradient
            from .guidance import _SDSLoss
            vae_in = vae_in.detach().requires_grad_(True)
            rsl = slice(self.rank * B, (self.rank + 1) * B) if rng_global else slice(None)
            cond_map = batch.get("condition_map")
            if cond_map is None:      # N1: the maps are a device-resident uint8 dataset; eager path gathers the float view of it
                cond_map = guid.maps.condition_map(batch["view_id"], batch["env_id"])
            lat = guid.encode_images(vae_in, rng["vae_eps"][rsl].to(dev) if rng is not None else None)
            self._mark("vae_fwd")
            grad, dlat, sums = guid.compute_grad_sds(lat, cond_map, ctx3, rng["t"][rsl].to(dev) if rng is not None else None,
                                                     rng["noise"][rsl].to(dev) if rng is not None else None)
            self._mark("unet_cn")
            loss_sds = _SDSLoss.apply(lat, dlat, sums[0] / B) * (B / Bg)          # mean over the GLOBAL batch of views
            (lam_sds * loss_sds).backward()
            self._mark("vae_bwd")
            dvae = vae_in.grad
        if resize:
            dcanvas = torch.empty(B, H * W, 3, device=dev)
            check(lib().dm_resize_bilinear(ptr(dvae.contiguous()), B, H, W, 512, 512, 3, ptr(dcanvas), 1, st), "dm_resize_bilinear")
        else:
            dcanvas = dvae.reshape(B, H * W, 3)
        nrms = sums.sqrt()    # the reference logs all of these every step (systems/dreammat.py:72-74 over compute_grad_sds' dict)
        gout = {"grad_norm": nrms[1], "uncond_m_noise_norm": nrms[2], "text_m_noise_norm": nrms[3], "text_m_uncond_norm": nrms[4],
                "text_m_null_norm": nrms[5], "null_m_uncond_norm": nrms[6], "noise_norm": nrms[7], "uncond_norm": nrms[8],
                "text_norm": nrms[9]}
        # backward into the hash grid / MLP
        geo.grads.zero_()
        dcolor_own = torch.empty(max(own_px, 1), 3, device=dev)
        o = 0
        for b, g in enumerate(gbs):
            n = g["pn"]
            aa = g.get("aa")
            k_aa = int(aa[0].shape[0]) if aa is not None else 0
            draw = torch.empty(H * W, 3, device=dev)
            check(lib().dm_antialias_bwd(ptr(dcanvas[b]), ptr(aa[0]) if k_aa else None, ptr(aa[1]) if k_aa else None,
                                         ptr(aa[2]) if k_aa else None, k_aa, H * W, 3, ptr(draw), st), "dm_antialias_bwd")
            check(lib().dm_gather_canvas_grad(ptr(draw), ptr(g["pix"]), n, 3, ptr(dcolor_own[o:o + n]), st), "gather")
            o += n
        # d loss / d colour back to the shading ranks (the forward all-to-all, transposed)
        dcolor_sh = exchange_rows(dcolor_own[:own_px], recv_counts, send_counts, self.world_size) if balanced else dcolor_own
        for (pts, pj, f, fj, jac, n, o) in saved:
            df = torch.empty(n, 5, device=dev); dfj = torch.empty(n, 5, device=dev)
            check(lib().dm_shade_bwd(C.byref(mat.mc_cfg if mat.cfg.use_raytracing else mat.ss_cfg), ptr(f), ptr(fj), ptr(dcolor_sh[o:o + n]), ptr(jac), lam_reg * 0.25 / total_pn,
                                     lam_reg * 0.1 / total_pn, n, ptr(df), ptr(dfj), st), "dm_shade_bwd")
            for pts_, d_ in ((pts, df), (pj, dfj)):
                check(lib().dm_hashgrid_mlp_bwd(C.byref(geo.hg), ptr(pts_), n, ptr(geo.grid), ptr(geo.W1), ptr(geo.W2), ptr(d_),
                                                ptr(geo.dgrid), ptr(geo.dW1), ptr(geo.dW2), st), "hashgrid bwd")
        loss_reg = (0.25 * reg_sums[0] + 0.1 * reg_sums[1]) / total_pn
        from .parallel import allreduce_gradients
        allreduce_gradients(geo.grads, self.world_size)          # the single large collective of the step (NVLink / NVSwitch)
        if apply_optimizer:       # False: the host framework (Lightning) steps its own optimizer on the same flat gradient
            self.optimizer_step()
        self._mark("render_bwd_adam")
        if self._steps_fused == 1 and dev.type == "cuda":
            self.reserve_step_scratch()
        self._steps_fused += 1
        return {"loss": lam_sds * loss_sds.detach() + lam_reg * loss_reg, "loss_sds": loss_sds.detach(),
                "loss_mat_reg": loss_reg, "comp_rgb": comp_rgb.detach(), **gout}
