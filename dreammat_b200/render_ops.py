"""torch-facing wrappers of the render-side C-ABI entry points (geometry, BVH, shading, canvas).

Each autograd.Function mirrors what Lightning's `loss.backward()` walks through in the
reference (SURVEY.md section 3.2), but every node is one hand-written kernel launch.
PyTorch supplies device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _cabi
from ._cabi import HashGridCfg, MaterialCfg, check, lib, ptr, stream_ptr


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# ----------------------------------------------------------------------------- geometry


def default_hashgrid_cfg(radius: float = 1.0, n_levels=16, log2_T=19, base=16, scale=1.447269237440378,
                         n_hidden=64, n_out=5) -> HashGridCfg:
    """configs/dreammat.yaml:41-50 + models/geometry/dreammat_mesh.py:93-121."""
    return HashGridCfg(n_levels, 2, log2_T, base, scale, -radius, radius, n_hidden, n_out)


def hashgrid_num_params(cfg: HashGridCfg):
    offs = (C.c_uint32 * (cfg.n_levels + 1))()
    total = lib().dm_hashgrid_layout(C.byref(cfg), offs)
    if total < 0:
        raise _cabi.DmError("dm_hashgrid_layout failed")
    return int(total) * cfg.n_features, [int(o) for o in offs]


class _HashGridMLP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, grid, W1, W2, cfg):
        points = _f32c(points)
        n = points.shape[0]
        out = torch.empty(n, cfg.n_out, device=points.device, dtype=torch.float32)
        check(lib().dm_hashgrid_mlp_fwd(C.byref(cfg), ptr(points), n, ptr(grid), ptr(W1), ptr(W2), ptr(out),
                                        stream_ptr()), "dm_hashgrid_mlp_fwd")
        ctx.save_for_backward(points, grid, W1, W2)
        ctx.cfg = cfg
        return out

    @staticmethod
    def backward(ctx, dout):
        points, grid, W1, W2 = ctx.saved_tensors
        dout = _f32c(dout)
        dgrid = torch.zeros_like(grid)
        dW1 = torch.zeros_like(W1)
        dW2 = torch.zeros_like(W2)
        check(lib().dm_hashgrid_mlp_bwd(C.byref(ctx.cfg), ptr(points), points.shape[0], ptr(grid), ptr(W1), ptr(W2),
                                        ptr(dout), ptr(dgrid), ptr(dW1), ptr(dW2), stream_ptr()),
              "dm_hashgrid_mlp_bwd")
        return None, dgrid, dW1, dW2, None


def hashgrid_mlp(points, grid, W1, W2, cfg):
    return _HashGridMLP.apply(points, grid, W1, W2, cfg)


def hashgrid_encode(points, grid, cfg):
    points = _f32c(points)
    enc = torch.empty(points.shape[0], cfg.n_levels * cfg.n_features, device=points.device)
    check(lib().dm_hashgrid_encode(C.byref(cfg), ptr(points), points.shape[0], ptr(grid), ptr(enc), stream_ptr()),
          "dm_hashgrid_encode")
    return enc


def jitter_positions(pos, nrm, rand_ang, normal_eps):
    pos, nrm = _f32c(pos), _f32c(nrm)
    out = torch.empty_like(pos)
    check(lib().dm_jitter_positions(ptr(pos), ptr(nrm), ptr(_f32c(rand_ang)), ptr(_f32c(normal_eps)), pos.shape[0],
                                    ptr(out), stream_ptr()), "dm_jitter_positions")
    return out


# ----------------------------------------------------------------------------- BVH / G-buffer


class Bvh:
    """Device BVH; stands in for `RayTracer` (models/renderers/raytracing_renderer.py:20-67)."""

    def __init__(self, vertices, triangles):
        v = np.ascontiguousarray(np.asarray(vertices.detach().cpu() if torch.is_tensor(vertices) else vertices,
                                            dtype=np.float32))
        t = np.ascontiguousarray(np.asarray(triangles.detach().cpu() if torch.is_tensor(triangles) else triangles,
                                            dtype=np.int32))
        assert t.shape[0] > 8, "BVH needs at least 8 triangles."  # raytracing_renderer.py:29
        h = C.c_void_p()
        check(lib().dm_bvh_build(v.ctypes.data, v.shape[0], t.ctypes.data, t.shape[0], C.byref(h)), "dm_bvh_build")
        self.h = h
        self.n_tris = t.shape[0]

    def __del__(self):
        if getattr(self, "h", None):
            try:
                lib().dm_bvh_free(self.h)
            except Exception:
                pass
            self.h = None

    def trace(self, rays_o, rays_d):
        """-> (t [N] (10 on miss), tri [N] int32 (-1 on miss), uv [N,2])."""
        rays_o, rays_d = _f32c(rays_o).view(-1, 3), _f32c(rays_d).view(-1, 3)
        n = rays_o.shape[0]
        t = torch.empty(n, device=rays_o.device)
        tri = torch.empty(n, device=rays_o.device, dtype=torch.int32)
        uv = torch.empty(n, 2, device=rays_o.device)
        check(lib().dm_bvh_trace(self.h, ptr(rays_o), ptr(rays_d), n, ptr(t), ptr(tri), ptr(uv), stream_ptr()),
              "dm_bvh_trace")
        return t, tri, uv


def raster_gbuffer(bvh: Bvh, v_pos, v_nrm, tris, rays_o, rays_d, mvp, w2c):
    B, H, W, _ = rays_d.shape
    dev = rays_d.device
    rast = torch.empty(B, H, W, 4, device=dev)
    gb_pos = torch.empty(B, H * W, 3, device=dev)
    gb_nrm = torch.empty(B, H * W, 3, device=dev)
    mask = torch.empty(B, H * W, device=dev, dtype=torch.uint8)
    comp_normal = torch.empty(B, H, W, 3, device=dev)
    check(lib().dm_raster_gbuffer(bvh.h, ptr(_f32c(v_pos)), ptr(_f32c(v_nrm)), ptr(tris.int().contiguous()),
                                  ptr(_f32c(rays_o)), ptr(_f32c(rays_d)), ptr(_f32c(mvp)), ptr(_f32c(w2c)), B, H, W,
                                  ptr(rast), ptr(gb_pos), ptr(gb_nrm), ptr(mask), ptr(comp_normal), stream_ptr()),
          "dm_raster_gbuffer")
    return rast, gb_pos, gb_nrm, mask, comp_normal


def compact_mask(mask):
    """Row-major indices of non-zero mask entries (order of `gb_pos[selector]`)."""
    mask = mask.contiguous().view(-1)
    idx = torch.empty(mask.numel(), device=mask.device, dtype=torch.int32)
    cnt = C.c_int64(0)
    check(lib().dm_compact_mask(ptr(mask), mask.numel(), ptr(idx), C.byref(cnt), stream_ptr()), "dm_compact_mask")
    return idx[:cnt.value].clone()


def gather_rows(src, idx):
    src = _f32c(src)
    c = src.shape[-1]
    out = torch.empty(idx.shape[0], c, device=src.device)
    check(lib().dm_gather_rows(ptr(src.view(-1, c)), ptr(idx), idx.shape[0], c, ptr(out), stream_ptr()),
          "dm_gather_rows")
    return out


def depth_normalize(rast, mask):
    n = mask.numel()
    out = torch.empty(n, device=rast.device)
    scratch = torch.empty(2, device=rast.device)
    check(lib().dm_depth_normalize(ptr(rast), ptr(mask.contiguous()), n, ptr(out), ptr(scratch), stream_ptr()),
          "dm_depth_normalize")
    return out


# ----------------------------------------------------------------------------- material


def direction_tables(n: int) -> torch.Tensor:
    """(ua, ue) Fibonacci tables of dreammat_material.py:89-102,389-398 (numpy fp64 -> fp32)."""
    ratio = 90 / 180
    num_points = int(n // (1 - ratio))
    phi = (np.sqrt(5) - 1.0) / 2.0
    k = np.arange(num_points - n, num_points, dtype=np.float64)
    z = 2.0 * k / num_points - 1.0
    az = (2 * np.pi * k * phi) % (2 * np.pi)
    el = np.arcsin(z)
    return torch.from_numpy(np.stack([az * 0.5 / np.pi, 1 - 2 * el / np.pi], -1).astype(np.float32))


def envmap_pack(rgb: torch.Tensor) -> torch.Tensor:
    rgb = _f32c(rgb)
    H, W, _ = rgb.shape
    out = torch.empty(H, W, 4, device=rgb.device)
    check(lib().dm_envmap_pack(ptr(rgb), H * W, ptr(out), stream_ptr()), "dm_envmap_pack")
    return out


AUX_KEYS = ("albedo", "roughness", "metalness", "specular_lights", "diffuse_lights", "specular_colors",
            "diffuse_colors")


def _alloc_aux(n, dev, want):
    if not want:
        return [None] * 7
    return [torch.empty(n, 3, device=dev), torch.empty(n, 1, device=dev), torch.empty(n, 1, device=dev),
            torch.empty(n, 3, device=dev), torch.empty(n, 3, device=dev), torch.empty(n, 3, device=dev),
            torch.empty(n, 3, device=dev)]


class _ShadeMC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, features_jitter, pts, normals, viewdirs, rand_d, rand_s, state, want_aux, reg_weight_n):
        cfg, bvh, env_rgba, tab_d, tab_s = state
        n = features.shape[0]
        dev = features.device
        features, features_jitter = _f32c(features), _f32c(features_jitter)
        color = torch.empty(n, 3, device=dev)
        jac = torch.empty(n, 9, device=dev)
        reg = torch.zeros(2, device=dev)
        aux = _alloc_aux(n, dev, want_aux)
        H, W, _ = env_rgba.shape
        check(lib().dm_shade_mc_fwd(C.byref(cfg), bvh.h, ptr(env_rgba), H, W, ptr(tab_d), ptr(tab_s), ptr(_f32c(pts)),
                                    ptr(_f32c(normals)), ptr(_f32c(viewdirs)), ptr(features), ptr(features_jitter),
                                    ptr(_f32c(rand_d).view(-1)), ptr(_f32c(rand_s).view(-1)), n, ptr(color), ptr(jac),
                                    ptr(reg), *[ptr(a) for a in aux], None, stream_ptr()), "dm_shade_mc_fwd")
        ctx.save_for_backward(features, features_jitter, jac)
        ctx.cfg = cfg
        ctx.inv_n = 1.0 / float(reg_weight_n if reg_weight_n else max(n, 1))
        mat_reg = (0.25 * reg[0] + 0.1 * reg[1]) * ctx.inv_n
        ctx.mark_non_differentiable(*[a for a in aux if a is not None])
        return (color, mat_reg, *[a if a is not None else torch.empty(0, device=dev) for a in aux])

    @staticmethod
    def backward(ctx, dcolor, dreg, *_):
        features, features_jitter, jac = ctx.saved_tensors
        n = features.shape[0]
        df = torch.empty_like(features)
        dfj = torch.empty_like(features_jitter)
        dcolor = _f32c(dcolor) if dcolor is not None else torch.zeros(n, 3, device=features.device)
        g = float(dreg) if dreg is not None else 0.0
        check(lib().dm_shade_bwd(C.byref(ctx.cfg), ptr(features), ptr(features_jitter), ptr(dcolor), ptr(jac),
                                 g * 0.25 * ctx.inv_n, g * 0.1 * ctx.inv_n, n, ptr(df), ptr(dfj), stream_ptr()),
              "dm_shade_bwd")
        return (df, dfj) + (None,) * 8


def shade_mc(features, features_jitter, pts, normals, viewdirs, rand_d, rand_s, cfg, bvh, env_rgba, tab_d, tab_s,
             want_aux=True, reg_weight_n=None):
    out = _ShadeMC.apply(features, features_jitter, pts, normals, viewdirs, rand_d, rand_s,
                         (cfg, bvh, env_rgba, tab_d, tab_s), want_aux, reg_weight_n)
    color, reg = out[0], out[1]
    aux = dict(zip(AUX_KEYS, out[2:])) if want_aux else {}
    return color, reg, aux


class _ShadeSplitSum(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, features_jitter, normals, viewdirs, state, want_aux, reg_weight_n):
        cfg, lut, dcube, mips = state
        n = features.shape[0]
        dev = features.device
        features, features_jitter = _f32c(features), _f32c(features_jitter)
        color = torch.empty(n, 3, device=dev)
        jac = torch.empty(n, 9, device=dev)
        reg = torch.zeros(2, device=dev)
        aux = _alloc_aux(n, dev, want_aux)
        arr = (C.c_void_p * len(mips))(*[m.data_ptr() for m in mips])
        check(lib().dm_shade_splitsum_fwd(C.byref(cfg), ptr(lut), lut.shape[0], ptr(dcube), dcube.shape[1], arr,
                                          len(mips), mips[0].shape[1], ptr(_f32c(normals)), ptr(_f32c(viewdirs)),
                                          ptr(features), ptr(features_jitter), n, ptr(color), ptr(jac), ptr(reg),
                                          *[ptr(a) for a in aux], stream_ptr()), "dm_shade_splitsum_fwd")
        ctx.save_for_backward(features, features_jitter, jac)
        ctx.cfg = cfg
        ctx.inv_n = 1.0 / float(reg_weight_n if reg_weight_n else max(n, 1))
        mat_reg = (0.25 * reg[0] + 0.1 * reg[1]) * ctx.inv_n
        ctx.mark_non_differentiable(*[a for a in aux if a is not None])
        return (color, mat_reg, *[a if a is not None else torch.empty(0, device=dev) for a in aux])

    @staticmethod
    def backward(ctx, dcolor, dreg, *_):
        grads = _ShadeMC.backward(ctx, dcolor, dreg)
        return grads[:2] + (None,) * 5


def shade_splitsum(features, features_jitter, normals, viewdirs, cfg, lut, dcube, mips, want_aux=True,
                   reg_weight_n=None):
    out = _ShadeSplitSum.apply(features, features_jitter, normals, viewdirs, (cfg, lut, dcube, list(mips)), want_aux,
                               reg_weight_n)
    color, reg = out[0], out[1]
    aux = dict(zip(AUX_KEYS, out[2:])) if want_aux else {}
    return color, reg, aux


# ----------------------------------------------------------------------------- canvas


class _ScatterCanvas(torch.autograd.Function):
    @staticmethod
    def forward(ctx, values, pix, n_pix):
        values = _f32c(values)
        c = values.shape[-1]
        canvas = torch.empty(n_pix, c, device=values.device)
        check(lib().dm_fill(ptr(canvas), canvas.numel(), 1.0, stream_ptr()), "dm_fill")
        check(lib().dm_scatter_canvas(ptr(values), ptr(pix), values.shape[0], c, ptr(canvas), stream_ptr()),
              "dm_scatter_canvas")
        ctx.save_for_backward(pix)
        ctx.c = c
        return canvas

    @staticmethod
    def backward(ctx, dcanvas):
        (pix,) = ctx.saved_tensors
        dcanvas = _f32c(dcanvas)
        dv = torch.empty(pix.shape[0], ctx.c, device=dcanvas.device)
        check(lib().dm_gather_canvas_grad(ptr(dcanvas.view(-1, ctx.c)), ptr(pix), pix.shape[0], ctx.c, ptr(dv),
                                          stream_ptr()), "dm_gather_canvas_grad")
        return dv, None, None


def scatter_canvas(values, pix, n_pix):
    """White canvas + index_put (raytracing_renderer.py:189-207)."""
    return _ScatterCanvas.apply(values, pix, n_pix)


# ----------------------------------------------------------------------------- optimiser / SDS


def adam_step(p, g, m, v, lr, beta1, beta2, eps, step, grad_scale=1.0):
    check(lib().dm_adam_step(ptr(p), ptr(g), ptr(m), ptr(v), p.numel(), lr, beta1, beta2, eps, int(step),
                             float(grad_scale), stream_ptr()), "dm_adam_step")


def fill_(t, value: float):
    """t[:] = value through the library (capturable into a CUDA graph, counted in dm_launch_count)."""
    assert t.is_contiguous() and t.dtype == torch.float32
    check(lib().dm_fill(ptr(t), t.numel(), float(value), stream_ptr()), "dm_fill")
    return t


def sds_grad(eps_pred, noise, w, c_text, c_uncond, c_null, c_noise):
    """eps_pred [3,B,C,H,W] fp32 -> (grad [B,C,H,W], dlatents, sums[10])."""
    eps_pred, noise, w = _f32c(eps_pred), _f32c(noise), _f32c(w)
    B = noise.shape[0]
    chw = noise[0].numel()
    grad = torch.empty_like(noise)
    dlat = torch.empty_like(noise)
    sums = torch.zeros(10, device=noise.device)
    check(lib().dm_sds_grad(ptr(eps_pred), ptr(noise), ptr(w), B, chw, c_text, c_uncond, c_null, c_noise, ptr(grad),
                            ptr(dlat), ptr(sums), stream_ptr()), "dm_sds_grad")
    return grad, dlat, sums


class _ResizeBilinear(torch.autograd.Function):
    """F.interpolate(x, (Ho, Wo), mode='bilinear', align_corners=False) on NHWC fp32 (dreammat_guidance.py:507-513)."""

    @staticmethod
    def forward(ctx, x, Ho, Wo):
        x = _f32c(x)
        n, Hi, Wi, c = x.shape
        out = torch.empty(n, Ho, Wo, c, device=x.device)
        check(lib().dm_resize_bilinear(ptr(x), n, Hi, Wi, Ho, Wo, c, ptr(out), 0, stream_ptr()), "dm_resize_bilinear")
        ctx.shape = (n, Hi, Wi, Ho, Wo, c)
        return out

    @staticmethod
    def backward(ctx, dout):
        n, Hi, Wi, Ho, Wo, c = ctx.shape
        dout = _f32c(dout)
        din = torch.empty(n, Hi, Wi, c, device=dout.device)
        check(lib().dm_resize_bilinear(ptr(dout), n, Hi, Wi, Ho, Wo, c, ptr(din), 1, stream_ptr()), "dm_resize_bilinear")
        return din, None, None


def resize_bilinear(x_bhwc, Ho, Wo):
    return _ResizeBilinear.apply(x_bhwc, Ho, Wo)
