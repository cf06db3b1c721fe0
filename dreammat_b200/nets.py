"""Device graphs of the three diffusers modules on the hot path, built from the C-ABI kernels.

    UNet            diffusers UNet2DConditionModel.forward   (dreammat_guidance.py:274-282)
    ControlNet      diffusers ControlNetModel.forward         (dreammat_guidance.py:218-229)
    VAEEncoder      AutoencoderKL.encode + its input-gradient (dreammat_guidance.py:285-292, 593-594)

Weights arrive as a flat dict with diffusers' state-dict names (fp32 or fp16) and are re-laid-out once
for the tensor-core kernel: conv [Cout,Cin,kh,kw] -> [Cout, kh*kw*Cin] (tap-major, channel-minor,
channels zero-padded to multiples of 64), q/k/v projections concatenated, all time-embedding
projections stacked into one GEMM.  Activations are NHWC, fp16 (or bf16) storage, fp32 accumulation.
No torch compute op is on the path: torch only owns the buffers.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from . import dense_ops as D


def _r64(c):
    return (c + 63) // 64 * 64


def _dst(into, **keys):
    """keyword arguments that make a dense_ops gradient call write into[key] (into: parameter name -> preallocated fp32
    tensor, e.g. the views of a flat gradient arena); none without `into`, and the call allocates as usual"""
    return {} if into is None else {arg: into[k] for arg, k in keys.items()}


class _Base:
    def __init__(self, w: Dict[str, torch.Tensor], device, dtype):
        self.dev, self.dt = device, dtype
        self.p: Dict[str, torch.Tensor] = {}
        self.conv_shape: Dict[str, tuple] = {}      # conv name -> diffusers [Cout, Cin, kh, kw] (before channel padding)
        self._src = w

    # ---- weight preparation
    def _vec(self, name, pad=0):
        v = self._src[name].float()
        if pad and pad > v.numel():
            v = torch.cat([v, torch.zeros(pad - v.numel(), device=v.device)])
        self.p[name] = v.to(self.dev, self.dt).contiguous()

    def _conv(self, name, cin_pad=0, cout_pad=0):
        w = self._src[name + ".weight"]
        self.conv_shape[name] = tuple(w.shape)
        self.p[name + ".w"] = D.conv_weight_to_gemm(w, cin_pad or _r64(w.shape[1]), cout_pad, self.dt).to(self.dev)
        if name + ".bias" in self._src:
            self._vec(name + ".bias", cout_pad)

    def _conv_dgrad(self, name, cin_pad=0, cout_pad=0):
        """weights of the input-gradient convolution: Wd[cin, (kh,kw), cout] = W[cout, cin, 2-kh, 2-kw]"""
        w = self._src[name + ".weight"].float()
        wd = w.flip(2, 3).permute(1, 0, 2, 3).contiguous()          # [Cin, Cout, kh, kw]
        self.p[name + ".wd"] = D.conv_weight_to_gemm(wd, cout_pad or _r64(w.shape[0]), cin_pad, self.dt).to(self.dev)

    def _lin(self, name, transpose_too=False):
        w = self._src[name + ".weight"].float()
        self.p[name + ".w"] = w.to(self.dev, self.dt).contiguous()
        if transpose_too:
            self.p[name + ".wt"] = w.t().contiguous().to(self.dev, self.dt)
        if name + ".bias" in self._src:
            self._vec(name + ".bias")

    def _norm(self, name):
        self._vec(name + ".weight")
        self._vec(name + ".bias")


# ================================================================================================ UNet / ControlNet


class _UNetCommon(_Base):
    def __init__(self, w, cfg, device, dtype):
        super().__init__(w, device, dtype)
        self.cfg = cfg
        self.tproj_names: List[str] = []

    def _prep_resnet(self, p, with_temb=True):
        self._norm(p + ".norm1"); self._conv(p + ".conv1")
        self._norm(p + ".norm2"); self._conv(p + ".conv2")
        if with_temb:
            self.tproj_names.append(p)
        if p + ".conv_shortcut.weight" in self._src:
            w = self._src[p + ".conv_shortcut.weight"]
            self.p[p + ".conv_shortcut.w"] = w.float().reshape(w.shape[0], w.shape[1]).to(self.dev, self.dt).contiguous()
            self._vec(p + ".conv_shortcut.bias")

    def _prep_transformer(self, p):
        self._norm(p + ".norm"); self._lin(p + ".proj_in"); self._lin(p + ".proj_out")
        b = p + ".transformer_blocks.0"
        for k in ("norm1", "norm2", "norm3"):
            self._norm(f"{b}.{k}")
        s = self._src
        self.p[b + ".attn1.qkv.w"] = torch.cat([s[f"{b}.attn1.to_q.weight"], s[f"{b}.attn1.to_k.weight"],
                                                s[f"{b}.attn1.to_v.weight"]], 0).float().to(self.dev, self.dt).contiguous()
        self._lin(b + ".attn1.to_out.0")
        self._lin(b + ".attn2.to_q")
        self.p[b + ".attn2.kv.w"] = torch.cat([s[f"{b}.attn2.to_k.weight"], s[f"{b}.attn2.to_v.weight"]],
                                              0).float().to(self.dev, self.dt).contiguous()
        self._lin(b + ".attn2.to_out.0")
        self._lin(b + ".ff.net.0.proj"); self._lin(b + ".ff.net.2")
        for k in (".w", ".bias"):      # value/gate rows interleaved for the fused GEGLU epilogue
            self.p[b + ".ff.net.0.proj" + k] = D.geglu_interleave(self.p[b + ".ff.net.0.proj" + k])

    def _prep_encoder_half(self):
        cfg = self.cfg
        self._conv("conv_in")
        self._lin("time_embedding.linear_1"); self._lin("time_embedding.linear_2")
        n = len(cfg.block_out_channels)
        for i in range(n):
            for j in range(cfg.layers_per_block):
                self._prep_resnet(f"down_blocks.{i}.resnets.{j}")
                if i < n - 1:
                    self._prep_transformer(f"down_blocks.{i}.attentions.{j}")
            if i < n - 1:
                self._conv(f"down_blocks.{i}.downsamplers.0.conv")
        self._prep_resnet("mid_block.resnets.0"); self._prep_transformer("mid_block.attentions.0")
        self._prep_resnet("mid_block.resnets.1")

    def _finish_tproj(self):
        ws, bs, self.tproj_off = [], [], {}
        off = 0
        for p in self.tproj_names:
            w = self._src[p + ".time_emb_proj.weight"].float()
            ws.append(w); bs.append(self._src[p + ".time_emb_proj.bias"].float())
            self.tproj_off[p] = (off, w.shape[0]); off += w.shape[0]
        self.p["tproj.w"] = torch.cat(ws, 0).to(self.dev, self.dt).contiguous()
        self.p["tproj.b"] = torch.cat(bs, 0).to(self.dev, self.dt).contiguous()
        self.tproj_total = off
        self._src = None  # drop the host copy

    # ---- forward pieces
    def time_embed(self, t_f32, tape=None):
        """Timesteps -> TimestepEmbedding -> SiLU -> every resnet's time_emb_proj in one GEMM.  With a tape (a dict) the
        three GEMM inputs are recorded for time_embed_bwd."""
        P = self.p
        e0 = D.timestep_embedding(t_f32, self.cfg.block_out_channels[0], self.dt)
        e1 = D.gemm(e0, P["time_embedding.linear_1.w"], bias=P["time_embedding.linear_1.bias"], act="silu")
        # SiLU(temb) is the only consumer of temb (class embedding disabled, dreammat_guidance.py:311-317)
        e2 = D.gemm(e1, P["time_embedding.linear_2.w"], bias=P["time_embedding.linear_2.bias"], act="silu")
        if tape is not None:
            tape.update(e0=e0, e1=e1, e2=e2)
        return D.gemm(e2, P["tproj.w"], bias=P["tproj.b"])   # [N, sum Cout]

    def time_embed_bwd(self, rec, d_tproj, into=None):
        """Backward of time_embed(t, tape=rec) for d_tproj [N, sum Cout] (every resnet_bwd has written its columns):
        gradients of tproj and both time_embedding linears.  The fused-SiLU GEMMs kept only their activated outputs, so
        each pre-activation is recomputed by the same GEMM without the activation (M is the batch).  `into`: see backward."""
        P, grads = self.p, {}
        grads["tproj.w"], grads["tproj.b"] = D.gemm_wgrad(d_tproj, rec["e2"], bias=True, **_dst(into, dw="tproj.w", db="tproj.b"))
        d = D.gemm_dgrad(d_tproj, P["tproj.w"])
        for name, xin in (("time_embedding.linear_2", rec["e1"]), ("time_embedding.linear_1", rec["e0"])):
            z = D.gemm(xin, P[name + ".w"], bias=P[name + ".bias"])
            dz = D.silu_bwd(z, d)
            grads[name + ".w"], grads[name + ".bias"] = D.gemm_wgrad(dz, xin, bias=True, **_dst(into, dw=name + ".w", db=name + ".bias"))
            if xin is not rec["e0"]:
                d = D.gemm_dgrad(dz, P[name + ".w"])
        return grads

    def resnet(self, p, x, tproj, out=None, tape=None):
        """ResnetBlock2D.  With a tape (a dict) it records what resnet_bwd needs: x, both GroupNorm statistics and conv1's
        output; the activated GroupNorm outputs are recomputed in the backward rather than kept."""
        P, G = self.p, self.cfg.norm_groups
        n, H, W, Cin = x.shape
        h, st1 = D.groupnorm(x, P[p + ".norm1.weight"], P[p + ".norm1.bias"], G, 1e-5, silu=True)
        off, co = self.tproj_off[p]
        h1 = D.conv2d(h, P[p + ".conv1.w"], 3, bias=P[p + ".conv1.bias"], rowvec=tproj[:, off:off + co])
        h, st2 = D.groupnorm(h1, P[p + ".norm2.weight"], P[p + ".norm2.bias"], G, 1e-5, silu=True)
        xs = x if x.is_contiguous() else x.contiguous()
        if p + ".conv_shortcut.w" in P:
            sc = D.gemm(xs.view(-1, Cin), P[p + ".conv_shortcut.w"], bias=P[p + ".conv_shortcut.bias"]).view(n, H, W, co)
        else:
            sc = x
        if tape is not None:
            tape.update(p=p, x=xs, st1=st1, h1=h1, st2=st2)
        return D.conv2d(h, P[p + ".conv2.w"], 3, bias=P[p + ".conv2.bias"], residual=sc, out=out)

    def resnet_bwd(self, rec, dout, d_tproj, dx_add=None, params=True, into=None):
        """Backward of resnet(p, x, tproj, tape=rec) for the output gradient dout [n, H, W, Cout]: returns (dx, grads) and
        writes this resnet's columns of d_tproj [n, sum Cout].  dx_add is a second gradient of x (x also fed a skip
        output): it rides on the shortcut's input-gradient GEMM as its residual, or costs one add when the shortcut is the
        identity.  params=False computes dx alone (a frozen block): no parameter or d_tproj gradient (d_tproj may be None),
        and none of the GroupNorm recomputations that only feed them; grads is then empty.  `into`: see ControlNet.backward."""
        P, G, p, x, h1 = self.p, self.cfg.norm_groups, rec["p"], rec["x"], rec["h1"]
        n, H, W, Cin = x.shape
        off, co = self.tproj_off[p]
        g1, b1, g2, b2 = (P[p + k] for k in (".norm1.weight", ".norm1.bias", ".norm2.weight", ".norm2.bias"))
        grads = {}
        dout = dout if dout.is_contiguous() else dout.contiguous()
        if params:
            a2, _ = D.groupnorm(h1, g2, b2, G, 1e-5, silu=True)                  # conv2's input, recomputed
            grads[p + ".conv2.w"], grads[p + ".conv2.bias"] = D.conv2d_wgrad(a2, dout, 3, bias=True, **_dst(into, dw=p + ".conv2.w", db=p + ".conv2.bias"))
        da2 = D.conv2d_dgrad(dout, P[p + ".conv2.w"], 3)
        dh1 = D.groupnorm_bwd(h1, da2, g2, b2, rec["st2"], G, 1e-5, silu=True)
        if params:
            grads[p + ".norm2.weight"], grads[p + ".norm2.bias"] = D.groupnorm_affine_grad(
                h1, da2, g2, b2, rec["st2"], G, silu=True, **_dst(into, dgamma=p + ".norm2.weight", dbeta=p + ".norm2.bias"))
            D.rowvec_grad(dh1, n, out=d_tproj[:, off:off + co])
            a1, _ = D.groupnorm(x, g1, b1, G, 1e-5, silu=True)                   # conv1's input, recomputed
            grads[p + ".conv1.w"], grads[p + ".conv1.bias"] = D.conv2d_wgrad(a1, dh1, 3, bias=True, **_dst(into, dw=p + ".conv1.w", db=p + ".conv1.bias"))
        da1 = D.conv2d_dgrad(dh1, P[p + ".conv1.w"], 3)
        if p + ".conv_shortcut.w" in P:
            if params:
                grads[p + ".conv_shortcut.w"], grads[p + ".conv_shortcut.bias"] = D.gemm_wgrad(
                    dout.view(-1, co), x.view(-1, Cin), bias=True, **_dst(into, dw=p + ".conv_shortcut.w", db=p + ".conv_shortcut.bias"))
            dsc = D.gemm_dgrad(dout.view(-1, co), P[p + ".conv_shortcut.w"],
                               residual=dx_add.view(-1, Cin) if dx_add is not None else None).view(n, H, W, Cin)
        elif dx_add is not None:
            dsc = D.axpby(dout.view(-1, co), 1.0, dx_add.view(-1, co), 1.0).view(n, H, W, co)
        else:
            dsc = dout
        dx = D.groupnorm_bwd(x, da1, g1, b1, rec["st1"], G, 1e-5, silu=True, dx_add=dsc)
        if params:
            grads[p + ".norm1.weight"], grads[p + ".norm1.bias"] = D.groupnorm_affine_grad(
                x, da1, g1, b1, rec["st1"], G, silu=True, **_dst(into, dgamma=p + ".norm1.weight", dbeta=p + ".norm1.bias"))
        return dx, grads

    def transformer(self, p, x, ctx, heads, tape=None):
        """Transformer2DModel (one BasicTransformerBlock).  With a tape (a dict) it also records what transformer_bwd
        needs; the output is the same bits either way (attention_lse writes attention's O)."""
        P, G = self.p, self.cfg.norm_groups
        n, H, W, C = x.shape
        M = n * H * W
        attn = D.attention if tape is None else D.attention_lse
        hN, stats = D.groupnorm(x, P[p + ".norm.weight"], P[p + ".norm.bias"], G, 1e-6, silu=False)
        h0 = D.gemm(hN.view(M, C), P[p + ".proj_in.w"], bias=P[p + ".proj_in.bias"])
        b = p + ".transformer_blocks.0"
        n1 = D.layernorm(h0, P[b + ".norm1.weight"], P[b + ".norm1.bias"])
        qkv = D.gemm(n1, P[b + ".attn1.qkv.w"]).view(n, H * W, 3 * C)
        o1 = attn(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads)
        o1, lse1 = o1 if tape is not None else (o1, None)
        h1 = D.gemm(o1.view(M, C), P[b + ".attn1.to_out.0.w"], bias=P[b + ".attn1.to_out.0.bias"], residual=h0)
        n2 = D.layernorm(h1, P[b + ".norm2.weight"], P[b + ".norm2.bias"])
        q = D.gemm(n2, P[b + ".attn2.to_q.w"]).view(n, H * W, C)
        kv = D.gemm(ctx.view(-1, ctx.shape[-1]), P[b + ".attn2.kv.w"]).view(n, ctx.shape[1], 2 * C)
        o2 = attn(q, kv[..., :C], kv[..., C:], heads)
        o2, lse2 = o2 if tape is not None else (o2, None)
        h2 = D.gemm(o2.view(M, C), P[b + ".attn2.to_out.0.w"], bias=P[b + ".attn2.to_out.0.bias"], residual=h1)
        n3 = D.layernorm(h2, P[b + ".norm3.weight"], P[b + ".norm3.bias"])
        f = D.gemm(n3, P[b + ".ff.net.0.proj.w"], bias=P[b + ".ff.net.0.proj.bias"], act="geglu")
        h3 = D.gemm(f, P[b + ".ff.net.2.w"], bias=P[b + ".ff.net.2.bias"], residual=h2)
        xs = x if x.is_contiguous() else x.contiguous()
        if tape is not None:
            tape.update(p=p, heads=heads, x=xs, ctx=ctx, hN=hN, stats=stats, h0=h0, n1=n1, qkv=qkv, o1=o1, lse1=lse1, h1=h1,
                        n2=n2, q=q, kv=kv, o2=o2, lse2=lse2, h2=h2, n3=n3, f=f, h3=h3)
        return D.gemm(h3, P[p + ".proj_out.w"], bias=P[p + ".proj_out.bias"], residual=xs.view(M, C)).view(n, H, W, C)

    def transformer_bwd(self, rec, dout, params=True, into=None):
        """Backward of transformer(p, x, ctx, heads, tape=rec) for the output gradient dout [n, H, W, C]: returns (dx,
        grads), grads mapping each prepared parameter name of the block to its fp32 gradient in the prepared layout (qkv /
        kv fused, ff.net.0.proj value / gate interleaved).  ctx gets no gradient (the text encoder is frozen).  The input
        gradients read the forward weights themselves (gemm_dgrad), and the GEGLU pre-activation is recomputed by one GEMM.
        params=False computes dx alone (a frozen block): no weight gradient and no GroupNorm affine gradient; grads is then
        empty (the LayerNorm kernel still forms its affine gradients, which are dropped).  `into`: see ControlNet.backward."""
        P, G, p, heads = self.p, self.cfg.norm_groups, rec["p"], rec["heads"]
        b = p + ".transformer_blocks.0"
        x = rec["x"]
        n, H, W, C = x.shape
        M = n * H * W
        grads = {}

        def lin(name, dy, xin, bias=True):
            if params:
                dw, db = D.gemm_wgrad(dy, xin, bias=bias, **(_dst(into, dw=name + ".w", db=name + ".bias") if bias else
                                                            _dst(into, dw=name + ".w")))
                grads[name + ".w"] = dw
                if bias:
                    grads[name + ".bias"] = db
            return D.gemm_dgrad(dy, P[name + ".w"])

        def ln(name, h, dn, dadd):
            dh, dg, db = D.layernorm_bwd(h, dn, P[name + ".weight"], dx_add=dadd,
                                         **(_dst(into, dgamma=name + ".weight", dbeta=name + ".bias") if params else {}))
            if params:
                grads[name + ".weight"], grads[name + ".bias"] = dg, db
            return dh

        dy = dout.contiguous().view(M, C)
        dh3 = lin(p + ".proj_out", dy, rec["h3"])
        df = lin(b + ".ff.net.2", dh3, rec["f"])
        g = D.gemm(rec["n3"], P[b + ".ff.net.0.proj.w"], bias=P[b + ".ff.net.0.proj.bias"])
        dn3 = lin(b + ".ff.net.0.proj", D.geglu_bwd(g, df), rec["n3"])
        dh2 = ln(b + ".norm3", rec["h2"], dn3, dh3)
        do2 = lin(b + ".attn2.to_out.0", dh2, rec["o2"]).view(n, H * W, C)
        kv = rec["kv"]
        d_kv = torch.empty_like(kv)
        dq2, _, _ = D.attention_bwd(rec["q"], kv[..., :C], kv[..., C:], rec["o2"], do2, rec["lse2"], heads,
                                    dk=d_kv[..., :C], dv=d_kv[..., C:])
        if params:
            grads[b + ".attn2.kv.w"], _ = D.gemm_wgrad(d_kv, rec["ctx"], **_dst(into, dw=b + ".attn2.kv.w"))
        dn2 = lin(b + ".attn2.to_q", dq2, rec["n2"], bias=False)
        dh1 = ln(b + ".norm2", rec["h1"], dn2, dh2)
        do1 = lin(b + ".attn1.to_out.0", dh1, rec["o1"]).view(n, H * W, C)
        qkv = rec["qkv"]
        d_qkv = torch.empty_like(qkv)
        D.attention_bwd(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], rec["o1"], do1, rec["lse1"], heads,
                        dq=d_qkv[..., :C], dk=d_qkv[..., C:2 * C], dv=d_qkv[..., 2 * C:])
        dn1 = lin(b + ".attn1.qkv", d_qkv, rec["n1"], bias=False)
        dh0 = ln(b + ".norm1", rec["h0"], dn1, dh1)
        dhN = lin(p + ".proj_in", dh0, rec["hN"].view(M, C)).view(n, H, W, C)
        gm, bt = P[p + ".norm.weight"], P[p + ".norm.bias"]
        dx = D.groupnorm_bwd(x, dhN, gm, bt, rec["stats"], G, 1e-6, dx_add=dout.contiguous())
        if params:
            grads[p + ".norm.weight"], grads[p + ".norm.bias"] = D.groupnorm_affine_grad(
                x, dhN, gm, bt, rec["stats"], G, **_dst(into, dgamma=p + ".norm.weight", dbeta=p + ".norm.bias"))
        return dx, grads

    def down_and_mid(self, sample, tproj, ctx, tape=None):
        """Down blocks and mid block.  With a tape (a list) every resnet / transformer / downsampler appends one record;
        a record whose input is also a skip output res[k] carries skip_in = k."""
        cfg = self.cfg
        res = [sample]
        n = len(cfg.block_out_channels)
        skip = [0]                      # index of the skip output that the next layer consumes, or None

        def rec(kind):
            if tape is None:
                return None
            tape.append(dict(kind=kind, skip_in=skip[0]))
            skip[0] = None
            return tape[-1]

        def push(s):
            res.append(s)
            skip[0] = len(res) - 1

        for i in range(n):
            for j in range(cfg.layers_per_block):
                sample = self.resnet(f"down_blocks.{i}.resnets.{j}", sample, tproj, tape=rec("resnet"))
                if i < n - 1:
                    sample = self.transformer(f"down_blocks.{i}.attentions.{j}", sample, ctx, cfg.heads[i], tape=rec("transformer"))
                push(sample)
            if i < n - 1:
                pn = f"down_blocks.{i}.downsamplers.0.conv"
                r = rec("down")
                if r is not None:
                    r.update(p=pn, x=sample)
                sample = D.conv2d(sample, self.p[pn + ".w"], 3, stride=2, pad=(1, 1), bias=self.p[pn + ".bias"])
                push(sample)
        sample = self.resnet("mid_block.resnets.0", sample, tproj, tape=rec("resnet"))
        sample = self.transformer("mid_block.attentions.0", sample, ctx, cfg.heads[-1], tape=rec("transformer"))
        sample = self.resnet("mid_block.resnets.1", sample, tproj, tape=rec("resnet"))
        return res, sample

    def down_and_mid_bwd(self, tape, d_res, d_mid, d_tproj, into=None):
        """Backward of down_and_mid(sample, tproj, ctx, tape=tape): d_res[k] is the gradient of skip output res[k] (None
        for none), d_mid that of the mid block's output.  Walks the tape in reverse; returns (d_sample, grads) with d_res[0]
        included in d_sample, and fills d_tproj.  Where an activation feeds a skip output and the next layer, the skip's
        gradient is the residual of that layer's input-gradient kernel (downsampler, resnet with a shortcut) or one add
        (resnet whose shortcut is the identity).  `into`: see ControlNet.backward."""
        grads = {}
        d = d_mid
        for r in reversed(tape):
            extra = d_res[r["skip_in"]] if r["skip_in"] is not None else None
            if r["kind"] == "resnet":
                d, g = self.resnet_bwd(r, d, d_tproj, dx_add=extra, into=into)
            elif r["kind"] == "transformer":
                assert extra is None      # a transformer's input is a resnet's output, never a skip output
                d, g = self.transformer_bwd(r, d, into=into)
            else:
                pn = r["p"]
                d = d if d.is_contiguous() else d.contiguous()
                g = {}
                g[pn + ".w"], g[pn + ".bias"] = D.conv2d_wgrad(r["x"], d, 3, stride=2, pad=(1, 1), bias=True,
                                                                **_dst(into, dw=pn + ".w", db=pn + ".bias"))
                d = D.conv2d_dgrad(D.upsample2x(d, zero_insert=True), self.p[pn + ".w"], 3, pad=(1, 1), residual=extra)
            grads.update(g)
        return d, grads

    def grads_to_state_dict(self, grads):
        """Prepared-layout gradients -> diffusers state-dict names and shapes (what a checkpoint or a stock optimizer
        consumes): convolutions back to [Cout, Cin, kh, kw] with the channel padding dropped, q / k / v split, the GEGLU
        projection de-interleaved, time_emb_proj un-stacked."""
        out = {}
        for k, v in grads.items():
            base = k.rsplit(".", 1)[0]
            if base in self.conv_shape:
                co, ci, kh, kw = self.conv_shape[base]
                if k.endswith(".w"):
                    out[base + ".weight"] = v.view(v.shape[0], kh, kw, -1)[:co, :, :, :ci].permute(0, 3, 1, 2).contiguous()
                else:
                    out[k] = v[:co]
            elif k in ("tproj.w", "tproj.b"):
                for p, (off, co) in self.tproj_off.items():
                    out[p + (".time_emb_proj.weight" if k == "tproj.w" else ".time_emb_proj.bias")] = v[off:off + co]
            elif k.endswith(".attn1.qkv.w"):
                C = v.shape[0] // 3
                for i, nm in enumerate(("to_q", "to_k", "to_v")):
                    out[f"{base[:-4]}.{nm}.weight"] = v[i * C:(i + 1) * C]
            elif k.endswith(".attn2.kv.w"):
                C = v.shape[0] // 2
                out[base[:-3] + ".to_k.weight"], out[base[:-3] + ".to_v.weight"] = v[:C], v[C:]
            elif base.endswith(".ff.net.0.proj"):
                D2 = v.shape[0] // 2                       # interleaved blocks of 32 value rows, then 32 gate rows
                blk = v.reshape(D2 // 32, 2, 32, *v.shape[1:])
                out[base + (".weight" if k.endswith(".w") else ".bias")] = torch.cat(
                    [blk[:, 0].reshape(D2, *v.shape[1:]), blk[:, 1].reshape(D2, *v.shape[1:])], 0)
            elif k.endswith(".w"):
                is_1x1 = base.endswith(".conv_shortcut") or base.startswith("controlnet_")
                out[base + ".weight"] = v[:, :, None, None] if is_1x1 else v
            else:
                out[k] = v
        return out


class UNet(_UNetCommon):
    def __init__(self, w, cfg, device="cuda", dtype=torch.float16):
        super().__init__(w, cfg, device, dtype)
        self._prep_encoder_half()
        n = len(cfg.block_out_channels)
        for i in range(n):
            for j in range(cfg.layers_per_block + 1):
                self._prep_resnet(f"up_blocks.{i}.resnets.{j}")
                if i > 0:
                    self._prep_transformer(f"up_blocks.{i}.attentions.{j}")
            if i < n - 1:
                self._conv(f"up_blocks.{i}.upsamplers.0.conv")
        self._norm("conv_norm_out"); self._conv("conv_out")
        # conv_out's weight with its 4 output rows zero-padded to 64, the Cout that conv2d_dgrad needs, for the decoder's
        # input gradient (backward_residuals).  A copy made once is valid only because the UNet is frozen, both in the
        # guidance loop and in ControlNet training; VAEEncoder's .wd copies rely on the same fact.
        w_out = self.p["conv_out.w"]
        self.conv_out_w64 = torch.zeros(64, w_out.shape[1], device=self.dev, dtype=self.dt)
        self.conv_out_w64[:w_out.shape[0]] = w_out
        self._finish_tproj()

    def forward(self, sample_nhwc, t_f32, ctx, down_res=None, mid_res=None, csd=None, tape=None):
        """sample [N,h,w,64] (4 real channels), ctx [N,77,D] -> eps [N,4,h,w] fp32 (values rounded to the
        storage dtype, as the reference's `.sample.to(input_dtype)`).
        csd = dict(noise, w1mac, coef, grad, dlat, norms[, eps_out]): conv_out runs with the CSD combination fused
        into its epilogue (D.conv2d_csd) and nothing is returned.
        With a tape (a dict) it records what backward_residuals needs, the decoder only (nothing upstream of the residuals
        is trainable); the output is the same bits either way.  A tape and csd exclude each other."""
        if tape is not None and csd is not None:
            raise ValueError("UNet.forward: a tape records eps for the training loss; the CSD epilogue returns none")
        cfg, P = self.cfg, self.p
        tproj = self.time_embed(t_f32)
        sample = D.conv2d(sample_nhwc, P["conv_in.w"], 3, bias=P["conv_in.bias"])
        res, sample = self.down_and_mid(sample, tproj, ctx)
        if mid_res is not None:
            sample = D.axpby(sample.view(-1, sample.shape[-1]), 1.0, mid_res.view(-1, sample.shape[-1]), 1.0).view(sample.shape)
        up = tape.setdefault("up", []) if tape is not None else None

        def rec(**kw):
            if up is None:
                return None
            up.append(kw)
            return kw
        if tape is not None:
            tape["n_res"] = len(res)
        n = len(cfg.block_out_channels)
        for i in range(n):
            for j in range(cfg.layers_per_block + 1):
                k = len(res) - 1
                skip = res.pop()
                N_, H, W, C1 = sample.shape
                C2 = skip.shape[-1]
                cat = torch.empty(N_, H, W, C1 + C2, device=self.dev, dtype=self.dt)
                c2 = cat.view(-1, C1 + C2)
                D.axpby(sample.view(-1, C1), 1.0, out=c2[:, :C1])
                # skip + ControlNet residual, fused into the concat copy
                D.axpby(skip.view(-1, C2), 1.0, down_res[k].view(-1, C2) if down_res is not None else None, 1.0,
                        out=c2[:, C1:])
                sample = self.resnet(f"up_blocks.{i}.resnets.{j}", cat, tproj, tape=rec(kind="resnet", C1=C1, k=k))
                if i > 0:
                    sample = self.transformer(f"up_blocks.{i}.attentions.{j}", sample, ctx, cfg.heads[n - 1 - i],
                                              tape=rec(kind="transformer"))
            if i < n - 1:
                pn = f"up_blocks.{i}.upsamplers.0.conv"
                rec(kind="upsample", p=pn)
                sample = D.conv2d(D.upsample2x(sample), P[pn + ".w"], 3, bias=P[pn + ".bias"])
        h, st = D.groupnorm(sample, P["conv_norm_out.weight"], P["conv_norm_out.bias"], cfg.norm_groups, 1e-5, silu=True)
        if tape is not None:
            tape["norm_out"] = (sample, st)
        N_, H, W, _ = h.shape
        if csd is not None:
            D.conv2d_csd(h, P["conv_out.w"], P["conv_out.bias"], **csd)
            return None
        out = torch.empty(N_, H, W, 8, device=self.dev, dtype=self.dt)
        D.conv2d(h, P["conv_out.w"], 3, bias=P["conv_out.bias"], out=out[..., :cfg.out_channels])
        return D.nhwc_to_nchw_f32(out, cfg.out_channels)

    def backward_residuals(self, tape, d_eps):
        """Input gradient of the decoder of forward(..., down_res, mid_res, tape=tape) for d_eps [N, h, w, 64] NHWC (the
        gradient of eps in its first 4 channels, zero padding; what mse_loss_grad writes): returns (d_down, d_mid), the
        gradients of the twelve ControlNet down residuals and of the mid residual in their shapes and storage type, ready
        for ControlNet.backward.  d_down[k] and d_mid are channel slices of an up resnet's input gradient: that resnet's
        input is cat(sample, skip + down_res[k]).  No parameter gradient is formed (the UNet is frozen)."""
        cfg, P = self.cfg, self.p
        x, st = tape["norm_out"]
        dh = D.conv2d_dgrad(d_eps, self.conv_out_w64, 3)
        d = D.groupnorm_bwd(x, dh, P["conv_norm_out.weight"], P["conv_norm_out.bias"], st, cfg.norm_groups, 1e-5, silu=True)
        d_down = [None] * tape["n_res"]
        for r in reversed(tape["up"]):
            if r["kind"] == "upsample":
                d = D.upsample2x_bwd(D.conv2d_dgrad(d, P[r["p"] + ".w"], 3))
            elif r["kind"] == "transformer":
                d, _ = self.transformer_bwd(r, d, params=False)
            else:
                dx, _ = self.resnet_bwd(r, d, None, params=False)
                d_down[r["k"]] = dx[..., r["C1"]:]
                d = dx[..., :r["C1"]].contiguous()
        return d_down, d


class ControlNet(_UNetCommon):
    def __init__(self, w, cfg, device="cuda", dtype=torch.float16):
        super().__init__(w, cfg, device, dtype)
        self._prep_encoder_half()
        ce = cfg.cond_embed_channels
        self._conv("controlnet_cond_embedding.conv_in", cin_pad=_r64(cfg.cond_channels), cout_pad=_r64(ce[0]))
        k = 0
        for i in range(len(ce) - 1):
            self._conv(f"controlnet_cond_embedding.blocks.{k}", cin_pad=_r64(ce[i]), cout_pad=_r64(ce[i])); k += 1
            self._conv(f"controlnet_cond_embedding.blocks.{k}", cin_pad=_r64(ce[i]), cout_pad=_r64(ce[i + 1])); k += 1
        self._conv("controlnet_cond_embedding.conv_out", cin_pad=_r64(ce[-1]))
        self.n_skips = 0
        i = 0
        while f"controlnet_down_blocks.{i}.weight" in self._src:
            w_ = self._src[f"controlnet_down_blocks.{i}.weight"]
            self.p[f"controlnet_down_blocks.{i}.w"] = w_.float().reshape(w_.shape[0], w_.shape[1]).to(self.dev, self.dt).contiguous()
            self._vec(f"controlnet_down_blocks.{i}.bias")
            i += 1
        self.n_skips = i
        w_ = self._src["controlnet_mid_block.weight"]
        self.p["controlnet_mid_block.w"] = w_.float().reshape(w_.shape[0], w_.shape[1]).to(self.dev, self.dt).contiguous()
        self._vec("controlnet_mid_block.bias")
        self._finish_tproj()

    def cond_embed(self, cond_nhwc, tape=None):
        """ControlNetConditioningEmbedding: cond [B,8h,8w,64] (22 real channels) -> [B,h,w,C0].  With a tape (a list) the
        input of every convolution is recorded for cond_embed_bwd."""
        P = self.p
        pe = "controlnet_cond_embedding."
        nb = 2 * (len(self.cfg.cond_embed_channels) - 1)
        layers = [(pe + "conv_in", 1, "silu")] + [(f"{pe}blocks.{i}", 1 + i % 2, "silu") for i in range(nb)] + [(pe + "conv_out", 1, None)]
        c = cond_nhwc
        for pn, stride, act in layers:
            if tape is not None:
                tape.append((pn, stride, act, c))
            c = D.conv2d(c, P[pn + ".w"], 3, stride=stride, pad=(1, 1), bias=P[pn + ".bias"], act=act)
        return c

    def cond_embed_bwd(self, tape, dc, into=None):
        """Backward of cond_embed(cond, tape=tape) for the embedding's gradient dc: gradients of its eight convolutions (the
        condition itself gets none).  The forward fuses SiLU into the convolution and keeps only the activated output, so
        each pre-activation is recomputed by the same convolution without the activation.  Padded channels (22 -> 64
        condition, 16 / 32 / 96 -> 64 / 64 / 128 widths) carry zero activations and zero weights, so their gradients come
        out exactly zero.  `into`: see backward."""
        P, grads = self.p, {}
        d = dc if dc.is_contiguous() else dc.contiguous()
        for k, (pn, stride, act, x) in reversed(list(enumerate(tape))):
            if act is not None:
                z = D.conv2d(x, P[pn + ".w"], 3, stride=stride, pad=(1, 1), bias=P[pn + ".bias"])
                d = D.silu_bwd(z, d)
            grads[pn + ".w"], grads[pn + ".bias"] = D.conv2d_wgrad(x, d, 3, stride=stride, pad=(1, 1), bias=True,
                                                                  **_dst(into, dw=pn + ".w", db=pn + ".bias"))
            if k > 0:
                d = D.conv2d_dgrad(D.upsample2x(d, zero_insert=True) if stride == 2 else d, P[pn + ".w"], 3, pad=(1, 1))
        return grads

    def forward(self, sample_nhwc, t_f32, ctx, cond_nhwc, conditioning_scale=1.0, tape=None):
        """Returns (down residuals, mid residual).  With a tape (a dict) it also records what backward() needs; the outputs
        are the same bits either way."""
        P = self.p
        rec = tape is not None
        tproj = self.time_embed(t_f32, tape=tape.setdefault("time", {}) if rec else None)
        c = self.cond_embed(cond_nhwc, tape=tape.setdefault("cond", []) if rec else None)
        N_ = sample_nhwc.shape[0]
        B = c.shape[0]
        rep = N_ // B
        c_rep = torch.empty(N_, *c.shape[1:], device=self.dev, dtype=self.dt)
        for k in range(rep):   # the embedding of view b is shared by its CFG branches (layout [branch][view])
            D.axpby(c.view(-1, c.shape[-1]), 1.0, out=c_rep[k * B:(k + 1) * B].view(-1, c.shape[-1]))
        sample = D.conv2d(sample_nhwc, P["conv_in.w"], 3, bias=P["conv_in.bias"], residual=c_rep)
        res, mid = self.down_and_mid(sample, tproj, ctx, tape=tape.setdefault("walk", []) if rec else None)
        if rec:
            res = [r if r.is_contiguous() else r.contiguous() for r in res]
            tape.update(sample_in=sample_nhwc, res=res, mid=mid, scale=conditioning_scale, n_cond=B, tproj_shape=tproj.shape)
        down = []
        for i, r in enumerate(res):
            n, H, W, C = r.shape
            rs = r if r.is_contiguous() else r.contiguous()
            down.append(D.gemm(rs.view(-1, C), P[f"controlnet_down_blocks.{i}.w"], bias=P[f"controlnet_down_blocks.{i}.bias"],
                               out_scale=conditioning_scale).view(n, H, W, C))
        n, H, W, C = mid.shape
        mid = D.gemm(mid.view(-1, C), P["controlnet_mid_block.w"], bias=P["controlnet_mid_block.bias"],
                     out_scale=conditioning_scale).view(n, H, W, C)
        return down, mid

    def backward(self, tape, d_down, d_mid, into=None):
        """Gradients of every parameter from the gradients of forward(..., tape=tape)'s fourteen outputs: d_down[i] / d_mid
        in the outputs' shapes and storage type.  Returns grads mapping EVERY key of self.p to an fp32 tensor in that key's
        prepared layout (grads_to_state_dict maps them to diffusers names).  The noisy latents, the condition, the
        timesteps and ctx get no gradient.
        into: a dict with a preallocated contiguous fp32 tensor of p[key]'s shape for every key of self.p (the views of a
        flat gradient arena).  Every gradient kernel then writes its output there: nothing is allocated for a parameter
        gradient, nothing is copied afterwards, and the returned dict is `into` itself."""
        P, scale = self.p, tape["scale"]
        grads = {}

        def zero_conv(name, dy, r):
            C = r.shape[-1]
            dy = dy.reshape(-1, C) if dy.is_contiguous() else dy.contiguous().view(-1, C)
            if scale != 1.0:      # out = scale * (W r + b): fold the scale into the gradient once
                dy = D.axpby(dy, scale)
            grads[name + ".w"], grads[name + ".bias"] = D.gemm_wgrad(dy, r.view(-1, C), bias=True,
                                                                     **_dst(into, dw=name + ".w", db=name + ".bias"))
            return D.gemm_dgrad(dy, P[name + ".w"]).view(r.shape)

        d_res = [zero_conv(f"controlnet_down_blocks.{i}", d_down[i], r) for i, r in enumerate(tape["res"])]
        d_m = zero_conv("controlnet_mid_block", d_mid, tape["mid"])
        d_tproj = torch.empty(tape["tproj_shape"], device=self.dev, dtype=self.dt)
        d_sample, g = self.down_and_mid_bwd(tape["walk"], d_res, d_m, d_tproj, into=into)
        grads.update(g)
        grads["conv_in.w"], grads["conv_in.bias"] = D.conv2d_wgrad(tape["sample_in"], d_sample, 3, bias=True,
                                                                    **_dst(into, dw="conv_in.w", db="conv_in.bias"))
        B = tape["n_cond"]
        dc = d_sample[:B]             # the embedding is shared by the rep copies of a view: its gradient is their sum
        for k in range(1, d_sample.shape[0] // B):
            dc = D.axpby(dc.reshape(-1, dc.shape[-1]), 1.0, d_sample[k * B:(k + 1) * B].view(-1, dc.shape[-1]), 1.0).view(dc.shape)
        grads.update(self.cond_embed_bwd(tape["cond"], dc, into=into))
        grads.update(self.time_embed_bwd(tape["time"], d_tproj, into=into))
        if into is None:
            return grads
        assert grads.keys() == into.keys() and all(grads[k] is into[k] for k in grads)
        return into


def controlnet_loss_and_grads(unet: UNet, controlnet: ControlNet, sample_nhwc, t, ctx, cond_nhwc, target,
                              conditioning_scale=1.0, grad_scale=1.0, into=None):
    """Loss and ControlNet gradients of one ControlNet training step (controlnet_train/diffusers_train_controlnet.py:
    F.mse_loss(unet(noisy, t, ctx, down_res, mid_res).float(), target.float()), then accelerator.backward(loss)), the UNet
    frozen.  sample_nhwc [N, h, w, 64] (the noisy latents, 4 real channels), cond_nhwc [Nc, 8h, 8w, 64], ctx [N, 77, D],
    target fp32 NCHW [N, 4, h, w] (the noise, for epsilon prediction).  Returns (loss, grads): loss a 0-dim fp32 device
    tensor, grads an fp32 tensor for every key of controlnet.p in its prepared layout, multiplied by grad_scale (a loss
    scale for fp16 storage, 1 for bf16).  With `into` (ControlNet.backward) the gradients are written there and grads is
    `into`.  No host synchronisation, so the call can be captured in a CUDA graph."""
    ctape, utape = {}, {}
    down, mid = controlnet.forward(sample_nhwc, t, ctx, cond_nhwc, conditioning_scale, tape=ctape)
    eps = unet.forward(sample_nhwc, t, ctx, down, mid, tape=utape)
    loss, d_eps = D.mse_loss_grad(eps, target, unet.dt, grad_scale=grad_scale)
    d_down, d_mid = unet.backward_residuals(utape, d_eps)
    del utape           # the decoder's activations are not needed by the ControlNet backward
    return loss, controlnet.backward(ctape, d_down, d_mid, into=into)


# ================================================================================================ VAE encoder


class VAEEncoder(_Base):
    """AutoencoderKL.encode with autograd w.r.t. the input image (weights frozen), as the reference
    differentiates through it every step (SURVEY.md F5)."""

    def __init__(self, w, cfg, device="cuda", dtype=torch.float16):
        from .weights import normalize_vae_keys
        super().__init__(normalize_vae_keys(w), device, dtype)     # legacy query/key/value/proj_attn names -> to_q/...
        self.cfg = cfg
        ch = cfg.block_out_channels
        self._conv("encoder.conv_in", cin_pad=64); self._conv_dgrad("encoder.conv_in", cin_pad=64)
        n = len(ch)
        for i in range(n):
            for j in range(cfg.layers_per_block):
                self._prep_resnet(f"encoder.down_blocks.{i}.resnets.{j}")
            if i < n - 1:
                pn = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                self._conv(pn); self._conv_dgrad(pn)
        self._prep_resnet("encoder.mid_block.resnets.0"); self._prep_resnet("encoder.mid_block.resnets.1")
        p = "encoder.mid_block.attentions.0"
        self._norm(p + ".group_norm")
        s = self._src
        wq = torch.cat([s[f"{p}.to_q.weight"], s[f"{p}.to_k.weight"], s[f"{p}.to_v.weight"]], 0).float()
        self.p[p + ".qkv.w"] = wq.to(device, dtype).contiguous()
        self.p[p + ".qkv.wt"] = wq.t().contiguous().to(device, dtype)
        self.p[p + ".qkv.bias"] = torch.cat([s[f"{p}.to_q.bias"], s[f"{p}.to_k.bias"], s[f"{p}.to_v.bias"]]).float().to(device, dtype)
        self._lin(p + ".to_out.0", transpose_too=True)
        self._norm("encoder.conv_norm_out")
        self._conv("encoder.conv_out", cout_pad=64); self._conv_dgrad("encoder.conv_out", cout_pad=64)
        # quant_conv 1x1 on the (padded to 64) moments
        L2 = 2 * cfg.latent_channels
        wq_ = torch.zeros(64, 64); wq_[:L2, :L2] = s["quant_conv.weight"].float().reshape(L2, L2)
        bq = torch.zeros(64); bq[:L2] = s["quant_conv.bias"].float()
        self.p["quant_conv.w"] = wq_.to(device, dtype); self.p["quant_conv.wt"] = wq_.t().contiguous().to(device, dtype)
        self.p["quant_conv.bias"] = bq.to(device, dtype)
        self._src = None

    def _prep_resnet(self, p):
        self._norm(p + ".norm1"); self._conv(p + ".conv1"); self._conv_dgrad(p + ".conv1")
        self._norm(p + ".norm2"); self._conv(p + ".conv2"); self._conv_dgrad(p + ".conv2")
        if p + ".conv_shortcut.weight" in self._src:
            w = self._src[p + ".conv_shortcut.weight"].float()
            w2 = w.reshape(w.shape[0], w.shape[1])
            self.p[p + ".conv_shortcut.w"] = w2.to(self.dev, self.dt).contiguous()
            self.p[p + ".conv_shortcut.wt"] = w2.t().contiguous().to(self.dev, self.dt)
            self._vec(p + ".conv_shortcut.bias")

    # ---- forward (saves what the backward needs in `tape`)
    def _resnet_fwd(self, p, x, tape):
        P, G = self.p, self.cfg.norm_groups
        n, H, W, Cin = x.shape
        a, st1 = D.groupnorm(x, P[p + ".norm1.weight"], P[p + ".norm1.bias"], G, 1e-6, silu=True)
        h1 = D.conv2d(a, P[p + ".conv1.w"], 3, bias=P[p + ".conv1.bias"])
        b, st2 = D.groupnorm(h1, P[p + ".norm2.weight"], P[p + ".norm2.bias"], G, 1e-6, silu=True)
        if p + ".conv_shortcut.w" in P:
            co = P[p + ".conv_shortcut.w"].shape[0]
            sc = D.gemm(x.view(-1, Cin), P[p + ".conv_shortcut.w"], bias=P[p + ".conv_shortcut.bias"]).view(n, H, W, co)
        else:
            sc = x
        out = D.conv2d(b, P[p + ".conv2.w"], 3, bias=P[p + ".conv2.bias"], residual=sc)
        if tape is not None:
            tape.append(("res", p, x, st1, h1, st2))
        return out

    def _resnet_bwd(self, rec, dout):
        _, p, x, st1, h1, st2 = rec
        P, G = self.p, self.cfg.norm_groups
        db = D.conv2d(dout, P[p + ".conv2.wd"], 3)
        dh1 = D.groupnorm_bwd(h1, db, P[p + ".norm2.weight"], P[p + ".norm2.bias"], st2, G, 1e-6, silu=True)
        da = D.conv2d(dh1, P[p + ".conv1.wd"], 3)
        if p + ".conv_shortcut.wt" in P:
            n, H, W, Co = dout.shape
            Ci = x.shape[-1]
            dsc = D.gemm(dout.view(-1, Co), P[p + ".conv_shortcut.wt"]).view(n, H, W, Ci)
        else:
            dsc = dout
        return D.groupnorm_bwd(x, da, P[p + ".norm1.weight"], P[p + ".norm1.bias"], st1, G, 1e-6, silu=True, dx_add=dsc)

    def _attn_fwd(self, x, tape):
        P, G = self.p, self.cfg.norm_groups
        p = "encoder.mid_block.attentions.0"
        B, H, W, C = x.shape
        N = H * W
        xn, st = D.groupnorm(x, P[p + ".group_norm.weight"], P[p + ".group_norm.bias"], G, 1e-6, silu=False)
        qkv = D.gemm(xn.view(-1, C), P[p + ".qkv.w"], bias=P[p + ".qkv.bias"]).view(B, N, 3 * C)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        scale = 1.0 / (C ** 0.5)
        S = D.gemm(q, k)                                  # [B, N, N] = q k^T
        Pm = D.softmax_rows(S, scale)
        vT = D.transpose(v)                               # [B, C, N]
        o = D.gemm(Pm, vT)                                # [B, N, C]
        out = D.gemm(o.view(-1, C), P[p + ".to_out.0.w"], bias=P[p + ".to_out.0.bias"], residual=x.view(-1, C)).view(B, H, W, C)
        if tape is not None:
            tape.append(("attn", x, st, qkv, Pm, vT))
        return out

    def _attn_bwd(self, rec, dout):
        _, x, st, qkv, Pm, vT = rec
        P, G = self.p, self.cfg.norm_groups
        p = "encoder.mid_block.attentions.0"
        B, H, W, C = x.shape
        N = H * W
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        scale = 1.0 / (C ** 0.5)
        do = D.gemm(dout.view(-1, C), P[p + ".to_out.0.wt"]).view(B, N, C)      # d o = dout W_o
        dqkv = torch.empty(B, N, 3 * C, device=self.dev, dtype=self.dt)
        PT = D.transpose(Pm)                                                    # [B, Nk, Nq]
        doT = D.transpose(do)                                                   # [B, C, Nq]
        D.gemm(PT, doT, out=dqkv[..., 2 * C:])                                  # dV = P^T dO
        dP = D.gemm(do, v)                                                      # dP = dO V^T   [B,Nq,Nk]
        dS = D.softmax_bwd(Pm, dP, scale)
        kT = D.transpose(k)                                                     # [B, C, Nk]
        D.gemm(dS, kT, out=dqkv[..., :C])                                       # dQ = dS K
        dST = D.transpose(dS)
        qT = D.transpose(q)
        D.gemm(dST, qT, out=dqkv[..., C:2 * C])                                 # dK = dS^T Q
        dxn = D.gemm(dqkv.view(-1, 3 * C), P[p + ".qkv.wt"]).view(B, H, W, C)
        return D.groupnorm_bwd(x, dxn, P[p + ".group_norm.weight"], P[p + ".group_norm.bias"], st, G, 1e-6, silu=False,
                               dx_add=dout)

    def encode_moments(self, x_nhwc, tape: Optional[list] = None):
        """x [B,H,W,64] (3 real channels, already 2*rgb-1) -> moments [B,H/8,W/8,64] (8 real channels)."""
        cfg, P = self.cfg, self.p
        h = D.conv2d(x_nhwc, P["encoder.conv_in.w"], 3, bias=P["encoder.conv_in.bias"])
        n = len(cfg.block_out_channels)
        for i in range(n):
            for j in range(cfg.layers_per_block):
                h = self._resnet_fwd(f"encoder.down_blocks.{i}.resnets.{j}", h, tape)
            if i < n - 1:
                pn = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                Hh, Ww = h.shape[1], h.shape[2]
                h = D.conv2d(h, P[pn + ".w"], 3, stride=2, pad=(0, 0), out_hw=(Hh // 2, Ww // 2), bias=P[pn + ".bias"])
                if tape is not None:
                    tape.append(("down", pn))
        h = self._resnet_fwd("encoder.mid_block.resnets.0", h, tape)
        h = self._attn_fwd(h, tape)
        h = self._resnet_fwd("encoder.mid_block.resnets.1", h, tape)
        a, st = D.groupnorm(h, P["encoder.conv_norm_out.weight"], P["encoder.conv_norm_out.bias"], cfg.norm_groups, 1e-6, silu=True)
        if tape is not None:
            tape.append(("norm_out", h, st))
        c = D.conv2d(a, P["encoder.conv_out.w"], 3, bias=P["encoder.conv_out.bias"])      # [B,h,w,64], 8 real
        B, Hh, Ww, _ = c.shape
        return D.gemm(c.view(-1, 64), P["quant_conv.w"], bias=P["quant_conv.bias"]).view(B, Hh, Ww, 64)

    def backward_input(self, tape: list, dmom):
        """dmom [B,h,w,64] -> d x_nhwc [B,H,W,64] (first 3 channels meaningful)."""
        cfg, P = self.cfg, self.p
        B, Hh, Ww, _ = dmom.shape
        d = D.gemm(dmom.view(-1, 64), P["quant_conv.wt"]).view(B, Hh, Ww, 64)
        d = D.conv2d(d, P["encoder.conv_out.wd"], 3)
        rec = tape.pop()
        assert rec[0] == "norm_out"
        d = D.groupnorm_bwd(rec[1], d, P["encoder.conv_norm_out.weight"], P["encoder.conv_norm_out.bias"], rec[2],
                            cfg.norm_groups, 1e-6, silu=True)
        while tape:
            rec = tape.pop()
            if rec[0] == "res":
                d = self._resnet_bwd(rec, d)
            elif rec[0] == "attn":
                d = self._attn_bwd(rec, d)
            elif rec[0] == "down":
                up = D.upsample2x(d, zero_insert=True)
                d = D.conv2d(up, P[rec[1] + ".wd"], 3, pad=(2, 2), out_hw=(up.shape[1], up.shape[2]))
        return D.conv2d(d, P["encoder.conv_in.wd"], 3)
