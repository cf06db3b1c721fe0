"""LayerNorm backward, the interleaved GEGLU backward and the GroupNorm affine gradients against float64 autograd.

Inputs are drawn and rounded to the storage type; the same values go to the kernel and to float64 autograd of
F.layer_norm / the GEGLU of diffusers / F.group_norm (+ SiLU).  dx / dh are computed in fp32 and rounded once, so they
must stay within SINGLE x their rounding floor (test_gpu_lowp.py); the fp32 affine gradients within ACC32.  Row counts are
ragged against every block / chunk size; widths are the model's."""
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_lowp import ACC32, DTYPES, SINGLE, Report, gen, randn, tname  # noqa: F401

pytestmark = pytest.mark.gpu


@DTYPES
def test_layernorm_bwd_matches_fp64(dt, gen):
    from dreammat_b200 import dense_ops as D
    rep = Report(f"layernorm_bwd {tname(dt)}")
    for C, M, add in ((320, 2 * 1024 + 3, True), (640, 513, False), (1280, 4 * 16 + 5, True), (320, 1, False)):
        x = randn(gen, M, C, scale=2.0, shift=0.5).to(dt)
        g, bt = (1 + 0.1 * randn(gen, C)).to(dt), (0.05 * randn(gen, C)).to(dt)
        dy = randn(gen, M, C).to(dt)
        dadd = randn(gen, M, C).to(dt) if add else None
        xd, gd, bd = (t.double().requires_grad_() for t in (x, g, bt))
        F.layer_norm(xd, (C,), gd, bd, 1e-5).backward(dy.double())
        dx, dg, db = D.layernorm_bwd(x, dy, g, dx_add=dadd)
        rep.cmp(f"C{C} M{M} dx", dx, xd.grad + (dadd.double() if add else 0), dt)
        rep.cmp(f"C{C} M{M} dgamma", dg, gd.grad, torch.float32)
        rep.cmp(f"C{C} M{M} dbeta", db, bd.grad, torch.float32)
    rep.check()


@DTYPES
def test_geglu_bwd_interleaved_matches_fp64(dt, gen):
    from dreammat_b200 import dense_ops as D
    rep = Report(f"geglu_bwd (interleaved) {tname(dt)}")
    for Dd, M in ((1280, 1024 + 7), (2560, 259), (5120, 21)):
        h = randn(gen, M, 2 * Dd).to(dt)              # [value | gate] halves, as diffusers' GEGLU.proj writes them
        dout = randn(gen, M, Dd).to(dt)
        hd = h.double().requires_grad_()
        a, gate = hd.chunk(2, -1)
        (a * F.gelu(gate)).backward(dout.double())
        hi = D.geglu_interleave(h.t()).t().contiguous()   # the fused epilogue's column order
        dh = D.geglu_bwd(hi, dout)
        rep.cmp(f"D{Dd} M{M} dh", dh, D.geglu_interleave(hd.grad.t()).t(), dt)
    rep.check()


@DTYPES
def test_groupnorm_affine_grad_matches_fp64(dt, gen):
    from dreammat_b200 import dense_ops as D
    rep = Report(f"groupnorm_affine_grad {tname(dt)}")
    for (n, H, W, C, silu) in ((2, 32, 32, 320, False), (2, 32, 32, 320, True), (2, 16, 16, 640, True),
                               (4, 4, 4, 1280, False), (3, 8, 8, 1280, True), (1, 5, 7, 640, False)):
        x = randn(gen, n, H, W, C, scale=1.5, shift=0.3).to(dt)
        g, bt = (1 + 0.1 * randn(gen, C)).to(dt), (0.05 * randn(gen, C)).to(dt)
        dz = randn(gen, n, H, W, C).to(dt)
        _, stats = D.groupnorm(x, g, bt, 32, 1e-5, silu=silu)
        gd, bd = (t.double().requires_grad_() for t in (g, bt))
        y = F.group_norm(x.double().permute(0, 3, 1, 2), 32, gd, bd, 1e-5)
        (F.silu(y) if silu else y).backward(dz.double().permute(0, 3, 1, 2))
        dg, db = D.groupnorm_affine_grad(x, dz, g, bt, stats, 32, silu=silu)
        rep.cmp(f"{n}x{H}x{W}x{C} silu={silu} dgamma", dg, gd.grad, torch.float32)
        rep.cmp(f"{n}x{H}x{W}x{C} silu={silu} dbeta", db, bd.grad, torch.float32)
    rep.check()
