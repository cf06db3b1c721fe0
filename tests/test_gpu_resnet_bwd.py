"""The streaming backward kernels (rowvec_grad, silu_bwd) against float64, and one ResnetBlock2D / the time embedding
differentiated by nets (resnet with a tape + resnet_bwd, time_embed + time_embed_bwd) against float64 autograd.

Kernel bound: 1.5x the rounding floor of the output type (the convention of test_gpu_norm_geglu_bwd.py).  Network bound:
2x the error of torch's own autograd in the storage type on the same rounded weights and inputs (the convention of
test_gpu_transformer_bwd.py).  The resnet reference is oracle.sd.resnet's own sequence of oracle.sd building blocks with
the time-embedding projection's output as a leaf, so that d_tproj itself can be compared."""
import pytest
import torch
import torch.nn.functional as F

from oracle import sd as O
from tests.test_gpu_lowp import DTYPES, Report, rel, tname

pytestmark = pytest.mark.gpu

P = "down_blocks.1.resnets.0"
RESNETS = [(320, 320, 32, 2), (960, 640, 16, 2)]        # (Cin, Cout, H = W, batch)


@DTYPES
def test_rowvec_grad_and_silu_bwd_match_float64(dt):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(5)
    rep = Report(f"rowvec_grad / silu_bwd {tname(dt)} (bound 1.5x rounding floor)")
    for n, rows, N in ((2, 1024, 320), (4, 16, 1280), (3, 100, 64)):
        dy = torch.randn(n * rows, N, device="cuda", generator=g).to(dt)
        rep.cmp(f"rowvec_grad {n}x{rows}x{N}", D.rowvec_grad(dy, n), dy.double().view(n, rows, N).sum(1), dt)
        wide = torch.zeros(n, N + 64, device="cuda", dtype=dt)
        D.rowvec_grad(dy.view(n, rows, N), n, out=wide[:, 64:])
        rep.exact(f"rowvec_grad {n}x{rows}x{N} into a column slice", wide[:, 64:], D.rowvec_grad(dy, n))
        assert not wide[:, :64].any()
    srcw = torch.randn(512, 128, device="cuda", generator=g).to(dt)
    rep.cmp("rowvec_grad of a column slice", D.rowvec_grad(srcw[:, 64:], 2), srcw[:, 64:].double().view(2, 256, 64).sum(1), dt)
    z = (torch.randn(4, 33, 320, device="cuda", generator=g) * 3).to(dt)
    dy = torch.randn(4, 33, 320, device="cuda", generator=g).to(dt)
    zd = z.double().requires_grad_()
    F.silu(zd).backward(dy.double())
    rep.cmp("silu_bwd", D.silu_bwd(z, dy), zd.grad, dt)
    rep.check()
    a, b = D.rowvec_grad(srcw, 2), D.rowvec_grad(srcw, 2)
    assert torch.equal(a, b)


def _resnet_ref(w, x, tp, dout, dtype):
    wd = {k: v.to("cuda", dtype).requires_grad_() for k, v in w.items() if "time_emb_proj" not in k}
    xd = x.to(dtype).permute(0, 3, 1, 2).contiguous().requires_grad_()
    tpd = tp.to(dtype).clone().requires_grad_()
    h = F.silu(O.gn(wd, P + ".norm1", xd, 32, 1e-5))
    h = O.conv(wd, P + ".conv1", h) + tpd[:, :, None, None]
    h = O.conv(wd, P + ".conv2", F.silu(O.gn(wd, P + ".norm2", h, 32, 1e-5)))
    sc = O.conv(wd, P + ".conv_shortcut", xd, padding=0) if P + ".conv_shortcut.weight" in wd else xd
    (sc + h).backward(dout.to(dtype).permute(0, 3, 1, 2))
    out = {k: v.grad for k, v in wd.items()}
    out["x"], out["tproj"] = xd.grad.permute(0, 2, 3, 1), tpd.grad
    return out


@DTYPES
def test_resnet_bwd_matches_fp64_autograd(dt):
    from dreammat_b200 import nets, weights
    rep = Report(f"ResnetBlock2D backward {tname(dt)} (bound 2x torch-autograd-in-{tname(dt)} floor)")
    for ci, co, S, B in RESNETS:
        g = torch.Generator().manual_seed(ci)
        w = {}
        O._rand_resnet(g, w, P, ci, co, 1280)
        w = {k: v.to(dt) for k, v in w.items()}
        net = nets._UNetCommon(w, weights.UNetConfig(), "cuda", dt)
        net._prep_resnet(P)
        net._finish_tproj()
        gc = torch.Generator(device="cuda").manual_seed(ci + 1)
        x = torch.randn(B, S, S, ci, device="cuda", generator=gc).to(dt)
        tp = torch.randn(B, co, device="cuda", generator=gc).to(dt)
        dout = torch.randn(B, S, S, co, device="cuda", generator=gc).to(dt)
        extra = torch.randn(B, S, S, ci, device="cuda", generator=gc).to(dt)
        tape = {}
        y = net.resnet(P, x, tp, tape=tape)
        assert torch.equal(y, net.resnet(P, x, tp))
        d_tproj = torch.zeros(B, co, device="cuda", dtype=dt)
        dx, grads = net.resnet_bwd(tape, dout, d_tproj)
        got = net.grads_to_state_dict(grads)
        got["x"], got["tproj"] = dx, d_tproj
        ref, flo = _resnet_ref(w, x, tp, dout, torch.float64), _resnet_ref(w, x, tp, dout, dt)
        assert set(got) == set(ref), set(ref) ^ set(got)
        for k in sorted(ref):
            rep.rows.append((f"{ci}->{co} {k}", rel(got[k], ref[k]), rel(flo[k], ref[k]), 2.0))
        # a second gradient of x: on the shortcut GEMM's residual (960 -> 640) or one add (320 -> 320)
        dx2, _ = net.resnet_bwd(tape, dout, d_tproj, dx_add=extra)
        rep.rows.append((f"{ci}->{co} x with a skip gradient", rel(dx2, ref["x"] + extra.double()), rel(flo["x"] + extra, ref["x"] + extra.double()), 2.0))
    rep.check()


@DTYPES
def test_time_embed_bwd_matches_fp64_autograd(dt):
    from dreammat_b200 import nets, weights
    cfg = weights.UNetConfig()
    g = torch.Generator().manual_seed(3)
    w = {}
    O._put(w, "time_embedding.linear_1", O._rand_lin(g, cfg.time_dim, 320))
    O._put(w, "time_embedding.linear_2", O._rand_lin(g, cfg.time_dim, cfg.time_dim))
    names = [("down_blocks.0.resnets.0", 320), ("down_blocks.1.resnets.0", 640), ("mid_block.resnets.0", 1280)]
    for p, co in names:
        O._put(w, p + ".time_emb_proj", O._rand_lin(g, co, cfg.time_dim))
    w = {k: v.to(dt) for k, v in w.items()}
    net = nets._UNetCommon(w, cfg, "cuda", dt)
    net._lin("time_embedding.linear_1"); net._lin("time_embedding.linear_2")
    net.tproj_names = [p for p, _ in names]
    net._finish_tproj()
    t = torch.tensor([20.0, 333.0, 700.0, 981.0])
    d_tproj = torch.randn(4, net.tproj_total, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4)).to(dt)
    tape = {}
    tproj = net.time_embed(t.cuda(), tape=tape)
    assert torch.equal(tproj, net.time_embed(t.cuda()))
    got = net.grads_to_state_dict(net.time_embed_bwd(tape, d_tproj))

    def ref(dtype):
        wd = {k: v.to("cuda", dtype).requires_grad_() for k, v in w.items()}
        temb = O._time_embed(wd, cfg, t, lambda v: v.to("cuda", dtype))
        out = torch.cat([O.linear(wd, p + ".time_emb_proj", F.silu(temb)) for p, _ in names], 1)
        out.backward(d_tproj.to(dtype))
        return {k: v.grad for k, v in wd.items()}, out

    (r64, _), (rdt, _) = ref(torch.float64), ref(dt)
    assert set(got) == set(r64), set(r64) ^ set(got)
    rep = Report(f"time embedding backward {tname(dt)} (bound 2x torch-autograd-in-{tname(dt)} floor)")
    for k in sorted(r64):
        rep.rows.append((k, rel(got[k], r64[k]), rel(rdt[k], r64[k]), 2.0))
    rep.check()
