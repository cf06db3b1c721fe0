"""The ControlNet training loss backpropagated through the frozen UNet: the two streaming kernels (upsample2x_bwd,
mse_loss_grad) against float64, resnet_bwd / transformer_bwd with params=False against params=True, the UNet decoder's
input gradient (UNet.forward with a tape + backward_residuals) against float64 autograd of oracle.sd.unet_forward with
respect to its residuals, and nets.controlnet_loss_and_grads against float64 autograd of the composed loss
F.mse_loss(unet_forward(..., *controlnet_forward(...)), target) for every ControlNet parameter.

Kernel bound: 1.5x the rounding floor of the output type (test_gpu_lowp.py).  Network bound: 2x the error of torch's own
autograd in the storage type on the same rounded weights and inputs (test_gpu_controlnet_bwd.py).  fp16 runs the loss at
grad_scale = numel / 2 (a loss scale, as torch's GradScaler: unscaled, 2 / numel is near fp16's smallest normal), bf16 at
1; the reference gradients are those of grad_scale * loss."""
import pytest
import torch
import torch.nn.functional as F

from oracle import sd as O
from tests.test_gpu_controlnet_bwd import _padding_is_zero
from tests.test_gpu_lowp import DTYPES, Report, rel, tname

pytestmark = pytest.mark.gpu

SMALL = dict(block_out_channels=(64, 128, 256, 256), heads=(1, 2, 4, 4), cross_attention_dim=128)


def _nchw(x, c=None):
    return (x if c is None else x[..., :c]).permute(0, 3, 1, 2)


def _skip_shapes(cfg, n, hw):
    sizes = [hw]
    for i in range(len(cfg.block_out_channels)):
        sizes += [sizes[-1]] * cfg.layers_per_block
        if i < len(cfg.block_out_channels) - 1:
            sizes.append(sizes[-1] // 2)
    chans = O.skip_channels(cfg)
    return [(n, s, s, c) for s, c in zip(sizes, chans)], (n, sizes[-1], sizes[-1], chans[-1])


# ------------------------------------------------------------------------------------------------ kernels


@DTYPES
def test_upsample2x_bwd_matches_float64_and_is_the_adjoint(dt):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(21)
    rep = Report(f"upsample2x_bwd {tname(dt)} (bound 1.5x rounding floor)")
    for n, H, W, C in ((2, 8, 8, 320), (1, 16, 12, 1280), (3, 5, 7, 64), (2, 32, 32, 640)):
        dy = torch.randn(n, 2 * H, 2 * W, C, device="cuda", generator=g).to(dt)
        ref = dy.double().view(n, H, 2, W, 2, C).sum((2, 4))
        got = D.upsample2x_bwd(dy)
        assert got.shape == (n, H, W, C) and got.dtype == dt
        rep.cmp(f"{n}x{H}x{W}x{C}", got, ref, dt)
        # <upsample2x(x), dy> = <x, upsample2x_bwd(dy)>, up to the rounding of got (Cauchy-Schwarz on got - ref)
        x = torch.randn(n, H, W, C, device="cuda", generator=g).to(dt)
        lhs = (D.upsample2x(x).double() * dy.double()).sum()
        rhs = (x.double() * got.double()).sum()
        bound = x.double().norm() * 1.5 * (ref.to(dt).double() - ref).norm() + 1e-9 * lhs.abs()
        assert (lhs - rhs).abs() <= bound, (n, H, W, C, float(lhs), float(rhs), float(bound))
        assert torch.equal(got, D.upsample2x_bwd(dy))
    rep.check()


@DTYPES
def test_mse_loss_grad_matches_float64_and_repeats(dt):
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(22)
    rep = Report(f"mse_loss_grad d_pred {tname(dt)} (bound 1.5x rounding floor)")
    for n, C, H, W, ld in ((2, 4, 16, 16, 64), (4, 4, 32, 32, 64), (3, 70, 5, 9, 128), (1, 4, 64, 64, 128)):
        numel = n * C * H * W
        gs = numel / 2 if dt == torch.float16 else 1.0
        pred = (torch.randn(n, C, H, W, device="cuda", generator=g) * 1.3).to(dt).float()   # as UNet.forward returns it
        target = torch.randn(n, C, H, W, device="cuda", generator=g)
        loss, d = D.mse_loss_grad(pred, target, dt, ld=ld, grad_scale=gs)
        assert loss.shape == () and loss.dtype == torch.float32 and d.shape == (n, H, W, ld) and d.dtype == dt
        diff = pred.double() - target.double()
        ref_loss = (diff * diff).mean()
        err = abs(float(loss) - float(ref_loss)) / float(ref_loss)
        print(f"\nmse_loss_grad loss {n}x{C}x{H}x{W}: rel err {err:.2e} (bound 1e-5)")
        assert err <= 1e-5
        rep.cmp(f"{n}x{C}x{H}x{W} ld {ld}", _nchw(d, C), gs * 2.0 / numel * diff, dt)
        assert not d[..., C:].any()
        loss2, d2 = D.mse_loss_grad(pred, target, dt, ld=ld, grad_scale=gs)
        assert torch.equal(loss, loss2) and torch.equal(d, d2)
    rep.check()


# ------------------------------------------------------------------------------------------------ params=False


@DTYPES
def test_dx_only_backward_equals_full_backward(dt):
    from dreammat_b200 import nets, weights
    cfg = weights.UNetConfig()
    g = torch.Generator().manual_seed(31)
    gc = torch.Generator(device="cuda").manual_seed(32)
    pr, pt = "up_blocks.1.resnets.0", "up_blocks.1.attentions.0"
    w = {}
    O._rand_resnet(g, w, pr, 1920, 1280, cfg.time_dim)
    O._rand_transformer(g, w, pt, 640, cfg.cross_attention_dim)
    w = {k: v.to(dt) for k, v in w.items()}
    net = nets._UNetCommon(w, cfg, "cuda", dt)
    net._prep_resnet(pr); net._prep_transformer(pt)
    net._finish_tproj()

    x = torch.randn(2, 8, 8, 1920, device="cuda", generator=gc).to(dt)
    tp = torch.randn(2, 1280, device="cuda", generator=gc).to(dt)
    dout = torch.randn(2, 8, 8, 1280, device="cuda", generator=gc).to(dt)
    tape = {}
    net.resnet(pr, x, tp, tape=tape)
    dx_full, g_full = net.resnet_bwd(tape, dout, torch.zeros(2, 1280, device="cuda", dtype=dt))
    dx_only, g_only = net.resnet_bwd(tape, dout, None, params=False)
    assert "up_blocks.1.resnets.0.conv_shortcut.w" in g_full and g_only == {}
    assert torch.equal(dx_full, dx_only)

    x = torch.randn(2, 16, 16, 640, device="cuda", generator=gc).to(dt)
    ctx = torch.randn(2, 77, cfg.cross_attention_dim, device="cuda", generator=gc).to(dt)
    dout = torch.randn(2, 16, 16, 640, device="cuda", generator=gc).to(dt)
    tape = {}
    net.transformer(pt, x, ctx, 10, tape=tape)
    dx_full, g_full = net.transformer_bwd(tape, dout)
    dx_only, g_only = net.transformer_bwd(tape, dout, params=False)
    assert len(g_full) > 10 and g_only == {}
    assert torch.equal(dx_full, dx_only)


# ------------------------------------------------------------------------------------------------ UNet decoder


def _unet_setup(cfg, dt, n, hw, seed):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import UNet
    w = {k: v.to(dt) for k, v in O.random_unet_weights(cfg, seed).items()}
    net = UNet(w, cfg, dtype=dt)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    zp = D.pad_convert(torch.randn(n, hw, hw, 4, device="cuda", generator=g), 64, dtype=dt)
    ctx = torch.randn(n, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    down_shapes, mid_shape = _skip_shapes(cfg, n, hw)
    down = [(0.5 * torch.randn(s, device="cuda", generator=g)).to(dt) for s in down_shapes]
    mid = (0.5 * torch.randn(mid_shape, device="cuda", generator=g)).to(dt)
    d_eps = torch.zeros(n, hw, hw, 64, device="cuda", dtype=dt)
    d_eps[..., :cfg.out_channels] = torch.randn(n, hw, hw, cfg.out_channels, device="cuda", generator=g).to(dt)
    return w, net, zp, ctx, down, mid, d_eps


def _unet_autograd(w, cfg, zp, t, ctx, down, mid, d_eps, dtype):
    wd = {k: v.to("cuda", dtype) for k, v in w.items()}
    dr = [_nchw(r).to(dtype).clone().requires_grad_() for r in down]
    mr = _nchw(mid).to(dtype).clone().requires_grad_()
    eps = O.unet_forward(wd, cfg, _nchw(zp, 4).to(dtype), t, ctx.to(dtype), dr, mr, q=lambda v: v.to("cuda", dtype))
    eps.backward(_nchw(d_eps, cfg.out_channels).to(dtype))
    return [r.grad.permute(0, 2, 3, 1) for r in dr], mr.grad.permute(0, 2, 3, 1)


@DTYPES
def test_full_size_unet_decoder_input_gradient_matches_fp64_autograd(dt, monkeypatch):
    from dreammat_b200 import dense_ops as D
    cfg = O.UNetConfig()
    w, net, zp, ctx, down, mid, d_eps = _unet_setup(cfg, dt, 2, 16, 41)
    t = torch.tensor([140.0, 820.0])
    tape = {}
    eps = net.forward(zp, t.cuda(), ctx, down, mid, tape=tape)
    assert torch.equal(eps, net.forward(zp, t.cuda(), ctx, down, mid))

    def forbidden(*_, **__):
        raise AssertionError("the frozen UNet's backward computed a parameter gradient")
    with monkeypatch.context() as m:
        for name in ("conv2d_wgrad", "gemm_wgrad", "groupnorm_affine_grad", "rowvec_grad"):
            m.setattr(D, name, forbidden)
        d_down, d_mid = net.backward_residuals(tape, d_eps)
    del tape
    assert len(d_down) == 12
    for got, r in zip(d_down + [d_mid], down + [mid]):
        assert got.shape == r.shape and got.dtype == dt
    ref_down, ref_mid = _unet_autograd(w, cfg, zp, t, ctx, down, mid, d_eps, torch.float64)
    flo_down, flo_mid = _unet_autograd(w, cfg, zp, t, ctx, down, mid, d_eps, dt)
    rep = Report(f"UNet decoder input gradient, full size, {tname(dt)} (bound 2x torch-autograd-in-{tname(dt)} floor)")
    for k in range(12):
        rep.rows.append((f"d_down[{k}] {tuple(down[k].shape)}", rel(d_down[k], ref_down[k]), rel(flo_down[k], ref_down[k]), 2.0))
    rep.rows.append(("d_mid", rel(d_mid, ref_mid), rel(flo_mid, ref_mid), 2.0))
    rep.check()


# ------------------------------------------------------------------------------------------------ end to end


def _e2e_setup(cfg, dt, n, n_cond, hw, seed, t):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import ControlNet, UNet
    wc = {k: v.to(dt) for k, v in O.random_controlnet_weights(cfg, seed).items()}
    wu = {k: v.to(dt) for k, v in O.random_unet_weights(cfg, seed + 1).items()}
    g = torch.Generator(device="cuda").manual_seed(seed + 2)
    zp = D.pad_convert(torch.randn(n, hw, hw, 4, device="cuda", generator=g), 64, dtype=dt)
    cp = D.pad_convert(torch.rand(n_cond, 8 * hw, 8 * hw, cfg.cond_channels, device="cuda", generator=g), 64, dtype=dt)
    ctx = torch.randn(n, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    target = torch.randn(n, cfg.out_channels, hw, hw, device="cuda", generator=g)
    gs = n * cfg.out_channels * hw * hw / 2 if dt == torch.float16 else 1.0
    return (wc, wu, UNet(wu, cfg, dtype=dt), ControlNet(wc, cfg, dtype=dt), zp, cp, ctx, torch.tensor(t, dtype=torch.float32),
            target, gs)


def _loss_autograd(wc, wu, cfg, zp, cp, ctx, t, target, scale, gs, dtype):
    q = lambda v: v.to("cuda", dtype)     # noqa: E731
    wcd = {k: v.to("cuda", dtype).requires_grad_() for k, v in wc.items()}
    wud = {k: v.to("cuda", dtype) for k, v in wu.items()}          # the UNet is frozen
    s = _nchw(zp, 4).to(dtype)
    down, mid = O.controlnet_forward(wcd, cfg, s, t, ctx.to(dtype), _nchw(cp, cfg.cond_channels).to(dtype), scale, q=q)
    eps = O.unet_forward(wud, cfg, s, t, ctx.to(dtype), down, mid, q=q)
    pred = eps.double() if dtype == torch.float64 else eps.float()
    loss = F.mse_loss(pred, target.to(pred.dtype))
    (gs * loss).backward()
    return loss.detach(), eps.detach(), {k: v.grad for k, v in wcd.items()}


def _check_e2e(title, cfg, dt, setup, scale):
    from dreammat_b200 import nets
    wc, wu, unet, cnet, zp, cp, ctx, t, target, gs = setup
    loss, grads = nets.controlnet_loss_and_grads(unet, cnet, zp, t.cuda(), ctx, cp, target, scale, gs)
    assert loss.shape == () and loss.dtype == torch.float32
    assert set(grads) == set(cnet.p) and _padding_is_zero(cnet, grads) >= 8
    for k, v in grads.items():
        assert v.dtype == torch.float32 and v.shape == cnet.p[k].shape, k
    got = cnet.grads_to_state_dict(grads)
    del grads
    l64, e64, ref = _loss_autograd(wc, wu, cfg, zp, cp, ctx, t, target, scale, gs, torch.float64)
    ldt, edt, flo = _loss_autograd(wc, wu, cfg, zp, cp, ctx, t, target, scale, gs, dt)
    assert set(got) == set(ref), set(ref) ^ set(got)
    rep = Report(title)
    # the loss is one number, so its error against torch's is a ratio of two random roundings; its floor is the larger of
    # torch's loss error and torch's error of eps itself
    rep.rows.append(("loss", rel(loss, l64), max(rel(ldt, l64), rel(edt, e64)), 2.0))
    for k in sorted(ref):
        assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
        rep.rows.append((k, rel(got[k], ref[k]), rel(flo[k], ref[k]), 2.0))
    rep.check()


@DTYPES
def test_full_size_controlnet_loss_and_grads_match_fp64_autograd(dt):
    cfg = O.UNetConfig()
    setup = _e2e_setup(cfg, dt, 2, 2, 16, 51, [90.0, 610.0])
    _check_e2e(f"ControlNet loss + gradients through the frozen UNet, full size, {tname(dt)} (bound 2x floor)", cfg, dt, setup, 1.0)


@DTYPES
def test_controlnet_loss_and_grads_conditioning_scale(dt):
    """conditioning_scale 0.5, and one condition embedding shared by two copies of each view, on a small configuration"""
    cfg = O.UNetConfig(**SMALL)
    setup = _e2e_setup(cfg, dt, 4, 2, 16, 61, [30.0, 400.0, 650.0, 990.0])
    _check_e2e(f"ControlNet loss + gradients, small, scale 0.5, {tname(dt)} (bound 2x floor)", cfg, dt, setup, 0.5)


@DTYPES
def test_controlnet_loss_and_grads_deterministic_and_graph_replay(dt):
    from dreammat_b200 import nets
    cfg = O.UNetConfig()
    _, _, unet, cnet, zp, cp, ctx, t, target, gs = _e2e_setup(cfg, dt, 2, 2, 16, 71, [250.0, 700.0])
    tc = t.cuda()

    def run():
        loss, grads = nets.controlnet_loss_and_grads(unet, cnet, zp, tc, ctx, cp, target, 1.0, gs)
        return [loss] + [grads[k] for k in sorted(grads)]

    one, two = run(), run()
    for a, b in zip(one, two):
        assert torch.equal(a, b)
    del two
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(one, captured):
        assert torch.equal(a, b)
