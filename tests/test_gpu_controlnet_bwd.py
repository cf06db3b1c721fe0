"""The whole ControlNet differentiated by nets (forward with a tape, then ControlNet.backward) against float64 autograd of
oracle.sd.controlnet_forward, for every parameter.

Weights come from oracle.sd.random_controlnet_weights (zero convolutions random, or nothing would flow) rounded to the
storage type; the same rounded weights, inputs and output gradients go to nets and to the references.  The floor of each
gradient is the error of torch's own autograd of the same oracle in the storage type on the GPU; nets must stay within 2x
that floor.  grads_to_state_dict maps the prepared layouts back to the oracle's (diffusers') names and drops the channel
padding; the padded parts of the prepared gradients are checked to be exactly zero."""
import pytest
import torch

from oracle import sd as O
from tests.test_gpu_lowp import DTYPES, Report, rel, tname

pytestmark = pytest.mark.gpu


def _setup(cfg, dt, n, n_cond, hw, seed, t):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import ControlNet
    w = {k: v.to(dt) for k, v in O.random_controlnet_weights(cfg, seed).items()}
    net = ControlNet(w, cfg, dtype=dt)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    z = torch.randn(n, hw, hw, 4, device="cuda", generator=g)
    cond = torch.rand(n_cond, 8 * hw, 8 * hw, cfg.cond_channels, device="cuda", generator=g)
    ctx = torch.randn(n, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    zp, cp = D.pad_convert(z, 64, dtype=dt), D.pad_convert(cond, 64, dtype=dt)
    chans = O.skip_channels(cfg)
    sizes = [hw]
    for i in range(len(cfg.block_out_channels)):
        sizes += [sizes[-1]] * cfg.layers_per_block
        if i < len(cfg.block_out_channels) - 1:
            sizes.append(sizes[-1] // 2)
    d_down = [torch.randn(n, s, s, c, device="cuda", generator=g).to(dt) for s, c in zip(sizes[:len(chans)], chans)]
    d_mid = torch.randn(n, sizes[-1], sizes[-1], chans[-1], device="cuda", generator=g).to(dt)
    return w, net, zp, cp, ctx, torch.tensor(t, dtype=torch.float32), d_down, d_mid


def _autograd(w, cfg, zp, cp, ctx, t, d_down, d_mid, scale, dtype):
    wd = {k: v.to("cuda", dtype).requires_grad_() for k, v in w.items()}
    nchw = lambda x, c=None: (x if c is None else x[..., :c]).to(dtype).permute(0, 3, 1, 2)   # noqa: E731
    down, mid = O.controlnet_forward(wd, cfg, nchw(zp, 4), t, ctx.to(dtype), nchw(cp, cfg.cond_channels), scale,
                                     q=lambda v: v.to("cuda", dtype))
    torch.autograd.backward(down + [mid], [nchw(d) for d in d_down] + [nchw(d_mid)])
    return {k: v.grad for k, v in wd.items()}


def _compare(title, net, got, ref, flo):
    assert set(got) == set(ref), set(ref) ^ set(got)
    rep = Report(title)
    for k in sorted(ref):
        assert got[k].shape == ref[k].shape, (k, got[k].shape, ref[k].shape)
        rep.rows.append((k, rel(got[k], ref[k]), rel(flo[k], ref[k]), 2.0))
    rep.check()


def _padding_is_zero(net, grads):
    """padded rows / columns of the prepared conv gradients (22 -> 64 condition, 4 -> 64 latents, 16 / 32 / 96 -> 64 / 64 /
    128 embedding widths) are exactly zero"""
    checked = 0
    for name, (co, ci, kh, kw) in net.conv_shape.items():
        g = grads[name + ".w"]
        g4 = g.view(g.shape[0], kh, kw, -1)
        if g4.shape[0] > co or g4.shape[3] > ci:
            assert not g4[co:].any() and not g4[..., ci:].any() and not grads[name + ".bias"][co:].any(), name
            checked += 1
    return checked


@DTYPES
def test_full_size_controlnet_backward_matches_fp64_autograd(dt):
    cfg = O.UNetConfig()
    w, net, zp, cp, ctx, t, d_down, d_mid = _setup(cfg, dt, 2, 2, 16, 11, [120.0, 760.0])
    tape = {}
    down, mid = net.forward(zp, t.cuda(), ctx, cp, tape=tape)
    plain_down, plain_mid = net.forward(zp, t.cuda(), ctx, cp)
    assert all(torch.equal(a, b) for a, b in zip(down + [mid], plain_down + [plain_mid]))
    grads = net.backward(tape, d_down, d_mid)
    assert set(grads) == set(net.p)
    for k, v in grads.items():
        assert v.dtype == torch.float32 and v.shape == net.p[k].shape, k
    assert _padding_is_zero(net, grads) >= 8
    got = net.grads_to_state_dict(grads)
    del tape, grads
    ref = _autograd(w, cfg, zp, cp, ctx, t, d_down, d_mid, 1.0, torch.float64)
    flo = _autograd(w, cfg, zp, cp, ctx, t, d_down, d_mid, 1.0, dt)
    _compare(f"ControlNet backward, full size, {tname(dt)} (bound 2x torch-autograd-in-{tname(dt)} floor)", net, got, ref, flo)


@DTYPES
def test_controlnet_backward_deterministic_and_graph_replay(dt):
    cfg = O.UNetConfig()
    w, net, zp, cp, ctx, t, d_down, d_mid = _setup(cfg, dt, 2, 2, 16, 13, [50.0, 900.0])
    tc = t.cuda()

    def run():
        tape = {}
        down, mid = net.forward(zp, tc, ctx, cp, tape=tape)
        grads = net.backward(tape, d_down, d_mid)
        return down + [mid] + [grads[k] for k in sorted(grads)]

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


@DTYPES
def test_conditioning_scale_and_shared_condition_embedding(dt):
    """conditioning_scale 0.5 and rep = 3 (one condition embedding shared by three copies of each view) on a small
    configuration"""
    cfg = O.UNetConfig(block_out_channels=(64, 128, 256, 256), heads=(1, 2, 4, 4), cross_attention_dim=128)
    w, net, zp, cp, ctx, t, d_down, d_mid = _setup(cfg, dt, 6, 2, 16, 17, [100.0, 700.0] * 3)
    tape = {}
    net.forward(zp, t.cuda(), ctx, cp, 0.5, tape=tape)
    grads = net.backward(tape, d_down, d_mid)
    assert set(grads) == set(net.p) and _padding_is_zero(net, grads) >= 8
    got = net.grads_to_state_dict(grads)
    ref = _autograd(w, cfg, zp, cp, ctx, t, d_down, d_mid, 0.5, torch.float64)
    flo = _autograd(w, cfg, zp, cp, ctx, t, d_down, d_mid, 0.5, dt)
    _compare(f"ControlNet backward, small, scale 0.5, rep 3, {tname(dt)} (bound 2x floor)", net, got, ref, flo)
