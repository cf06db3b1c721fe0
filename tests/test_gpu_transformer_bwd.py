"""A whole Transformer2DModel differentiated by nets (transformer with a tape, then transformer_bwd) against float64
autograd of the oracle's own oracle.sd.transformer, for the input and every parameter.

Weights come from oracle.sd._rand_transformer and are rounded to the storage type; the same rounded weights, x, ctx
(77 x 1024) and dout go to nets and to the reference.  The floor of each gradient is the error of the same
oracle.sd.transformer run through torch's own autograd on the GPU in the storage type, i.e. what stock PyTorch in fp16 /
bf16 produces; nets must stay within 2x that floor for every gradient.  The prepared layouts are mapped back: qkv / kv
split into to_q / to_k / to_v, ff.net.0.proj de-interleaved."""
import pytest
import torch

from oracle import sd as O
from tests.test_gpu_lowp import DTYPES, Report, rel, tname

pytestmark = pytest.mark.gpu

SHAPES = [(320, 5, 32, 2), (640, 10, 16, 2), (1280, 20, 4, 4)]   # (C, heads, H = W, batch)
P = "mid_block.attentions.0"


def _setup(C, heads, S, B, dt, seed):
    from dreammat_b200 import nets, weights
    g = torch.Generator().manual_seed(seed)
    w = {}
    O._rand_transformer(g, w, P, C, 1024)
    w = {k: v.to(dt) for k, v in w.items()}
    net = nets._UNetCommon(w, weights.UNetConfig(), "cuda", dt)
    net._prep_transformer(P)
    gc = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn(B, S, S, C, device="cuda", generator=gc).to(dt)
    ctx = torch.randn(B, 77, 1024, device="cuda", generator=gc).to(dt)
    dout = torch.randn(B, S, S, C, device="cuda", generator=gc).to(dt)
    return w, net, x, ctx, dout


def _autograd(w, x, ctx, dout, heads, dtype):
    wd = {k: v.to("cuda", dtype).requires_grad_() for k, v in w.items()}
    xd = x.to(dtype).permute(0, 3, 1, 2).contiguous().requires_grad_()
    y = O.transformer(wd, P, xd, ctx.to(dtype), heads, 32, O.Ident)
    y.backward(dout.to(dtype).permute(0, 3, 1, 2))
    out = {k: v.grad for k, v in wd.items()}
    out["x"] = xd.grad.permute(0, 2, 3, 1)
    return out


def _to_oracle_names(grads, dx, C):
    b = P + ".transformer_blocks.0"
    out = {"x": dx}
    for k, v in grads.items():
        if k == b + ".attn1.qkv.w":
            for i, nm in enumerate(("to_q", "to_k", "to_v")):
                out[f"{b}.attn1.{nm}.weight"] = v[i * C:(i + 1) * C]
        elif k == b + ".attn2.kv.w":
            out[b + ".attn2.to_k.weight"], out[b + ".attn2.to_v.weight"] = v[:C], v[C:]
        elif k.startswith(b + ".ff.net.0.proj"):
            D2 = v.shape[0] // 2                       # interleaved blocks of 32 value rows, then 32 gate rows
            blk = v.reshape(D2 // 32, 2, 32, *v.shape[1:])
            out[k.replace(".w", ".weight")] = torch.cat([blk[:, 0].reshape(D2, *v.shape[1:]), blk[:, 1].reshape(D2, *v.shape[1:])], 0)
        else:
            out[k[:-2] + ".weight" if k.endswith(".w") else k] = v
    return out


@DTYPES
def test_transformer_bwd_matches_fp64_autograd(dt):
    rep = Report(f"Transformer2DModel backward {tname(dt)} (bound 2x torch-autograd-in-{tname(dt)} floor)")
    for C, heads, S, B in SHAPES:
        w, net, x, ctx, dout = _setup(C, heads, S, B, dt, seed=C)
        tape = {}
        y = net.transformer(P, x, ctx, heads, tape=tape)
        dx, grads = net.transformer_bwd(tape, dout)
        got = _to_oracle_names(grads, dx, C)
        ref = _autograd(w, x, ctx, dout, heads, torch.float64)
        flo = _autograd(w, x, ctx, dout, heads, dt)
        assert set(got) == set(ref), set(ref) ^ set(got)
        for k in sorted(ref):
            rep.rows.append((f"C{C} {k}", rel(got[k], ref[k]), rel(flo[k], ref[k]), 2.0))
        assert y.shape == x.shape
    rep.check()


@DTYPES
def test_transformer_tape_keeps_output_deterministic_and_graph_replay(dt):
    C, heads, S, B = SHAPES[1]
    w, net, x, ctx, dout = _setup(C, heads, S, B, dt, seed=7)
    plain = net.transformer(P, x, ctx, heads)

    def run():
        tape = {}
        y = net.transformer(P, x, ctx, heads, tape=tape)
        dx, grads = net.transformer_bwd(tape, dout)
        return [y, dx] + [grads[k] for k in sorted(grads)]

    one, two = run(), run()
    assert torch.equal(one[0], plain)
    for a, b in zip(one, two):
        assert torch.equal(a, b)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(one, captured):
        assert torch.equal(a, b)
