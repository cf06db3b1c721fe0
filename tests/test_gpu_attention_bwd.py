"""The attention backward (dm_attention_bwd) and the lse forward (dm_attention_lse) against float64 references.

Inputs are drawn, rounded to the storage type, and the same rounded values go to the kernels and to the float64 reference,
as in test_gpu_lowp.py; errors are relative L2.  lse is checked against float64 logsumexp within fp32 accumulation
(ACC32), and O against dm_attention bit for bit.

The gradients are checked against float64 math of the backward the kernel defines.  Like every FlashAttention-style
backward (torch's included), it takes delta = rowsum(dO o O) from the 16-bit O the forward stored.  Where P is nearly
one-hot, the part of O that dS depends on is smaller than O's rounding, so the float64 reference takes delta from that same
O (which is what autograd computes in a 16-bit model); where it does not matter the two agree to O's rounding floor.

Bound: the kernel rounds P and dS to 16 bits before their products and rounds each output once.  Each of those roundings
gets its own measured floor, as test_gpu_lowp.py measures one: the relative error that rounding alone causes in the
output, e.g. for dQ = scale dS K, rel(scale round(dS) K, scale dS K).  A measured floor follows cancellation: in
dQ = scale dS K the rows of dS sum to 0, and with a large common component in K (a large common logit) one rounding of dS
moves dQ by far more than dQ's own rounding does.  The kernel's roundings are these same roundings of (fp32 rather than
float64) values, so its error is at most their sum up to fp32 accumulation; the bound is BWD_MULT = 1.5 times that sum:
  dV: out + P;   dK, dQ: out + P + dS + fp32.
The fp32 term is what computing dP - delta in fp32 (rather than float64) changes, measured the same way: where P is
nearly one-hot, dP - delta of the dominant key is a cancellation of two fp32 sums far below their size.
On the shape list (random logits, P far from one-hot) the gradients are also compared with float64 autograd of SDPA itself,
with exact delta, so that a mistake shared by the kernel and the hand-written reference cannot pass: the kernel makes four
16-bit roundings on the dQ / dK path (P, dS, O inside delta, the output), each about one output floor; AUTOGRAD_MULT = 8 is
twice that count.
Where the exact dQ / dK is 0 (one key: dP = delta exactly), the kernel's dP - delta is the difference of two fp32 sums of
the same 64 products taken in different orders; those cases check an absolute bound.
"""
import pytest
import torch

from tests.test_gpu_lowp import ACC32, DTYPES, Report, _attn_pack, _attn_ref, gen, randn, rel, tname  # noqa: F401

pytestmark = pytest.mark.gpu

BWD_MULT = 1.5
AUTOGRAD_MULT = 8.0
SENTINEL = 7.0

CASES = [  # (layout, B, heads, Nq, Nk): the shape list of test_attention_layouts_and_shapes_match_fp64
    ("self", 1, 1, 1, 1), ("self", 3, 5, 63, 63), ("self", 1, 20, 64, 64), ("self", 3, 5, 65, 65),
    ("self", 3, 1, 129, 129), ("self", 1, 20, 300, 300), ("self", 3, 5, 1024, 1024), ("self", 1, 5, 4096, 4096),
    ("cross", 3, 1, 1, 77), ("cross", 1, 1, 127, 77), ("cross", 3, 5, 128, 77), ("cross", 1, 5, 129, 77),
    ("cross", 3, 20, 300, 77), ("cross", 1, 20, 1024, 77), ("cross", 3, 5, 4096, 77),
    ("contig", 3, 5, 300, 129), ("contig", 1, 20, 1, 1024), ("contig", 3, 1, 129, 65), ("contig", 1, 5, 127, 4096),
    ("contig", 3, 20, 128, 64), ("contig", 1, 1, 300, 63), ("contig", 3, 5, 4096, 1), ("contig", 1, 5, 64, 1),
]


def _grad_bufs(layout, B, Nq, Nk, Cc, dt):
    """dq / dk / dv as the model holds them: column slices of one [B, N, 3C] (self) or [B, Nk, 2C] (cross) buffer, each
    with 64 extra sentinel columns that must stay untouched; contiguous tensors otherwise.  Returns (dq, dk, dv, bands)."""
    if layout == "self":
        buf = torch.full((B, Nq, 3 * Cc + 64), SENTINEL, device="cuda", dtype=dt)
        return buf[..., :Cc], buf[..., Cc:2 * Cc], buf[..., 2 * Cc:3 * Cc], [buf[..., 3 * Cc:]]
    if layout == "cross":
        buf = torch.full((B, Nk, 2 * Cc + 64), SENTINEL, device="cuda", dtype=dt)
        return None, buf[..., :Cc], buf[..., Cc:2 * Cc], [buf[..., 2 * Cc:]]
    return None, None, None, []


def _bwd_ref(q, k, v, o16, do, heads, dt):
    """float64 gradients of the backward with delta from the stored 16-bit O, and the measured floor of each rounding:
    returns {name: (ref, floor_out + floor_P [+ floor_dS + floor_fp32])} in the [B, N, heads*64] layout"""
    B, Nq, Nk = q.shape[0], q.shape[1], k.shape[1]
    sp = lambda t, n: t.double().reshape(B, n, heads, 64).transpose(1, 2)  # noqa: E731
    mg = lambda t: t.transpose(1, 2).reshape(B, t.shape[2], heads * 64)  # noqa: E731
    Q, K, V, O, dO = sp(q, Nq), sp(k, Nk), sp(v, Nk), sp(o16, Nq), sp(do, Nq)
    P = torch.softmax((Q @ K.transpose(-1, -2)) / 8.0, -1)
    dP = dO @ V.transpose(-1, -2)
    delta = (dO * O).sum(-1, keepdim=True)
    dS = P * (dP - delta)
    Pr = P.to(dt).double() - P                     # what rounding P to 16 bits changes
    dSr = Pr * (dP - delta)                        # ... in dS (which is computed from the rounded P)
    dSr2 = dS.to(dt).double() - dS                 # rounding dS itself
    f = lambda t: t.float()  # noqa: E731
    assert not torch.backends.cuda.matmul.allow_tf32
    dSf = P * ((f(dO) @ f(V).transpose(-1, -2) - (f(dO) * f(O)).sum(-1, keepdim=True)).double() - (dP - delta))
    out = {}
    for name, ref, via in (("dQ", mg((dS @ K) / 8.0), [mg((e @ K) / 8.0) for e in (dSr, dSr2, dSf)]),
                           ("dK", mg((dS.transpose(-1, -2) @ Q) / 8.0), [mg((e.transpose(-1, -2) @ Q) / 8.0) for e in (dSr, dSr2, dSf)]),
                           ("dV", mg(P.transpose(-1, -2) @ dO), [mg(Pr.transpose(-1, -2) @ dO)])):
        nr = float(ref.norm()) + 1e-30
        out[name] = (ref, rel(ref.to(dt), ref) + sum(float(e.norm()) / nr for e in via))
    return out


def _sdpa_autograd(q, k, v, do, heads):
    qd, kd, vd = (t.detach().double().requires_grad_() for t in (q, k, v))
    _attn_ref(qd, kd, vd, heads).backward(do.double())
    return qd.grad, kd.grad, vd.grad


def _lse_ref(q, k, heads):
    B, Nq, Nk = q.shape[0], q.shape[1], k.shape[1]
    sq = q.double().reshape(B, Nq, heads, 64).transpose(1, 2)
    sk = k.double().reshape(B, Nk, heads, 64).transpose(1, 2)
    return torch.logsumexp((sq @ sk.transpose(-1, -2)) / 8.0, -1)


def _check_case(rep, name, q, k, v, heads, layout, dt, g, autograd_bound=None):
    from dreammat_b200 import dense_ops as D
    B, Nq, Cc = q.shape
    Nk = k.shape[1]
    o, lse = D.attention_lse(q, k, v, heads)
    rep.exact(f"{name} O == attention()", o, D.attention(q, k, v, heads))
    rep.rows.append((f"{name} lse", rel(lse, _lse_ref(q, k, heads)), None, ACC32))
    do = randn(g, B, Nq, Cc).to(dt)
    dq, dk, dv, bands = _grad_bufs(layout, B, Nq, Nk, Cc, dt)
    dq, dk, dv = D.attention_bwd(q, k, v, o, do, lse, heads, dq=dq, dk=dk, dv=dv)
    ref = _bwd_ref(q, k, v, o, do, heads, dt)
    for nm, got in (("dQ", dq), ("dK", dk), ("dV", dv)):
        r, fl = ref[nm]
        if Nk == 1 and nm != "dV":      # exact 0; the kernel leaves fp32 residue of dP - delta (module docstring)
            amax = float(got.float().abs().max())
            rep.rows.append((f"{name} {nm} max |value| (exact 0, absolute bound)", amax, None, 1e-3))
        else:
            rep.rows.append((f"{name} {nm}", rel(got, r), fl, BWD_MULT))
    if autograd_bound:      # independent check: float64 autograd of SDPA, exact delta (see test docstring)
        for nm, got, r in zip(("dQ", "dK", "dV"), (dq, dk, dv), _sdpa_autograd(q, k, v, do, heads)):
            if not (Nk == 1 and nm != "dV"):
                rep.cmp(f"{name} {nm} vs SDPA autograd", got, r, dt, autograd_bound)
    for band in bands:
        rep.exact(f"{name} other columns untouched", band, torch.full_like(band, SENTINEL))


@DTYPES
def test_attention_bwd_layouts_and_shapes_match_fp64(dt, gen):
    """lse within fp32 accumulation of float64 logsumexp, O bit-identical to attention(), and dQ / dK / dV against
    float64 autograd of SDPA over the model's layouts, ragged query tiles and key blocks, 1 / 5 / 20 heads."""
    rep = Report(f"attention backward {tname(dt)} (bound {BWD_MULT}x summed rounding floors)")
    for (layout, B, heads, Nq, Nk) in CASES:
        Cc = heads * 64
        q, k, v = _attn_pack(randn(gen, B, Nq, Cc), randn(gen, B, Nk, Cc), randn(gen, B, Nk, Cc), layout, dt)
        _check_case(rep, f"{layout} B{B} h{heads} {Nq}x{Nk}", q, k, v, heads, layout, dt, gen, AUTOGRAD_MULT)
    rep.check()


@DTYPES
def test_attention_bwd_stress_matches_fp64(dt, gen):
    """A large common logit (40) with no spread, a maximum only in the ragged last key block, and a maximum rising by
    tens of units from block to block.  Head h's logit offset rides on column 64h of q (1) and k (8 x offset)."""
    rep = Report(f"attention backward stress {tname(dt)} (bound {BWD_MULT}x summed rounding floors)")
    B, heads, Nq = 3, 5, 300
    Cc = heads * 64
    for pattern, Nk, layout in (("last", 129, "contig"), ("last", 77, "cross"), ("last", 65, "contig"),
                                ("rising", 1024, "contig")):
        q, k, v = randn(gen, B, Nq, Cc, scale=0.5), randn(gen, B, Nk, Cc, scale=0.5), randn(gen, B, Nk, Cc)
        blk = torch.arange(Nk, device="cuda") // 64
        off = (15.0 * (blk == blk[-1]) if pattern == "last" else 20.0 * blk) + randn(gen, B, Nk)
        for h in range(heads):
            q[..., 64 * h] = 1.0
            k[..., 64 * h] = 8.0 * off
        qq, kk, vv = _attn_pack(q, k, v, layout, dt)
        _check_case(rep, f"{pattern} Nk={Nk} {layout}", qq, kk, vv, heads, layout, dt, gen)
    for Nk in (77, 1024):
        q, k = torch.zeros(B, Nq, Cc, device="cuda"), torch.zeros(B, Nk, Cc, device="cuda")
        q[..., ::64], k[..., ::64] = 1.0, 320.0
        qq, kk, vv = _attn_pack(q, k, randn(gen, B, Nk, Cc), "contig", dt)
        _check_case(rep, f"constant logit 40 Nk={Nk}", qq, kk, vv, heads, "contig", dt, gen)
    rep.check()


@DTYPES
def test_attention_bwd_deterministic_and_graph_replay(dt, gen):
    """Two eager runs give the same bits, and so does the same sequence captured in a CUDA graph (after one warm call)."""
    from dreammat_b200 import dense_ops as D
    B, heads, N, Cc = 2, 5, 1024, 320
    q, k, v = _attn_pack(randn(gen, B, N, Cc), randn(gen, B, N, Cc), randn(gen, B, N, Cc), "self", dt)
    do = randn(gen, B, N, Cc).to(dt)

    def run():
        o, lse = D.attention_lse(q, k, v, heads)
        return (o, lse, *D.attention_bwd(q, k, v, o, do, lse, heads))

    one, two = run(), run()
    for a, b in zip(one, two):
        assert torch.equal(a, b)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = run()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(one, captured):
        assert torch.equal(a, b)
