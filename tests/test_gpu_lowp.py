"""The 16-bit dense path (fp16 and bf16 storage, fp32 accumulation) against plain fp64 references of the same operation.

Every op-level test runs for both storage types.  Inputs are drawn, rounded to the storage type, and the same rounded
values go to the kernel and to the fp64 reference (torch on the GPU in float64).  The bound of an op that rounds its
output once is set by the rounding floor of the output type, measured in the test: floor = rel(ref.to(dt), ref), and the
kernel must satisfy err <= 1.5 * floor.  Round-to-nearest sits at about 1x the floor and a truncating store at about 2x,
so the bound tells the two apart; fp32 accumulation error (~1e-6) is far below either 16-bit floor.  Ops that round more
than once (attention rounds P before PV) get a documented multiple of the floor.  Pure copies must be bit-exact.  Every
case prints its error next to its floor.

The network tests compare bf16 storage against the bf16-emulating oracle (weights and activations rounded where the
reference rounds them) within 2x the oracle's own floor, bf16 emulation against pure fp32, measured in the test.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import sd as O

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
SINGLE = 1.5        # ops that round their output once
ATTN = 3.0          # attention: P rounded to the storage type before PV, then the output (two roundings per path)
ACC32 = 2e-5        # fp32 outputs (out_f32): what fp32 accumulation on the tensor cores gives, as in test_gpu_hp.py
TINY = 1e-7         # absolute slack for outputs whose floor is 0 (exactly representable results)
QB = lambda x: x.bfloat16().float()  # noqa: E731


def rel(a, b):
    a, b = a.detach().double().reshape(-1), b.detach().double().reshape(-1)
    assert a.numel() == b.numel()
    a = a.to(b.device)
    return float((a - b).norm() / (b.norm() + 1e-30))


def floor_of(ref, dt):
    """relative L2 error of rounding the exact result to the output type: the best any kernel can do"""
    return rel(ref.to(dt), ref)


def nchw(x_nhwc, c=None):
    x = x_nhwc.permute(0, 3, 1, 2)
    return x if c is None else x[:, :c]


def tname(dt):
    return {torch.float16: "fp16", torch.bfloat16: "bf16", torch.float32: "fp32"}[dt]


class Report:
    """collects (case, error, floor, multiple) rows, prints them all, then fails on every row over its bound"""

    def __init__(self, title):
        self.title, self.rows = title, []

    def cmp(self, name, got, ref, dt, mult=SINGLE, exact_result=None):
        """got is the kernel output (storage type dt, or fp32); ref the fp64 reference.  Where ref already emulates the
        op's rounding of intermediates, exact_result is the unrounded final value the floor is measured on."""
        if dt == torch.float32:
            self.rows.append((name, rel(got, ref), None, ACC32))
        else:
            self.rows.append((name, rel(got, ref), floor_of(ref if exact_result is None else exact_result, dt), mult))

    def exact(self, name, got, ref):
        self.rows.append((name, 0.0 if torch.equal(got, ref) else float("inf"), 0.0, 0.0))

    def check(self):
        print(f"\n{self.title}:")
        bad = []
        for name, e, f, m in self.rows:
            if m == 0.0:
                print(f"  {name}: {'bit-exact' if e == 0.0 else 'DIFFERS'} (must be bit-exact)")
                ok = e == 0.0
            elif f is None:
                print(f"  {name}: err {e:.2e} (fp32 output, bound {m:.0e})")
                ok = e <= m
            else:
                print(f"  {name}: err {e:.2e} floor {f:.2e} ratio {e / f if f > 0 else 0.0:.2f} (bound {m}x)")
                ok = e <= m * f + TINY
            if not ok:
                bad.append((name, e, f, m))
        assert not bad, bad


@pytest.fixture
def gen():
    return torch.Generator(device="cuda").manual_seed(1234)


def randn(g, *shape, scale=1.0, shift=0.0):
    return torch.randn(*shape, device="cuda", generator=g) * scale + shift


# ------------------------------------------------------------------------------------------------ A. GEMM / convolution


def gemm_ref(a, b, bias=None, rowvec=None, rows_per_vec=1, residual=None, alpha=1.0, out_scale=1.0, act=None):
    """out = out_scale * (act(alpha * a b^T + bias + rowvec[m // rows_per_vec]) + residual), in fp64 (tc_gemm.cu epilogue)"""
    f = alpha * (a.double() @ b.double().transpose(-1, -2))
    if bias is not None:
        f = f + bias.double()
    if rowvec is not None:
        f = f + rowvec.double().repeat_interleave(rows_per_vec, 0)[:f.shape[-2]]
    if act == "silu":
        f = F.silu(f)
    if residual is not None:
        f = f + residual.double()
    return f * out_scale


@DTYPES
def test_gemm_epilogues_match_fp64(dt, gen):
    """Each epilogue alone, all together, GEGLU, fp32 output and a channel-slice output, over both tile widths, M on
    both sides of the 128-row tile and N ragged against both tile widths."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"gemm epilogues {tname(dt)}")
    r = lambda *s, **k: randn(gen, *s, **k).to(dt)  # noqa: E731
    M, N, K = 300, 200, 192
    a, b = r(M, K), r(N, K, scale=K ** -0.5)
    bias, res, rv = r(N), r(M, N), r(math.ceil(M / 64), N)
    variants = {
        "plain": {}, "bias": dict(bias=bias), "residual": dict(residual=res), "rowvec": dict(rowvec=rv, rows_per_vec=64),
        "silu": dict(act="silu"), "alpha_scale": dict(alpha=0.37, out_scale=2.5),
        "all": dict(bias=bias, rowvec=rv, rows_per_vec=64, act="silu", residual=res, alpha=0.8, out_scale=0.5),
    }
    for bn in (64, 128):
        for vn, kw in variants.items():
            rep.cmp(f"{vn} bn{bn}", D.gemm(a, b, bn=bn, **kw), gemm_ref(a, b, **kw), dt)
        kw = variants["all"]
        rep.cmp(f"all out_f32 bn{bn}", D.gemm(a, b, bn=bn, out_f32=True, **kw), gemm_ref(a, b, **kw), torch.float32)
        # output into a channel slice of a wider buffer (skip concatenation): ldc = N + 96, neighbours untouched
        wide = torch.full((M, N + 96), 7.0, device="cuda", dtype=dt)
        D.gemm(a, b, bn=bn, out=wide[:, 32:32 + N], **kw)
        rep.cmp(f"all ldc>N bn{bn}", wide[:, 32:32 + N], gemm_ref(a, b, **kw), dt)
        rep.exact(f"ldc>N neighbours bn{bn}", torch.cat([wide[:, :32], wide[:, 32 + N:]], 1),
                  torch.full((M, 96), 7.0, device="cuda", dtype=dt))
    # shapes: M around the 128-row tile, ragged N, K up to 5120 (the long-K ones take the split-K path)
    for Mi in (1, 127, 128, 129, 300, 4096):
        for (Ni, Ki) in ((200, 192), (328, 640), (1280, 5120)):
            if Mi == 4096 and Ki == 5120:
                continue
            ai, bi = r(Mi, Ki), r(Ni, Ki, scale=Ki ** -0.5)
            kw = dict(bias=r(Ni), residual=r(Mi, Ni), act="silu", rowvec=r(math.ceil(Mi / 100), Ni), rows_per_vec=100)
            for bn in (64, 128):
                rep.cmp(f"{Mi}x{Ni}x{Ki} bn{bn}", D.gemm(ai, bi, bn=bn, **kw), gemm_ref(ai, bi, **kw), dt)
    # GEGLU epilogue (value * gelu(gate), interleaved weight rows), with alpha / out_scale
    for (Mi, Dh) in ((300, 256), (129, 640), (4096, 320)):
        ai, w, bb = r(Mi, 320), r(2 * Dh, 320, scale=320 ** -0.5), r(2 * Dh)
        pr = 0.9 * (ai.double() @ w.double().t()) + bb.double()
        ref = pr[:, :Dh] * F.gelu(pr[:, Dh:]) * 1.5
        for bn in (64, 128):
            out = D.gemm(ai, D.geglu_interleave(w), bias=D.geglu_interleave(bb), act="geglu", alpha=0.9, out_scale=1.5, bn=bn)
            rep.cmp(f"geglu {Mi}x{Dh} bn{bn}", out, ref, dt)
    rep.check()


@DTYPES
def test_gemm_batched_and_shared_b_match_fp64(dt, gen):
    """Batched GEMM on strided slices of one fused buffer (the VAE mid-block attention: q k^T, P V^T with residual), and
    the shared-B path that folds the batch into M."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"batched gemm {tname(dt)}")
    r = lambda *s, **k: randn(gen, *s, **k).to(dt)  # noqa: E731
    B, Nt, Cc = 3, 320, 128
    qkv = r(B, Nt, 3 * Cc)
    q, k, v = qkv[..., :Cc], qkv[..., Cc:2 * Cc], qkv[..., 2 * Cc:]
    rep.cmp("q k^T strided", D.gemm(q, k), gemm_ref(q, k), dt)
    Pm = torch.softmax(r(B, Nt, Nt).float(), -1).to(dt)
    vT = v.transpose(1, 2).contiguous()
    res, bias = r(B, Nt, Cc), r(Cc)
    rep.cmp("P V + bias + residual", D.gemm(Pm, vT, bias=bias, residual=res), gemm_ref(Pm, vT, bias=bias, residual=res), dt)
    # into a channel slice of a fused buffer (the backward writes dQ / dK / dV into one [B, N, 3C] tensor)
    dqkv = torch.zeros(B, Nt, 3 * Cc, device="cuda", dtype=dt)
    D.gemm(Pm, vT, out=dqkv[..., Cc:2 * Cc])
    rep.cmp("P V into slice", dqkv[..., Cc:2 * Cc], gemm_ref(Pm, vT), dt)
    rep.exact("slice neighbours", dqkv[..., :Cc].abs().sum() + dqkv[..., 2 * Cc:].abs().sum(), torch.zeros((), device="cuda", dtype=dt))
    # shared B: [B, M, K] x [N, K] folded into one [B*M, K] GEMM (bias / residual / silu)
    for (Bb, Mi, Ni, Ki) in ((3, 300, 200, 192), (6, 77, 640, 128), (2, 4096, 320, 320)):
        a, w = r(Bb, Mi, Ki), r(Ni, Ki, scale=Ki ** -0.5)
        kw = dict(bias=r(Ni), residual=r(Bb, Mi, Ni), act="silu")
        rep.cmp(f"shared B {Bb}x{Mi}x{Ni}x{Ki}", D.gemm(a, w, **kw), gemm_ref(a, w, **kw), dt)
    # shared B over row-strided slices that are still stacked at M * lda per batch: folded as well
    w = r(64, Cc, scale=Cc ** -0.5)
    rep.cmp("shared B strided q", D.gemm(q, w), gemm_ref(q, w), dt)
    rep.check()
    # batches that are not stacked at M * lda cannot be folded: refused, not computed wrongly
    with pytest.raises(RuntimeError, match="densely stacked"):
        D.gemm(r(B, Nt + 8, Cc)[:, :Nt], w)


def _plan(M, N, K, act=0):
    from dreammat_b200._cabi import lib
    kk, bb, ss = C.c_int(), C.c_int(), C.c_int()
    assert lib().dm_gemm_plan(M, N, K, act, 0, C.byref(kk), C.byref(bb), C.byref(ss)) == 0
    return bb.value, ss.value


@DTYPES
def test_splitk_on_off_match_fp64_and_repeat(dt, gen):
    """Few-tile, long-K shapes: the plan must choose split-K (> 1) so the comparison is not vacuous.  Split-K on and off
    both match fp64; two split-K calls give identical bits (the workspace slices are rewritten every call)."""
    from dreammat_b200 import dense_ops as D
    from dreammat_b200._cabi import check, lib
    D._ensure_workspace()
    rep = Report(f"split-K {tname(dt)}")
    r = lambda *s, **k: randn(gen, *s, **k).to(dt)  # noqa: E731
    cases = []
    for (Mi, Ni, Ki) in ((192, 1280, 5120), (77, 640, 2560), (300, 328, 5120)):
        a, b = r(Mi, Ki), r(Ni, Ki, scale=Ki ** -0.5)
        kw = dict(bias=r(Ni), residual=r(Mi, Ni), act="silu", rowvec=r(math.ceil(Mi / 64), Ni), rows_per_vec=64,
                  alpha=0.7, out_scale=1.3)
        wide = torch.zeros(Mi, Ni + 64, device="cuda", dtype=dt)

        def run(a=a, b=b, kw=kw, wide=wide, Ni=Ni):
            D.gemm(a, b, out=wide[:, :Ni], **kw)
            return wide[:, :Ni].clone()
        cases.append((f"gemm {Mi}x{Ni}x{Ki}", _plan(Mi, Ni, Ki, 1)[1], run, gemm_ref(a, b, **kw)))
    for (n, hw, ci, co) in ((3, 8, 1280, 1280), (1, 8, 2560, 1280), (3, 16, 1280, 640)):
        x, w = r(n, hw, hw, ci), r(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
        tp, res = r(n, co), r(n, hw, hw, co)
        wg = D.conv_weight_to_gemm(w, dtype=dt)

        def run(x=x, wg=wg, tp=tp, res=res):
            return D.conv2d(x, wg, 3, rowvec=tp, residual=res)
        ref = nchw_to_nhwc(F.conv2d(nchw(x.double()), w.double(), padding=1) + tp.double()[:, :, None, None]) + res.double()
        cases.append((f"conv {n}x{hw}x{hw} {ci}->{co}", _plan(n * hw * hw, co, 9 * ci)[1], run, ref))
    try:
        for name, split, run, ref in cases:
            assert split > 1, (name, split)
            on1, on2 = run(), run()
            rep.exact(f"{name} split-K twice (split {split})", on1, on2)
            rep.cmp(f"{name} split-K on", on1, ref, dt)
        check(lib().dm_tune_gemm(20), "dm_tune_gemm")
        for name, _, run, ref in cases:
            rep.cmp(f"{name} split-K off", run(), ref, dt)
        assert _plan(192, 1280, 5120)[1] == 1
    finally:
        check(lib().dm_tune_gemm(21), "dm_tune_gemm")
    rep.check()


def nchw_to_nhwc(x):
    return x.permute(0, 2, 3, 1)


@DTYPES
def test_conv_shapes_and_epilogues_match_fp64(dt, gen):
    """Implicit-GEMM convolution: 3x3 stride 1, 3x3 stride 2 with the VAE's (0,1,0,1) padding and the UNet's (1,1), 1x1;
    output widths whose 128-row tile spans several rows or several images (some ragged past the last image); the
    channel counts of the SD layers; bias / per-image rowvec / residual / SiLU / out_scale; a channel-slice output."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"conv {tname(dt)}")
    r = lambda *s, **k: randn(gen, *s, **k).to(dt)  # noqa: E731
    # (n_img, H, Cin, Cout, k, stride, pad, epilogue)
    cases = [
        (1, 8, 2560, 1280, 3, 1, (1, 1), "rowvec"), (3, 8, 1280, 1280, 3, 1, (1, 1), "all"),
        (6, 8, 640, 320, 3, 1, (1, 1), "bias"), (3, 8, 64, 4, 3, 1, (1, 1), "slice"),
        (1, 16, 320, 640, 3, 1, (1, 1), "all"), (3, 16, 1280, 1280, 1, 1, (0, 0), "residual"),
        (6, 16, 64, 200, 3, 1, (1, 1), "silu"), (3, 32, 640, 640, 3, 1, (1, 1), "slice"),
        (1, 64, 320, 320, 3, 1, (1, 1), "all"), (3, 64, 64, 128, 3, 1, (1, 1), "plain"),
        (6, 64, 64, 64, 1, 1, (0, 0), "all"),
        (3, 16, 320, 320, 3, 2, (0, 0), "bias"), (1, 128, 128, 128, 3, 2, (0, 0), "plain"),
        (6, 16, 640, 640, 3, 2, (1, 1), "all"), (3, 32, 64, 320, 3, 2, (1, 1), "slice"),
    ]
    for (n, H, ci, co, ks, st, pad, ep) in cases:
        x, w = r(n, H, H, ci), r(co, ci, ks, ks, scale=(ks * ks * ci) ** -0.5)
        wg = D.conv_weight_to_gemm(w, dtype=dt)
        xd = nchw(x.double())
        if st == 2 and pad == (0, 0):        # VAE downsampler: F.pad (0, 1, 0, 1) then a valid stride-2 conv
            ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), w.double(), stride=2)
            out_hw = (H // 2, H // 2)
        else:
            ref = F.conv2d(xd, w.double(), stride=st, padding=pad[0])
            out_hw = None
        Ho, Wo = ref.shape[-2:]
        kw, post = {}, {}
        if ep in ("bias", "all"):
            kw["bias"] = r(co)
            ref = ref + kw["bias"].double()[None, :, None, None]
        if ep in ("rowvec", "all"):
            kw["rowvec"] = r(n, co)
            ref = ref + kw["rowvec"].double()[:, :, None, None]
        if ep in ("silu", "all"):
            kw["act"] = "silu"
            ref = F.silu(ref)
        ref = nchw_to_nhwc(ref)
        if ep in ("residual", "all"):
            kw["residual"] = r(n, Ho, Wo, co)
            ref = ref + kw["residual"].double()
        if ep == "all":
            kw["out_scale"] = 0.75
            ref = ref * 0.75
        name = f"{n}x{H}x{H}x{ci}->{co} k{ks}s{st}p{pad[0]} Wo{Wo} {ep}"
        if ep == "slice":
            wide = torch.full((n, Ho, Wo, co + 64), 3.0, device="cuda", dtype=dt)
            D.conv2d(x, wg, ks, stride=st, pad=pad, out_hw=out_hw, out=wide[..., 16:16 + co])
            rep.cmp(name, wide[..., 16:16 + co], ref, dt)
            rep.exact(name + " neighbours", torch.cat([wide[..., :16], wide[..., 16 + co:]], -1),
                      torch.full((n, Ho, Wo, 64), 3.0, device="cuda", dtype=dt))
        else:
            for bn in ((64, 128) if co > 64 else (0,)):
                rep.cmp(f"{name} bn{bn}", D.conv2d(x, wg, ks, stride=st, pad=pad, out_hw=out_hw, bn=bn, **kw), ref, dt)
    rep.check()


@DTYPES
def test_rejected_shapes_fail_loudly(dt, gen):
    """Shapes the tensor-core kernels do not handle are refused with an error, never computed wrongly."""
    from dreammat_b200 import dense_ops as D
    r = lambda *s: randn(gen, *s).to(dt)  # noqa: E731
    with pytest.raises(RuntimeError, match="multiple of 64"):
        D.gemm(r(300, 100), r(200, 100))                          # K % 64
    with pytest.raises(RuntimeError, match="multiple of 64"):
        D.conv2d(r(1, 8, 8, 96), r(64, 9 * 96), 3)                # Cin % 64
    with pytest.raises(RuntimeError, match="GEGLU"):
        D.gemm(r(300, 64), r(96, 64), act="geglu")               # GEGLU needs whole 64-row value/gate blocks
    for Wo in (24, 40, 96):                                       # output widths that do not tile into 128-pixel boxes
        with pytest.raises(RuntimeError, match="128-pixel"):
            D.conv2d(r(1, Wo, Wo, 64), r(64, 9 * 64), 3)


# ------------------------------------------------------------------------------------------------ B. fused attention


def _attn_pack(q, k, v, layout, dt):
    """fp32 q [B,Nq,C], k/v [B,Nk,C] -> rounded views in the model's layouts: 'self' = column slices of one [B, N, 3C]
    buffer, 'cross' = q alone and k/v slices of one [B, Nk, 2C] buffer, 'contig' = three tensors"""
    Cc = q.shape[-1]
    if layout == "self":
        qkv = torch.cat([q, k, v], -1).to(dt)
        return qkv[..., :Cc], qkv[..., Cc:2 * Cc], qkv[..., 2 * Cc:]
    if layout == "cross":
        kv = torch.cat([k, v], -1).to(dt)
        return q.to(dt), kv[..., :Cc], kv[..., Cc:]
    return q.to(dt), k.to(dt), v.to(dt)


def _attn_ref(q, k, v, heads):
    B, Nq, Nk = q.shape[0], q.shape[1], k.shape[1]
    sp = lambda t, n: t.double().reshape(B, n, heads, 64).transpose(1, 2)  # noqa: E731
    return F.scaled_dot_product_attention(sp(q, Nq), sp(k, Nk), sp(v, Nk)).transpose(1, 2).reshape(B, Nq, heads * 64)


@DTYPES
def test_attention_layouts_and_shapes_match_fp64(dt, gen):
    """The model's own layouts (q/k/v as column slices of the fused projection buffers) and the contiguous one, over
    ragged key blocks (Nk around 64, 77 text tokens), ragged query tiles, 1 / 5 / 20 heads and batch 1 / 3."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"attention {tname(dt)} (bound {ATTN}x floor)")
    cases = [  # (layout, B, heads, Nq, Nk)
        ("self", 1, 1, 1, 1), ("self", 3, 5, 63, 63), ("self", 1, 20, 64, 64), ("self", 3, 5, 65, 65),
        ("self", 3, 1, 129, 129), ("self", 1, 20, 300, 300), ("self", 3, 5, 1024, 1024), ("self", 1, 5, 4096, 4096),
        ("cross", 3, 1, 1, 77), ("cross", 1, 1, 127, 77), ("cross", 3, 5, 128, 77), ("cross", 1, 5, 129, 77),
        ("cross", 3, 20, 300, 77), ("cross", 1, 20, 1024, 77), ("cross", 3, 5, 4096, 77),
        ("contig", 3, 5, 300, 129), ("contig", 1, 20, 1, 1024), ("contig", 3, 1, 129, 65), ("contig", 1, 5, 127, 4096),
        ("contig", 3, 20, 128, 64), ("contig", 1, 1, 300, 63), ("contig", 3, 5, 4096, 1), ("contig", 1, 5, 64, 1),
    ]
    for (layout, B, heads, Nq, Nk) in cases:
        Cc = heads * 64
        q, k, v = _attn_pack(randn(gen, B, Nq, Cc), randn(gen, B, Nk, Cc), randn(gen, B, Nk, Cc), layout, dt)
        rep.cmp(f"{layout} B{B} h{heads} {Nq}x{Nk}", D.attention(q, k, v, heads), _attn_ref(q, k, v, heads), dt, ATTN)
    rep.check()


@DTYPES
def test_attention_online_softmax_stress_matches_fp64(dt, gen):
    """Logits shaped to exercise the running-max rescale: a maximum that rises by tens of units from one 64-key block
    to the next, a maximum in the first block only, a maximum only in the ragged last block, and near-constant rows
    (also with a large common logit).  Head h's logit offset is carried by column 64h of q (set to 1) and k (8 x offset,
    the kernel scale being 1/8)."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"attention online-softmax stress {tname(dt)} (bound {ATTN}x floor)")
    B, heads, Nq = 3, 5, 300
    Cc = heads * 64

    def offsets(Nk, pattern):
        blk = torch.arange(Nk, device="cuda") // 64
        nb = int(blk[-1]) + 1
        jit = randn(gen, B, Nk)
        if pattern == "rising":
            return 20.0 * blk + jit
        if pattern == "rising_slow":           # earlier blocks still carry weight: the rescale factor must be right
            return 1.5 * blk + jit
        if pattern == "first":
            return 12.0 * (blk == 0) + jit
        if pattern == "last":
            return 15.0 * (blk == nb - 1) + jit
        raise ValueError(pattern)

    for pattern, Nk, layout in (("rising", 1024, "contig"), ("rising", 129, "contig"), ("rising_slow", 1024, "contig"),
                                ("first", 1024, "contig"), ("first", 300, "self"), ("last", 129, "contig"),
                                ("last", 77, "cross"), ("last", 65, "contig")):
        q, k, v = randn(gen, B, Nq, Cc, scale=0.5), randn(gen, B, Nk, Cc, scale=0.5), randn(gen, B, Nk, Cc)
        off = offsets(Nk, pattern)
        for h in range(heads):
            q[..., 64 * h] = 1.0
            k[..., 64 * h] = 8.0 * off
        if layout == "self":
            k, v = k[:, :Nq], v[:, :Nq]
        qq, kk, vv = _attn_pack(q, k, v, layout, dt)
        rep.cmp(f"{pattern} Nk={kk.shape[1]} {layout}", D.attention(qq, kk, vv, heads), _attn_ref(qq, kk, vv, heads), dt, ATTN)
    for Nk in (77, 1024):
        # near-constant rows: tiny logits, and a large common logit (40) with no spread at all
        q, k, v = _attn_pack(randn(gen, B, Nq, Cc, scale=1e-3), randn(gen, B, Nk, Cc), randn(gen, B, Nk, Cc), "contig", dt)
        rep.cmp(f"near-constant Nk={Nk}", D.attention(q, k, v, heads), _attn_ref(q, k, v, heads), dt, ATTN)
        q, k = torch.zeros(B, Nq, Cc, device="cuda"), torch.zeros(B, Nk, Cc, device="cuda")
        q[..., ::64], k[..., ::64] = 1.0, 320.0
        q, k, v = _attn_pack(q, k, randn(gen, B, Nk, Cc), "contig", dt)
        rep.cmp(f"constant logit 40 Nk={Nk}", D.attention(q, k, v, heads), _attn_ref(q, k, v, heads), dt, ATTN)
    rep.check()


# ------------------------------------------------------------------------------------------------ C. streaming kernels


def _gn_ref(x, gm, bt, G, eps, silu):
    y = F.group_norm(nchw(x), G, gm.double(), bt.double(), eps)
    return nchw_to_nhwc(F.silu(y) if silu else y)


GN_SHAPES = [  # (n_img, H, W, C): the slab / chunk mappings the SD layers produce, 8x8 latents up to the VAE's first level
    (3, 8, 8, 2560), (6, 8, 8, 1280), (1, 8, 8, 64), (3, 16, 16, 1920), (1, 16, 16, 1280), (6, 16, 16, 64),
    (1, 32, 32, 960), (3, 32, 32, 640), (6, 32, 32, 320), (3, 64, 64, 320), (1, 64, 64, 512), (3, 64, 64, 128),
    (1, 128, 128, 256), (1, 256, 256, 256), (1, 512, 512, 128),
]


def _gn_case(rep, D, dt, g, n, H, W, Cc, silu, shift, eps=1e-6, G=32):
    """forward from a channel slice (ld > C) into a channel slice (ldy > C), backward with and without dx_add"""
    xw = randn(g, n, H, W, Cc + 64, shift=shift).to(dt)
    x = xw[..., 32:32 + Cc]
    gm, bt = randn(g, Cc, scale=0.1, shift=1.0).to(dt), randn(g, Cc, scale=0.1).to(dt)
    yw = torch.zeros(n, H, W, Cc + 16, device="cuda", dtype=dt)
    _, st = D.groupnorm(x, gm, bt, G, eps, silu=silu, out=yw[..., 8:8 + Cc])
    x64 = x.double().requires_grad_(True)
    ref = _gn_ref(x64, gm, bt, G, eps, silu)
    tag = f"{n}x{H}x{W}x{Cc} silu={int(silu)} mean/std={shift:g}"
    rep.cmp(f"fwd {tag}", yw[..., 8:8 + Cc], ref, dt)
    assert float(yw[..., :8].abs().sum()) == 0 and float(yw[..., 8 + Cc:].abs().sum()) == 0, tag
    dz, add = randn(g, n, H, W, Cc).to(dt), randn(g, n, H, W, Cc).to(dt)
    (gx,) = torch.autograd.grad(ref, x64, dz.double())
    xc = x.contiguous()
    rep.cmp(f"bwd {tag}", D.groupnorm_bwd(xc, dz, gm, bt, st, G, eps, silu=silu), gx, dt)
    rep.cmp(f"bwd+dx_add {tag}", D.groupnorm_bwd(xc, dz, gm, bt, st, G, eps, silu=silu, dx_add=add), gx + add.double(), dt)


@DTYPES
def test_groupnorm_16bit_matches_fp64(dt, gen):
    from dreammat_b200 import dense_ops as D
    rep = Report(f"groupnorm {tname(dt)}")
    for i, (n, H, W, Cc) in enumerate(GN_SHAPES):
        _gn_case(rep, D, dt, gen, n, H, W, Cc, silu=bool(i % 2), shift=0.0)
    rep.check()


@DTYPES
@pytest.mark.parametrize("mean_over_std", [0.0, 10.0, 100.0, 1000.0])
def test_groupnorm_mean_offset_matches_fp64(dt, mean_over_std, gen):
    """Groups whose mean is far from zero relative to their spread: the statistics must not lose the variance to
    cancellation (the one-pass E[x^2] - mean^2 in fp32 does, from mean/std ~ 100 on)."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"groupnorm mean/std={mean_over_std:g} {tname(dt)}")
    for (n, H, W, Cc) in ((1, 512, 512, 128), (3, 16, 16, 1920), (6, 8, 8, 64)):
        for silu in (False, True):
            _gn_case(rep, D, dt, gen, n, H, W, Cc, silu=silu, shift=mean_over_std)
    rep.check()


@DTYPES
def test_groupnorm_16bit_bit_repeatable(dt, gen):
    """Same inputs, same bits: forward output and statistics, backward output."""
    from dreammat_b200 import dense_ops as D
    for (n, H, W, Cc) in ((1, 512, 512, 128), (3, 8, 8, 2560), (6, 32, 32, 320)):
        x = randn(gen, n, H, W, Cc, shift=3.0).to(dt)
        gm, bt = randn(gen, Cc, scale=0.1, shift=1.0).to(dt), randn(gen, Cc, scale=0.1).to(dt)
        dz, add = randn(gen, n, H, W, Cc).to(dt), randn(gen, n, H, W, Cc).to(dt)
        runs = []
        for _ in range(2):
            y, st = D.groupnorm(x, gm, bt, 32, 1e-6, silu=True)
            dx = D.groupnorm_bwd(x, dz, gm, bt, st, 32, 1e-6, silu=True, dx_add=add)
            runs.append((y, st, dx))
        for a, b in zip(*runs):
            assert torch.equal(a, b), (n, H, W, Cc)


@DTYPES
def test_streaming_kernels_16bit_match_fp64(dt, gen):
    """The 16-bit instantiations of the remaining streaming kernels (the fp32 mode runs different kernels)."""
    from dreammat_b200 import dense_ops as D
    rep = Report(f"streaming kernels {tname(dt)}")
    r = lambda *s, **k: randn(gen, *s, **k).to(dt)  # noqa: E731
    for Cc in (320, 640, 1280):
        for M in (77, 300, 4097):
            h, gm, bt = r(M, Cc, shift=0.5), r(Cc, scale=0.1, shift=1.0), r(Cc, scale=0.1)
            rep.cmp(f"layernorm {M}x{Cc}", D.layernorm(h, gm, bt), F.layer_norm(h.double(), (Cc,), gm.double(), bt.double(), 1e-5), dt)
    for (M, Dh) in ((300, 320), (4096, 1280), (77, 640)):
        hh = r(M, 2 * Dh)
        rep.cmp(f"geglu {M}x{Dh}", D.geglu(hh), hh[:, :Dh].double() * F.gelu(hh[:, Dh:].double()), dt)
    for shape in ((3, 8, 8, 1280), (1, 32, 32, 320), (2, 64, 64, 64)):
        xs = r(*shape)
        ref = nchw_to_nhwc(F.interpolate(nchw(xs.double()), scale_factor=2.0, mode="nearest")).to(dt)
        rep.exact(f"upsample2x {shape}", D.upsample2x(xs), ref)
        zi = torch.zeros(shape[0], 2 * shape[1], 2 * shape[2], shape[3], device="cuda", dtype=dt)
        zi[:, ::2, ::2] = xs
        rep.exact(f"zero-insert {shape}", D.upsample2x(xs, zero_insert=True), zi)
    # axpby: strided sources, into a channel slice of a wider buffer; a = 1 without s2 is a plain copy
    src = r(300, 3 * 320)
    for (a, b) in ((1.0, 0.5), (-0.7, 1.3)):
        cat = torch.full((300, 960), 5.0, device="cuda", dtype=dt)
        D.axpby(src[:, :320], a, src[:, 640:], b, out=cat[:, 320:640])
        rep.cmp(f"axpby a={a} b={b}", cat[:, 320:640], a * src[:, :320].double() + b * src[:, 640:].double(), dt)
        rep.exact(f"axpby neighbours a={a}", torch.cat([cat[:, :320], cat[:, 640:]], 1), torch.full((300, 640), 5.0, device="cuda", dtype=dt))
    cp = torch.zeros(300, 640, device="cuda", dtype=dt)
    D.axpby(src[:, 320:640], out=cp[:, 320:])
    rep.exact("axpby copy", cp[:, 320:], src[:, 320:640])
    rep.cmp("axpby scale only", D.axpby(src[:, :320], 0.3), 0.3 * src[:, :320].double(), dt)
    # transpose: ragged extents, and a strided column slice of a fused buffer (the VAE attention's v)
    for shape in ((2, 70, 50), (3, 130, 66), (1, 4096, 128), (2, 2, 4096)):
        t3 = r(*shape)
        rep.exact(f"transpose {shape}", D.transpose(t3), t3.transpose(1, 2).contiguous())
    qkv = r(2, 320, 3 * 128)
    rep.exact("transpose strided slice", D.transpose(qkv[..., 256:]), qkv[..., 256:].transpose(1, 2).contiguous())
    for cols in (77, 333, 4096):
        sm, dP = r(64, cols, scale=3.0), r(64, cols)
        P = D.softmax_rows(sm, 0.3)
        rep.cmp(f"softmax {cols}", P, torch.softmax(sm.double() * 0.3, -1), dt)
        Pd = P.double()
        rep.cmp(f"softmax_bwd {cols}", D.softmax_bwd(P, dP, 0.3), 0.3 * Pd * (dP.double() - (Pd * dP.double()).sum(-1, keepdim=True)), dt)
    # layout / dtype conversions at the fp32 boundaries
    for (cin, cpad) in ((3, 64), (22, 64), (4, 8)):
        xf = torch.rand(2, 16, 16, cin, device="cuda", generator=gen)
        pc = D.pad_convert(xf, cpad, 2.0, -1.0, dt)
        ref = torch.zeros(2, 16, 16, cpad, device="cuda", dtype=torch.float64)
        ref[..., :cin] = xf.double() * 2 - 1
        rep.cmp(f"pad_convert {cin}->{cpad}", pc, ref, dt)
        rep.cmp(f"unpad_convert {cpad}->{cin}", D.unpad_convert(pc, cin, 0.5), pc[..., :cin].double() * 0.5, torch.float32)
        rep.exact(f"nhwc_to_nchw_f32 {cpad}->{cin}", D.nhwc_to_nchw_f32(pc, cin), nchw(pc[..., :cin]).float().contiguous())
    # posterior sample: diffusers rounds std, eps and the pre-scale sample to the weights dtype; the reference does too
    mom = r(3, 16, 16, 64, scale=2.0)
    mom[0, 0, :4, 4:8] = torch.tensor([25.0, -35.0, 15.0, -29.0], device="cuda").to(dt)   # logvar outside / inside the clamp
    eps = randn(gen, 3, 4, 16, 16)
    md = nchw(mom.double())
    mean, lv = md[:, :4], md[:, 4:8].clamp(-30, 20)
    rd = lambda t: t.to(dt).double()  # noqa: E731
    smp = rd(mean + rd(torch.exp(0.5 * lv)) * rd(eps.double()))
    rep.cmp("vae_sample", D.vae_sample(mom, eps, 0.18215), rd(smp * 0.18215), dt, exact_result=smp * 0.18215)
    dz = randn(gen, 3, 4, 16, 16)
    inside = (md[:, 4:8] >= -30) & (md[:, 4:8] <= 20)
    dref = torch.zeros(3, 64, 16, 16, device="cuda", dtype=torch.float64)
    dref[:, :4] = dz.double() * 0.18215
    dref[:, 4:8] = torch.where(inside, dz.double() * 0.18215 * eps.double() * 0.5 * torch.exp(0.5 * md[:, 4:8]), 0.0)
    rep.cmp("vae_sample_bwd", D.vae_sample_bwd(mom, eps, dz, 0.18215), nchw_to_nhwc(dref), dt)
    # add_noise with the CFG replication, timestep embedding, silu
    z, nz = randn(gen, 2, 4, 16, 16), randn(gen, 2, 4, 16, 16)
    ac = torch.tensor([0.9, 0.2], device="cuda")
    out = D.add_noise(z, nz, ac.sqrt(), (1 - ac).sqrt(), 3, 64, dt)
    mix = nchw_to_nhwc(ac.double().sqrt()[:, None, None, None] * z.double() + (1 - ac.double()).sqrt()[:, None, None, None] * nz.double())
    ref = torch.zeros(6, 16, 16, 64, device="cuda", dtype=torch.float64)
    ref[..., :4] = mix.repeat(3, 1, 1, 1)
    rep.cmp("add_noise", out, ref, dt)
    t = torch.tensor([1.0, 37.0, 250.0, 500.0, 999.0], device="cuda")
    for dim in (320, 64):
        half = dim // 2
        fr = torch.exp(-math.log(10000.0) * torch.arange(half, device="cuda", dtype=torch.float64) / half)
        ang = t.double()[:, None] * fr[None]
        rep.cmp(f"timestep_embedding {dim}", D.timestep_embedding(t, dim, dt), torch.cat([ang.cos(), ang.sin()], -1), dt)
    xs = r(3, 16, 16, 320, scale=3.0)
    rep.cmp("silu", D.silu(xs), F.silu(xs.double()), dt)
    rep.check()


# ------------------------------------------------------------------------------------------------ D. fused CSD epilogue


def test_fused_csd_epilogue_bf16_matches_unfused(gen):
    """dm_conv2d_csd with bf16 activations and weights: the noise predictions it emits equal conv_out (D.conv2d) +
    layout change up to fp32 summation order before the bf16 rounding, and grad / dlatents / the ten logged sums equal
    their closed form applied to those predictions.  The eps bound is the fp16 test's scaled by the ratio of the two
    unit roundoffs (8); the other bounds are fp32 reduction order and stay as they are."""
    from dreammat_b200 import dense_ops as D
    dt = torch.bfloat16
    rn = lambda *s_: randn(gen, *s_)  # noqa: E731
    for (B, hw, Cin) in ((2, 16, 64), (4, 8, 128), (1, 32, 320), (8, 64, 320)):
        assert D.csd_supported(dt, B, hw, hw)
        x = rn(3 * B, hw, hw, Cin).to(dt)
        w4 = (rn(4, Cin, 3, 3) / (3 * Cin ** 0.5)).to(dt)
        wg = D.conv_weight_to_gemm(w4, dtype=dt)
        bias = (rn(4) * 0.1).to(dt)
        noise, w1mac = rn(B, 4, hw, hw), torch.rand(B, device="cuda", generator=gen)
        coef = torch.tensor([1.05, -0.7, -0.2, 0.1, 0.37], device="cuda")
        grad, dlat, sums = torch.empty_like(noise), torch.empty_like(noise), torch.zeros(10, device="cuda")
        eps = torch.empty(3, B, 4, hw, hw, device="cuda")
        D.conv2d_csd(x, wg, bias, noise, w1mac, coef, grad, dlat, sums, eps)
        out = torch.empty(3 * B, hw, hw, 8, device="cuda", dtype=dt)
        D.conv2d(x, wg, 3, bias=bias, out=out[..., :4])
        eps_ref = D.nhwc_to_nchw_f32(out, 4).view(3, B, 4, hw, hw)
        conv64 = F.conv2d(nchw(x.double()), w4.double(), padding=1) + bias.double()[None, :, None, None]
        et, eu, en = eps[0], eps[1], eps[2]
        gref = torch.nan_to_num(w1mac.view(-1, 1, 1, 1) * (1.05 * et - 0.7 * eu - 0.2 * en + 0.1 * noise))
        sref = torch.stack([0.5 * (gref ** 2).sum(), (gref ** 2).sum(), ((eu - noise) ** 2).sum(), ((et - noise) ** 2).sum(),
                            ((et - eu) ** 2).sum(), ((et - en) ** 2).sum(), ((en - eu) ** 2).sum(), (noise ** 2).sum(), (eu ** 2).sum(),
                            (et ** 2).sum()])
        errs = dict(eps=rel(eps, eps_ref), grad=rel(grad, gref), dlat=rel(dlat, gref * 0.37),
                    sums=float(((sums - sref).abs() / sref.abs().clamp_min(1e-20)).max()))
        e64, f64 = rel(eps, conv64.view(3, B, 4, hw, hw)), floor_of(conv64, dt)
        print(f"\nfused CSD epilogue bf16 B={B} {hw}x{hw} Cin={Cin}: " + " ".join(f"{k}={v:.1e}" for k, v in errs.items())
              + f" eps-vs-fp64={e64:.2e} (floor {f64:.2e})")
        assert errs["eps"] < 8e-4 and errs["grad"] < 1e-6 and errs["dlat"] < 1e-6 and errs["sums"] < 1e-5, errs
        assert e64 <= SINGLE * f64, (e64, f64)


# ------------------------------------------------------------------------------------------------ E. networks in bf16


@pytest.fixture(scope="module")
def small_bf16():
    ucfg = O.UNetConfig(block_out_channels=(64, 128, 256, 256), heads=(1, 2, 4, 4), cross_attention_dim=128)
    vcfg = O.VAEConfig(block_out_channels=(64, 64, 128, 128))
    wu = O.round_weights(O.random_unet_weights(ucfg, 0), torch.bfloat16)
    wc = O.round_weights(O.random_controlnet_weights(ucfg, 1), torch.bfloat16)
    wv = O.round_weights(O.random_vae_weights(vcfg, 2), torch.bfloat16)
    return ucfg, vcfg, wu, wc, wv


def test_unet_bf16_matches_oracle(small_bf16):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import UNet
    ucfg, _, wu, _, _ = small_bf16
    g = torch.Generator().manual_seed(3)
    z, t = torch.randn(3, 4, 32, 32, generator=g), torch.tensor([37, 500, 940])
    ctx = torch.randn(3, 77, ucfg.cross_attention_dim, generator=g)
    ref16 = O.unet_forward(wu, ucfg, QB(z), t, QB(ctx), q=QB)
    ref32 = O.unet_forward(wu, ucfg, QB(z), t, QB(ctx))
    net = UNet(wu, ucfg, dtype=torch.bfloat16)
    out = net.forward(D.pad_convert(z.permute(0, 2, 3, 1).contiguous().cuda(), 64, dtype=torch.bfloat16), t.float().cuda(),
                      ctx.bfloat16().cuda())
    e, f = rel(out, ref16), rel(ref16, ref32)
    print(f"\nunet small bf16: rel err vs bf16-emulating oracle {e:.2e} (bf16 floor {f:.2e}, bound 2x)")
    assert e < 2 * f


def test_controlnet_bf16_matches_oracle(small_bf16):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import ControlNet
    ucfg, _, _, wc, _ = small_bf16
    g = torch.Generator().manual_seed(4)
    B, hw = 2, 16
    z, t = torch.randn(3 * B, 4, hw, hw, generator=g), torch.tensor([100, 700] * 3)
    ctx = torch.randn(3 * B, 77, ucfg.cross_attention_dim, generator=g)
    cond = torch.rand(B, 22, 8 * hw, 8 * hw, generator=g)
    d16, m16 = O.controlnet_forward(wc, ucfg, QB(z), t, QB(ctx), QB(cond), 0.8, q=QB)
    d32, m32 = O.controlnet_forward(wc, ucfg, QB(z), t, QB(ctx), QB(cond), 0.8)
    net = ControlNet(wc, ucfg, dtype=torch.bfloat16)
    down, mid = net.forward(D.pad_convert(z.permute(0, 2, 3, 1).contiguous().cuda(), 64, dtype=torch.bfloat16), t.float().cuda(),
                            ctx.bfloat16().cuda(), D.pad_convert(cond.permute(0, 2, 3, 1).contiguous().cuda(), 64, dtype=torch.bfloat16), 0.8)
    errs = [rel(nchw(a.float()), b) for a, b in zip(down, d16)] + [rel(nchw(mid.float()), m16)]
    floors = [rel(a, b) for a, b in zip(d16, d32)] + [rel(m16, m32)]
    print("\ncontrolnet small bf16 (err / floor):", " ".join(f"{e:.1e}/{f:.1e}" for e, f in zip(errs, floors)))
    assert len(down) == 12
    assert all(e < 2 * f for e, f in zip(errs, floors)), list(zip(errs, floors))


def test_vae_encoder_bf16_forward_backward_match_oracle(small_bf16):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import VAEEncoder
    _, vcfg, _, _, wv = small_bf16
    g = torch.Generator().manual_seed(5)
    B, R = 2, 128
    rgb, eps = torch.rand(B, R, R, 3, generator=g), torch.randn(B, 4, R // 8, R // 8, generator=g)
    dz = torch.randn(B, 4, R // 8, R // 8, generator=g)
    ref = {}
    for name, q in (("bf16", QB), ("fp32", O.Ident)):
        x = (rgb * 2 - 1).permute(0, 3, 1, 2).clone().requires_grad_(True)
        mom_r = O.vae_encode_moments(wv, vcfg, q(x), q=q)
        z_r = O.vae_sample(mom_r, eps, vcfg.scaling_factor, q)
        z_r.backward(dz)
        ref[name] = (mom_r.detach(), z_r.detach(), x.grad.clone())
    vae = VAEEncoder(wv, vcfg, dtype=torch.bfloat16)
    tape = []
    mom = vae.encode_moments(D.pad_convert(rgb.cuda(), 64, 2.0, -1.0, torch.bfloat16), tape)
    z = D.vae_sample(mom, eps.cuda(), vcfg.scaling_factor)
    dx = vae.backward_input(tape, D.vae_sample_bwd(mom, eps.cuda(), dz.cuda(), vcfg.scaling_factor))
    got = (nchw(mom.float(), 8), z, nchw(dx.float(), 3))
    names = ("moments", "latents", "input-grad")
    errs = [rel(a, b) for a, b in zip(got, ref["bf16"])]
    floors = [rel(a, b) for a, b in zip(ref["bf16"], ref["fp32"])]
    print("\nvae small bf16: " + " ".join(f"{n} {e:.2e} (floor {f:.2e})" for n, e, f in zip(names, errs, floors)))
    assert all(e < 2 * f for e, f in zip(errs, floors)), list(zip(names, errs, floors))


def test_guidance_step_bf16_matches_oracle(small_bf16):
    """The a7-a9 slice in bf16 storage (rgb -> VAE -> add_noise -> ControlNet + UNet x3 -> CSD grad -> loss -> d rgb), with
    the conv_out + CSD epilogue fused and unfused.  Each output within 2x the bf16 floor of the oracle; the loss is half the
    squared norm of the SDS gradient, so its relative error is bounded by twice the gradient's."""
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.guidance import PromptProcessorOutput, StableDiffusionLightGuidance, _SDSLoss
    ucfg, vcfg, wu, wc, wv = small_bf16
    g = torch.Generator().manual_seed(6)
    B, R = 2, 128
    Dm = ucfg.cross_attention_dim
    rgb, cond = torch.rand(B, R, R, 3, generator=g), torch.rand(B, R, R, 22, generator=g)
    vd, uvd, null = torch.randn(4, 77, Dm, generator=g), torch.randn(4, 77, Dm, generator=g), torch.randn(1, 77, Dm, generator=g)
    pu = PromptProcessorOutput(vd[:1], uvd[:1], null, vd, uvd)
    el, az, dist = torch.tensor([10.0, 70.0]), torch.tensor([20.0, -170.0]), torch.tensor([3.5, 3.5])
    t = torch.tensor([321, 777])
    noise, veps = torch.randn(B, 4, R // 8, R // 8, generator=g), torch.randn(B, 4, R // 8, R // 8, generator=g)
    ctx3 = pu.get_text_embeddings(el, az, dist, True, return_null_text_embeddings=True)
    ref = {}
    for name, q in (("bf16", QB), ("fp32", O.Ident)):
        x = rgb.clone().requires_grad_(True)
        loss_o, grad_o, z_o = O.guidance_step(wv, wc, wu, ucfg, vcfg, x, cond, QB(ctx3), t, noise, veps,
                                              scales=(1.05, -0.7, -0.2, 0.0), cond_scale=1.0, q=q)
        loss_o.backward()
        ref[name] = (z_o.detach(), grad_o.detach(), float(loss_o.detach()), x.grad.clone())
    fl = dict(latents=rel(ref["bf16"][0], ref["fp32"][0]), sds_grad=rel(ref["bf16"][1], ref["fp32"][1]),
              d_rgb=rel(ref["bf16"][3], ref["fp32"][3]))
    fl["loss"] = 2 * fl["sds_grad"]
    cfg = dict(use_controlnet=True, control_types=["light"], condition_scales=[1.0], cond_scale=1.05, uncond_scale=-0.7,
               null_scale=-0.2, noise_scale=0.0)
    guid = StableDiffusionLightGuidance(cfg, ucfg, vcfg, wu, wc, wv, dtype=torch.bfloat16)
    assert guid.weights_dtype == torch.bfloat16 and D.csd_supported(torch.bfloat16, B, R // 8, R // 8)
    bad = []
    for fuse in (True, False):
        guid.fuse_csd = fuse
        rgb_c = rgb.cuda().requires_grad_(True)
        lat = guid.encode_images(rgb_c, veps.cuda())
        grad, dlat, sums = guid.compute_grad_sds(lat, cond.cuda(), ctx3, t.cuda(), noise.cuda())
        loss = _SDSLoss.apply(lat, dlat, sums[0] / B)
        loss.backward()
        e = dict(latents=rel(lat, ref["bf16"][0]), sds_grad=rel(grad, ref["bf16"][1]),
                 loss=abs(float(loss.detach()) - ref["bf16"][2]) / abs(ref["bf16"][2]), d_rgb=rel(rgb_c.grad, ref["bf16"][3]))
        print(f"\nguidance small bf16 fuse_csd={fuse}: " + " ".join(f"{k} {v:.2e} (floor {fl[k]:.2e})" for k, v in e.items()))
        bad += [(fuse, k, v, fl[k]) for k, v in e.items() if not v < 2 * fl[k]]
    assert not bad, bad


@pytest.mark.slow
def test_unet_full_size_bf16_matches_oracle():
    """SD-2.1-base topology (random init), one view = 3 CFG samples at 64x64 latents, bf16 storage, within 2x the oracle's
    bf16 floor."""
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.nets import UNet
    ucfg = O.UNetConfig()
    wu = O.round_weights(O.random_unet_weights(ucfg, 7), torch.bfloat16)
    g = torch.Generator().manual_seed(8)
    z, t = torch.randn(3, 4, 64, 64, generator=g), torch.tensor([250, 250, 250])
    ctx = torch.randn(3, 77, 1024, generator=g)
    with torch.no_grad():
        ref16 = O.unet_forward(wu, ucfg, QB(z), t, QB(ctx), q=QB)
        ref32 = O.unet_forward(wu, ucfg, QB(z), t, QB(ctx))
    net = UNet(wu, ucfg, dtype=torch.bfloat16)
    out = net.forward(D.pad_convert(z.permute(0, 2, 3, 1).contiguous().cuda(), 64, dtype=torch.bfloat16), t.float().cuda(),
                      ctx.bfloat16().cuda())
    e, f = rel(out, ref16), rel(ref16, ref32)
    print(f"\nunet full-size bf16: rel err vs bf16-emulating oracle {e:.2e} (bf16 floor {f:.2e}, bound 2x)")
    assert e < 2 * f
