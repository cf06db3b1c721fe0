"""The ControlNet optimizer's kernels on flat buffers: dm_grad_sumsq against a float64 sum, dm_adamw_prepare + dm_adamw_step
against torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW on fp32 tensors fed the same gradients, the dropped step on a
non-finite gradient, and lr read from device memory by a captured graph.

Bounds (relative L2 against torch's fp32 result after 10 steps): master weights 1e-6, m and v 2e-6, grad_norm 1e-6.
Measured on an H100 80GB HBM3: master 2.9e-8, m 8.9e-8, v 1.1e-7 (the values are printed).  The 16-bit copy must equal
master.to(dtype) bit for bit."""
import pytest
import torch

from tests.test_gpu_lowp import DTYPES, rel, tname

pytestmark = pytest.mark.gpu

BETAS, EPS = (0.9, 0.999), 1e-8


def _ints(state):
    return state.view(torch.int32)


def test_grad_sumsq_matches_float64_and_repeats():
    from dreammat_b200 import dense_ops as D
    g = torch.Generator(device="cuda").manual_seed(1)
    for n in (1, 3, 7, 1023, 1025, 256 * 4 * 1056 + 5, 3_000_001, 40_000_003):
        x = torch.randn(n, device="cuda", generator=g) * 3.0
        got, again = D.grad_sumsq(x), D.grad_sumsq(x)
        ref = (x.double() ** 2).sum()
        err = abs(float(got) - float(ref)) / float(ref)
        print(f"\ngrad_sumsq n={n}: rel err {err:.2e} (bound 1e-6)")
        assert err <= 1e-6 and torch.equal(got, again)


class _Ours:
    def __init__(self, p0, dt, lr, wd, max_norm, gscale):
        from dreammat_b200 import dense_ops as D
        self.D, self.wd, self.max_norm, self.gscale = D, wd, max_norm, gscale
        self.master, self.m, self.v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
        self.w16 = p0.to(dt)
        self.state = D.adamw_state(lr, "cuda")
        self.sumsq = torch.zeros((), device="cuda")

    def step(self, g):
        """g is the scaled gradient, as the backward leaves it in the arena"""
        D = self.D
        D.grad_sumsq(g, out=self.sumsq)
        D.adamw_prepare(self.sumsq, self.state, BETAS, self.max_norm, 1.0 / self.gscale)
        D.adamw_step(self.master, self.m, self.v, g, self.w16, self.state, BETAS, EPS, self.wd)


class _Torch:
    def __init__(self, p0, lr, wd, max_norm):
        self.p = p0.clone().requires_grad_()
        self.opt = torch.optim.AdamW([self.p], lr=lr, betas=BETAS, eps=EPS, weight_decay=wd)
        self.max_norm = max_norm

    def step(self, g_unscaled):
        self.p.grad = g_unscaled.clone()
        norm = torch.nn.utils.clip_grad_norm_([self.p], float("inf") if self.max_norm is None else self.max_norm)
        self.opt.step()
        return norm

    @property
    def moments(self):
        st = self.opt.state[self.p]
        return st["exp_avg"], st["exp_avg_sq"]


@DTYPES
@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("max_norm", [1.0, 1e4, None], ids=["clipped", "unclipped", "noclip"])
def test_ten_steps_match_torch_adamw(dt, wd, max_norm):
    n = 1_000_003                      # not a multiple of 4 or 8
    gen = torch.Generator(device="cuda").manual_seed(5)
    p0 = torch.randn(n, device="cuda", generator=gen) * 0.05
    gscale = 1024.0 if dt == torch.float16 else 1.0
    ours, ref = _Ours(p0, dt, 1e-3, wd, max_norm, gscale), _Torch(p0, 1e-3, wd, max_norm)
    for k in range(10):
        g = torch.randn(n, device="cuda", generator=gen) * 0.01      # norm 10: max_norm 1 clips, 1e4 does not
        norm = ref.step(g)
        ours.step(g * gscale)
        assert abs(float(ours.state[4]) - float(norm)) <= 1e-6 * float(norm), (k, float(ours.state[4]), float(norm))
        assert torch.equal(ours.w16, ours.master.to(dt))
    m_ref, v_ref = ref.moments
    errs = dict(master=rel(ours.master, ref.p), m=rel(ours.m, m_ref), v=rel(ours.v, v_ref))
    print(f"\nadamw 10 steps {tname(dt)} wd {wd} max_norm {max_norm}: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    assert errs["master"] <= 1e-6 and errs["m"] <= 2e-6 and errs["v"] <= 2e-6, errs
    assert int(_ints(ours.state)[1]) == 10 and int(_ints(ours.state)[2]) == 0
    assert rel(ours.master, p0) > 1e-3         # the weights did move


@DTYPES
def test_zero_elements_stay_exactly_zero_under_weight_decay(dt):
    n = 4099
    gen = torch.Generator(device="cuda").manual_seed(6)
    p0 = torch.randn(n, device="cuda", generator=gen)
    pad = torch.arange(n, device="cuda") % 3 == 0            # the channel padding of a prepared weight: zero, zero gradient
    p0[pad] = 0
    ours = _Ours(p0, dt, 1e-2, 1e-2, 1.0, 1.0)
    for _ in range(5):
        g = torch.randn(n, device="cuda", generator=gen)
        g[pad] = 0
        ours.step(g)
    for t in (ours.master, ours.m, ours.v, ours.w16):
        assert not t[pad].any()
        assert (t[pad].view(torch.int32 if t.dtype == torch.float32 else torch.int16) == 0).all()      # +0, not -0
    assert ours.master[~pad].ne(p0[~pad]).all()


@DTYPES
def test_non_finite_gradient_drops_the_step(dt):
    n = 10_001
    gen = torch.Generator(device="cuda").manual_seed(7)
    p0 = torch.randn(n, device="cuda", generator=gen)
    for bad in (float("inf"), float("nan")):
        ours, ref = _Ours(p0, dt, 1e-3, 1e-2, 1.0, 1.0), _Torch(p0, 1e-3, 1e-2, 1.0)
        g = torch.randn(n, device="cuda", generator=gen)
        g_bad = g.clone()
        g_bad[n - 2] = bad
        before = [t.clone() for t in (ours.master, ours.m, ours.v, ours.w16)]
        ours.step(g_bad)
        for a, b in zip(before, (ours.master, ours.m, ours.v, ours.w16)):
            assert torch.equal(a, b)
        assert _ints(ours.state)[1:4].tolist() == [0, 1, 1]             # step, skipped_steps, skip
        ours.step(g)
        ref.step(g)
        assert _ints(ours.state)[1:4].tolist() == [1, 1, 0]
        assert rel(ours.master, ref.p) <= 1e-6 and rel(ours.m, ref.moments[0]) <= 2e-6 and rel(ours.v, ref.moments[1]) <= 2e-6


def test_lr_in_device_memory_reaches_a_captured_graph():
    n = 5003
    gen = torch.Generator(device="cuda").manual_seed(8)
    p0 = torch.randn(n, device="cuda", generator=gen)
    g = torch.randn(n, device="cuda", generator=gen)
    ours, ref = _Ours(p0, torch.bfloat16, 1e-3, 0.0, None, 1.0), _Torch(p0, 1e-3, 0.0, None)
    ours.step(g)                       # sizes the library scratch before the capture
    ref.step(g)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ours.step(g)
    moved = []
    for lr in (1e-3, 5e-2):
        ours.state[:1].fill_(lr)
        ref.opt.param_groups[0]["lr"] = lr
        prev = ours.master.clone()
        graph.replay()
        ref.step(g)
        moved.append(float((ours.master - prev).abs().mean()))
        assert rel(ours.master, ref.p) <= 1e-6
    assert int(_ints(ours.state)[1]) == 3 and moved[1] > 10 * moved[0]
