"""controlnet_train.ControlNetTrainer: the flat arenas leave the ControlNet's forward bit-identical, the backward writes its
gradients in place, one step equals clip_grad_norm_ + torch.optim.AdamW applied to that step's own gradients (the gradients
themselves are pinned by test_gpu_unet_bwd.py), the channel padding stays zero, steps repeat bit for bit eagerly and as a
replayed CUDA graph, training lowers the loss on a fixed batch without touching the UNet, and the checkpoint round trip is
exact.  fp16 runs at a loss scale of numel / 2 (as test_gpu_unet_bwd.py), bf16 at 1.

Per-step comparisons start from identical state: free-running trajectories of two optimizers separate for reasons that
have nothing to do with kernel accuracy (test_gpu_config1.py)."""
import pytest
import torch

from oracle import sd as O
from tests.test_gpu_lowp import DTYPES, rel, tname
from tests.test_gpu_unet_bwd import SMALL

pytestmark = pytest.mark.gpu


def _setup(dt, cfg=None, n=2, hw=16, seed=81, **kw):
    from dreammat_b200 import dense_ops as D
    from dreammat_b200.controlnet_train import ControlNetTrainer
    from dreammat_b200.nets import ControlNet, UNet
    cfg = cfg or O.UNetConfig(**SMALL)
    wc = {k: v.to(dt) for k, v in O.random_controlnet_weights(cfg, seed).items()}
    wu = {k: v.to(dt) for k, v in O.random_unet_weights(cfg, seed + 1).items()}
    unet, cnet = UNet(wu, cfg, dtype=dt), ControlNet(wc, cfg, dtype=dt)
    g = torch.Generator(device="cuda").manual_seed(seed + 2)
    batch = dict(latents=torch.randn(n, 4, hw, hw, device="cuda", generator=g),
                 cond=D.pad_convert(torch.rand(n, 8 * hw, 8 * hw, cfg.cond_channels, device="cuda", generator=g), 64, dtype=dt),
                 ctx=torch.randn(n, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt),
                 noise=torch.randn(n, 4, hw, hw, device="cuda", generator=g),
                 timesteps=torch.tensor([40, 870, 333, 601][:n], device="cuda"))
    kw.setdefault("grad_scale", n * 4 * hw * hw / 2 if dt == torch.float16 else 1.0)

    def trainer():
        return ControlNetTrainer(unet, cnet, **kw)
    return cfg, wc, unet, cnet, batch, trainer


def _step(tr, b, **kw):
    return tr.step(b["latents"], b["cond"], b["ctx"], noise=kw.get("noise", b["noise"]), timesteps=kw.get("timesteps", b["timesteps"]))


def _forward(cnet, b):
    from dreammat_b200 import dense_ops as D
    zp = D.pad_convert(b["latents"].permute(0, 2, 3, 1).contiguous(), 64, dtype=cnet.dt)
    down, mid = cnet.forward(zp, b["timesteps"].float(), b["ctx"], b["cond"])
    return down + [mid]


def _pad_mask(tr):
    """True where the flat arenas hold channel padding of a prepared convolution or an alignment gap"""
    real = torch.zeros(tr.n, device="cuda", dtype=torch.bool)
    for key in tr.shapes:
        for idx in tr._index_map(key).values():
            real[idx.reshape(-1)] = True
    return ~real


@DTYPES
def test_construction_keeps_forward_bits_and_backward_writes_in_place(dt, monkeypatch):
    from dreammat_b200 import dense_ops as D, nets
    cfg, _, unet, cnet, b, trainer = _setup(dt)
    before = _forward(cnet, b)
    old = dict(cnet.p)
    tr = trainer()
    assert set(cnet.p) == set(old)
    for k, v in cnet.p.items():
        assert v.data_ptr() == tr.w16.data_ptr() + 2 * tr.offsets[k] and v.data_ptr() % 16 == 0
        assert v.shape == old[k].shape and v.dtype == dt and torch.equal(v, old[k])
    for x, y in zip(before, _forward(cnet, b)):
        assert torch.equal(x, y)
    assert torch.equal(tr.master, tr.w16.float()) and int(_pad_mask(tr).sum()) > 0

    zp = D.pad_convert(b["latents"].permute(0, 2, 3, 1).contiguous(), 64, dtype=dt)
    args = (unet, cnet, zp, b["timesteps"].float(), b["ctx"], b["cond"], b["noise"], 1.0, tr.grad_scale)
    loss_a, fresh = nets.controlnet_loss_and_grads(*args)
    tr.grad.fill_(float("nan"))
    alloc, frozen_decoder = D._f32_out, unet.backward_residuals
    trainable = [True]

    def no_alloc(t, shape, like):
        assert t is not None or not trainable[0], "a parameter gradient was allocated although `into` was given"
        return alloc(t, shape, like)

    def decoder(*a):      # the frozen UNet's LayerNorm backward forms affine gradients and drops them: not parameters' gradients
        trainable[0] = False
        try:
            return frozen_decoder(*a)
        finally:
            trainable[0] = True
    with monkeypatch.context() as mp:
        mp.setattr(D, "_f32_out", no_alloc)
        mp.setattr(unet, "backward_residuals", decoder)
        loss_b, got = nets.controlnet_loss_and_grads(*args, into=tr.grad_views)
    assert got is tr.grad_views and torch.equal(loss_a, loss_b) and set(got) == set(fresh)
    for k in fresh:
        assert torch.equal(fresh[k], got[k]), k
    assert not tr.grad[~_pad_mask(tr)].isnan().any()            # every parameter's slice was written


def _reference_step(tr, master, m, v, t):
    """clip_grad_norm_ + AdamW on the flat master copy with the gradient the step left in the arena"""
    p = master.clone().requires_grad_()
    opt = torch.optim.AdamW([p], lr=float(tr.state[0]), betas=tr.betas, eps=tr.eps, weight_decay=tr.weight_decay)
    if t:
        opt.state[p] = dict(step=torch.tensor(float(t)), exp_avg=m.clone(), exp_avg_sq=v.clone())
    p.grad = tr.grad / tr.grad_scale
    norm = torch.nn.utils.clip_grad_norm_([p], tr.max_grad_norm)
    opt.step()
    return p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], float(norm)


def _check_steps(dt, cfg, n, hw, steps, title):
    _, _, unet, cnet, b, trainer = _setup(dt, cfg=cfg, n=n, hw=hw, lr=1e-4)
    tr = trainer()
    for t in range(steps):
        if t:       # the second step is clipped for certain, later ones are not
            tr.max_grad_norm = tr.grad_norm / 2 if t == 1 else tr.grad_norm * 1e3
        state = [x.clone() for x in (tr.master, tr.m, tr.v)]
        loss = _step(tr, b)
        p, m, v, norm = _reference_step(tr, *state, t)
        errs = (rel(tr.master, p), rel(tr.m, m), rel(tr.v, v), abs(tr.grad_norm - norm) / norm)
        print(f"\n{title} {tname(dt)} step {t + 1}: loss {float(loss):.5f} grad_norm {tr.grad_norm:.4f} "
              f"errors master {errs[0]:.2e} m {errs[1]:.2e} v {errs[2]:.2e} norm {errs[3]:.2e}")
        assert errs[0] <= 1e-6 and errs[1] <= 2e-6 and errs[2] <= 2e-6 and errs[3] <= 1e-6, errs
        assert torch.equal(tr.w16, tr.master.to(dt)) and rel(tr.master, state[0]) > 0
    assert tr.steps == steps and tr.skipped_steps == 0


@DTYPES
def test_step_equals_torch_adamw_on_the_same_gradients(dt):
    _check_steps(dt, None, 2, 16, 3, "small")


@DTYPES
def test_full_size_step_equals_torch_adamw_on_the_same_gradients(dt):
    _check_steps(dt, O.UNetConfig(), 2, 16, 3, "full size")


@DTYPES
def test_padding_stays_zero_and_runs_repeat_bit_for_bit_eagerly_and_as_a_graph(dt):
    _, _, unet, cnet, b, trainer = _setup(dt, lr=1e-4)
    tr = trainer()
    start = tr.state_dict()
    pad = _pad_mask(tr)

    def run(captured):
        tr.load_state_dict(start)
        losses = [_step(tr, b).clone() for _ in range(5)]
        assert tr.steps == 5 and (not captured or tr._graph is not None)
        return losses + [tr.master.clone(), tr.w16.clone(), tr.m.clone(), tr.v.clone()]

    one = run(False)
    assert not tr.master[pad].any() and not tr.w16[pad].any() and not tr.m[pad].any() and not tr.grad[pad].any()
    assert float(one[4]) != float(one[0])
    two = run(False)
    tr.capture(b["latents"], b["cond"], b["ctx"])
    three = run(True)
    for x, y, z in zip(one, two, three):
        assert torch.equal(x, y) and torch.equal(x, z)
    # drawn noise / timesteps: the replayed step still trains and stays finite
    loss = tr.step(b["latents"], b["cond"], b["ctx"])
    assert tr.steps == 6 and torch.isfinite(loss) and tr.skipped_steps == 0


@DTYPES
def test_training_lowers_the_loss_and_leaves_the_unet_alone(dt):
    _, _, unet, cnet, b, trainer = _setup(dt, lr=1e-4)
    frozen = {k: v.clone() for k, v in unet.p.items()}
    w64 = unet.conv_out_w64.clone()
    tr = trainer()
    losses = [float(_step(tr, b)) for _ in range(20)]
    print(f"\n20 steps at lr 1e-4, {tname(dt)}: loss {losses[0]:.5f} -> {losses[-1]:.5f}")
    assert losses[-1] < losses[0] and tr.steps == 20
    assert all(torch.equal(v, frozen[k]) for k, v in unet.p.items()) and torch.equal(unet.conv_out_w64, w64)


@DTYPES
def test_state_dict_round_trip_is_exact_with_diffusers_names(dt):
    from dreammat_b200 import weights
    cfg, wc, unet, cnet, b, trainer = _setup(dt, lr=1e-4)
    tr = trainer()
    sd0 = tr.state_dict()
    names = weights.random_controlnet(cfg, "cuda")
    assert set(sd0["weights"]) == set(names) == set(wc)
    for k, v in sd0["weights"].items():
        assert v.shape == names[k].shape and v.dtype == torch.float32, k
        assert torch.equal(v, wc[k].float().cuda()), k            # the master copy starts from the 16-bit weights
    for _ in range(2):
        _step(tr, b)
    tr.set_lr(3e-5)
    sd = tr.state_dict()
    assert sd["step"] == 2 and sd["lr"] == float(torch.tensor(3e-5, dtype=torch.float32))
    kept = [t.clone() for t in (tr.master, tr.m, tr.v, tr.w16, tr.state[:3])]
    tr.step(b["latents"], b["cond"], b["ctx"])                     # move away (noise and timesteps drawn), then come back
    assert tr.steps == 3
    tr.load_state_dict(sd)
    for a, c in zip(kept, (tr.master, tr.m, tr.v, tr.w16, tr.state[:3])):
        assert torch.equal(a, c)
    again = tr.state_dict()
    for part in ("weights", "exp_avg", "exp_avg_sq"):
        assert set(again[part]) == set(sd[part]) and all(torch.equal(again[part][k], sd[part][k]) for k in sd[part])
    assert (again["step"], again["skipped_steps"], again["lr"]) == (sd["step"], sd["skipped_steps"], sd["lr"])
    # fp32 source weights, when given, become the master copy
    hi = {k: v + 1e-4 * torch.randn_like(v) for k, v in sd["weights"].items()}
    _, _, _, _, _, trainer2 = _setup(dt, master_weights=hi)
    tr2 = trainer2()
    got = tr2.state_dict()["weights"]
    assert all(torch.equal(got[k], hi[k]) for k in hi) and torch.equal(tr2.w16, tr2.master.to(dt))
