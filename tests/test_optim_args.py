"""Host side of the ControlNet optimizer (no GPU): argument checks of dm_grad_sumsq / dm_adamw_prepare / dm_adamw_step (the
library returns before touching the device, so the pointers here are never dereferenced), the bucketed gradient all-reduce
under gloo with two processes, and the layout of the flat parameter arenas."""
import ctypes as C
import os
import socket

import torch
import torch.multiprocessing as mp

DM_EINVAL = -1
A, M, V, G, W, S = (C.c_void_p(a) for a in (0x10000, 0x30000, 0x40000, 0x50000, 0x60000, 0x70000))
ODD2, ODD8 = C.c_void_p(0x10002), C.c_void_p(0x10008)
INF, NAN = float("inf"), float("nan")


def _sumsq(g=G, n=1001, out=S):
    from dreammat_b200._cabi import lib
    return lib().dm_grad_sumsq(g, n, out, None)


def _prepare(sumsq=S, state=A, b1=0.9, b2=0.999, max_norm=1.0, inv=1.0):
    from dreammat_b200._cabi import lib
    return lib().dm_adamw_prepare(sumsq, state, b1, b2, max_norm, inv, None)


def _step(bf16=1, master=A, m=M, v=V, g=G, w16=W, n=1001, state=S, b1=0.9, b2=0.999, eps=1e-8, wd=1e-2):
    from dreammat_b200._cabi import lib
    return lib().dm_adamw_step(bf16, master, m, v, g, w16, n, state, b1, b2, eps, wd, None)


def test_grad_sumsq_rejects_bad_arguments():
    from dreammat_b200._cabi import lib
    for kw in (dict(g=None), dict(out=None), dict(n=0), dict(n=-4), dict(g=ODD8), dict(out=ODD2)):
        assert _sumsq(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


def test_adamw_prepare_rejects_bad_arguments():
    from dreammat_b200._cabi import lib
    for kw in (dict(sumsq=None), dict(state=None), dict(sumsq=ODD2), dict(state=ODD2), dict(b1=1.0), dict(b1=-0.1), dict(b2=1.0),
               dict(b2=1.5), dict(b1=NAN), dict(max_norm=-1.0), dict(max_norm=NAN), dict(inv=0.0), dict(inv=-1.0), dict(inv=INF),
               dict(inv=NAN)):
        assert _prepare(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


def test_adamw_step_rejects_bad_arguments():
    from dreammat_b200._cabi import lib
    for kw in (dict(bf16=2), dict(bf16=-1), dict(master=None), dict(m=None), dict(v=None), dict(g=None), dict(w16=None),
               dict(state=None), dict(n=0), dict(n=-8), dict(master=ODD8), dict(m=ODD8), dict(v=ODD8), dict(g=ODD8), dict(w16=ODD8),
               dict(state=ODD2), dict(b1=1.0), dict(b1=-0.5), dict(b2=1.0), dict(b2=NAN), dict(eps=-1e-8), dict(wd=-0.1)):
        assert _step(**kw) == DM_EINVAL, (kw, lib().dm_last_error())


# ------------------------------------------------------------------------------------------------ all-reduce


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_FLAT = 10008


def _rank_grad(rank):
    return torch.randn(N_FLAT, generator=torch.Generator().manual_seed(7 + rank))


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    from dreammat_b200.parallel import allreduce_mean_buckets
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mean = sum(_rank_grad(r) for r in range(world)) / world
    # buckets that divide the buffer (8 x 1251 elements, the whole buffer), ones that do not, one larger than the buffer
    for bucket_bytes in (4 * 1251, 4 * N_FLAT, 4 * 1000, 4 * 4096, 1 << 20):
        flat = _rank_grad(rank)
        scale = allreduce_mean_buckets(flat, world, bucket_bytes=bucket_bytes)
        ret[(rank, bucket_bytes)] = (scale, float((flat * scale - mean).abs().max()))
    dist.barrier()
    dist.destroy_process_group()


def test_bucketed_allreduce_equals_single_process_mean():
    from dreammat_b200.parallel import allreduce_mean_buckets
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    assert len(ret) == 10
    for key, (scale, err) in ret.items():
        assert scale == 0.5 and err <= 1e-6, (key, scale, err)
    flat = _rank_grad(0)
    assert allreduce_mean_buckets(flat, 1) == 1.0 and torch.equal(flat, _rank_grad(0))     # world 1: no collective


# ------------------------------------------------------------------------------------------------ arena layout


def test_arena_offsets_are_16_byte_aligned_and_views_tile_the_arena_without_overlap():
    from dreammat_b200.controlnet_train import ARENA_ALIGN, arena_layout, arena_views
    shapes = {"conv.w": (64, 9 * 64), "conv.bias": (64,), "odd.w": (5, 3), "one": (1,), "norm.weight": (321,), "tproj.w": (37, 11),
              "last": (7,)}
    off, n = arena_layout(shapes)
    assert list(off) == list(shapes) and n % ARENA_ALIGN == 0
    for dt in (torch.float16, torch.bfloat16, torch.float32):
        flat = torch.zeros(n, dtype=dt)
        views = arena_views(flat, shapes, off)
        assert set(views) == set(shapes)
        for k, v in views.items():
            assert tuple(v.shape) == shapes[k] and v.is_contiguous()
            assert (v.data_ptr() - flat.data_ptr()) == off[k] * flat.element_size()
            assert (off[k] * 2) % 16 == 0                       # 16 bytes in the 16-bit arena, so also in the fp32 ones
            v += 1                                              # every element of every view exactly once
        covered = int(flat.float().sum())
        assert covered == sum(v.numel() for v in views.values()) and float(flat.float().max()) == 1.0
        assert n - covered < ARENA_ALIGN * len(shapes)          # only alignment gaps are left, and they are untouched
