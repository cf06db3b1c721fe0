"""View-parallel data parallelism for the SDS step (SURVEY.md section 8e).

Views are independent up to the parameter gradient, so the global batch of V views is split into
contiguous shards of V / world views; SD / ControlNet / VAE weights, env maps, the BVH and the G-buffer
cache are replicated.  The only exchange is ONE all-reduce(SUM) of the flat [hash grid | W1 | W2] gradient
(12 602 288 fp32 = 50.4 MB) per step, after which every rank applies the identical fused Adam update.

Normalisation that keeps the sharded step equal to the single-process one:
  * loss_sds is a mean over the GLOBAL batch of views (dreammat_guidance.py:594 `/ batch_size`), so each
    rank scales its d loss / d latents by 1 / V_global;
  * loss_mat_reg is a mean over the covered pixels of the WHOLE batch (dreammat_material.py:116-117), so
    each rank normalises its pixel sums by the global pixel count.  Every rank holds the full G-buffer
    cache, so that count is known locally -- no extra collective.
"""
from __future__ import annotations

import gc
from typing import List, Sequence, Tuple

import torch


def quiesce_host_gc() -> None:
    """Move everything alive now (torch, the nets, the scene: ~170 k objects) to the permanent generation.  With one process per
    GPU every step ends in a collective, so the step is as slow as the slowest rank's HOST, and a full generation-2 collection
    of this process takes 32-40 ms (measured) against a 25 ms 8-GPU step.  After the freeze a full collection only walks what
    was allocated since (microseconds).  Insurance, not a measured win: the 300-step A/B runs on 1 and 2 GPUs
    saw no step hit by a collection either way -- the step allocates few container objects.
    No reference counterpart."""
    gc.collect()
    gc.freeze()


def shard_slice(n_views: int, rank: int, world: int) -> slice:
    if n_views % world != 0:
        raise ValueError(f"global view batch {n_views} must divide over {world} ranks")
    per = n_views // world
    return slice(rank * per, (rank + 1) * per)


def global_pixel_count(pn_per_view: Sequence[int], view_ids: Sequence[int]) -> int:
    return int(sum(int(pn_per_view[int(v)]) for v in view_ids))


def allreduce_gradients(flat_grad: torch.Tensor, world: int):
    """The single collective of the step.  NCCL over NVLink/NVSwitch on GPUs, gloo in the CPU tests."""
    if world > 1:
        import torch.distributed as dist
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)
    return flat_grad


# ---------------------------------------------------------------------------------------------------------------------
# Pixel-balanced shading (multi-GPU).  One view per rank leaves the ranks with 57 k .. 198 k covered pixels (x 328 rays):
# the step waits for the largest view.  The Monte-Carlo shading is per-pixel independent and every rank holds the BVH,
# the hash grid and the whole G-buffer cache, so the covered pixels of the GLOBAL batch are laid out in one line
# (views in global batch order, pixels in G-buffer order) and cut into `world` equal intervals.  Rank r shades interval
# r, then ONE all-to-all returns the colours to the ranks that own the views (whole images are needed for the
# antialias blend, the VAE and the UNet); in the backward the same all-to-all, transposed, carries d loss / d colour
# back to the shading ranks, whose hash-grid gradients meet in the existing gradient all-reduce.

def pixel_partition(pn_global: Sequence[int], world: int) -> Tuple[List[List[Tuple[int, int, int]]], List[List[int]]]:
    """pn_global[g] = covered pixels of view g of the global batch (rank-major order, V_local views per rank).

    Returns (segments, counts): segments[r] = [(g, start, stop), ...] pieces of views that rank r shades (in global
    order), counts[r][o] = number of pixels rank r shades for views owned by rank o (all-to-all split sizes)."""
    V = len(pn_global)
    if V % world != 0:
        raise ValueError(f"global view batch {V} must divide over {world} ranks")
    per = V // world
    off = [0]
    for n in pn_global:
        off.append(off[-1] + int(n))
    P = off[-1]
    segments: List[List[Tuple[int, int, int]]] = []
    counts: List[List[int]] = []
    for r in range(world):
        lo, hi = r * P // world, (r + 1) * P // world
        segs, cnt = [], [0] * world
        for g in range(V):
            a, b = max(lo, off[g]), min(hi, off[g + 1])
            if b > a:
                segs.append((g, a - off[g], b - off[g]))
                cnt[g // per] += b - a
        segments.append(segs)
        counts.append(cnt)
    return segments, counts


def warm_exchange(max_rows: int, world: int, device) -> None:
    """Run the row exchange once per message-size decade before the step loop.  NCCL sets up point-to-point channels lazily
    and uses more of them for larger messages, while the per-step counts vary with the sampled views, so a size class first
    seen inside the loop can pay a connection setup there.  A candidate for the single 350 ms step seen in one 300-step run on
    2 GPUs; not separated from the allocator cause handled by
    DreamMat.reserve_step_scratch()."""
    if world == 1:
        return
    rows = 16
    while True:
        rows = min(rows, max(int(max_rows), 16))
        for c in (3, 9):
            buf = torch.zeros(rows * world, c, device=device)
            exchange_rows(buf, [rows] * world, [rows] * world, world)
        if rows >= max_rows:
            break
        rows *= 4


def exchange_rows(send: torch.Tensor, send_counts: Sequence[int], recv_counts: Sequence[int], world: int) -> torch.Tensor:
    """all_to_all of row blocks: `send` [sum(send_counts), C] grouped by destination rank in rank order ->
    [sum(recv_counts), C] grouped by source rank.  NCCL on GPUs, gloo in the CPU tests."""
    recv = send.new_empty((int(sum(recv_counts)),) + tuple(send.shape[1:]))
    if world == 1:
        recv.copy_(send)
        return recv
    import torch.distributed as dist
    dist.all_to_all_single(recv, send.contiguous(), [int(c) for c in recv_counts], [int(c) for c in send_counts])
    return recv
