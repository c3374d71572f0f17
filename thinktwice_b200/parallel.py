"""Data-parallel sharding of independent frames + the path's single collective (SURVEY.md §8e).

Frames of a batch are split into contiguous chunks, one per rank (one process per GPU); weights are replicated;
after the forward ONE all-gather returns every rank's waypoints `(B_local, K+1, 4, 2)` — a few hundred bytes, i.e.
a latency-bound NCCL call issued on the compute stream right after the last decoder kernel.  No kernel has a
collective to fuse with.  NOTE (SURVEY fact 4): in the default mode the reference's Look module couples the frames of one
forward call, so sharded results equal the reference run with the SAME per-rank chunk, not the un-sharded batch.  With
`model.enable_independent_frames()` every frame is computed as if alone, so a sharded batch equals the un-sharded batch frame
for frame.  A list of per-frame clouds in batch['points'] is sliced like the other per-frame lists.
"""
import torch
import torch.distributed as dist


def shard_range(total, rank, world):
    """contiguous chunk [lo, hi) of `total` frames owned by `rank` (remainder spread over the first ranks)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(batch, rank, world):
    """slice every per-frame entry of a reference-format batch dict (tensors on dim 0, img_metas list)."""
    B = batch['img'].shape[0]
    lo, hi = shard_range(B, rank, world)
    out = {}
    for k, v in batch.items():
        if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == B:
            out[k] = v[lo:hi]
        elif isinstance(v, list) and len(v) == B:
            out[k] = v[lo:hi]
        else:
            out[k] = v
    return out


def gather_waypoints(pred_wp, world=None, out=None):
    """all-gather of the local waypoints; returns (B_total, K+1, 4, 2) ordered by rank (== frame order of
    shard_batch).  Equal chunk sizes use one all_gather_into_tensor; ragged chunks fall back to all_gather."""
    if not (dist.is_available() and dist.is_initialized()):
        return pred_wp
    world = world or dist.get_world_size()
    wp = pred_wp.contiguous()
    sizes = [None] * world
    if out is not None:                                            # equal chunks, preallocated (graph-friendly)
        dist.all_gather_into_tensor(out, wp)
        return out
    n = torch.tensor([wp.shape[0]], device=wp.device)
    counts = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(counts, n)
    counts = [int(c) for c in counts]
    if len(set(counts)) == 1:
        out = wp.new_empty((world * counts[0],) + tuple(wp.shape[1:]))
        dist.all_gather_into_tensor(out, wp)
        return out
    m = max(counts)
    pad = wp.new_zeros((m,) + tuple(wp.shape[1:]))
    pad[:wp.shape[0]] = wp
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.cat([p[:c] for p, c in zip(parts, counts)], 0)
