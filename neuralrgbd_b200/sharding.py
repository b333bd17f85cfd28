"""Multi-GPU plumbing of the inference path (SURVEY §8e): one process per GPU, trajectories /
windows sharded across ranks, weights broadcast once, no per-frame collective.

Replaces what `torch.nn.DataParallel` does implicitly in the reference (`test_KVNet.py:163-164`,
`train_KVNet.py:261-262`: replicate weights every forward, scatter one video per GPU, gather).
Backend-agnostic (`nccl` on the GPU machines, `gloo` in the CPU tests)."""
import torch
import torch.distributed as dist


def shard_indices(n_items, rank, world):
    """Round-robin ownership `r, r+world, ...` (SURVEY §8e). Every item belongs to exactly one rank."""
    return list(range(rank, n_items, world))


def chunk_trajectory(n_frames, t_win_r, n_chunks):
    """Split the valid reference indices [t_win_r, n_frames - t_win_r) of one trajectory into
    n_chunks contiguous chunks. Each chunk restarts the K-Net recursion with BV_predict=None at its
    head (the reference does the same at trajectory starts / invalid poses, test_KVNet.py:197-198,
    241-246) and reads a t_win_r halo of frames on both sides."""
    lo, hi = t_win_r, n_frames - t_win_r
    n = max(hi - lo, 0)
    out = []
    for c in range(n_chunks):
        a = lo + (n * c) // n_chunks
        b = lo + (n * (c + 1)) // n_chunks
        if b > a:
            out.append({'ref_begin': a, 'ref_end': b, 'frame_begin': a - t_win_r, 'frame_end': b + t_win_r})
    return out


def broadcast_module(module, src=0):
    """One broadcast per floating-point parameter/buffer (21 MB total for KVNET): the only collective
    on the inference path, executed once at start-up."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 0
    n = 0
    seen = set()
    for t in list(module.parameters()) + list(module.buffers()):
        if t.data_ptr() in seen or not t.is_floating_point():
            continue
        seen.add(t.data_ptr())
        dist.broadcast(t.data, src=src)
        n += t.numel()
    return n


def max_over_ranks(value, device=None):
    """Max of a scalar over ranks (the bench's step time is the slowest rank's)."""
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
