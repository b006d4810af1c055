"""Multi-GPU host logic of the inference path: independent sequences shard across ranks with no data-path
collective (SURVEY.md §8e); the only exchanges are the timing reduction and an optional gather of results."""
from __future__ import annotations


def shard_indices(n_items: int, world_size: int, rank: int) -> list[int]:
    """Round-robin: sequence s runs on rank s % world_size (the reference's samplers slice per rank the same way,
    spann3r/datasets/__init__.py:27-39)."""
    if not (0 <= rank < world_size):
        raise ValueError(f"rank {rank} outside world of {world_size}")
    return list(range(rank, n_items, world_size))


def max_over_ranks(value_ms: float, device=None) -> float:
    """Max of a per-rank scalar (CUDA-event milliseconds) over the process group; identity without one."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value_ms)
    t = torch.tensor([value_ms], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_objects(obj):
    """All ranks' small python objects on every rank (per-rank frame counts / timings)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [obj]
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def run_sharded(forward, sequences, per_gpu_batch: int = 1, rank: int | None = None, world_size: int | None = None,
                independent: bool = False):
    """BASELINE config[2] as a function: `sequences` (a list of equal-length lists of view dicts {'img': [1, 3, H, W]},
    the SAME list on every rank) are dealt round-robin to the ranks (`shard_indices`); each rank advances up to
    `per_gpu_batch` of its sequences in lockstep as one batched call of `forward` (= `Spann3R.forward`; sequences in a
    batch must share frame count and resolution) and returns {sequence index: preds of that sequence} for ITS sequences.
    No collective on the data path; use `gather_objects` for small per-rank summaries.

    independent=True: `forward` is `Spann3R.forward_sequences`, called once with all of the rank's sequences and
    max_batch = per_gpu_batch; each sequence then runs with its own memory, as at batch 1, and sequences may differ in
    length and resolution."""
    import torch
    import torch.distributed as dist
    if world_size is None:
        world_size = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
    if rank is None:
        rank = dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0
    if per_gpu_batch < 1:
        raise ValueError("per_gpu_batch must be >= 1")
    mine = shard_indices(len(sequences), world_size, rank)
    if independent:
        res = forward([sequences[i] for i in mine], per_gpu_batch)
        return {i: r[0] for i, r in zip(mine, res)}
    out = {}
    for s0 in range(0, len(mine), per_gpu_batch):
        ids = mine[s0: s0 + per_gpu_batch]
        seqs = [sequences[i] for i in ids]
        n_frames = len(seqs[0])
        if any(len(q) != n_frames for q in seqs):
            raise ValueError("sequences advanced in lockstep must have the same number of frames")
        if any(tuple(q[f]["img"].shape) != tuple(seqs[0][f]["img"].shape) for q in seqs for f in range(n_frames)):
            raise ValueError("sequences advanced in lockstep must share one resolution")
        frames = [{"img": torch.cat([q[f]["img"] for q in seqs], dim=0)} for f in range(n_frames)]
        preds = forward(frames)[0]
        for j, i in enumerate(ids):
            out[i] = [{k: v[j: j + 1] for k, v in p.items()} for p in preds]
    return out
