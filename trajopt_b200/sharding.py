"""Batch sharding over ranks (SURVEY.md §8e): trajectories never interact, so a batch is cut into contiguous
shards, one per GPU / process, with no collective on the data path.  The only exchanges are the report's
reductions (converged count, max device time) and, when one caller wants the whole batch back, a gather of the
per-trajectory results in rank order.  A multi-start batch (group_size G > 1) is cut on group boundaries: the seeds of one
problem interact (group_stop) and are selected together, so a group is never split across ranks."""
import numpy as np


def shard_bounds(total, rank, world, group_size=0):
    """[b0, b1) of `rank`: contiguous shards, the first `total % world` ranks get one extra trajectory.  With
    group_size G > 1 the groups are shared out that way instead, and the bounds are whole groups."""
    G = max(int(group_size), 1)
    if not (0 <= rank < world) or total < 0 or total % G:
        raise ValueError("bad rank/world/total/group_size")
    base, extra = divmod(total // G, world)
    g0 = rank * base + min(rank, extra)
    return g0 * G, (g0 + base + (1 if rank < extra else 0)) * G


def shard(desc, rank, world):
    b0, b1 = shard_bounds(desc.B, rank, world, desc.c.group_size)
    return desc.slice(b0, b1)


def converged_count(status, group_size=0):
    """The report's converged count: trajectories that ended OPT_CONVERGED, or with groups (G > 1) problems with at
    least one converged seed."""
    ok = np.asarray(status) == 0
    G = max(int(group_size), 1)
    return int(ok.sum()) if G == 1 else int(ok.reshape(-1, G).any(axis=1).sum())


def gather_results(local, total, dist=None, group_size=0):
    """All ranks receive the full-batch results (rank order = trajectory order).  `local` maps names to arrays
    whose first axis is the shard (of a batch sharded with `group_size`); `dist` is torch.distributed (None = single
    process).  Per-group arrays gather with total = the number of groups and no group_size."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return {k: np.asarray(v) for k, v in local.items()}
    import torch
    world = dist.get_world_size()
    out = {}
    for k in sorted(local):
        v = np.ascontiguousarray(local[k])
        parts = []
        for r in range(world):  # shards may differ in length by one: broadcast each rank's piece
            b0, b1 = shard_bounds(total, r, world, group_size)
            buf = torch.from_numpy(v.copy() if r == dist.get_rank() else np.zeros((b1 - b0,) + v.shape[1:], v.dtype))
            dist.broadcast(buf, src=r)
            parts.append(buf.numpy())
        out[k] = np.concatenate(parts, axis=0)
    return out


def reduce_report(converged, seconds, dist=None):
    """(sum of converged trajectories, max of the per-rank device time) — the numbers bench.py reports."""
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return float(converged), float(seconds)
    import torch
    c = torch.tensor([float(converged)], dtype=torch.float64)
    s = torch.tensor([float(seconds)], dtype=torch.float64)
    dist.all_reduce(c, op=dist.ReduceOp.SUM)
    dist.all_reduce(s, op=dist.ReduceOp.MAX)
    return float(c.item()), float(s.item())
