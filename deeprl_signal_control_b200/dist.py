"""Replica sharding across ranks (one process per GPU).  Replicas are independent, so the
simulation path has no collective; the learner all-reduces (SUM) its flat gradient once per update
after each rank scaled its local sum by 1 / (n_step * total_replicas).

Used by the product path: `BatchedTrainer.start_episode` (episode_seeds), `BatchedA2C.backward` (grad_scale,
allreduce_sum_), the training driver `agents/train.py` (replica_range, gather_traces, sum_partials) and bench.py (shard_replicas)."""
from __future__ import annotations

import numpy as np


def replica_range(rank: int, world: int, total_replicas: int):
    """(replica0, n_local) of `rank` when `total_replicas` global replicas are split evenly over `world` ranks: rank k
    owns [k*R/W, (k+1)*R/W).  Raises ValueError unless world divides total_replicas, so that every rank rejects a bad
    split alike, before any collective."""
    rank, world, total = int(rank), int(world), int(total_replicas)
    if world < 1 or not 0 <= rank < world:
        raise ValueError("rank %d is not in a world of %d" % (rank, world))
    if total % world:
        raise ValueError("%d replicas cannot be split evenly over %d ranks" % (total, world))
    n = total // world
    return rank * n, n


def gather_traces(trace, group=None, dst: int = 0):
    """Host-side gather of every rank's [T, r] trace (the same r on every rank) to group rank `dst`, in global replica
    order: rank k's columns land at [k*r, (k+1)*r) of the result.  `trace` is a host array or CPU tensor, so the group
    must take CPU tensors (gloo).  Returns the float32 [T, world*r] numpy array on `dst`, None on every other rank."""
    import torch
    import torch.distributed as dist
    t = torch.as_tensor(np.ascontiguousarray(trace, dtype=np.float32))
    parts = [torch.empty_like(t) for _ in range(dist.get_world_size(group))] \
        if dist.get_rank(group) == dst else None
    dist.gather(t, parts, group=group, group_dst=dst)
    return None if parts is None else torch.cat(parts, 1).numpy()


def sum_partials(x, group=None, dst: int = 0):
    """Host-side sum over the ranks of `group` (gloo) of every rank's same-shape float array, to group rank `dst`:
    gathered as float32, added in float64 in rank order.  Returns the float64 numpy sum on `dst`, None on every other
    rank.  The training driver adds the A2C loss terms with it, each rank's being its partial sum already scaled by
    1 / (n_step * R_total)."""
    import torch
    import torch.distributed as dist
    t = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32))
    parts = [torch.empty_like(t) for _ in range(dist.get_world_size(group))] \
        if dist.get_rank(group) == dst else None
    dist.gather(t, parts, group=group, group_dst=dst)
    if parts is None:
        return None
    out = np.zeros(t.shape, np.float64)
    for p in parts:
        out += p.numpy()
    return out


def shard_replicas(rank: int, world: int, replicas_per_rank: int, seed0: int):
    """Global replica ids and first-episode seeds of one rank: rank k owns [k*R, (k+1)*R)."""
    replica0 = rank * replicas_per_rank
    ids = np.arange(replicas_per_rank, dtype=np.int64) + replica0
    seeds = episode_seeds(seed0, 0, replica0, replicas_per_rank, world * replicas_per_rank)
    return replica0, ids, seeds


def episode_seeds(seed0: int, episode: int, replica0: int, n_local: int, total_replicas: int) -> np.ndarray:
    """Seeds of this rank's replicas for its `episode`-th episode.  The reference re-seeds SUMO with `seed += 1` per
    episode (envs/env.py:560); with R_total lock-stepped replicas the counter advances by R_total per episode, so that
    the seed sets of all (rank, episode) pairs are disjoint: seed = seed0 + episode * R_total + global replica id."""
    ids = np.arange(n_local, dtype=np.int64) + int(replica0)
    return (ids + int(seed0) + int(episode) * int(total_replicas)).astype(np.uint64)


def grad_scale(n_step: int, world: int, replicas_per_rank: int) -> float:
    return 1.0 / (n_step * world * replicas_per_rank)


def allreduce_sum_(flat_grad, group=None):
    import torch.distributed as dist
    dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
    return flat_grad


def bind_to_gpu_numa(device_index: int):
    """Restrict this process to the host cores of the GPU's NUMA node (nvidia-smi topo 'CPU Affinity'), BEFORE any
    page-locked buffer is allocated: pinned pages are then first-touched on the local node, so a rank's H2D / D2H
    traffic does not cross the inter-socket link.  On an 8-GPU box GPUs 0-3 and 4-7 hang off different sockets; four
    ranks sharing one socket's PCIe root is what limited the host-buffer (e2e) path at N = 4 in round 1.
    Returns the cpu list it bound to, or None when NVML / the affinity call is unavailable (nothing is changed then)."""
    import os
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(int(device_index))
        n_words = (os.cpu_count() + 63) // 64
        mask = nv.nvmlDeviceGetCpuAffinity(h, n_words)
        cpus = {64 * w + b for w, word in enumerate(mask) for b in range(64) if (int(word) >> b) & 1}
        cpus &= set(os.sched_getaffinity(0))
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return sorted(cpus)
    except Exception:
        return None
