"""Node-axis sharding across GPUs (SURVEY §8e): one process per GPU, tasks/jobs/queues replicated,
nodes split in contiguous NodeList blocks.  The dense pass needs exactly two small exchanges:

  1. MAX all-reduce of the per-group gradient statistics (does any idle-fit / future-fit node exist, max
     soft-taint count) so every shard scores against the same candidate set;
  2. a fold of the per-task best (score, node) pairs — all-gather of T x 12 bytes per rank, then the
     canonical arg-max (highest score, lowest NodeList index).

torch.distributed is the plumbing (NCCL on GPUs, gloo in the CPU tests); tensors wrap the library's own
device buffers, nothing is computed by torch on the hot path besides the tiny fold.
"""
from __future__ import annotations

from typing import Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_nodes: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous block of the node axis for `rank`; block starts are multiples of 64 (mask words)."""
    per = -(-n_nodes // world)
    per = -(-per // 64) * 64
    b = min(n_nodes, rank * per)
    e = min(n_nodes, b + per)
    return b, e


def fold_best(best_score: torch.Tensor, best_node: torch.Tensor, group=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Cross-shard arg-max of per-task (score f64, node i32; -1 = no candidate in this shard)."""
    world = dist.get_world_size(group)
    scores = [torch.empty_like(best_score) for _ in range(world)]
    nodes = [torch.empty_like(best_node) for _ in range(world)]
    dist.all_gather(scores, best_score, group=group)
    dist.all_gather(nodes, best_node, group=group)
    s = torch.stack(scores)  # [W, T]
    n = torch.stack(nodes).to(torch.int64)
    valid = n >= 0
    neg_inf = torch.full_like(s, float("-inf"))
    s_m = torch.where(valid, s, neg_inf)
    top = s_m.max(dim=0).values
    big = torch.iinfo(torch.int64).max
    cand = torch.where(valid & (s_m == top.unsqueeze(0)), n, torch.full_like(n, big))
    node = cand.min(dim=0).values
    none = node == big
    node = torch.where(none, torch.full_like(node, -1), node).to(torch.int32)
    score = torch.where(none, torch.zeros_like(top), top)
    return score, node


def reduce_group_stats(stats: torch.Tensor, group=None) -> torch.Tensor:
    """MAX all-reduce of the int32 [G,4] gradient statistics (flags are 0/1, counts are maxima)."""
    dist.all_reduce(stats, op=dist.ReduceOp.MAX, group=group)
    return stats


class _CudaBuffer:
    """__cuda_array_interface__ view of a device pointer owned by libvcalloc."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 3}


def device_tensor(ptr: int, shape, dtype: torch.dtype, device) -> torch.Tensor:
    typestr = {torch.float64: "<f8", torch.int32: "<i4"}[dtype]
    return torch.as_tensor(_CudaBuffer(ptr, shape, typestr), device=device)


def sharded_dense_best(eng, world: int, rank: int, device, materialize: bool = False):
    """Node-sharded dense pass on an uploaded Engine: returns the global per-task best (score, node)."""
    b, e = shard_bounds(eng.snap.N, world, rank)
    eng.set_shard(b, e)
    eng.dense_begin()
    ptr, count = eng.dense_stats_ptr()
    if count:
        reduce_group_stats(device_tensor(ptr, (count,), torch.int32, device))
        # NCCL returns once the reduction is queued and orders only torch's current stream after it; the library's
        # stream is non-blocking, so the scoring kernels of dense_finish would otherwise read the shard's local stats
        torch.cuda.current_stream(device).synchronize()
    eng.dense_finish(materialize)
    ps, pn = eng.dense_best_ptrs()
    T = eng.snap.T
    return fold_best(device_tensor(ps, (T,), torch.float64, device), device_tensor(pn, (T,), torch.int32, device))
