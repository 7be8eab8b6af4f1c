"""Multi-GPU sharding of a batch of independent frame-pair alignments (SURVEY.md section 8e).

Each alignment reads only its own two pyramids and writes its own Result (the reference runs them as
independent TBB tasks, dvo_slam/src/local_tracker.cpp:180-184, keyframe_graph.cpp:587-590), so the
batch shards by contiguous ranges of pair indices with no data-path collective; the only exchange is
one all-gather of fixed-size result records at the end.  Works with any torch.distributed backend
(NCCL on GPUs; gloo in the CPU unit tests).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
import torch.distributed as dist

from .engine import CResult

RESULT_BYTES = C.sizeof(CResult)


def shard_range(total: int, world_size: int, rank: int) -> tuple[int, int]:
    """Contiguous shard [begin, end) of pair indices owned by ``rank`` (remainder spread over the first ranks)."""
    base, rem = divmod(total, world_size)
    begin = rank * base + min(rank, rem)
    return begin, begin + base + (1 if rank < rem else 0)


def results_to_tensor(results, device) -> torch.Tensor:
    """ctypes array of dvo_b200_result -> uint8 tensor [n, RESULT_BYTES] on ``device``."""
    n = len(results)
    buf = np.frombuffer(memoryview(results), dtype=np.uint8).reshape(n, RESULT_BYTES)
    return torch.from_numpy(buf.copy()).to(device)


def tensor_to_results(t: torch.Tensor):
    arr = t.detach().cpu().contiguous().numpy()
    n = arr.shape[0]
    out = (CResult * n)()
    C.memmove(out, arr.ctypes.data, n * RESULT_BYTES)
    return out


def all_gather_results(local: torch.Tensor, total: int) -> torch.Tensor:
    """All-gather per-rank rows [n_r, m] into [total, m] in pair order, rank r holding the rows of shard_range(total, ws, r):
    any dtype and any m, padded to the largest shard.  The result records [n_r, RESULT_BYTES] uint8, and the other per-pair
    outputs of Engine.match_batch_modes_device as rows: (alpha, beta) [n_r, 2] float64, best as [n_r, 1] int32 and the
    scores [n_r, k] float64."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local
    ws = dist.get_world_size()
    sizes = [shard_range(total, ws, r) for r in range(ws)]
    nmax = max(e - b for b, e in sizes)
    pad = torch.zeros((nmax, local.shape[1]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    gathered = [torch.empty_like(pad) for _ in range(ws)]
    dist.all_gather(gathered, pad)
    return torch.cat([g[: e - b] for g, (b, e) in zip(gathered, sizes)], 0)
