"""Multi-GPU plumbing for the scoring path: one process per GPU (torchrun), documents / passages sharded
row-wise over ranks, ONE exchange step -- an all-gather of each rank's per-query top-k (score, global id)
over NCCL (NVLink 5 / NVSwitch) -- followed by a k-way merge on every rank.

The reference does this inside faiss (``GpuMultipleClonerOptions.shard = True``,
matchmaker/retrieval/faiss_indices.py:61-67: per-shard search, host-side merge); there is no
torch.distributed call anywhere in the reference.  Works with the ``gloo`` backend on CPU tensors too, which
is how the N>1 logic is tested without GPUs.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous row range [lo, hi) of rank `rank` (first n_items % world ranks get one extra row)."""
    per, rem = divmod(n_items, world)
    lo = rank * per + min(rank, rem)
    return lo, lo + per + (1 if rank < rem else 0)


def passage_shard_bounds(doc_offsets, rank: int, world: int) -> Tuple[int, int, int, int]:
    """Passage-aligned split of a ragged token store: passage d owns rows [doc_offsets[d], doc_offsets[d+1]).
    Returns (first passage, end passage, first row, end row) of rank `rank`.  Every passage lands on exactly one rank
    and rank r's range starts at the first passage that begins at or after row shard_bounds(n_rows, r, world)[0], so
    row ranges are contiguous, cover every row and are balanced up to one passage; a rank may get no passage."""
    import numpy as np
    off = np.asarray(doc_offsets, dtype=np.int64).reshape(-1)
    n_docs, n_rows = len(off) - 1, int(off[-1])

    def start(r: int) -> int:
        if r >= world:
            return n_docs
        return int(min(n_docs, np.searchsorted(off, shard_bounds(n_rows, r, world)[0], side="left")))

    d_lo, d_hi = start(rank), start(rank + 1)
    return d_lo, d_hi, int(off[d_lo]), int(off[d_hi])


def rank_topk(scores: torch.Tensor, ids: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Top-k per row under the project-wide total order (score descending, id ascending).
    scores [Nq, n] f32, ids [Nq, n] or [n] i64."""
    if ids.dim() == 1:
        ids = ids.unsqueeze(0).expand(scores.shape[0], -1)
    k = min(k, scores.shape[1])
    oi = torch.argsort(ids, dim=1, stable=True)
    s1 = torch.gather(scores, 1, oi)
    i1 = torch.gather(ids, 1, oi)
    os_ = torch.argsort(s1, dim=1, descending=True, stable=True)[:, :k]
    return torch.gather(s1, 1, os_), torch.gather(i1, 1, os_)


def all_gather_merge(local_scores: torch.Tensor, local_ids: torch.Tensor, k: int,
                     group: Optional[dist.ProcessGroup] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """All-gather per-rank top-k lists [Nq, k_local] (scores f32, global ids i64) and merge to the global
    top-k on every rank.  Message per rank: Nq * k_local * 12 bytes."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return rank_topk(local_scores, local_ids, k)
    world = dist.get_world_size(group)
    nq, kl = local_scores.shape
    # ONE collective: (score bits, id) packed as int64 pairs -> [world * nq, kl, 2]
    packed = torch.stack([local_scores.contiguous().view(torch.int32).to(torch.int64), local_ids.contiguous()], dim=-1)
    gathered = torch.empty((world * nq, kl, 2), dtype=torch.int64, device=packed.device)
    dist.all_gather_into_tensor(gathered, packed, group=group)  # rank-major concatenation
    gs = gathered[..., 0].to(torch.int32).view(torch.float32)
    gi = gathered[..., 1]
    cs = gs.reshape(world, nq, kl).permute(1, 0, 2).reshape(nq, world * kl)
    ci = gi.reshape(world, nq, kl).permute(1, 0, 2).reshape(nq, world * kl)
    if cs.is_cuda:  # k-way merge on the GPU kernel (mmb200_topk_merge); torch ops only for the gloo/CPU tests
        from . import interaction
        return interaction.topk_merge(cs, ci, min(k, world * kl))
    return rank_topk(cs, ci, k)


def topk_all_gather_merge(local_scores: torch.Tensor, k: int, id_base: int,
                          group: Optional[dist.ProcessGroup] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Scores of this rank's document shard [Nq, n_local] -> global per-query top-k.  Document j of the
    shard has global id ``id_base + j``."""
    nq, n = local_scores.shape
    ids = torch.arange(id_base, id_base + n, device=local_scores.device, dtype=torch.int64)
    if local_scores.is_cuda:
        from . import interaction
        ls, li = interaction.topk_merge(local_scores, ids.unsqueeze(0).expand(nq, -1), min(k, n))
    else:
        ls, li = rank_topk(local_scores, ids, k)
    return all_gather_merge(ls, li, k, group)
