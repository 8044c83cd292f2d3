"""Exact (brute-force) maximum-inner-product index with id mapping on the H100 kernels.

Drop-in for ``FaissIdIndexer`` (matchmaker/retrieval/faiss_indices.py:49-74) as driven by
dense_retrieval.py:328 (``index``) and :391 (``search``): same constructor config keys (``token_dim``,
``faiss_use_gpu``, ``token_dtype``), same method signatures, numpy in / numpy out.

Multi-GPU: the reference shards through faiss (``GpuMultipleClonerOptions.shard = True``) inside one process.
Here every rank of a ``torch.distributed`` job keeps one contiguous slab of the passages in its GPU's HBM
(fp16, 1 536 B per 768-d passage: 8.8 M passages = 13.5 GB, 1.7 GB per GPU on 8), searches it with the fused
GEMM + top-k kernel, and the per-query top-k lists are exchanged with ONE NCCL all-gather and merged.
"""
from __future__ import annotations

from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction, sharding
from .base_index import GPUIndexer


class FlatIPIndexer(GPUIndexer):
    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.passages: Optional[torch.Tensor] = None   # [n_local, dim] fp16 on self.device
        self.ids: Optional[torch.Tensor] = None        # [n_local] int64
        self.n_total = 0
        self.split_scale = None

    def index(self, ids: List[numpy.ndarray], data_chunks: List[numpy.ndarray]):
        """ids: list of int64 arrays; data_chunks: list of [n_i, token_dim] arrays (the fp16 memmaps of
        dense_retrieval.py:297-302).  Every rank is given the same lists and keeps rows shard_bounds(n, rank, world).
        The rows go to HBM through token_storage.blocks_to_device: file-backed memmaps are read by the native loader
        (pread -> pinned staging -> cudaMemcpyAsync), only the byte range this rank owns is touched."""
        from .token_storage import blocks_to_device
        rank, world = self._world()
        n = int(sum(len(x) for x in ids))
        lo, hi = sharding.shard_bounds(n, rank, world)
        self.n_total, self.lo, self.hi = n, lo, hi
        if hi > lo:
            with torch.cuda.device(self.device):
                vecs = blocks_to_device(data_chunks, lo, hi, self.device)
            self._set_passages(vecs)
            id_parts, off = [], 0
            for i_arr in ids:
                a, b = max(lo, off), min(hi, off + len(i_arr))
                if a < b:
                    id_parts.append(torch.from_numpy(numpy.ascontiguousarray(i_arr[a - off:b - off]).astype(numpy.int64)))
                off += len(i_arr)
            self.ids = torch.cat(id_parts).to(self.device)
        else:
            self._set_passages(torch.empty((0, self.token_dim), dtype=self.store_dtype, device=self.device))
            self.ids = torch.empty(0, dtype=torch.int64, device=self.device)

    def _set_passages(self, vecs: torch.Tensor):
        """fp16 storage as is; fp32 storage (token_dtype float32, faiss without useFloat16) as the fp16 hi / lo split the
        kernel consumes -- same bytes per passage as fp32, 22 mantissa bits per value."""
        if self.store_dtype == torch.float16:
            self.passages, self.split_scale = vecs.to(torch.float16), None
        else:
            self.passages, self.split_scale = interaction.flat_ip_split_f32(vecs.float(), "passages")

    def search(self, query_vec: numpy.ndarray, top_n: int):
        if self.passages is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        if query_vec.ndim == 1:
            query_vec = query_vec[numpy.newaxis, :]
        q = torch.from_numpy(numpy.ascontiguousarray(query_vec)).to(
            self.device, dtype=torch.float16 if self.store_dtype == torch.float16 else torch.float32)
        scores, ids = self.search_device(q, top_n)
        return scores.cpu().numpy(), ids.cpu().numpy()

    def search_device(self, q: torch.Tensor, top_n: int):
        """Same as search() but device tensors in/out (no host round trip)."""
        rank, world = self._world()
        if top_n > interaction.FLAT_IP_MAX_K:
            raise _lib.MatchmakerB200Error(f"top_n > {interaction.FLAT_IP_MAX_K} is not supported by the fused top-k kernel")
        k_local = top_n
        if self.passages.shape[0] > 0:
            s, i = interaction.flat_ip_topk(q, self.passages, k_local, ids=self.ids, split_scale=self.split_scale)
        else:
            s = torch.full((q.shape[0], k_local), -3.4028234663852886e38, device=self.device)
            i = torch.full((q.shape[0], k_local), -1, dtype=torch.int64, device=self.device)
        if world > 1:
            s, i = sharding.all_gather_merge(s, i, top_n, self.group)
        return s, i

    def search_unique(self, query_vec: numpy.ndarray, top_n: int, index_hit_top_n: int):
        """The ``maxP->bert_dot`` aggregation (dense_retrieval.py:414-427): search ``index_hit_top_n`` vector hits and
        keep the ``top_n`` best distinct ids, each at its best hit's score -- on the device, after the cross-rank merge,
        so a passage whose vectors straddle two ranks is still counted once.  Missing results are
        (-3.4028235e38, -1)."""
        if self.passages is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        if query_vec.ndim == 1:
            query_vec = query_vec[numpy.newaxis, :]
        q = torch.from_numpy(numpy.ascontiguousarray(query_vec)).to(
            self.device, dtype=torch.float16 if self.store_dtype == torch.float16 else torch.float32)
        s, i = self.search_device(q, index_hit_top_n)
        s, i = interaction.topk_unique(s, i, top_n)
        return s.cpu().numpy(), i.cpu().numpy()

    def save(self, path: str):
        """dense_retrieval.py calls indexer.save(run_folder/faiss.index) after index().  One file per rank
        (`<path>.rank<r>of<w>` when the job has more than one rank -- every rank owns a different slab, so they must
        not write the same file), each recording its row range and the world size it was cut for."""
        rank, world = self._world()
        torch.save({"passages": self.passages.cpu(), "split_scale": self.split_scale, "ids": self.ids.cpu(), "n_total": self.n_total,
                    "lo": getattr(self, "lo", 0), "hi": getattr(self, "hi", self.n_total), "world": world, "rank": rank,
                    "token_dtype": str(self.store_dtype)}, self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        blob = self._load_shard(self._shard_path(path))
        lo, hi = sharding.shard_bounds(blob["n_total"], *self._world())
        self.passages, self.split_scale = blob["passages"].to(self.device), blob.get("split_scale")
        self.ids = blob["ids"].to(self.device)
        self.n_total, self.lo, self.hi = blob["n_total"], lo, hi
