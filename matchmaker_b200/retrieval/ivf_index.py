"""Inverted-file (IVF) maximum-inner-product index on the H100 kernels.

Drop-in for ``FaissIVFIndexer`` (matchmaker/retrieval/faiss_indices.py:106-145), selected by
``faiss_index_type: "ivf"`` in dense_retrieval.py: same config keys (``token_dim``, ``faiss_use_gpu``, ``token_dtype``,
``faiss_ivf_list_count`` = nlist, ``faiss_ivf_search_probe_count`` = nprobe), same methods, numpy in / numpy out.

- Coarse quantizer: ``nlist`` unit-norm centroids, trained by spherical k-means (``prepare``).  fp16 storage keeps fp16
  centroids and fp16 lists (faiss IndexIVFScalarQuantizer QT_fp16); fp32 storage keeps both as the fp16 hi / lo split
  (IndexIVFFlat over IndexFlatIP).
- Lists: the rows sorted by their argmax-inner-product centroid (ties to the lowest list id), with their int64 ids.
- Search: the ``nprobe`` best centroids per query (flat_ip_topk), then the exact top-k over the union of the probed
  lists (interaction.ivf_search), merged across ranks.

Multi-GPU: every rank is given the same chunks; training runs on rank 0 and the centroids are broadcast, so all ranks
probe the same lists; each rank lists its shard_bounds rows, and the per-rank top-k lists are merged with one
all-gather.
"""
from __future__ import annotations

from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction, sharding
from .base_index import GPUIndexer

KMEANS_ITERATIONS = 10
KMEANS_MAX_POINTS_PER_LIST = 256     # training uses at most this many points per list (a seeded subsample)
KMEANS_SEED = 1234
_SPLIT_EPS = 1.0 / 1024.0            # relative perturbation when an empty list takes half of a populated one
_NO_RESULT = -3.4028234663852886e38


class IVFIndexer(GPUIndexer):
    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.nlist = int(config["faiss_ivf_list_count"])
        self.nprobe = int(config["faiss_ivf_search_probe_count"])
        if self.nlist < 1 or self.nprobe < 1:
            raise _lib.MatchmakerB200Error("faiss_ivf_list_count and faiss_ivf_search_probe_count must be >= 1")
        self.centroids: Optional[torch.Tensor] = None    # [nlist, dim] f32, unit rows
        self.rows: Optional[torch.Tensor] = None         # [n_local, dim] fp16 or [n_local, 2*dim] split, sorted by list
        self.split_scale = None
        self.ids: Optional[torch.Tensor] = None          # [n_local] int64, in list order
        self.list_offsets: Optional[torch.Tensor] = None  # [nlist + 1] int64
        self.max_list_len = 0
        self.n_total = 0
        self.train_objective: List[float] = []           # sum of the assigned inner products, per iteration
        self.train_splits: List[int] = []                # empty lists re-seeded after each iteration

    # ------------------------------------------------------------------ training
    def prepare(self, data_chunks: List[numpy.ndarray], subsample=-1):
        """Train the coarse quantizer on the vectors of `data_chunks` (`subsample` is ignored, as in the reference):
        rank 0 trains, every other rank receives its centroids."""
        rank, world = self._world()
        if rank == 0:
            cents = self.train(data_chunks)
        else:
            cents = torch.empty((self.nlist, self.token_dim), dtype=torch.float32, device=self.device)
        if world > 1:
            import torch.distributed as dist
            dist.broadcast(cents, 0, group=self.group)
        self.set_centroids(cents)

    def _training_points(self, data_chunks):
        """(points [n_train, dim] in the storage dtype, rows of the initial centroids): a seeded permutation picks both."""
        from .token_storage import blocks_to_device
        n = int(sum(len(c) for c in data_chunks))
        if n < self.nlist:
            raise _lib.MatchmakerB200Error(f"IVF training needs at least nlist = {self.nlist} points, got {n}")
        n_train = min(n, KMEANS_MAX_POINTS_PER_LIST * self.nlist)
        perm = numpy.random.RandomState(KMEANS_SEED).permutation(n)
        if n_train == n:
            with torch.cuda.device(self.device):
                x = blocks_to_device(data_chunks, 0, n, self.device)
            init = perm[:self.nlist]
        else:
            sel = numpy.sort(perm[:n_train])
            parts, off = [], 0
            for c in data_chunks:
                lo, hi = numpy.searchsorted(sel, [off, off + len(c)])
                if hi > lo:
                    parts.append(torch.from_numpy(numpy.ascontiguousarray(numpy.asarray(c)[sel[lo:hi] - off])))
                off += len(c)
            x = torch.cat(parts).to(self.device)
            init = numpy.searchsorted(sel, perm[:self.nlist])
        x = x.to(self.store_dtype)
        return x, torch.from_numpy(init.astype(numpy.int64)).to(self.device)

    def train(self, data_chunks, niter: int = KMEANS_ITERATIONS, init_centroids: Optional[torch.Tensor] = None):
        """Spherical k-means: `niter` rounds of (assign every point to its argmax-inner-product centroid, replace each
        centroid by the normalised mean of its points).  Deterministic: the same data gives bit-identical centroids."""
        x, init = self._training_points(data_chunks)
        return self.train_points(x, init, niter, init_centroids)

    def train_points(self, x: torch.Tensor, init: torch.Tensor, niter: int = KMEANS_ITERATIONS,
                     init_centroids: Optional[torch.Tensor] = None):
        """`train` on the points `_training_points` returned, for callers that use the sample again."""
        if init_centroids is None:
            c = torch.nn.functional.normalize(x[init].float(), dim=1)
        else:
            c = init_centroids.to(self.device, torch.float32)
        self.train_objective, self.train_splits = [], []
        rng = numpy.random.RandomState(KMEANS_SEED + 1)
        for _ in range(niter):
            c, _, score = self.kmeans_step(x, c)
            self.train_objective.append(float(score))
            c, n_split = self._split_empty(c, rng)
            self.train_splits.append(n_split)
        return c

    def kmeans_step(self, x: torch.Tensor, c: torch.Tensor):
        """One iteration: (new centroids, assignment, objective with the old centroids)."""
        store, scale = self._centroid_store(c)
        s, a = interaction.flat_ip_topk(x, store, 1, split_scale=scale)
        a = a[:, 0]
        perm, offsets = self._layout(a)
        self._counts = offsets[1:] - offsets[:-1]
        return interaction.ivf_list_means(x, perm, offsets), a, s.double().sum().item()

    def _layout(self, assign: torch.Tensor):
        """Stable sort of the rows by list id -> (row order, list_offsets [nlist + 1])."""
        perm = torch.sort(assign, stable=True).indices
        counts = torch.bincount(assign, minlength=self.nlist)
        offsets = torch.zeros(self.nlist + 1, dtype=torch.int64, device=assign.device)
        offsets[1:] = torch.cumsum(counts, 0)
        return perm, offsets

    def _split_empty(self, c: torch.Tensor, rng):
        """Re-seed every empty list by splitting a populated one, picked with probability proportional to (size - 1): the
        two get the same centroid with opposite +-eps perturbations, then both are normalised."""
        counts = self._counts.cpu().numpy().astype(numpy.int64)
        empty = numpy.nonzero(counts == 0)[0]
        if len(empty) == 0:
            return c, 0
        sign = torch.ones(c.shape[1], device=c.device)
        sign[0::2] = -1.0
        c = c.clone()
        for ci in empty:
            w = numpy.maximum(counts - 1, 0).astype(numpy.float64)   # one vectorised draw per empty list
            cj = int(rng.choice(self.nlist, p=w / w.sum()))
            base = c[cj].clone()
            c[ci] = base * (1.0 + _SPLIT_EPS * sign)
            c[cj] = base * (1.0 - _SPLIT_EPS * sign)
            counts[ci] = counts[cj] // 2
            counts[cj] -= counts[ci]
        return torch.nn.functional.normalize(c, dim=1), len(empty)

    def _centroid_store(self, c: torch.Tensor):
        if self.store_dtype == torch.float16:
            return c.to(torch.float16).contiguous(), None
        return interaction.flat_ip_split_f32(c, "passages")

    def set_centroids(self, cents: torch.Tensor):
        self.centroids = cents.to(self.device, torch.float32).contiguous()
        if self.centroids.shape != (self.nlist, self.token_dim):
            raise _lib.MatchmakerB200Error(f"centroids must be [{self.nlist}, {self.token_dim}], got "
                                           f"{tuple(self.centroids.shape)}")
        self.c_store, self.c_scale = self._centroid_store(self.centroids)

    # ------------------------------------------------------------------ adding
    def index(self, ids: List[numpy.ndarray], data_chunks: List[numpy.ndarray]):
        """ids: list of int64 arrays; data_chunks: list of [n_i, token_dim] arrays.  Every rank is given the same lists
        and keeps rows shard_bounds(n, rank, world), sorted into their lists."""
        from .token_storage import blocks_to_device
        if self.centroids is None:
            raise _lib.MatchmakerB200Error("index() before prepare(): the IVF index has no centroids")
        rank, world = self._world()
        n = int(sum(len(x) for x in ids))
        lo, hi = sharding.shard_bounds(n, rank, world)
        self.n_total, self.lo, self.hi = n, lo, hi
        if hi > lo:
            with torch.cuda.device(self.device):
                vecs = blocks_to_device(data_chunks, lo, hi, self.device).to(self.store_dtype)
            id_parts, off = [], 0
            for i_arr in ids:
                a, b = max(lo, off), min(hi, off + len(i_arr))
                if a < b:
                    id_parts.append(torch.from_numpy(numpy.ascontiguousarray(i_arr[a - off:b - off]).astype(numpy.int64)))
                off += len(i_arr)
            self.add_sorted(vecs, torch.cat(id_parts).to(self.device))
        else:
            self.add_sorted(torch.empty((0, self.token_dim), dtype=self.store_dtype, device=self.device),
                            torch.empty(0, dtype=torch.int64, device=self.device))

    def add_sorted(self, vecs: torch.Tensor, ids: torch.Tensor):
        """Assign `vecs` to their lists and store them in list order (replaces the index content)."""
        if vecs.shape[0] > 0:
            _, a = interaction.flat_ip_topk(vecs, self.c_store, 1, split_scale=self.c_scale)
            perm, offsets = self._layout(a[:, 0])
            vecs, ids = vecs[perm], ids[perm]
        else:
            offsets = torch.zeros(self.nlist + 1, dtype=torch.int64, device=self.device)
        self.list_offsets, self.ids = offsets, ids.contiguous()
        self.max_list_len = int((offsets[1:] - offsets[:-1]).max().item())
        if self.store_dtype == torch.float16:
            self.rows, self.split_scale = vecs.to(torch.float16).contiguous(), None
        else:
            self.rows, self.split_scale = interaction.flat_ip_split_f32(vecs.float(), "passages")

    # ------------------------------------------------------------------ search
    def _to_device_queries(self, query_vec: numpy.ndarray) -> torch.Tensor:
        if self.rows is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        if query_vec.ndim == 1:
            query_vec = query_vec[numpy.newaxis, :]
        return torch.from_numpy(numpy.ascontiguousarray(query_vec)).to(
            self.device, dtype=torch.float16 if self.store_dtype == torch.float16 else torch.float32)

    def search(self, query_vec: numpy.ndarray, top_n: int):
        s, i = self.search_device(self._to_device_queries(query_vec), top_n)
        return s.cpu().numpy(), i.cpu().numpy()

    def coarse(self, q: torch.Tensor) -> torch.Tensor:
        """The min(nprobe, nlist) lists every query probes: [nq, nprobe] int64, best centroid first."""
        return interaction.flat_ip_topk(q, self.c_store, min(self.nprobe, self.nlist), split_scale=self.c_scale)[1]

    def search_device(self, q: torch.Tensor, top_n: int):
        """Same as search() but device tensors in/out.  No host synchronisation with fp16 storage (fp32 storage reads
        the query scale when it splits the queries).  Returns the ids given to index()."""
        rank, world = self._world()
        if top_n > interaction.FLAT_IP_MAX_K:
            raise _lib.MatchmakerB200Error(f"top_n > {interaction.FLAT_IP_MAX_K} is not supported by the fused top-k kernel")
        if self.rows.shape[0] > 0:
            s, i = interaction.ivf_search(q, self.rows, self.ids, self.list_offsets, self.coarse(q), top_n,
                                          self.max_list_len, split_scale=self.split_scale)
        else:
            s = torch.full((q.shape[0], top_n), _NO_RESULT, device=self.device)
            i = torch.full((q.shape[0], top_n), -1, dtype=torch.int64, device=self.device)
        if world > 1:
            s, i = sharding.all_gather_merge(s, i, top_n, self.group)
        return s, i

    def search_unique(self, query_vec: numpy.ndarray, top_n: int, index_hit_top_n: int):
        """The ``maxP->bert_dot`` aggregation, as FlatIPIndexer.search_unique: ``index_hit_top_n`` hits, the ``top_n``
        best distinct ids at their best score."""
        s, i = self.search_device(self._to_device_queries(query_vec), index_hit_top_n)
        s, i = interaction.topk_unique(s, i, top_n)
        return s.cpu().numpy(), i.cpu().numpy()

    # ------------------------------------------------------------------ persistence
    def save(self, path: str):
        """One file per rank (`<path>.rank<r>of<w>` with more than one rank), holding its row range, the world size it
        was cut for and the centroids."""
        rank, world = self._world()
        torch.save({"centroids": self.centroids.cpu(), "rows": self.rows.cpu(), "split_scale": self.split_scale,
                    "ids": self.ids.cpu(), "list_offsets": self.list_offsets.cpu(), "max_list_len": self.max_list_len,
                    "n_total": self.n_total, "lo": getattr(self, "lo", 0), "hi": getattr(self, "hi", self.n_total),
                    "world": world, "rank": rank, "token_dtype": str(self.store_dtype), "nlist": self.nlist,
                    "nprobe": self.nprobe}, self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        """nprobe comes from config_overwrites["faiss_ivf_search_probe_count"] when given, else from the file."""
        blob = self._load_shard(self._shard_path(path))
        lo, hi = sharding.shard_bounds(blob["n_total"], *self._world())
        self.nlist = int(blob["nlist"])
        self.nprobe = int(blob["nprobe"])
        if config_overwrites and "faiss_ivf_search_probe_count" in config_overwrites:
            self.nprobe = int(config_overwrites["faiss_ivf_search_probe_count"])
        self.set_centroids(blob["centroids"])
        self.rows, self.split_scale = blob["rows"].to(self.device), blob["split_scale"]
        self.ids, self.list_offsets = blob["ids"].to(self.device), blob["list_offsets"].to(self.device)
        self.max_list_len = int(blob["max_list_len"])
        self.n_total, self.lo, self.hi = blob["n_total"], lo, hi
