"""Graph index for approximate maximum-inner-product search on the H100 kernels.

Drop-in for ``FaissHNSWIndexer`` (matchmaker/retrieval/faiss_indices.py:76-104), selected by
``faiss_index_type: "hnsw"`` in dense_retrieval.py: same config keys (``token_dim``, ``token_dtype``,
``faiss_hnsw_graph_neighbors`` = M, ``faiss_hnsw_efConstruction``, ``faiss_hnsw_efSearch``), same methods, numpy in /
numpy out.  ``faiss_use_gpu`` is ignored: the reference's HNSW always runs on the CPU (its example config sets it to
False), and this index always runs on the GPU.

The graph is not faiss's multi-layer HNSW but one flat graph after CAGRA (Ootomo et al., ICDE 2024):
- build: the exact k-NN graph (flat_ip_topk, K = max(2M, efConstruction)), rank-based detour pruning to R = 2M edges
  per node (interaction.graph_prune), then reverse edges merged in;
- search: an exact scan of a seeded sample of rows picks each query's starting list, then a beam search with list size
  L = max(efSearch, top_n) rounded up to 32 (interaction.graph_search, one CTA per query).

Storage: fp16 rows (queries rounded to fp16), or fp32 rows read directly by the search kernel (the fp16 hi / lo split
exists only for the k-NN stage and the entry sample).  Graph edges are int32 row positions within the shard; user ids
stay int64.  Multi-GPU: each rank builds a graph over its shard_bounds rows, and the per-rank top-k lists are merged
with one all-gather (faiss IndexShards semantics).
"""
from __future__ import annotations

from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction, sharding
from .base_index import GPUIndexer

GRAPH_SEED = 1234
KNN_WORKSPACE_CAP = 2 << 30   # device scratch of one k-NN batch of flat_ip_topk
_NO_RESULT = -3.4028234663852886e38


def graph_degrees(M: int, ef_construction: int):
    """(R, K): out-degree 2M (faiss's level-0 degree) and k-NN degree max(R, efConstruction), within the kernels'
    limits R <= 1024, K <= 1023."""
    R = 2 * int(M)
    K = max(R, int(ef_construction))
    if not 1 <= R <= interaction.GRAPH_MAX_DEGREE:
        raise _lib.MatchmakerB200Error(f"faiss_hnsw_graph_neighbors = {M} gives out-degree 2M = {R}; the graph index "
                                       f"needs 1 <= 2M <= {interaction.GRAPH_MAX_DEGREE}")
    if K > interaction.GRAPH_MAX_KNN:
        key = "faiss_hnsw_efConstruction" if int(ef_construction) > R else "faiss_hnsw_graph_neighbors"
        raise _lib.MatchmakerB200Error(f"{key}: the k-NN degree max(2M, efConstruction) = {K} is above the limit "
                                       f"{interaction.GRAPH_MAX_KNN}")
    return R, K


def search_list_size(ef_search: int, top_n: int) -> int:
    """L = max(efSearch, top_n) rounded up to 32, at most 1024."""
    L = (max(int(ef_search), int(top_n), 1) + 31) // 32 * 32
    if L > interaction.GRAPH_MAX_LIST:
        key = "faiss_hnsw_efSearch" if int(ef_search) >= int(top_n) else "top_n"
        raise _lib.MatchmakerB200Error(f"{key}: the search list size max(efSearch, top_n) rounded up to 32 = {L} is "
                                       f"above the limit {interaction.GRAPH_MAX_LIST}")
    return L


def entry_positions(n: int) -> numpy.ndarray:
    """E = min(n, max(1024, n // 128)) row positions from a seeded permutation: every query's starting list is picked
    among them by an exact scan (the job of HNSW's upper layers)."""
    e = min(n, max(1024, n // 128))
    return numpy.random.RandomState(GRAPH_SEED).permutation(n)[:e].astype(numpy.int64)


def knn_graph(rows: torch.Tensor, K: int, cap: int = KNN_WORKSPACE_CAP) -> torch.Tensor:
    """Exact k-NN graph [n, K] int32 of rows [n, dim] (fp16, or fp32 searched through the fp16 hi / lo split): each
    row's K best other rows under (score desc, position asc), -1 where the shard has fewer.  flat_ip_topk(rows, rows,
    K + 1) runs in row batches whose scratch fits `cap`; a row is dropped from its own list wherever it lands (with
    duplicate rows it need not come first)."""
    n = rows.shape[0]
    out = torch.empty((n, K), dtype=torch.int32, device=rows.device)
    if n == 0:
        return out
    if rows.dtype == torch.float16:
        store, scale = rows, None
    else:
        store, scale = interaction.flat_ip_split_f32(rows.float(), "passages")
    lib = _lib.load()
    with torch.cuda.device(rows.device):
        b = interaction.ivf_query_batch(n, lambda nb: lib.mmb200_flat_ip_workspace_bytes(nb, n, K + 1), cap)
    for b0 in range(0, n, b):
        b1 = min(n, b0 + b)
        _, nb = interaction.flat_ip_topk(rows[b0:b1], store, K + 1, split_scale=scale)
        nb = nb.to(torch.int32)
        own = nb == torch.arange(b0, b1, dtype=torch.int32, device=rows.device).unsqueeze(1)
        keep = torch.sort(own.to(torch.int8), dim=1, stable=True).indices[:, :K]   # the other rows, in rank order
        out[b0:b1] = torch.gather(nb, 1, keep)
    return out


def reverse_merge(pruned: torch.Tensor) -> torch.Tensor:
    """Final lists [n, R] int32 from the pruned lists: the first ceil(R/2) pruned edges of u; then every w with u among
    the first ceil(R/2) pruned edges of w, ordered by (that rank, w); then the rest of u's pruned list; duplicates
    skipped, cut at R, -1 padded.  Stable sorts on the device."""
    n, R = pruned.shape
    dev = pruned.device
    if n == 0:
        return pruned.clone()
    H = (R + 1) // 2
    P = pruned.to(torch.int64)
    u = torch.arange(n, device=dev).unsqueeze(1).expand(n, R)
    r = torch.arange(R, device=dev).unsqueeze(0).expand(n, R)
    head, tail = (r < H) & (P >= 0), (r >= H) & (P >= 0)
    # reverse edges, flattened in (w, r) order, then stably sorted to (u, r, w)
    rv_u, rv_w, rv_r = P[head], u[head], r[head]
    o = torch.sort(rv_r, stable=True).indices
    o = o[torch.sort(rv_u[o], stable=True).indices]
    rv_u, rv_w = rv_u[o], rv_w[o]
    starts = torch.cumsum(torch.bincount(rv_u, minlength=n), 0) - torch.bincount(rv_u, minlength=n)
    rv_order = H + torch.arange(rv_u.numel(), device=dev) - starts[rv_u]
    cu = torch.cat([u[head], rv_u, u[tail]])
    cv = torch.cat([P[head], rv_w, P[tail]])
    co = torch.cat([r[head], rv_order, H + n + r[tail]])
    # keep each (u, v) once, at its first place
    o = torch.sort(co, stable=True).indices
    cu, cv, co = cu[o], cv[o], co[o]
    o = torch.sort(cu * n + cv, stable=True).indices
    cu, cv, co = cu[o], cv[o], co[o]
    first = torch.ones_like(cu, dtype=torch.bool)
    first[1:] = (cu[1:] != cu[:-1]) | (cv[1:] != cv[:-1])
    cu, cv, co = cu[first], cv[first], co[first]
    # order each node's list by place and cut at R
    o = torch.sort(co, stable=True).indices
    cu, cv = cu[o], cv[o]
    o = torch.sort(cu, stable=True).indices
    cu, cv = cu[o], cv[o]
    counts = torch.bincount(cu, minlength=n)
    pos = torch.arange(cu.numel(), device=dev) - (torch.cumsum(counts, 0) - counts)[cu]
    keep = pos < R
    out = torch.full((n, R), -1, dtype=torch.int32, device=dev)
    out[cu[keep], pos[keep]] = cv[keep].to(torch.int32)
    return out


class GraphIndexer(GPUIndexer):
    """faiss_index_type "hnsw" on the GPU.  ``faiss_use_gpu`` is read and ignored (see the module docstring)."""
    gpu_only = False

    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.M = int(config["faiss_hnsw_graph_neighbors"])
        self.ef_construction = int(config["faiss_hnsw_efConstruction"])
        self.ef_search = int(config["faiss_hnsw_efSearch"])
        self.R, self.K = graph_degrees(self.M, self.ef_construction)
        search_list_size(self.ef_search, 1)
        self.rows: Optional[torch.Tensor] = None         # [n_local, dim] fp16 / fp32
        self.ids: Optional[torch.Tensor] = None          # [n_local] int64
        self.graph: Optional[torch.Tensor] = None        # [n_local, R] int32 row positions, -1 padded
        self.entry_pos: Optional[torch.Tensor] = None    # [E] int64 row positions
        self.entry_store, self.entry_scale = None, None  # the entry rows as flat_ip_topk reads them
        self.n_total = 0

    def prepare(self, data_chunks: List[numpy.ndarray], subsample=-1):
        """Nothing to train (the reference's prepare only trains faiss's fp16 scalar quantizer)."""

    def index(self, ids: List[numpy.ndarray], data_chunks: List[numpy.ndarray]):
        """ids: list of int64 arrays; data_chunks: list of [n_i, token_dim] arrays.  Every rank is given the same lists
        and builds the graph over its rows shard_bounds(n, rank, world)."""
        from .token_storage import blocks_to_device
        rank, world = self._world()
        n = int(sum(len(x) for x in ids))
        lo, hi = sharding.shard_bounds(n, rank, world)
        self.n_total, self.lo, self.hi = n, lo, hi
        if hi > lo:
            with torch.cuda.device(self.device):
                vecs = blocks_to_device(data_chunks, lo, hi, self.device)
            id_parts, off = [], 0
            for i_arr in ids:
                a, b = max(lo, off), min(hi, off + len(i_arr))
                if a < b:
                    id_parts.append(torch.from_numpy(numpy.ascontiguousarray(i_arr[a - off:b - off]).astype(numpy.int64)))
                off += len(i_arr)
            self.build(vecs, torch.cat(id_parts).to(self.device))
        else:
            self.build(torch.empty((0, self.token_dim), device=self.device),
                       torch.empty(0, dtype=torch.int64, device=self.device))

    def build(self, vecs: torch.Tensor, ids: torch.Tensor):
        """Replace the index content by a graph over `vecs` [n, dim] with user ids `ids` [n]."""
        self.rows = vecs.to(self.device, self.store_dtype).contiguous()
        self.ids = ids.to(self.device, torch.int64).contiguous()
        knn = knn_graph(self.rows, self.K)
        pruned = interaction.graph_prune(knn, self.R) if self.rows.shape[0] else knn.new_empty((0, self.R))
        self.graph = reverse_merge(pruned)
        self._set_entries(torch.from_numpy(entry_positions(self.rows.shape[0])).to(self.device))

    def _set_entries(self, pos: torch.Tensor):
        self.entry_pos = pos
        if self.store_dtype == torch.float16:
            self.entry_store, self.entry_scale = self.rows[pos].contiguous(), None
        elif pos.numel():
            self.entry_store, self.entry_scale = interaction.flat_ip_split_f32(self.rows[pos], "passages")

    # ------------------------------------------------------------------ search
    def _to_device_queries(self, query_vec: numpy.ndarray) -> torch.Tensor:
        if self.rows is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        if query_vec.ndim == 1:
            query_vec = query_vec[numpy.newaxis, :]
        return torch.from_numpy(numpy.ascontiguousarray(query_vec)).to(self.device, dtype=self.store_dtype)

    def search(self, query_vec: numpy.ndarray, top_n: int):
        s, i = self.search_device(self._to_device_queries(query_vec), top_n)
        return s.cpu().numpy(), i.cpu().numpy()

    def entries(self, q: torch.Tensor, L: int) -> torch.Tensor:
        """The min(L, E) entry rows of best score for every query: [nq, min(L, E)] int64 row positions."""
        m = min(L, self.entry_pos.numel())
        return interaction.flat_ip_topk(q, self.entry_store, m, ids=self.entry_pos, split_scale=self.entry_scale)[1]

    def search_device(self, q: torch.Tensor, top_n: int):
        """Same as search() but device tensors in/out.  No host synchronisation with fp16 storage (fp32 storage reads the
        query scale when the entry scan splits the queries).  Returns the ids given to index()."""
        rank, world = self._world()
        if top_n > interaction.FLAT_IP_MAX_K:
            raise _lib.MatchmakerB200Error(f"top_n > {interaction.FLAT_IP_MAX_K} is not supported by the graph index")
        L = search_list_size(self.ef_search, top_n)
        if self.rows.shape[0] > 0:
            s, i = interaction.graph_search(q, self.rows, self.ids, self.graph, self.entries(q, L), top_n, L)
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
        was cut for, the graph and the entry sample."""
        rank, world = self._world()
        torch.save({"rows": self.rows.cpu(), "ids": self.ids.cpu(), "graph": self.graph.cpu(),
                    "entry_pos": self.entry_pos.cpu(), "n_total": self.n_total, "lo": getattr(self, "lo", 0),
                    "hi": getattr(self, "hi", self.n_total), "world": world, "rank": rank,
                    "token_dtype": str(self.store_dtype), "M": self.M, "ef_construction": self.ef_construction,
                    "ef_search": self.ef_search}, self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        """efSearch comes from config_overwrites["faiss_hnsw_efSearch"] when given, else from the file."""
        blob = self._load_shard(self._shard_path(path))
        lo, hi = sharding.shard_bounds(blob["n_total"], *self._world())
        self.M, self.ef_construction, self.ef_search = int(blob["M"]), int(blob["ef_construction"]), int(blob["ef_search"])
        if config_overwrites and "faiss_hnsw_efSearch" in config_overwrites:
            self.ef_search = int(config_overwrites["faiss_hnsw_efSearch"])
        self.R, self.K = graph_degrees(self.M, self.ef_construction)
        search_list_size(self.ef_search, 1)
        self.rows, self.ids = blob["rows"].to(self.device), blob["ids"].to(self.device)
        self.graph = blob["graph"].to(self.device)
        self._set_entries(blob["entry_pos"].to(self.device))
        self.n_total, self.lo, self.hi = blob["n_total"], lo, hi
