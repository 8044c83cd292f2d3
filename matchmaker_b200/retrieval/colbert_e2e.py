"""Exact (brute-force) ColBERT end-to-end retrieval over the encoded token store.

The ColBERT paper's two-stage search with exact token search in place of its approximate index:

1. candidate generation -- every live query token is searched against all token rows of the store (``flat_ip_topk``,
   the rows' passage ids as ids), keeping its ``token_top_k`` best rows; the candidate passages of a query are the
   union of those rows' passages (``topk_unique``);
2. exact scoring -- the query against each candidate with ``forward_aggregation`` semantics (colbert.py:100-112):
   sum over query tokens of the max over the passage's stored rows (``maxsim_store``, no padding in HBM);
3. ranking -- the ``top_n`` best per query under (score desc, id asc), merged across ranks.

Everything is enqueued on the current stream without a host synchronisation between the stages.  Candidate lists
have a static width ``C = min(Lq * token_top_k, 4096)`` with void entries.  Candidate cap: the candidate set is the
exact union of the token hits whenever ``Lq * token_top_k <= 4096``; beyond that, the 4096 distinct passages with the
highest single-token score (ties by passage id) are kept.

The store is what the reference's encode loop writes (``token_reps_N.npy`` + ``doc_infos.npz``, read by
``token_storage.load_token_storage``): each passage keeps only its real token rows (dense_retrieval.py:244), and the
``id_mapping`` value of a row is its passage's position in ``seq_ids`` -- which is also the id this index returns.
Multi-GPU: one process per GPU, each rank owns a contiguous range of whole passages (``sharding.passage_shard_bounds``)
and the per-rank top lists are merged with ``sharding.all_gather_merge``.

The token store's format (dense rows, E4M3 or residual codes) is ``colbert_store``'s: the indexer holds one store
and runs both stages through it.
"""
from __future__ import annotations

from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction, sharding
from . import colbert_store
from .base_index import GPUIndexer
from .colbert_store import fp8_store_scale  # noqa: F401  (public name of this module)

CANDIDATE_CAP = 4096          # candidate passages per query and rank (the topk_unique limit)
_VOID_SCORE = -3.4028234663852886e38


def doc_offsets_from_id_mapping(id_mapping: List[numpy.ndarray]) -> numpy.ndarray:
    """Row offsets [n_docs + 1] of the passages of a token store from its per-block ``id_mapping`` (row -> passage
    position in ``seq_ids``): passage d is rows [off[d], off[d+1]), n_docs = 1 + the largest position.  Passages whose
    rows were all stripped get an empty range.  Raises on a mapping that is not non-decreasing (the reference's writer
    appends passages in order, so anything else is malformed input)."""
    rows = numpy.concatenate([numpy.asarray(x, dtype=numpy.int64).reshape(-1) for x in id_mapping]) if id_mapping \
        else numpy.zeros(0, dtype=numpy.int64)
    if rows.size and (rows[0] < 0 or (numpy.diff(rows) < 0).any()):
        raise _lib.MatchmakerB200Error("id_mapping must be non-negative and non-decreasing over the concatenated blocks "
                                       "(rows of one passage are contiguous, passages in seq_ids order)")
    n_docs = int(rows[-1]) + 1 if rows.size else 0
    return numpy.searchsorted(rows, numpy.arange(n_docs + 1, dtype=numpy.int64), side="left").astype(numpy.int64)


def token_store_attribute(name: str, doc: str) -> property:
    """An attribute of the indexer's token store (``tokens``), read and set under the indexer's name."""
    return property(lambda self: getattr(self.tokens, name), lambda self, v: setattr(self.tokens, name, v), doc=doc)


class ColBERTEndToEndIndexer(GPUIndexer):
    residual = False   # the store keeps residual codes (ColBERTResidualIndexer)
    plaid_capable = False   # accepts the PLAID search keys (an IVF token index: ColBERTIVFIndexer)
    store = token_store_attribute("rows", "[rows of this rank, ...] the stored rows as the kernels read them")
    store_scale = token_store_attribute("scale", "s_d of an E4M3 store, else None")
    chunk_rows = token_store_attribute("slab_rows", "rows per slab of a streamed build")

    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        if not self.plaid_capable and any(config.get(k) is not None for k in
                                          ("colbert_plaid_ndocs", "colbert_plaid_centroid_score_threshold")):
            raise _lib.MatchmakerB200Error("PLAID search (colbert_plaid_*) needs the centroids of an IVF token index: "
                                           "ColBERTIVFIndexer or ColBERTResidualIndexer")
        self.tokens = colbert_store.select(config, self.token_dim, self.store_dtype, self.device, process_group,
                                           self.residual)
        self.row_ids: Optional[torch.Tensor] = None     # [rows] int64 passage id (seq_ids position) of every row
        self.offsets: Optional[torch.Tensor] = None     # [passages of this rank + 1] int64, local row offsets
        self.max_doc_len = 1
        self.d_lo = self.d_hi = 0
        self.n_docs = 0

    @property
    def fp8(self) -> bool:
        """The store holds E4M3 rows (``colbert_store_dtype: "float8_e4m3"``)."""
        return isinstance(self.tokens, colbert_store.E4M3TokenStore)

    def index(self, id_mapping: List[numpy.ndarray], storage: List[numpy.ndarray]):
        """id_mapping, storage: the first two results of ``token_storage.load_token_storage`` (per-block row -> passage
        position arrays, and the [rows, token_dim] blocks).  Every rank is given the same lists and keeps its passage
        range; its rows reach HBM through ``token_storage.blocks_to_device``."""
        from .token_storage import blocks_to_device
        if len(id_mapping) != len(storage) or any(len(a) != len(b) for a, b in zip(id_mapping, storage)):
            raise _lib.MatchmakerB200Error("id_mapping and storage must have one entry per stored row, block by block")
        if storage and storage[0].shape[1] != self.token_dim:
            raise _lib.MatchmakerB200Error(f"storage rows have dim {storage[0].shape[1]}, config token_dim is "
                                           f"{self.token_dim}")
        off = doc_offsets_from_id_mapping(id_mapping)
        rank, world = self._world()
        self.n_docs = len(off) - 1
        d_lo, d_hi, r_lo, r_hi = sharding.passage_shard_bounds(off, rank, world) if self.n_docs else (0, 0, 0, 0)

        def load(a, b):
            with torch.cuda.device(self.device):
                return blocks_to_device(storage, r_lo + a, r_lo + b, self.device)
        # every rank builds, with or without rows: the E4M3 store scale is an all-reduce
        self._build(load, r_hi - r_lo, off[d_lo:d_hi + 1] - r_lo, d_lo)

    def index_device(self, rows: torch.Tensor, doc_offsets: numpy.ndarray, first_doc: int = 0):
        """Index this rank's passages from a device tensor: rows [n_rows, token_dim]; passage first_doc + d is rows
        [doc_offsets[d], doc_offsets[d+1]) (int64 [n + 1], non-decreasing, from 0 to n_rows)."""
        off = numpy.asarray(doc_offsets, dtype=numpy.int64)
        if rows.dim() != 2 or rows.shape[1] != self.token_dim or off[0] != 0 or off[-1] != rows.shape[0] or \
                (numpy.diff(off) < 0).any():
            raise _lib.MatchmakerB200Error("index_device: rows [n_rows, token_dim] and non-decreasing offsets from 0")
        self._build(lambda a, b: rows[a:b].to(self.device), rows.shape[0], off, first_doc)

    def _build(self, load, n: int, off: numpy.ndarray, first_doc: int):
        """The store of this rank's n rows (``load(a, b)``: rows [a, b) on the device), and its passages: passage
        first_doc + d is rows [off[d], off[d+1])."""
        self.tokens.build(load, n)
        self._set_passages(off, first_doc)

    def _set_passages(self, off: numpy.ndarray, first_doc: int):
        lens = torch.from_numpy(numpy.diff(off)).to(self.device)
        self.offsets = torch.from_numpy(off).to(self.device)
        self.max_doc_len = max(1, int(numpy.diff(off).max())) if len(off) > 1 else 1
        self.row_ids = torch.repeat_interleave(torch.arange(first_doc, first_doc + len(off) - 1, device=self.device), lens)
        self.d_lo, self.d_hi = first_doc, first_doc + len(off) - 1

    def search(self, query_vec: numpy.ndarray, top_n: int, token_top_k: Optional[int] = None):
        """query_vec [Nq, Lq, dim] (the query_encode output of ColBERT.forward_representation: padded tokens are
        all-zero rows).  Returns (scores [Nq, top_n] f32, ids [Nq, top_n] i64): ids are positions in ``seq_ids``,
        missing results (-3.4028235e38, -1)."""
        if self.tokens.rows is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        q = torch.from_numpy(numpy.ascontiguousarray(query_vec))
        if q.dim() == 2:
            q = q.unsqueeze(0)
        scores, ids = self.search_device(q.to(self.device), top_n, token_top_k)
        return scores.cpu().numpy(), ids.cpu().numpy()

    def search_device(self, q: torch.Tensor, top_n: int, token_top_k: Optional[int] = None):
        """search() with device tensors in and out.  token_top_k (k') defaults to min(top_n, 1024)."""
        if self.tokens.rows is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        if q.dim() != 3 or q.shape[-1] != self.token_dim:
            raise _lib.MatchmakerB200Error(f"expected queries [Nq, Lq, {self.token_dim}], got {tuple(q.shape)}")
        kp = min(top_n, interaction.FLAT_IP_MAX_K) if token_top_k is None else int(token_top_k)
        if not 1 <= kp <= interaction.FLAT_IP_MAX_K:
            raise _lib.MatchmakerB200Error(f"token_top_k must be in [1, {interaction.FLAT_IP_MAX_K}], got {kp}")
        if not 1 <= top_n <= CANDIDATE_CAP:
            raise _lib.MatchmakerB200Error(f"top_n must be in [1, {CANDIDATE_CAP}], got {top_n}")
        rank, world = self._world()
        nq, lq, dim = q.shape
        q = q.to(self.device, self.store_dtype).contiguous()
        if self.tokens.rows.shape[0] == 0:
            s = torch.full((nq, top_n), _VOID_SCORE, device=self.device)
            i = torch.full((nq, top_n), -1, dtype=torch.int64, device=self.device)
        else:
            s, i = self._search_local(q, top_n, kp)
        if world > 1:
            s, i = sharding.all_gather_merge(s, i, top_n, self.group)
        return s, i

    def candidates_device(self, q: torch.Tensor, kp: int, qs: Optional[torch.Tensor] = None):
        """Stage 1 on this rank: (best single-token score, passage id) [Nq, C] of every candidate passage, best first;
        void entries are (-3.4028235e38, -1).  q [Nq, Lq, dim] in the store dtype on the device; qs what the scan
        reads (``tokens.queries(q)[0]``, computed here when not given).  With an E4M3 store the scores are in the
        scaled domain of each query."""
        nq, lq, dim = q.shape
        toks = q.reshape(nq * lq, dim)
        stoks = (self.tokens.queries(q)[0] if qs is None else qs).reshape(nq * lq, dim)
        hs, hi = self._scan(toks, stoks, kp)
        c = min(lq * kp, CANDIDATE_CAP)
        return interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c)

    def _scan(self, toks, stoks, kp: int):
        """The kp best (score, passage id) of every query token (toks as given, stoks as the store reads them):
        token hits -> passage ids; all-zero query rows are padding and their hits are voided."""
        hs, hi = self.tokens.scan(stoks, kp, self.row_ids)
        pad = (toks == 0).all(dim=1, keepdim=True)
        return hs.masked_fill(pad, float("-inf")), hi

    def _search_local(self, q: torch.Tensor, top_n: int, kp: int):
        nq = q.shape[0]
        qs, sq = self.tokens.queries(q)
        _, cand = self.candidates_device(q, kp, qs)
        c = cand.shape[1]
        # stage 2: exact max-sim of every candidate; void candidates (id -1) are skipped and score -inf
        pair_d = torch.where(cand >= 0, cand - self.d_lo, torch.full_like(cand, -1))
        pair_q = torch.arange(nq, device=self.device, dtype=torch.int32).repeat_interleave(c)
        scores = self.tokens.maxsim(qs, self.offsets, pair_q, pair_d, self.max_doc_len).view(nq, c)
        s, i = interaction.topk_merge(scores, cand, top_n)
        return self.tokens.unscale(s, sq), i
