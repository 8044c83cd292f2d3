"""Re-ranking with TK and TK-Sparse over a document store that was encoded once.

TK's document contextualisation (positions, the transformer, the mixer) does not depend on the query
(ecai20_tk.py:87-124), and it is nearly all of TK's inference cost.  ``ECAI20_TK.encode_documents`` /
``CIKM20_TK_Sparse.encode_documents`` run it once per passage; the rows go into the reference's encode folder
(``token_reps_N.npy`` + ``doc_infos.npz`` with ``token_dtype: float32``, through :class:`TKStoreWriter`), and
:class:`TKDocumentStore` keeps them in HBM and scores candidates with the store mode of the kernel-pooling kernels
(``interaction.kernel_pool_store``): the cosine -> RBF -> pooling stage only.

TK-Sparse's gate multiplies every kernel activation of its term, so a term whose gate is 0 adds exactly 0 to every score:
such rows are not stored (a passage whose terms are all gated 0 keeps one, so that it scores as in ``forward``).  The
gates of the stored rows go into a parallel file per block, ``gate_reps_N.npy`` ([token_block_size] float32, written
and read like the token blocks).

Multi-GPU: one process per GPU, each rank owns a contiguous range of whole passages (``sharding.passage_shard_bounds``),
scores the candidates it owns (-inf, id -1 for the others) and one ``sharding.all_gather_merge`` ranks them.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import numpy
import torch

from .. import _lib, interaction, sharding
from .base_index import GPUIndexer
from .colbert_e2e import doc_offsets_from_id_mapping
from .token_storage import TokenStorageWriter

GATE_FILE = "gate_reps_{}.npy"


class TKStoreWriter(TokenStorageWriter):
    """:class:`TokenStorageWriter` (float32 rows) plus, with ``gated=True``, one gate value per stored row in
    ``gate_reps_N.npy`` beside ``token_reps_N.npy``.  Without gates the folder is exactly the writer's."""

    def __init__(self, folder: str, token_dim: int, token_block_size: int, gated: bool = False):
        self.gated = gated
        self.gates: List[numpy.memmap] = []
        super().__init__(folder, token_dim, token_block_size, "float32")

    def _new_block(self):
        super()._new_block()
        if self.gated:
            path = os.path.join(self.folder, GATE_FILE.format(len(self.gates)))
            self.gates.append(numpy.memmap(path, dtype=numpy.float32, mode="w+", shape=(self.block_size,)))

    def add(self, seq_id: str, vectors: numpy.ndarray, gate: Optional[numpy.ndarray] = None):
        """vectors [n_rows, dim] and, for a gated store, gate [n_rows]; all-zero rows are dropped with their gate."""
        v = numpy.asarray(vectors, dtype=numpy.float32).reshape(-1, self.dim)
        if self.gated != (gate is not None):
            raise _lib.MatchmakerB200Error("TKStoreWriter.add: a gate for every passage of a gated store, none otherwise")
        super().add(seq_id, v)
        if self.gated:
            g = numpy.asarray(gate, dtype=numpy.float32).reshape(-1)
            if len(g) != len(v):
                raise _lib.MatchmakerB200Error("TKStoreWriter.add: one gate value per row")
            b, lo, hi = self.doc_infos[seq_id]
            self.gates[b][lo:hi] = g[numpy.abs(v).sum(-1) > 0]

    def close(self):
        for g in self.gates:
            g.flush()
        super().close()


def load_gates(folder: str, token_block_size: int, storage: List[numpy.ndarray]) -> List[numpy.ndarray]:
    """The gate blocks of a gated encode folder, cut like ``storage`` (the blocks of ``load_token_storage``)."""
    out = []
    for f, blk in enumerate(storage):
        path = os.path.join(folder, GATE_FILE.format(f))
        if not os.path.isfile(path):
            raise _lib.MatchmakerB200Error(f"{folder}: no {GATE_FILE.format(f)}; the store was written without gates")
        out.append(numpy.memmap(path, dtype=numpy.float32, mode="r", shape=(token_block_size,))[:len(blk)])
    return out


def local_pairs(candidates: torch.Tensor, d_lo: int, d_hi: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(pair_d, ids) of candidates [Nq, C] (store positions, -1 = none) on the rank owning passages [d_lo, d_hi):
    pair_d is the local passage or -1, ids the position or -1 where this rank does not own the candidate."""
    mine = (candidates >= d_lo) & (candidates < d_hi)
    return (torch.where(mine, candidates - d_lo, -1).to(torch.int32).reshape(-1),
            torch.where(mine, candidates, -1).to(torch.int64))


def merge(scores: torch.Tensor, ids: torch.Tensor, k: int, group=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The top k of every row of this rank's scores [Nq, C] under (score desc, id asc), merged across ranks; missing
    entries are (-inf, -1)."""
    if scores.is_cuda:
        s, i = interaction.topk_merge(scores, ids, k)
    else:   # the gloo tests of the merge run on the CPU
        s, i = sharding.rank_topk(scores, ids, k)
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        s, i = sharding.all_gather_merge(s, i, k, group)
    # topk_merge fills missing results as faiss does, (-FLT_MAX, -1); a re-ranked candidate list reports them with the
    # score of a candidate that is not there, -inf
    return s.masked_fill(i < 0, float("-inf")), i


class TKDocumentStore(GPUIndexer):
    """The rows ``encode_documents`` of ``model`` (an ``ECAI20_TK`` or ``CIKM20_TK_Sparse``) made for every passage,
    HBM-resident in fp32 (config ``token_dtype: "float32"``, ``token_dim`` = the model's width), and ``rerank`` over them.
    Passage ids are positions in the encode folder's ``seq_ids``."""

    def __init__(self, config, model, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        if self.store_dtype != torch.float32:
            raise _lib.MatchmakerB200Error("TKDocumentStore keeps fp32 rows (token_dtype: float32): the cosine needs "
                                           "fp32 inputs")
        self.model = model
        self.gated = hasattr(model, "stop_word_reducer")   # CIKM20_TK_Sparse
        self.rows: Optional[torch.Tensor] = None      # [rows of this rank, D] fp32
        self.gate: Optional[torch.Tensor] = None      # [rows of this rank] fp32 (TK-Sparse)
        self.offsets: Optional[torch.Tensor] = None   # [passages of this rank + 1] int64, local row offsets
        self.doc_offsets: Optional[numpy.ndarray] = None   # [n_docs + 1] int64 of the whole store
        self.max_doc_len = 1
        self.d_lo = self.d_hi = 0

    def index(self, id_mapping: List[numpy.ndarray], storage: List[numpy.ndarray],
              gates: Optional[List[numpy.ndarray]] = None):
        """id_mapping, storage: the first two results of ``token_storage.load_token_storage``; gates (TK-Sparse): the
        result of :func:`load_gates`.  Every rank is given the same lists and keeps its passage range."""
        from .token_storage import blocks_to_device
        if len(id_mapping) != len(storage) or any(len(a) != len(b) for a, b in zip(id_mapping, storage)):
            raise _lib.MatchmakerB200Error("id_mapping and storage must have one entry per stored row, block by block")
        if not storage or storage[0].shape[1] != self.token_dim or storage[0].dtype != numpy.float32:
            raise _lib.MatchmakerB200Error(f"storage must be float32 rows of token_dim {self.token_dim}")
        if self.gated != (gates is not None):
            raise _lib.MatchmakerB200Error("TK-Sparse stores need their gates (load_gates); TK stores have none")
        if gates is not None and [len(g) for g in gates] != [len(b) for b in storage]:
            raise _lib.MatchmakerB200Error("gates must hold one value per stored row, block by block")
        off = doc_offsets_from_id_mapping(id_mapping)
        rank, world = self._world()
        d_lo, d_hi, r_lo, r_hi = sharding.passage_shard_bounds(off, rank, world)
        with torch.cuda.device(self.device):
            rows = blocks_to_device(storage, r_lo, r_hi, self.device)
        gate = None
        if gates is not None:
            gate = torch.from_numpy(numpy.concatenate([numpy.asarray(g) for g in gates])[r_lo:r_hi]).to(self.device)
        self._set(off, d_lo, d_hi, rows, gate)

    def _set(self, off: numpy.ndarray, d_lo: int, d_hi: int, rows: torch.Tensor, gate: Optional[torch.Tensor]):
        local = off[d_lo:d_hi + 1] - off[d_lo]
        self.doc_offsets = off
        self.d_lo, self.d_hi = d_lo, d_hi
        self.rows, self.gate = rows.to(self.device, torch.float32).contiguous(), None if gate is None else gate.to(self.device)
        self.offsets = torch.from_numpy(numpy.ascontiguousarray(local)).to(self.device)
        self.max_doc_len = max(1, int(numpy.diff(local).max())) if len(local) > 1 else 1

    @torch.no_grad()
    def rerank(self, query_ctx: torch.Tensor, query_mask: torch.Tensor, candidates: torch.Tensor,
               top_n: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """query_ctx [Nq, Lq, D]: the contextualised queries (the model's ``forward_representation`` with
        ``positional_features_q``), query_mask [Nq, Lq]; candidates [Nq, C] store positions, -1 = none.  Returns
        (scores [Nq, k], ids [Nq, k]) with k = min(top_n, C), sorted by (score desc, id asc); missing entries are
        (-inf, -1).  Enqueued without a host synchronisation."""
        if self.rows is None:
            raise _lib.MatchmakerB200Error("rerank() before index()")
        nq, c = candidates.shape
        k = c if top_n is None else min(int(top_n), c)
        cand = candidates.to(self.device, torch.int64)
        pair_d, ids = local_pairs(cand, self.d_lo, self.d_hi)
        pair_q = torch.arange(nq, device=self.device, dtype=torch.int32).repeat_interleave(c)
        if self.rows.shape[0] == 0:   # a rank without passages owns no candidate
            scores = torch.full((nq, c), float("-inf"), device=self.device)
        else:
            extra = {"gate": self.gate} if self.gated else {}
            scores = self.model.score_store(query_ctx.to(self.device), query_mask.to(self.device), self.rows,
                                            self.offsets, pair_q, pair_d, max_doc_len=self.max_doc_len,
                                            **extra).view(nq, c)
        return merge(scores, ids, k, self.group)

    def save(self, path: str):
        """One file per rank (``<path>.rank<r>of<w>`` with more than one rank): this rank's rows (and gates), its
        passage range and the store's passage offsets."""
        if self.rows is None:
            raise _lib.MatchmakerB200Error("save() before index()")
        rank, world = self._world()
        torch.save({"rows": self.rows.cpu(), "gate": None if self.gate is None else self.gate.cpu(),
                    "doc_offsets": torch.from_numpy(self.doc_offsets), "d_lo": self.d_lo, "d_hi": self.d_hi,
                    "token_dtype": str(self.store_dtype), "world": world, "rank": rank}, self._shard_path(path))

    def load(self, path: str):
        """Restore this rank's share; refused unless the file was written by this rank of a job of this world size for
        the passage range this rank owns, and with gates exactly for a TK-Sparse model."""
        blob = self._load_shard(self._shard_path(path), row_range=False)
        off = blob["doc_offsets"].numpy()
        rank, world = self._world()
        d_lo, d_hi, _, _ = sharding.passage_shard_bounds(off, rank, world)
        if (blob["d_lo"], blob["d_hi"]) != (d_lo, d_hi):
            raise _lib.MatchmakerB200Error(f"store file holds passages [{blob['d_lo']},{blob['d_hi']}), this rank owns "
                                           f"[{d_lo},{d_hi}) -- re-index or load with the same world size")
        if (blob["gate"] is not None) != self.gated:
            raise _lib.MatchmakerB200Error("store file gates do not match the model (TK-Sparse stores carry gates)")
        self._set(off, d_lo, d_hi, blob["rows"], blob["gate"])
