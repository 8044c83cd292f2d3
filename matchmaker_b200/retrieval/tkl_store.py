"""Re-ranking with TKL over a document store that was encoded once.

TKL contextualises every packed 50-position chunk of a document alone, with the same positional features
(sigir20_tkl.py:142-175), so a chunk depends neither on the query nor on the rest of the batch, and the transformer
over ~28 chunks of an 1 100-token document is nearly all of TKL's inference cost.  ``TKL_sigir20.encode_documents`` runs
it once per passage; :class:`TKLStoreWriter` puts the packed chunks into the reference's encode folder
(``token_reps_N.npy`` + ``doc_infos.npz``, ``token_dtype: float32``), 40 consecutive rows per chunk, masked rows kept as
zeros (the reference writer's all-zero-row strip would shift positions, and TKL's windows are positional).  A sidecar per
block, ``tkl_chunks_N.npy``, holds one record per chunk: its 40 mask bytes and its slot within its passage.
:class:`TKLDocumentStore` keeps the chunks in HBM and scores candidates with the store mode of the TKL window-score
kernels (``interaction.tkl_store_window_scores``) and the top-3 window selection: the interaction stage only.

Every passage is scored with C = ``chunk_slots(model.max_length)`` chunk slots: a pair scores what ``forward`` gives its
document padded to ``max_doc_length`` (the hill selection depends on the window count W in corner cases).  A pair whose
passage has no packed chunk (an empty passage) scores -inf with id -1, like a candidate that is missing.

Multi-GPU: one process per GPU, each rank owns a contiguous range of whole passages (``sharding.passage_shard_bounds``),
scores the candidates it owns (-inf, id -1 for the others) and one ``sharding.all_gather_merge`` ranks them.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import numpy
import torch

from .. import _lib, sharding
from ..rankers.tkl import chunk_slots
from .base_index import GPUIndexer
from .colbert_e2e import doc_offsets_from_id_mapping
from .tk_store import local_pairs, merge
from .token_storage import TokenStorageWriter

CHUNK = 40
CHUNK_FILE = "tkl_chunks_{}.npy"
# one record per stored chunk: the mask byte of each of its 40 rows and its slot within its passage
CHUNK_RECORD = numpy.dtype([("mask", numpy.uint8, (CHUNK,)), ("slot", "<i4")])


def _check_block_size(token_block_size: int):
    if token_block_size % CHUNK != 0:
        raise _lib.MatchmakerB200Error(f"a TKL store needs token_block_size % {CHUNK} == 0 so that no chunk straddles a "
                                       f"block; got {token_block_size}")


class TKLStoreWriter(TokenStorageWriter):
    """The reference's encode folder (float32 rows) of TKL's packed chunks, plus a ``tkl_chunks_N.npy`` sidecar per
    block with each chunk's mask and slot.  A passage's chunks stay in one block, so a passage holds at most
    token_block_size / 40 chunks."""

    def __init__(self, folder: str, token_dim: int, token_block_size: int):
        _check_block_size(token_block_size)
        self.meta: List[numpy.memmap] = []
        super().__init__(folder, token_dim, token_block_size, "float32")

    def _new_block(self):
        super()._new_block()
        path = os.path.join(self.folder, CHUNK_FILE.format(len(self.meta)))
        self.meta.append(numpy.memmap(path, dtype=CHUNK_RECORD, mode="w+", shape=(self.block_size // CHUNK,)))

    def add(self, seq_id: str, chunks: numpy.ndarray, chunk_mask: numpy.ndarray, slots: numpy.ndarray):
        """One passage: chunks [n, 40, dim], chunk_mask [n, 40], slots [n] (strictly increasing), the passage's part of
        ``TKL_sigir20.encode_documents``; n = 0 for a passage without a packed chunk.  Masked rows are stored as zeros."""
        m = numpy.asarray(chunk_mask).reshape(-1, CHUNK) != 0
        v = numpy.asarray(chunks, dtype=numpy.float32).reshape(-1, CHUNK, self.dim)
        s = numpy.asarray(slots, dtype=numpy.int64).reshape(-1)
        if not len(v) == len(m) == len(s):
            raise _lib.MatchmakerB200Error("TKLStoreWriter.add: one mask row and one slot per chunk")
        if len(s) and (s[0] < 0 or (numpy.diff(s) <= 0).any()):
            raise _lib.MatchmakerB200Error("TKLStoreWriter.add: slots must be non-negative and strictly increasing")
        n = len(v) * CHUNK
        if n > self.block_size:
            raise _lib.MatchmakerB200Error(f"TKLStoreWriter.add: {len(v)} chunks do not fit a block of "
                                           f"{self.block_size} rows")
        if self.filled[-1] + n > self.block_size:
            self._new_block()
        b = len(self.storage) - 1
        lo = self.filled[b]
        self.storage[b][lo:lo + n] = (v * m[..., None]).reshape(n, self.dim)
        rec = self.meta[b][lo // CHUNK:(lo + n) // CHUNK]
        rec["mask"] = m
        rec["slot"] = s
        self.filled[b] = lo + n
        self.doc_infos[seq_id] = (b, lo, lo + n)
        self.id_mapping[b].extend([len(self.seq_ids)] * n)
        self.seq_ids.append(seq_id)

    def close(self):
        for m in self.meta:
            m.flush()
        super().close()


def load_chunk_meta(folder: str, token_block_size: int, storage: List[numpy.ndarray]) -> List[numpy.ndarray]:
    """The chunk records (``CHUNK_RECORD``) of a TKL encode folder, block by block, cut like ``storage`` (the blocks of
    ``load_token_storage``)."""
    _check_block_size(token_block_size)
    out = []
    for f, blk in enumerate(storage):
        path = os.path.join(folder, CHUNK_FILE.format(f))
        if not os.path.isfile(path):
            raise _lib.MatchmakerB200Error(f"{folder}: no {CHUNK_FILE.format(f)}; not a TKL store (TKLStoreWriter)")
        if len(blk) % CHUNK:
            raise _lib.MatchmakerB200Error(f"{folder}: block {f} holds {len(blk)} rows, not whole {CHUNK}-row chunks")
        out.append(numpy.memmap(path, dtype=CHUNK_RECORD, mode="r", shape=(token_block_size // CHUNK,))[:len(blk) // CHUNK])
    return out


def void_pairs(scores: torch.Tensor, ids: torch.Tensor, live: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(scores, ids) [Nq, C] of this rank with every pair that is not ``live`` -- a candidate this rank does not own, or
    a passage without a packed chunk -- set to (-inf, -1): ranked like a missing candidate."""
    return scores.masked_fill(~live, float("-inf")), ids.masked_fill(~live, -1)


class TKLDocumentStore(GPUIndexer):
    """The packed chunks ``encode_documents`` of ``model`` (a ``TKL_sigir20``) made for every passage, HBM-resident in fp32
    (config ``token_dtype: "float32"``, ``token_dim`` = the model's width), and ``rerank`` over them.  Passage ids are
    positions in the encode folder's ``seq_ids``."""

    def __init__(self, config, model, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        if self.store_dtype != torch.float32:
            raise _lib.MatchmakerB200Error("TKLDocumentStore keeps fp32 chunks (token_dtype: float32): the cosine needs "
                                           "fp32 inputs")
        self.model = model
        self.C = chunk_slots(int(model.max_length))   # chunk slots of a document padded to max_doc_length
        self.chunks: Optional[torch.Tensor] = None      # [chunks of this rank, 40, D] fp32
        self.chunk_mask: Optional[torch.Tensor] = None  # [chunks of this rank, 40] uint8
        self.slots: Optional[torch.Tensor] = None       # [chunks of this rank] int32, slot within the passage
        self.doc_slots: Optional[torch.Tensor] = None   # [passages of this rank, C] int32, local chunk index or -1
        self.live: Optional[torch.Tensor] = None        # [passages of this rank] bool: has a packed chunk
        self.doc_offsets: Optional[numpy.ndarray] = None   # [n_docs + 1] int64 row offsets of the whole store
        self.d_lo = self.d_hi = 0

    def index(self, id_mapping: List[numpy.ndarray], storage: List[numpy.ndarray], chunk_meta: List[numpy.ndarray]):
        """id_mapping, storage: the first two results of ``token_storage.load_token_storage``; chunk_meta: the result of
        :func:`load_chunk_meta`.  Every rank is given the same lists and keeps its passage range."""
        from .token_storage import blocks_to_device
        if len(id_mapping) != len(storage) or any(len(a) != len(b) for a, b in zip(id_mapping, storage)):
            raise _lib.MatchmakerB200Error("id_mapping and storage must have one entry per stored row, block by block")
        if not storage or storage[0].shape[1] != self.token_dim or storage[0].dtype != numpy.float32:
            raise _lib.MatchmakerB200Error(f"storage must be float32 rows of token_dim {self.token_dim}")
        if [len(m) * CHUNK for m in chunk_meta] != [len(b) for b in storage]:
            raise _lib.MatchmakerB200Error("chunk_meta must hold one record per 40 stored rows, block by block")
        off = doc_offsets_from_id_mapping(id_mapping)
        if (off % CHUNK).any():
            raise _lib.MatchmakerB200Error("every passage must be whole 40-row chunks (a TKLStoreWriter folder)")
        rank, world = self._world()
        d_lo, d_hi, r_lo, r_hi = sharding.passage_shard_bounds(off, rank, world)
        with torch.cuda.device(self.device):
            rows = blocks_to_device(storage, r_lo, r_hi, self.device)
        rec = numpy.concatenate([numpy.asarray(m) for m in chunk_meta])[r_lo // CHUNK:r_hi // CHUNK]
        self._set(off, d_lo, d_hi, rows.view(-1, CHUNK, self.token_dim), torch.from_numpy(rec["mask"].copy()),
                  torch.from_numpy(rec["slot"].copy()))

    def _set(self, off: numpy.ndarray, d_lo: int, d_hi: int, chunks: torch.Tensor, mask: torch.Tensor,
             slots: torch.Tensor):
        counts = numpy.diff(off[d_lo:d_hi + 1]) // CHUNK
        s = slots.numpy().astype(numpy.int64)
        doc = numpy.repeat(numpy.arange(len(counts)), counts)
        if len(s) and (s.min() < 0 or s.max() >= self.C or (numpy.diff(s)[doc[1:] == doc[:-1]] <= 0).any()):
            raise _lib.MatchmakerB200Error(f"chunk slots must be strictly increasing within a passage and below C = "
                                           f"{self.C}, the slots of max_doc_length {self.model.max_length}")
        self.doc_offsets = off
        self.d_lo, self.d_hi = d_lo, d_hi
        dev = self.device
        self.chunks = chunks.to(dev, torch.float32).contiguous()
        self.chunk_mask = mask.to(dev, torch.uint8).contiguous()
        self.slots = slots.to(dev, torch.int32)
        n_docs = d_hi - d_lo
        cnt = torch.from_numpy(counts).to(dev)
        self.live = cnt > 0
        # the [n_docs, C] slot table, built on the device: slot s of passage d holds its chunk's local index
        self.doc_slots = torch.full((max(n_docs, 1), self.C), -1, dtype=torch.int32, device=dev)
        if len(s):
            doc = torch.repeat_interleave(torch.arange(n_docs, device=dev), cnt)
            self.doc_slots[doc, self.slots.long()] = torch.arange(len(s), dtype=torch.int32, device=dev)

    @torch.no_grad()
    def rerank(self, query_ctx: torch.Tensor, query_mask: torch.Tensor, candidates: torch.Tensor,
               top_n: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """query_ctx [Nq, Lq, D]: the contextualised queries (the model's ``forward_representation`` with
        ``positional_features_q``, its first result), query_mask [Nq, Lq]; candidates [Nq, C] store positions, -1 =
        none.  Returns (scores [Nq, k], ids [Nq, k]) with k = min(top_n, C), sorted by (score desc, id asc); missing
        entries and passages without a packed chunk are (-inf, -1).  Enqueued without a host synchronisation."""
        if self.chunks is None:
            raise _lib.MatchmakerB200Error("rerank() before index()")
        nq, c = candidates.shape
        k = c if top_n is None else min(int(top_n), c)
        cand = candidates.to(self.device, torch.int64)
        pair_d, ids = local_pairs(cand, self.d_lo, self.d_hi)
        if self.chunks.shape[0] == 0:   # a rank without packed chunks owns no scorable candidate
            scores, ids = void_pairs(torch.full((nq, c), float("-inf"), device=self.device), ids,
                                     torch.zeros_like(ids, dtype=torch.bool))
        else:
            live = ((pair_d >= 0) & self.live[pair_d.clamp(min=0).long()]).view(nq, c)
            pair_q = torch.arange(nq, device=self.device, dtype=torch.int32).repeat_interleave(c)
            s = self.model.score_store(query_ctx.to(self.device), query_mask.to(self.device), self.chunks,
                                       self.chunk_mask, self.doc_slots, pair_q, torch.where(live.view(-1), pair_d, -1))
            scores, ids = void_pairs(s.view(nq, c), ids, live)
        return merge(scores, ids, k, self.group)

    def save(self, path: str):
        """One file per rank (``<path>.rank<r>of<w>`` with more than one rank): this rank's chunks, masks and slots, its
        passage range, the store's row offsets and C."""
        if self.chunks is None:
            raise _lib.MatchmakerB200Error("save() before index()")
        rank, world = self._world()
        torch.save({"chunks": self.chunks.cpu(), "chunk_mask": self.chunk_mask.cpu(), "slots": self.slots.cpu(),
                    "doc_offsets": torch.from_numpy(self.doc_offsets), "d_lo": self.d_lo, "d_hi": self.d_hi,
                    "C": self.C, "token_dtype": str(self.store_dtype), "world": world, "rank": rank},
                   self._shard_path(path))

    def load(self, path: str):
        """Restore this rank's share; refused unless the file was written by this rank of a job of this world size for
        the passage range this rank owns, and for a model with this max_doc_length's chunk slot count."""
        blob = self._load_shard(self._shard_path(path), row_range=False)
        off = blob["doc_offsets"].numpy()
        rank, world = self._world()
        d_lo, d_hi, _, _ = sharding.passage_shard_bounds(off, rank, world)
        if (blob["d_lo"], blob["d_hi"]) != (d_lo, d_hi):
            raise _lib.MatchmakerB200Error(f"store file holds passages [{blob['d_lo']},{blob['d_hi']}), this rank owns "
                                           f"[{d_lo},{d_hi}) -- re-index or load with the same world size")
        if blob["C"] != self.C:
            raise _lib.MatchmakerB200Error(f"store file was indexed with C = {blob['C']} chunk slots, this model's "
                                           f"max_doc_length gives {self.C}")
        self._set(off, d_lo, d_hi, blob["chunks"], blob["chunk_mask"], blob["slots"])
