"""ColBERT end-to-end retrieval with an inverted-file (IVF) token index: ``faiss_index_type: "ivf"`` for ColBERT.

Stage 1 of ``ColBERTEndToEndIndexer`` (every live query token against every token row of the store) becomes the
ColBERT paper's approximate token search: each live token probes its ``nprobe`` nearest lists of a spherical k-means
quantizer and keeps its ``token_top_k`` best rows of the union of those lists.  Stages 2 and 3 (exact max-sim of the
candidate passages, ranking, merge across ranks), sharding, ``token_top_k`` and the candidate cap are inherited.

The rows are not copied into list order: stage 2 reads them in passage order, and a second copy would double the
store's HBM.  Instead the index keeps ``row_index`` (int64, one per row: the rows of list l are
``row_index[list_offsets[l]:list_offsets[l+1]]``, ascending within a list) and the scan gathers each tile's rows out of
the passage-ordered store (``interaction.ivf_search(..., row_index=...)``).  Device memory beyond the exact indexer's:
8 bytes per row plus the centroids and list offsets.

Config: ``faiss_ivf_list_count`` = nlist, ``faiss_ivf_search_probe_count`` = nprobe, as ``IVFIndexer`` reads them.  The
quantizer is ``IVFIndexer``'s: same sampling, k-means and empty-list splits; rank 0 trains and broadcasts.

With ``colbert_store_dtype: "float8_e4m3"`` the rows are assigned to their lists as given (before they are quantized),
so the lists and the layout are those of the fp16 indexer, and the gather scan reads the e4m3 store.
"""
from __future__ import annotations

from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction
from .colbert_e2e import CANDIDATE_CAP, ColBERTEndToEndIndexer
from .ivf_index import IVFIndexer

ASSIGN_BATCH = 1 << 20      # rows per assignment call: bounds the flat_ip_topk scratch (~12 bytes * kpad per row)


class ColBERTIVFIndexer(ColBERTEndToEndIndexer):
    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.ivf = IVFIndexer(config, device=self.device, process_group=process_group)   # quantizer + k-means
        self.row_index: Optional[torch.Tensor] = None      # [rows] int64 store row of every list position
        self.list_offsets: Optional[torch.Tensor] = None   # [nlist + 1] int64
        self.max_list_len = 0
        self._saved_layout = None                          # (fingerprint, row_index, list_offsets) from load()
        self._fp8_lists: Optional[torch.Tensor] = None     # fp8 index(): list of every row, assigned chunk by chunk

    @property
    def nlist(self) -> int:
        return self.ivf.nlist

    @property
    def nprobe(self) -> int:
        return self.ivf.nprobe

    # ------------------------------------------------------------------ build
    def prepare(self, storage: List[numpy.ndarray], subsample=-1):
        """Train the coarse quantizer on the token rows (the blocks of ``token_storage.load_token_storage``)."""
        self.ivf.prepare(storage, subsample)

    def _fingerprint(self):
        return {"n_rows": int(self.store.shape[0]) if self.store is not None else 0, "d_lo": int(self.d_lo),
                "d_hi": int(self.d_hi), "world": int(self._world()[1])}

    def index(self, id_mapping: List[numpy.ndarray], storage: List[numpy.ndarray]):
        if self.ivf.centroids is None:
            raise _lib.MatchmakerB200Error("index() before prepare() or load(): the IVF token index has no centroids")
        super().index(id_mapping, storage)
        if self.store.shape[0] == 0:
            self._set_layout(torch.zeros(0, dtype=torch.int64, device=self.device),
                             torch.zeros(self.nlist + 1, dtype=torch.int64, device=self.device))
        elif self.fp8:   # the parent streamed the rows itself (index_device was not called)
            self._layout_from(self._take_fp8_lists)

    def index_device(self, rows: torch.Tensor, doc_offsets: numpy.ndarray, first_doc: int = 0):
        if self.ivf.centroids is None:
            raise _lib.MatchmakerB200Error("index() before prepare() or load(): the IVF token index has no centroids")
        super().index_device(rows, doc_offsets, first_doc)
        self._layout_from(self._take_fp8_lists if self.fp8 else lambda: self.assign(self.store))

    def _fp8_chunk(self, rows: torch.Tensor, a: int, b: int, n: int):
        if self._saved_layout is not None:   # load() restored the layout: nothing to assign
            return
        if a == 0:
            self._fp8_lists = torch.empty(n, dtype=torch.int64, device=self.device)
        self._fp8_lists[a:b] = self.assign(rows.to(self.store_dtype))

    def _take_fp8_lists(self) -> torch.Tensor:
        lists, self._fp8_lists = self._fp8_lists, None
        return lists

    def _layout_from(self, lists):
        """The layout from the rows' lists (``lists()``), or the one load() restored without assigning anything."""
        if self._saved_layout is None:
            self._set_layout(*self.ivf._layout(lists()))   # stable: ascending store rows per list
        else:
            self._set_layout(self._saved_layout[1].to(self.device), self._saved_layout[2].to(self.device))

    def assign(self, rows: torch.Tensor) -> torch.Tensor:
        """List id of every row: its argmax-inner-product centroid (ties to the lowest list id)."""
        out = torch.empty(rows.shape[0], dtype=torch.int64, device=self.device)
        for a in range(0, rows.shape[0], ASSIGN_BATCH):
            b = min(rows.shape[0], a + ASSIGN_BATCH)
            out[a:b] = interaction.flat_ip_topk(rows[a:b], self.ivf.c_store, 1, split_scale=self.ivf.c_scale)[1][:, 0]
        return out

    def _set_layout(self, row_index: torch.Tensor, list_offsets: torch.Tensor):
        if self._saved_layout is not None and self._saved_layout[0] != self._fingerprint():
            raise _lib.MatchmakerB200Error(f"the loaded IVF token layout was built for {self._saved_layout[0]}, this "
                                           f"store is {self._fingerprint()}: re-index without load()")
        if list_offsets.numel() != self.nlist + 1 or row_index.numel() != int(list_offsets[-1]) or \
                row_index.numel() != self.store.shape[0]:
            raise _lib.MatchmakerB200Error("IVF token layout does not cover the store's rows")
        self.row_index, self.list_offsets = row_index.contiguous(), list_offsets.contiguous()
        self.max_list_len = int((list_offsets[1:] - list_offsets[:-1]).max().item()) if self.nlist else 0

    # ------------------------------------------------------------------ stage 1
    def candidates_device(self, q: torch.Tensor, kp: int, qs: Optional[torch.Tensor] = None):
        """Stage 1 on this rank with the token index: every live token probes its nprobe lists and keeps its kp best
        rows of their union (passage ids as ids); all-zero padding tokens probe nothing.  Then the parent's de-duplicated
        candidate lists [Nq, C], best first, void entries (-3.4028235e38, -1).  q and qs as the parent's: the coarse
        search reads q, the list scan qs."""
        nq, lq, dim = q.shape
        toks = q.reshape(nq * lq, dim)
        stoks = (self._score_queries(q)[0] if qs is None else qs).reshape(nq * lq, dim)
        pad = (toks == 0).all(dim=1, keepdim=True)
        probes = self.ivf.coarse(toks).masked_fill(pad, -1)
        hs, hi = interaction.ivf_search(stoks, self.flat, self.row_ids, self.list_offsets, probes, kp, self.max_list_len,
                                        split_scale=self.split_scale, row_index=self.row_index)
        c = min(lq * kp, CANDIDATE_CAP)
        return interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c)

    # ------------------------------------------------------------------ persistence
    def _shard_path(self, path: str) -> str:
        rank, world = self._world()
        return path if world == 1 else f"{path}.rank{rank}of{world}"

    def save(self, path: str):
        """One file per rank (``<path>.rank<r>of<w>`` with more than one rank): the centroids, this rank's layout, nlist,
        nprobe, the token dtype, the store dtype and scale, and the fingerprint of the store it was built for.  The rows
        are not written: they come back from the encoded token store through ``index()``."""
        if self.row_index is None:
            raise _lib.MatchmakerB200Error("save() before index()")
        rank, world = self._world()
        torch.save({"centroids": self.ivf.centroids.cpu(), "row_index": self.row_index.cpu(),
                    "list_offsets": self.list_offsets.cpu(), "nlist": self.nlist, "nprobe": self.nprobe,
                    "token_dtype": str(self.store_dtype), "store_dtype": "float8_e4m3" if self.fp8 else None,
                    "store_scale": self.store_scale, "fingerprint": self._fingerprint(), "rank": rank},
                   self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        """Restore the quantizer and this rank's layout; the following ``index()`` on the same store reuses the layout
        (and raises if the store is not the one it was built for).  nprobe comes from
        config_overwrites["faiss_ivf_search_probe_count"] when given, else from the file."""
        import os
        rank, world = self._world()
        if not os.path.isfile(self._shard_path(path)):
            raise _lib.MatchmakerB200Error(f"no index file {self._shard_path(path)} for rank {rank} of {world}: was the "
                                           "index saved with another world size?")
        blob = torch.load(self._shard_path(path))
        fp = blob["fingerprint"]
        if fp["world"] != world or blob["rank"] != rank:
            raise _lib.MatchmakerB200Error(f"index file {self._shard_path(path)} was written by rank {blob['rank']} of "
                                           f"{fp['world']}; this job is rank {rank} of {world} -- re-index or load with "
                                           "the same world size")
        if blob["token_dtype"] != str(self.store_dtype):
            raise _lib.MatchmakerB200Error(f"index file was written with token_dtype {blob['token_dtype']}, this indexer "
                                           f"is configured for {self.store_dtype}")
        store_dtype = "float8_e4m3" if self.fp8 else None
        if blob.get("store_dtype") != store_dtype:
            raise _lib.MatchmakerB200Error(f"index file was written with colbert_store_dtype {blob.get('store_dtype')}, "
                                           f"this indexer is configured for {store_dtype}")
        self.saved_store_scale = blob.get("store_scale")
        self.ivf.nlist = int(blob["nlist"])
        self.ivf.nprobe = int(blob["nprobe"])
        if config_overwrites and "faiss_ivf_search_probe_count" in config_overwrites:
            self.ivf.nprobe = int(config_overwrites["faiss_ivf_search_probe_count"])
        self.ivf.set_centroids(blob["centroids"])
        self._saved_layout = (fp, blob["row_index"], blob["list_offsets"])
        self.row_index = self.list_offsets = None
