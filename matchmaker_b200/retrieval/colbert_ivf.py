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

The store assigns the rows to their lists as it builds (``colbert_store``): E4M3 rows as given, before they are
quantized, so the lists and the layout are those of the fp16 indexer, and the gather scan reads the e4m3 store.
"""
from __future__ import annotations

from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction
from . import colbert_plaid
from .colbert_e2e import ColBERTEndToEndIndexer
from .ivf_index import IVFIndexer

ASSIGN_BATCH = 1 << 20      # rows per assignment call: bounds the flat_ip_topk scratch (~12 bytes * kpad per row)


class ColBERTIVFIndexer(ColBERTEndToEndIndexer):
    plaid_capable = True

    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.ivf = IVFIndexer(config, device=self.device, process_group=process_group)   # quantizer + k-means
        keys = colbert_plaid.config_keys(config)
        if keys is not None:
            colbert_plaid.check_envelope(self.ivf.nlist, self.token_dim)
        self.plaid = None if keys is None else colbert_plaid.PLAIDSearch(*keys)   # PLAID search, when configured
        self.row_index: Optional[torch.Tensor] = None      # [rows] int64 store row of every list position
        self.list_offsets: Optional[torch.Tensor] = None   # [nlist + 1] int64
        self.max_list_len = 0
        self._saved_layout = None                          # (fingerprint, row_index, list_offsets) from load()

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
        n_rows = int(self.tokens.rows.shape[0]) if self.tokens.rows is not None else 0
        return {"n_rows": n_rows, "d_lo": int(self.d_lo), "d_hi": int(self.d_hi), "world": int(self._world()[1])}

    def _build(self, load, n: int, off: numpy.ndarray, first_doc: int):
        """The parent's store and passages, then the layout: from the lists the store's build assigned, or the one
        load() restored without assigning anything."""
        if self.ivf.centroids is None:
            raise _lib.MatchmakerB200Error("index() before prepare() or load(): the IVF token index has no centroids")
        saved = self._saved_layout
        lists = self.tokens.build(load, n, None if saved else lambda rows: self.assign(rows.to(self.store_dtype)))
        self._set_passages(off, first_doc)
        if saved is None:
            self._set_layout(*self.ivf._layout(lists))   # stable: ascending store rows per list
        else:
            self._set_layout(saved[1].to(self.device), saved[2].to(self.device))

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
                row_index.numel() != self.tokens.rows.shape[0]:
            raise _lib.MatchmakerB200Error("IVF token layout does not cover the store's rows")
        self.row_index, self.list_offsets = row_index.contiguous(), list_offsets.contiguous()
        self.max_list_len = int((list_offsets[1:] - list_offsets[:-1]).max().item()) if self.nlist else 0
        if self.plaid is not None:
            self.plaid.set_layout(self)

    # ------------------------------------------------------------------ search
    def search_device(self, q: torch.Tensor, top_n: int, token_top_k: Optional[int] = None):
        """search() with device tensors in and out.  With PLAID search, top_n <= colbert_plaid_ndocs // 4 and
        token_top_k must not be given."""
        if self.plaid is not None:
            if token_top_k is not None:
                raise _lib.MatchmakerB200Error("token_top_k has no meaning in a PLAID search (colbert_plaid_ndocs)")
            if top_n > self.plaid.ndocs // 4:
                raise _lib.MatchmakerB200Error(f"PLAID search needs top_n <= colbert_plaid_ndocs // 4 = "
                                               f"{self.plaid.ndocs // 4}, got {top_n}")
            if q.dim() == 3 and q.shape[1] > interaction.PLAID_MAX_LQ:
                raise _lib.MatchmakerB200Error(f"PLAID search needs Lq <= {interaction.PLAID_MAX_LQ}, got {q.shape[1]}")
        return super().search_device(q, top_n, token_top_k)

    def _search_local(self, q: torch.Tensor, top_n: int, kp: int):
        if self.plaid is None:
            return super()._search_local(q, top_n, kp)
        return self.plaid.search(self, q, top_n)

    # ------------------------------------------------------------------ stage 1
    def _scan(self, toks, stoks, kp: int):
        """Stage 1 with the token index: every live token probes its nprobe lists (the coarse search reads toks) and
        keeps its kp best rows of their union (the list scan reads stoks); all-zero padding tokens probe nothing."""
        pad = (toks == 0).all(dim=1, keepdim=True)
        probes = self.ivf.coarse(toks).masked_fill(pad, -1)
        return self.tokens.ivf_scan(stoks, self.row_ids, self.row_index, self.list_offsets, probes, kp, self.max_list_len)

    # ------------------------------------------------------------------ persistence
    def save(self, path: str):
        """One file per rank (``<path>.rank<r>of<w>`` with more than one rank): the centroids, this rank's layout, nlist,
        nprobe, the token dtype, the store dtype and scale, and the fingerprint of the store it was built for.  The rows
        are not written: they come back from the encoded token store through ``index()``."""
        if self.row_index is None:
            raise _lib.MatchmakerB200Error("save() before index()")
        torch.save({"centroids": self.ivf.centroids.cpu(), "row_index": self.row_index.cpu(),
                    "list_offsets": self.list_offsets.cpu(), "nlist": self.nlist, "nprobe": self.nprobe,
                    "token_dtype": str(self.store_dtype), **self.tokens.state(), "fingerprint": self._fingerprint(),
                    "rank": self._world()[0]}, self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        """Restore the quantizer and this rank's layout; the following ``index()`` on the same store reuses the layout
        (and raises if the store is not the one it was built for).  nprobe comes from
        config_overwrites["faiss_ivf_search_probe_count"] when given, else from the file."""
        blob = self._load_shard(self._shard_path(path), row_range=False)
        self.tokens.restore(blob)
        self.ivf.nlist = int(blob["nlist"])
        self.ivf.nprobe = int(blob["nprobe"])
        if config_overwrites and "faiss_ivf_search_probe_count" in config_overwrites:
            self.ivf.nprobe = int(config_overwrites["faiss_ivf_search_probe_count"])
        self.ivf.set_centroids(blob["centroids"])
        self._saved_layout = (blob["fingerprint"], blob["row_index"], blob["list_offsets"])
        self.row_index = self.list_offsets = None
