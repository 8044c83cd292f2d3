"""ColBERT IVF retrieval over a residual-compressed token store (``colbert_residual_bits``, DESIGN 3.4g).

``ColBERTIVFIndexer`` keeps every token row in HBM at full width.  This indexer keeps each row as its IVF list's base
vector plus ``b`` bits per dimension (ColBERTv2 / PLAID residual compression) and decodes the codes where the rows are
consumed: inside the probed-list scan of stage 1 (``interaction.ivf_search_residual``) and inside the max-sim of
stage 2 (``interaction.maxsim_store_residual``).  Everything else -- the spherical k-means quantizer, the list layout
over the passage-ordered store, ``token_top_k``, the candidate cap, ranking and the merge across ranks -- is
``ColBERTIVFIndexer``'s.

Format (``csrc/residual.cuh``): row x of list l has codes code[d] = #{i : cutoff[d][i] <= float(x[d]) -
float(base[l][d])} and decodes to fp16_rn(float(base[l][d]) + float(weight[d][code[d]])).
- base[l]: the un-normalised mean (fp64 sums in ascending row order, stored as fp16) of the list's rows in the
  k-means training sample (``IVFIndexer``'s seeded sample, up to 256 rows per list), zero for a list without sample rows;
- cutoff[d] (2^b - 1, fp32) and weight[d] (2^b, fp16): the i / 2^b and (i + 0.5) / 2^b quantiles (nearest rank) in
  dimension d of the residuals of ``TABLE_SAMPLE_ROWS`` rows drawn from that sample by a seeded permutation.

Device memory per row: dim * b / 8 bytes of codes and a 4-byte list id, plus the inherited ``row_index`` and
``row_ids`` (16 bytes); no fp16 rows.  ``index()`` streams the rank's rows through the device in slabs of
``INDEX_SLAB_ROWS``.  Envelope: ``token_dtype: "float16"``, dim % 64 == 0, 64 <= dim <= 1024, b in {1, 2}.
"""
from __future__ import annotations

import os
from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction, sharding
from .colbert_e2e import CANDIDATE_CAP, doc_offsets_from_id_mapping
from .colbert_ivf import ColBERTIVFIndexer

INDEX_SLAB_ROWS = 1 << 20    # rows per slab of index(): peak device memory is the codes plus one fp16 slab
TABLE_SAMPLE_ROWS = 1 << 17  # residuals behind the per-dimension quantiles, drawn from the k-means training sample
TABLE_SEED = 4321
MEAN_CHUNK_ROWS = 1 << 16    # rows per host chunk of the fp64 list sums (whole lists per chunk)


def list_means_f16(x: torch.Tensor, assign: torch.Tensor, nlist: int) -> numpy.ndarray:
    """[nlist, dim] fp16: the mean of the rows x [n, dim] of each list (``assign`` [n]), summed in fp64 in ascending row
    order on the host, zero for an empty list.  The rows move to the host in chunks of whole lists, so each list's sum
    is one sequential reduction and the result does not depend on the chunking."""
    perm = torch.sort(assign, stable=True).indices
    counts = torch.bincount(assign, minlength=nlist).cpu().numpy()
    off = numpy.concatenate([[0], numpy.cumsum(counts)])
    sums = numpy.zeros((nlist, x.shape[1]), dtype=numpy.float64)
    l0 = 0
    while l0 < nlist:
        l1 = l0 + 1   # whole lists, at least one, up to MEAN_CHUNK_ROWS rows
        while l1 < nlist and off[l1 + 1] - off[l0] <= MEAN_CHUNK_ROWS:
            l1 += 1
        live = l0 + numpy.nonzero(counts[l0:l1])[0]
        if len(live):
            xs = x[perm[off[l0]:off[l1]]].cpu().numpy().astype(numpy.float64)
            # axis-0 reductions of a C-ordered array add the rows one after the other
            sums[live] = numpy.add.reduceat(xs, off[live] - off[l0], axis=0)
        l0 = l1
    return (sums / numpy.maximum(counts, 1)[:, None]).astype(numpy.float16)


class ColBERTResidualIndexer(ColBERTIVFIndexer):
    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.bits = int(config.get("colbert_residual_bits", 0))
        if self.bits not in interaction.RESIDUAL_BITS:
            raise _lib.MatchmakerB200Error(f"colbert_residual_bits must be 1 or 2, got {self.bits}")
        if self.store_dtype != torch.float16:
            raise _lib.MatchmakerB200Error('the residual token store needs token_dtype: "float16"')
        if self.token_dim % 64 or not 64 <= self.token_dim <= 1024:
            raise _lib.MatchmakerB200Error(f"the residual token store needs token_dim % 64 == 0 and 64 <= token_dim <= "
                                           f"1024, got {self.token_dim}")
        self.slab_rows = INDEX_SLAB_ROWS
        self.base: Optional[torch.Tensor] = None      # [nlist, dim] fp16
        self.weight: Optional[torch.Tensor] = None    # [dim, 2^b] fp16
        self.cutoff: Optional[torch.Tensor] = None    # [dim, 2^b - 1] fp32
        self.list_ids: Optional[torch.Tensor] = None  # [rows] int32
        # self.store holds the codes [rows, dim * b / 8] uint8: the inherited checks (indexed, row count) read it

    # ------------------------------------------------------------------ training
    def prepare(self, storage: List[numpy.ndarray], subsample=-1):
        """Train the quantizer, then the bases and level tables, on rank 0; every other rank receives all three."""
        rank, world = self._world()
        dim, nlev = self.token_dim, 1 << self.bits
        if rank == 0:
            x, init = self.ivf._training_points(storage)
            cents = self.ivf.train_points(x, init)
            self.ivf.set_centroids(cents)
            base, weight, cutoff = self.train_tables(x)
        else:
            cents = torch.empty((self.nlist, dim), dtype=torch.float32, device=self.device)
            base = torch.empty((self.nlist, dim), dtype=torch.float16, device=self.device)
            weight = torch.empty((dim, nlev), dtype=torch.float16, device=self.device)
            cutoff = torch.empty((dim, nlev - 1), dtype=torch.float32, device=self.device)
        if world > 1:
            import torch.distributed as dist
            for t in (cents, base, weight, cutoff):
                dist.broadcast(t, 0, group=self.group)
        self.ivf.set_centroids(cents)
        self.base, self.weight, self.cutoff = base, weight, cutoff

    def train_tables(self, x: torch.Tensor):
        """(base [nlist, dim] fp16, weight [dim, 2^b] fp16, cutoff [dim, 2^b - 1] fp32) from the training sample
        x [n, dim] under the current centroids: the bases from every row of x (``list_means_f16``), the quantiles from
        the residuals of min(n, TABLE_SAMPLE_ROWS) rows picked by a permutation seeded with TABLE_SEED.
        Bit-reproducible: fp64 sums in a fixed order, nearest-rank picks from a sort."""
        x = x.to(self.device, torch.float16).contiguous()
        a = self.assign(x)
        base = torch.from_numpy(list_means_f16(x, a, self.nlist)).to(self.device)
        pick_rows = torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(TABLE_SEED))[:TABLE_SAMPLE_ROWS]
        pick_rows = pick_rows.to(self.device)
        r = x[pick_rows].float() - base[a[pick_rows]].float()
        rs = torch.sort(r, dim=0).values
        n, nlev = r.shape[0], 1 << self.bits

        def pick(fr):
            return rs[min(n - 1, int(fr * n))]
        cutoff = torch.stack([pick(i / nlev) for i in range(1, nlev)], dim=1).contiguous()
        weight = torch.stack([pick((i + 0.5) / nlev) for i in range(nlev)], dim=1).to(torch.float16).contiguous()
        return base, weight, cutoff

    # ------------------------------------------------------------------ build
    def _require_tables(self):
        if self.ivf.centroids is None or self.base is None:
            raise _lib.MatchmakerB200Error("index() before prepare() or load(): the residual token index has no tables")

    def _encode(self, rows: torch.Tensor):
        """(list ids int32, codes) of fp16 rows on the device."""
        a = self.assign(rows)
        return a.to(torch.int32), interaction.residual_encode(rows, a, self.base, self.cutoff, self.bits)

    def index(self, id_mapping: List[numpy.ndarray], storage: List[numpy.ndarray]):
        """As ``ColBERTEndToEndIndexer.index``, but the rank's rows pass through the device in slabs of
        ``self.slab_rows``: each slab is assigned, encoded and freed."""
        from .token_storage import blocks_to_device
        self._require_tables()
        if len(id_mapping) != len(storage) or any(len(a) != len(b) for a, b in zip(id_mapping, storage)):
            raise _lib.MatchmakerB200Error("id_mapping and storage must have one entry per stored row, block by block")
        if storage and storage[0].shape[1] != self.token_dim:
            raise _lib.MatchmakerB200Error(f"storage rows have dim {storage[0].shape[1]}, config token_dim is "
                                           f"{self.token_dim}")
        off = doc_offsets_from_id_mapping(id_mapping)
        rank, world = self._world()
        self.n_docs = len(off) - 1
        d_lo, d_hi, r_lo, r_hi = sharding.passage_shard_bounds(off, rank, world) if self.n_docs else (0, 0, 0, 0)
        codes = torch.empty((r_hi - r_lo, self.token_dim * self.bits // 8), dtype=torch.uint8, device=self.device)
        lids = torch.empty(r_hi - r_lo, dtype=torch.int32, device=self.device)
        for a in range(r_lo, r_hi, self.slab_rows):
            b = min(r_hi, a + self.slab_rows)
            with torch.cuda.device(self.device):
                rows = blocks_to_device(storage, a, b, self.device).to(torch.float16)
            lids[a - r_lo:b - r_lo], codes[a - r_lo:b - r_lo] = self._encode(rows)
            del rows
        self._set_codes(codes, lids, off[d_lo:d_hi + 1] - r_lo if self.n_docs else numpy.zeros(1, numpy.int64), d_lo)

    def index_device(self, rows: torch.Tensor, doc_offsets: numpy.ndarray, first_doc: int = 0):
        """Index this rank's passages from a device tensor rows [n_rows, token_dim] (encoded in slabs, not kept)."""
        self._require_tables()
        off = numpy.asarray(doc_offsets, dtype=numpy.int64)
        if rows.dim() != 2 or rows.shape[1] != self.token_dim or off[0] != 0 or off[-1] != rows.shape[0] or \
                (numpy.diff(off) < 0).any():
            raise _lib.MatchmakerB200Error("index_device: rows [n_rows, token_dim] and non-decreasing offsets from 0")
        n = rows.shape[0]
        codes = torch.empty((n, self.token_dim * self.bits // 8), dtype=torch.uint8, device=self.device)
        lids = torch.empty(n, dtype=torch.int32, device=self.device)
        for a in range(0, n, self.slab_rows):
            b = min(n, a + self.slab_rows)
            lids[a:b], codes[a:b] = self._encode(rows[a:b].to(self.device, torch.float16).contiguous())
        self._set_codes(codes, lids, off, first_doc)

    def _set_codes(self, codes: torch.Tensor, lids: torch.Tensor, off: numpy.ndarray, first_doc: int, layout=None):
        self.store, self.flat, self.split_scale = codes, None, None
        self.list_ids = lids
        lens = torch.from_numpy(numpy.diff(off)).to(self.device)
        self.offsets = torch.from_numpy(off).to(self.device)
        self.max_doc_len = max(1, int(numpy.diff(off).max())) if len(off) > 1 else 1
        self.row_ids = torch.repeat_interleave(torch.arange(first_doc, first_doc + len(off) - 1, device=self.device), lens)
        self.d_lo, self.d_hi = first_doc, first_doc + len(off) - 1
        # stable sort: ascending store rows per list (load() passes the saved one)
        row_index, list_offsets = self.ivf._layout(lids.to(torch.int64)) if layout is None else layout
        self.row_index, self.list_offsets = row_index.contiguous(), list_offsets.contiguous()
        self.max_list_len = int((list_offsets[1:] - list_offsets[:-1]).max().item())

    def decoded_store(self) -> torch.Tensor:
        """The fp16 rows the codes decode to [rows, dim] (what both stages score against)."""
        return interaction.residual_decode(self.store, self.list_ids, self.base, self.weight, self.bits)

    # ------------------------------------------------------------------ stages 1 and 2
    def candidates_device(self, q: torch.Tensor, kp: int):
        """``ColBERTIVFIndexer.candidates_device`` with the list scan decoding the codes."""
        nq, lq, dim = q.shape
        toks = q.reshape(nq * lq, dim)
        pad = (toks == 0).all(dim=1, keepdim=True)
        probes = self.ivf.coarse(toks).masked_fill(pad, -1)
        hs, hi = interaction.ivf_search_residual(toks, self.store, self.base, self.weight, self.bits, self.row_ids,
                                                 self.row_index, self.list_offsets, probes, kp, self.max_list_len)
        c = min(lq * kp, CANDIDATE_CAP)
        return interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c)

    def _search_local(self, q: torch.Tensor, top_n: int, kp: int):
        nq = q.shape[0]
        _, cand = self.candidates_device(q, kp)
        c = cand.shape[1]
        pair_d = torch.where(cand >= 0, cand - self.d_lo, torch.full_like(cand, -1))
        pair_q = torch.arange(nq, device=self.device, dtype=torch.int32).repeat_interleave(c)
        scores = interaction.maxsim_store_residual(q, self.store, self.list_ids, self.base, self.weight, self.bits,
                                                   self.offsets, pair_q, pair_d, self.max_doc_len).view(nq, c)
        return interaction.topk_merge(scores, cand, top_n)

    # ------------------------------------------------------------------ persistence
    def save(self, path: str):
        """One file per rank (``<path>.rank<r>of<w>`` with more than one rank) with everything a search needs: the
        centroids, bases, level tables, bits, this rank's codes, list ids, layout and passage offsets."""
        if self.row_index is None:
            raise _lib.MatchmakerB200Error("save() before index()")
        rank, world = self._world()
        torch.save({"centroids": self.ivf.centroids.cpu(), "base": self.base.cpu(), "weight": self.weight.cpu(),
                    "cutoff": self.cutoff.cpu(), "bits": self.bits, "dim": self.token_dim, "codes": self.store.cpu(),
                    "list_ids": self.list_ids.cpu(), "row_index": self.row_index.cpu(),
                    "list_offsets": self.list_offsets.cpu(), "offsets": self.offsets.cpu(), "d_lo": int(self.d_lo),
                    "n_docs": int(self.n_docs), "nlist": self.nlist, "nprobe": self.nprobe, "rank": rank,
                    "world": world}, self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        """Restore a searchable index written by ``save`` (no ``index()`` needed).  Raises when the file was written
        for another rank, world size, bit count or dim.  nprobe comes from
        config_overwrites["faiss_ivf_search_probe_count"] when given, else from the file."""
        rank, world = self._world()
        fn = self._shard_path(path)
        if not os.path.isfile(fn):
            raise _lib.MatchmakerB200Error(f"no index file {fn} for rank {rank} of {world}: was the index saved with "
                                           "another world size?")
        blob = torch.load(fn)
        if blob["world"] != world or blob["rank"] != rank:
            raise _lib.MatchmakerB200Error(f"index file {fn} was written by rank {blob['rank']} of {blob['world']}; "
                                           f"this job is rank {rank} of {world}")
        if blob["bits"] != self.bits or blob["dim"] != self.token_dim:
            raise _lib.MatchmakerB200Error(f"index file {fn} holds {blob['bits']}-bit codes of dim {blob['dim']}; this "
                                           f"indexer is configured for {self.bits} bits, dim {self.token_dim}")
        self.ivf.nlist = int(blob["nlist"])
        self.ivf.nprobe = int(blob["nprobe"])
        if config_overwrites and "faiss_ivf_search_probe_count" in config_overwrites:
            self.ivf.nprobe = int(config_overwrites["faiss_ivf_search_probe_count"])
        self.ivf.set_centroids(blob["centroids"])
        dev = self.device
        self.base, self.weight, self.cutoff = blob["base"].to(dev), blob["weight"].to(dev), blob["cutoff"].to(dev)
        self.n_docs = int(blob["n_docs"])
        self._set_codes(blob["codes"].to(dev), blob["list_ids"].to(dev), blob["offsets"].numpy(), int(blob["d_lo"]),
                        (blob["row_index"].to(dev), blob["list_offsets"].to(dev)))
