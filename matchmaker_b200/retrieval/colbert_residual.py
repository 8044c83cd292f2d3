"""ColBERT IVF retrieval over a residual-compressed token store (``colbert_residual_bits``, DESIGN 3.4g).

``ColBERTIVFIndexer`` keeps every token row in HBM at full width.  This indexer keeps each row as its IVF list's base
vector plus ``b`` bits per dimension (ColBERTv2 / PLAID residual compression) and decodes the codes where the rows are
consumed: inside the probed-list scan of stage 1 (``interaction.ivf_search_residual``) and inside the max-sim of
stage 2 (``interaction.maxsim_store_residual``).  Everything else -- the spherical k-means quantizer, the list layout
over the passage-ordered store, ``token_top_k``, the candidate cap, ranking and the merge across ranks -- is
``ColBERTIVFIndexer``'s.

The codes, their tables and both decoding stages are ``colbert_store.ResidualTokenStore``'s; this indexer trains the
tables in ``prepare`` and saves the whole index.  Tables:
- base[l]: the un-normalised mean (fp64 sums in ascending row order, stored as fp16) of the list's rows in the
  k-means training sample (``IVFIndexer``'s seeded sample, up to 256 rows per list), zero for a list without sample
  rows;
- cutoff[d] (2^b - 1, fp32) and weight[d] (2^b, fp16): the i / 2^b and (i + 0.5) / 2^b quantiles (nearest rank) in
  dimension d of the residuals of ``TABLE_SAMPLE_ROWS`` rows drawn from that sample by a seeded permutation.

``index()`` streams the rank's rows through the device in slabs of ``colbert_store.SLAB_ROWS``.  Envelope:
``token_dtype: "float16"``, dim % 64 == 0, 64 <= dim <= 1024, b in {1, 2}.
"""
from __future__ import annotations

from typing import List

import numpy
import torch

from .. import _lib
from .colbert_e2e import token_store_attribute
from .colbert_ivf import ColBERTIVFIndexer

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
    residual = True
    slab_rows = token_store_attribute("slab_rows", "rows per slab of index(): the codes plus one fp16 slab in HBM")
    list_ids = token_store_attribute("list_ids", "[rows] int32 list of every stored row")
    base = token_store_attribute("base", "[nlist, dim] fp16 list bases")
    weight = token_store_attribute("weight", "[dim, 2^b] fp16 decoded levels")
    cutoff = token_store_attribute("cutoff", "[dim, 2^b - 1] fp32 level cutoffs")
    bits = property(lambda self: self.tokens.bits, doc="code bits per dimension")

    def decoded_store(self) -> torch.Tensor:
        """The fp16 rows the codes decode to [rows, dim] (what both stages score against)."""
        return self.tokens.decoded()

    # ------------------------------------------------------------------ training
    def prepare(self, storage: List[numpy.ndarray], subsample=-1):
        """Train the quantizer, then the bases and level tables, on rank 0; every other rank receives all four."""
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

    # ------------------------------------------------------------------ persistence
    def save(self, path: str):
        """One file per rank (``<path>.rank<r>of<w>`` with more than one rank) with everything a search needs: the
        centroids, bases, level tables, bits, this rank's codes, list ids, layout and passage offsets."""
        if self.row_index is None:
            raise _lib.MatchmakerB200Error("save() before index()")
        rank, world = self._world()
        torch.save({"centroids": self.ivf.centroids.cpu(), **self.tokens.state(), "row_index": self.row_index.cpu(),
                    "list_offsets": self.list_offsets.cpu(), "offsets": self.offsets.cpu(), "d_lo": int(self.d_lo),
                    "n_docs": int(self.n_docs), "nlist": self.nlist, "nprobe": self.nprobe, "rank": rank,
                    "world": world}, self._shard_path(path))

    def load(self, path: str, config_overwrites=None):
        """Restore a searchable index written by ``save`` (no ``index()`` needed).  Raises when the file was written
        for another rank, world size, bit count or dim.  nprobe comes from
        config_overwrites["faiss_ivf_search_probe_count"] when given, else from the file."""
        blob = self._load_shard(self._shard_path(path), row_range=False)
        self.tokens.restore(blob)
        self.ivf.nlist = int(blob["nlist"])
        self.ivf.nprobe = int(blob["nprobe"])
        if config_overwrites and "faiss_ivf_search_probe_count" in config_overwrites:
            self.ivf.nprobe = int(config_overwrites["faiss_ivf_search_probe_count"])
        self.ivf.set_centroids(blob["centroids"])
        self.n_docs = int(blob["n_docs"])
        self._set_passages(blob["offsets"].numpy(), int(blob["d_lo"]))
        self._set_layout(blob["row_index"].to(self.device), blob["list_offsets"].to(self.device))
