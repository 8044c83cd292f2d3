"""The token store of ColBERT end-to-end retrieval: one class per format, selected once from the config.

- ``DenseTokenStore``: the rows as fp16, or as fp32 (scanned through the fp16 hi / lo split);
- ``E4M3TokenStore`` (``colbert_store_dtype: "float8_e4m3"``, DESIGN 3.4i): row x held as e4m3(x * 2^s_d), with s_d the
  scale rule (``interaction.fp8_scale_log2``) over the largest |x| of the whole store (a MAX all-reduce over the ranks,
  so the stored values do not depend on the world size); each query is quantized with its own scale s_q and the scores
  are multiplied by 2^-(s_q + s_d);
- ``ResidualTokenStore`` (``colbert_residual_bits``, DESIGN 3.4g): each row as its IVF list's base vector plus ``b``
  bits per dimension, decoded inside the list scan and the max-sim.

Every store answers the same questions: ``build`` from the rank's rows, ``queries`` (the operand the kernels read and
its per-query scale), ``unscale``, the stage-1 scans (``scan``: exact, ``ivf_scan``: probed lists gathered out of the
passage-ordered store), the stage-2 ``maxsim``, and what it adds to a saved file (``state`` / ``restore``).
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from .. import _lib, interaction

STORE_DTYPES = ("float8_e4m3",)   # values of colbert_store_dtype
SLAB_ROWS = 1 << 20          # rows per slab of a streamed build: peak device memory is the store plus one slab


def select(config, token_dim: int, dtype: torch.dtype, device: torch.device, group=None, residual: bool = False):
    """The store the config selects (``residual``: the indexer keeps residual codes).  Raises on a configuration
    outside the formats' envelopes."""
    sd = config.get("colbert_store_dtype")
    if sd is not None:
        if sd not in STORE_DTYPES:
            raise _lib.MatchmakerB200Error(f"colbert_store_dtype must be one of {STORE_DTYPES}, got {sd!r}")
        if token_dim % 128 or not 128 <= token_dim <= 1024:
            raise _lib.MatchmakerB200Error(f"the float8_e4m3 token store needs token_dim % 128 == 0 and 128 <= "
                                           f"token_dim <= 1024, got {token_dim}")
        if config.get("colbert_residual_bits") is not None:
            raise _lib.MatchmakerB200Error("colbert_store_dtype and colbert_residual_bits are two different token "
                                           "store formats: configure one of them")
        return E4M3TokenStore(token_dim, dtype, device, group)
    if residual:
        bits = int(config.get("colbert_residual_bits", 0))
        if bits not in interaction.RESIDUAL_BITS:
            raise _lib.MatchmakerB200Error(f"colbert_residual_bits must be 1 or 2, got {bits}")
        if dtype != torch.float16:
            raise _lib.MatchmakerB200Error('the residual token store needs token_dtype: "float16"')
        if token_dim % 64 or not 64 <= token_dim <= 1024:
            raise _lib.MatchmakerB200Error(f"the residual token store needs token_dim % 64 == 0 and 64 <= token_dim <= "
                                           f"1024, got {token_dim}")
        return ResidualTokenStore(token_dim, dtype, device, bits)
    return DenseTokenStore(token_dim, dtype, device)


class _TokenStore:
    """What every format shares: the streamed build and the unscaled queries."""
    scale: Optional[int] = None   # the store scale s_d of an E4M3 store

    def __init__(self, dim: int, dtype: torch.dtype, device: torch.device):
        self.dim, self.dtype, self.device = dim, dtype, device   # dtype: of the rows (and queries) as given
        self.slab_rows = SLAB_ROWS
        self.rows: Optional[torch.Tensor] = None   # [rows of this rank, ...] what the max-sim reads

    def _stream(self, load, n: int, assign, put, slab_rows: int):
        """Rows [0, n) slab by slab: ``put(a, b, rows, lists)`` gets each slab as ``load`` returns it and, with
        ``assign``, its lists.  Returns the lists of all n rows (None without ``assign``)."""
        lists = torch.empty(n, dtype=torch.int64, device=self.device) if assign is not None else None
        for a in range(0, n, slab_rows):
            b = min(n, a + slab_rows)
            rows = load(a, b)
            if assign is not None:
                lists[a:b] = assign(rows)
            put(a, b, rows, None if lists is None else lists[a:b])
            del rows
        return lists

    def queries(self, q: torch.Tensor):
        """(what the kernels read, per-query scale or None) of queries q in the given dtype."""
        return q, None

    def unscale(self, scores: torch.Tensor, sq) -> torch.Tensor:
        return scores


class DenseTokenStore(_TokenStore):
    """fp16 rows, or fp32 rows plus their fp16 hi / lo split (``flat``, ``split_scale``) for the scans."""
    store_dtype = None   # the colbert_store_dtype a saved file records

    def __init__(self, dim: int, dtype: torch.dtype, device: torch.device):
        super().__init__(dim, dtype, device)
        self.flat: Optional[torch.Tensor] = None   # what the scans read
        self.split_scale = None

    def build(self, load: Callable, n: int, assign: Optional[Callable] = None) -> Optional[torch.Tensor]:
        """The store of this rank's n rows: ``load(a, b)`` returns rows [a, b) on the device, ``assign(rows)`` (IVF)
        the list of every row given.  Returns the lists of the n rows (None without ``assign``).  One slab of all n
        rows: fp16 rows given on the device are the store, not a copy of it."""
        self.rows = torch.empty((0, self.dim), dtype=self.dtype, device=self.device)

        def put(a, b, rows, lists):
            self.rows = rows
        lists = self._stream(lambda a, b: load(a, b).to(self.dtype), n, assign, put, max(n, 1))
        if self.dtype == torch.float16 or n == 0:
            self.flat, self.split_scale = self.rows, None
        else:
            self.flat, self.split_scale = interaction.flat_ip_split_f32(self.rows, "passages")
        return lists

    def scan(self, stoks: torch.Tensor, kp: int, row_ids: torch.Tensor):
        """Stage 1, exact: the kp best rows of every query token (passage ids as ids)."""
        return interaction.flat_ip_topk(stoks, self.flat, kp, ids=row_ids, split_scale=self.split_scale)

    def ivf_scan(self, stoks, row_ids, row_index, list_offsets, probes, kp: int, max_list_len: int):
        """Stage 1, IVF: the kp best rows of the probed lists of every query token."""
        return interaction.ivf_search(stoks, self.flat, row_ids, list_offsets, probes, kp, max_list_len,
                                      split_scale=self.split_scale, row_index=row_index)

    def maxsim(self, qs, offsets, pair_q, pair_d, max_doc_len: int):
        """Stage 2: the max-sim of every (query, passage) pair."""
        return interaction.maxsim_store(qs, self.rows, offsets, pair_q, pair_d, max_doc_len)

    def state(self) -> dict:
        """What a saved IVF token layout records about the store."""
        return {"store_dtype": self.store_dtype, "store_scale": None}

    def restore(self, blob: dict):
        """Check a saved IVF token layout against this store's format."""
        if blob.get("store_dtype") != self.store_dtype:
            raise _lib.MatchmakerB200Error(f"index file was written with colbert_store_dtype {blob.get('store_dtype')}, "
                                           f"this indexer is configured for {self.store_dtype}")


def fp8_store_scale(local_amax: torch.Tensor, group=None) -> int:
    """The store scale s_d from this rank's largest |x| (a one-element fp32 tensor on the rank's device): the MAX
    all-reduce over the ranks of ``group`` when torch.distributed is initialized, then the scale rule.  Raises on a
    non-finite maximum."""
    import torch.distributed as dist
    amax = local_amax.reshape(1).to(torch.float32).clone()
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(amax, op=dist.ReduceOp.MAX, group=group)
    return interaction.fp8_store_scale(float(amax.item()))


class E4M3TokenStore(DenseTokenStore):
    """e4m3 rows under the store scale ``scale`` (s_d); scanned and max-simmed on the FP8 tensor cores."""
    store_dtype = "float8_e4m3"

    def __init__(self, dim: int, dtype: torch.dtype, device: torch.device, group=None):
        super().__init__(dim, dtype, device)
        self.group = group
        self.loaded_scale: Optional[int] = None   # s_d of a loaded IVF token layout: a re-index must reproduce it

    def build(self, load: Callable, n: int, assign: Optional[Callable] = None) -> Optional[torch.Tensor]:
        """Streamed in slabs of ``slab_rows``: pass 1 takes the largest |x|, the all-reduce over ``group`` (which every
        rank joins, with or without rows) makes it the store's, pass 2 quantizes each slab into the preallocated store.
        ``assign`` sees each slab as given, before it is quantized.  Peak device memory: the store plus one slab and
        its fp32 copy."""
        amax = torch.zeros((), dtype=torch.float32, device=self.device)
        for a in range(0, n, self.slab_rows):
            lo, hi = torch.aminmax(load(a, min(n, a + self.slab_rows)))
            amax = torch.maximum(amax, torch.maximum(hi, -lo).float())
        s = fp8_store_scale(amax, self.group)
        if self.loaded_scale is not None and s != self.loaded_scale:
            raise _lib.MatchmakerB200Error(f"the loaded index was built for an fp8 store with scale 2^{self.loaded_scale}"
                                           f", these rows give 2^{s}: re-index without load()")
        self.rows = torch.empty((n, self.dim), dtype=torch.float8_e4m3fn, device=self.device)

        def put(a, b, rows, lists):
            self.rows[a:b] = interaction.fp8_quantize(rows, s)
        lists = self._stream(load, n, assign, put, self.slab_rows)
        self.flat, self.split_scale, self.scale = self.rows, None, s
        return lists

    def queries(self, q: torch.Tensor):
        """Each query quantized under the scale of its own largest |x| (on the device, no host synchronisation)."""
        sq = interaction.fp8_scale_log2(q.abs().amax(dim=(1, 2)))
        return interaction.fp8_quantize(q, sq), sq

    def unscale(self, scores: torch.Tensor, sq) -> torch.Tensor:
        """A positive per-query factor: the ranking of the scaled scores is the unscaled one."""
        return interaction.fp8_unscale(scores, sq + self.scale)

    def state(self) -> dict:
        return {"store_dtype": self.store_dtype, "store_scale": self.scale}

    def restore(self, blob: dict):
        super().restore(blob)
        self.loaded_scale = blob.get("store_scale")


class ResidualTokenStore(_TokenStore):
    """Residual codes (ColBERTv2 / PLAID residual compression, format in ``csrc/residual.cuh``): row x of list l has
    codes code[d] = #{i : cutoff[d][i] <= float(x[d]) - float(base[l][d])} and decodes to
    fp16_rn(float(base[l][d]) + float(weight[d][code[d]])).
    - base[l]: the un-normalised mean (fp64 sums in ascending row order, stored as fp16) of the list's rows in the
      k-means training sample, zero for a list without sample rows;
    - cutoff[d] (2^b - 1, fp32) and weight[d] (2^b, fp16): the i / 2^b and (i + 0.5) / 2^b quantiles (nearest rank) in
      dimension d of the residuals of sample rows drawn by a seeded permutation (``ColBERTResidualIndexer.prepare``).
    Device memory per row: dim * b / 8 bytes of codes (``rows``) and a 4-byte list id; no fp16 rows."""

    def __init__(self, dim: int, dtype: torch.dtype, device: torch.device, bits: int):
        super().__init__(dim, dtype, device)
        self.bits = bits
        # self.rows holds the codes [rows, dim * b / 8] uint8
        self.list_ids: Optional[torch.Tensor] = None   # [rows] int32
        self.base: Optional[torch.Tensor] = None       # [nlist, dim] fp16
        self.weight: Optional[torch.Tensor] = None     # [dim, 2^b] fp16
        self.cutoff: Optional[torch.Tensor] = None     # [dim, 2^b - 1] fp32

    def build(self, load: Callable, n: int, assign: Callable) -> torch.Tensor:
        """Streamed in slabs of ``slab_rows``: each slab, as fp16, is assigned to its lists, encoded and freed."""
        if self.base is None:
            raise _lib.MatchmakerB200Error("index() before prepare() or load(): the residual token index has no tables")
        self.rows = torch.empty((n, self.dim * self.bits // 8), dtype=torch.uint8, device=self.device)

        def put(a, b, rows, lists):
            self.rows[a:b] = interaction.residual_encode(rows, lists, self.base, self.cutoff, self.bits)
        lists = self._stream(lambda a, b: load(a, b).to(torch.float16).contiguous(), n, assign, put, self.slab_rows)
        self.list_ids = lists.to(torch.int32)
        return lists

    def decoded(self) -> torch.Tensor:
        """The fp16 rows the codes decode to [rows, dim] (what both stages score against)."""
        return interaction.residual_decode(self.rows, self.list_ids, self.base, self.weight, self.bits)

    def ivf_scan(self, stoks, row_ids, row_index, list_offsets, probes, kp: int, max_list_len: int):
        return interaction.ivf_search_residual(stoks, self.rows, self.base, self.weight, self.bits, row_ids, row_index,
                                               list_offsets, probes, kp, max_list_len)

    def maxsim(self, qs, offsets, pair_q, pair_d, max_doc_len: int):
        return interaction.maxsim_store_residual(qs, self.rows, self.list_ids, self.base, self.weight, self.bits, offsets,
                                                 pair_q, pair_d, max_doc_len)

    def state(self) -> dict:
        return {"base": self.base.cpu(), "weight": self.weight.cpu(), "cutoff": self.cutoff.cpu(), "bits": self.bits,
                "dim": self.dim, "codes": self.rows.cpu(), "list_ids": self.list_ids.cpu()}

    def restore(self, blob: dict):
        if blob["bits"] != self.bits or blob["dim"] != self.dim:
            raise _lib.MatchmakerB200Error(f"index file holds {blob['bits']}-bit codes of dim {blob['dim']}; this "
                                           f"indexer is configured for {self.bits} bits, dim {self.dim}")
        dev = self.device
        self.base, self.weight, self.cutoff = blob["base"].to(dev), blob["weight"].to(dev), blob["cutoff"].to(dev)
        self.rows, self.list_ids = blob["codes"].to(dev), blob["list_ids"].to(dev)
