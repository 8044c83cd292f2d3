"""Shared cases of the flat-IP envelope tests (no GPU): the routing rules of the inner-product top-k, the shape matrix
that runs every compiled instantiation of its kernel body ``flat_ip_tc_body``, seeded integer inputs on which every
kernel's fp32 arithmetic is exact, and one fp64 oracle.

Routing (``csrc/flat_ip.cu``):

- list width ``epl_for_k`` (:50): EPL = 32 for k <= 256 (1024 list entries per query row), else 64 (2048).
- ``make_plan`` (:731-770), flat mode only: ``n_qblocks = ceil(nq / 128)``, ``n_tiles = ceil(n / 128)``; cluster size
  CL = 2 when ``n_qblocks`` is even or >= 9, else 1, and ``MMB200_FLATIP_CLUSTER`` = 1, 2 or 4 overrides it.  The range
  count is the smallest r <= min(32, n_tiles) whose item grid fills >= 88 % of the ``sm_count / CL`` cluster slots
  (or the best fill there is); ``MMB200_FLATIP_RANGES`` overrides it when 1 <= r <= min(32, n_tiles).  Then
  ``tiles_per_range = ceil(n_tiles / r)`` and the range count actually run is ``ceil(n_tiles / tiles_per_range)``.
- kernels (:1020-1030, :1184-1197): ``flat_ip_topk`` runs ``flat_ip_tc_kernel<T, CL, EPL, false>`` with T = __half
  for fp16 and the fp32 split, __nv_bfloat16 for bf16; ``ivf_search`` runs ``flat_ip_tc_kernel<T, 1, EPL, true>``,
  with ``row_index`` ``flat_ip_tc_gather_kernel<T, EPL>``; ``ivf_search_residual`` runs
  ``flat_ip_tc_residual_kernel<EPL, bits>``.  E4M3 (dtype "e4m3", both operands float8_e4m3fn, flat_ip.cu:1054-1062,
  :1231-1232): ``flat_ip_topk`` runs ``flat_ip_tc_fp8_kernel<CL, EPL>`` under the same plan; ``ivf_search`` only with
  ``row_index``, on ``flat_ip_tc_gather_fp8_kernel<EPL>`` (without it the call is refused).
- merge (:792, :795-849): ``topk_merge_kernel`` sorts at most 8192 candidates at once; more (flat mode: ``n_ranges *
  kpad``, IVF: ``nprobe * kslot``) are cut to their k best in groups and merged again.

Inputs are small integers (fp16), integers of magnitude <= 4 (bf16), integer queries against passages a + b * 2^-10
(the fp32 split: q_lo = 0, hi and lo exact), and residual codes over integer base and weight tables.  ``make_case``
asserts that sum_i |q_i p_i| < 2^24 grains for every (query, row) pair, so every fp32 sum is exact in any order: then
(score desc, signed id asc) is a total order and ids and scores are bit-exact, including the (-FLT_MAX, -1) tail.  The
e4m3 rows hold integers e4m3 holds exactly with sum_i |q_i p_i| < 2^11, the bound under which the FP8 MMA's own
accumulation is exact (test_maxsim_envelope_gpu.py::test_fp8_mma_accumulates_exactly)."""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

import colbert_residual_oracle as RO
import ivf_oracle

FLAT, IVF_GATHER, RESIDUAL = "flat_ip_tc_kernel", "flat_ip_tc_gather_kernel", "flat_ip_tc_residual_kernel"
FLAT_FP8, GATHER_FP8 = "flat_ip_tc_fp8_kernel", "flat_ip_tc_gather_fp8_kernel"
KERNELS = (FLAT, IVF_GATHER, RESIDUAL, FLAT_FP8, GATHER_FP8)
E4M3_EXACT_GRAINS = 2 ** 11   # the e4m3 rows' bound (maxsim_cases.E4M3_EXACT_GRAINS)
TNAME = {"f16": "__half", "split": "__half", "bf16": "__nv_bfloat16"}
BM = BN = 128
MAX_RANGES = 32
MERGE_SEG = 8192
SM_COUNT_H100 = 132
NO_RESULT = -3.4028234663852886e38
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def inst(kernel: str, *args) -> str:
    """Canonical instantiation name, e.g. ``flat_ip_tc_kernel<__half,4,64,false>``."""
    return kernel + "<" + ",".join(str(a).lower() if isinstance(a, bool) else str(a) for a in args) + ">"


def epl_for_k(k: int) -> int:
    return 32 if k <= 256 else 64


def plan(nq: int, n: int, k: int, sm_count: int, cluster: Optional[int] = None, ranges: Optional[int] = None) -> dict:
    """make_plan and workspace_bytes (flat_ip.cu:731-779) with the two environment overrides."""
    n_qblocks, n_tiles, kpad = -(-nq // BM), -(-n // BN), -(-k // 32) * 32
    cl = 2 if (n_qblocks % 2 == 0 or n_qblocks >= 9) else 1
    if cluster in (1, 2, 4):
        cl = cluster
    n_qgroups = -(-n_qblocks // cl)
    max_clusters = max(1, sm_count // cl)
    max_r = max(1, min(MAX_RANGES, n_tiles))
    effs, best_r, best_eff = {}, 1, -1.0
    for r in range(1, max_r + 1):
        items = n_qgroups * r
        g = min(max_clusters, items)
        waves = -(-items // g)
        effs[r] = items / (waves * max_clusters)
        if effs[r] > best_eff + 1e-9:
            best_eff, best_r = effs[r], r
    for r in range(1, max_r + 1):
        if effs[r] >= 0.88 or effs[r] >= best_eff - 1e-9:
            best_r = r
            break
    if ranges is not None and 1 <= ranges <= max_r:
        best_r = ranges
    tpr = -(-n_tiles // best_r)
    n_ranges = -(-n_tiles // tpr)
    grid = cl * min(max_clusters, n_qgroups * n_ranges)

    def a256(v):
        return -(-v // 256) * 256
    ws = (a256(nq * 4) + a256(grid * BM * 32 * epl_for_k(k) * 8) + a256(nq * n_ranges * kpad * 4)
          + a256(nq * n_ranges * kpad * 8))
    return {"n_qblocks": n_qblocks, "n_tiles": n_tiles, "n_ranges": n_ranges, "tiles_per_range": tpr, "grid": grid,
            "cl": cl, "kpad": kpad, "workspace": ws}


@dataclass(frozen=True)
class Row:
    mode: str              # "flat" (flat_ip_topk), "ivf" (ivf_search with and without row_index), "residual"
    dtype: str             # "f16", "bf16", "split" (fp32 storage as fp16 hi / lo), "e4m3"; residual rows are "f16"
    nq: int
    n: int                 # flat: passages; ivf / residual: rows in the lists (the store has padding rows besides)
    dim: int
    k: int
    seed: int
    why: str
    cl: Optional[int] = None       # MMB200_FLATIP_CLUSTER (flat mode)
    ranges: Optional[int] = None   # MMB200_FLATIP_RANGES (flat mode)
    regime: str = "rand"   # "rand"; "neg": every candidate scores < 0; "tie": a run of equal rows straddles rank k
    ids: str = "perm"      # "perm": shuffled, some negative; "extreme": also INT64_MIN / MAX and -1; "implicit"
    id_base: int = 0
    run: int = 0           # tie regime: length of the run of equal rows
    lists: tuple = ()      # ivf / residual: list lengths
    nprobe: int = 0
    bits: int = 0          # residual code bits

    def __str__(self):
        s = f"{self.mode}-{self.dtype}-nq{self.nq}-n{self.n}-d{self.dim}-k{self.k}-{self.regime}-{self.ids}"
        if self.mode == "flat":
            s += f"-cl{self.cl or 'auto'}-r{self.ranges or 'auto'}"
        else:
            s += f"-nlist{len(self.lists)}-np{self.nprobe}" + (f"-b{self.bits}" if self.bits else "")
        return s

    @property
    def max_list_len(self) -> int:
        return max(self.lists)

    def plan(self, sm_count: int = SM_COUNT_H100) -> dict:
        return plan(self.nq, self.n, self.k, sm_count, self.cl, self.ranges)

    def env(self) -> dict:
        """The plan overrides of the row as environment variables (unset ones are removed)."""
        return {"MMB200_FLATIP_CLUSTER": None if self.cl is None else str(self.cl),
                "MMB200_FLATIP_RANGES": None if self.ranges is None else str(self.ranges)}

    def merge_candidates(self, sm_count: int = SM_COUNT_H100) -> int:
        if self.mode == "flat":
            pl = self.plan(sm_count)
            return pl["n_ranges"] * pl["kpad"]
        kslot = -(-min(self.k, max(1, self.max_list_len)) // 32) * 32
        return self.nprobe * kslot


def dispatched(row: Row) -> frozenset:
    """The instantiations the envelope test runs for a row."""
    e = epl_for_k(row.k)
    if row.mode == "flat":
        return frozenset({flat_inst(row.dtype, row.plan()["cl"], e)})
    if row.dtype == "e4m3":
        return frozenset({inst(GATHER_FP8, e)})   # e4m3 IVF runs through row_index only
    if row.mode == "ivf":
        return frozenset({inst(FLAT, TNAME[row.dtype], 1, e, True), inst(IVF_GATHER, TNAME[row.dtype], e)})
    return frozenset({inst(RESIDUAL, e, row.bits)})


def flat_inst(dtype: str, cl: int, epl: int) -> str:
    """The flat_ip_topk kernel of a dtype at a cluster size and list width."""
    return inst(FLAT_FP8, cl, epl) if dtype == "e4m3" else inst(FLAT, TNAME[dtype], cl, epl, False)


def _big_lists():
    g = torch.Generator().manual_seed(77)
    return tuple(int(v) for v in torch.randint(0, 7, (1100,), generator=g))


BIG_LISTS = _big_lists()

MATRIX = (
    # ---- flat_ip_topk: T x CL x EPL, 12 instantiations, plus the fp32 split on the __half kernels
    Row("flat", "f16", 1, 1, 64, 33, 1, "one query, one passage, k > n; implicit ids from a negative id_base",
        ids="implicit", id_base=-7),
    Row("flat", "bf16", 127, 127, 64, 31, 2, "bf16 <1,32>: 127 queries against 127 passages, every score < 0: the TMA "
        "zero fill of the last tile's row 127 would win", regime="neg"),
    Row("flat", "f16", 128, 4095, 128, 257, 3, "<1,64>: 32 ranges forced at n = 128 * 32 - 1: cross-range tau and a "
        "two-pass merge (32 * 288 candidates); INT64 edge ids", ranges=32, ids="extreme"),
    Row("flat", "bf16", 129, 4097, 64, 1000, 4, "bf16 <2,64>: 129 queries (two blocks, CL 2 on its own); n = 128 * 32 + "
        "1 with 32 ranges asked: 17 run, merged in three groups", ranges=32),
    Row("flat", "f16", 300, 3000, 64, 256, 5, "<2,32> forced with 3 query blocks (an idle cluster slot); a run of 1500 "
        "equal rows (over the 1024-entry list) straddles k = 256, ids not monotone, -1 and INT64_MIN in the run",
        cl=2, regime="tie", ids="extreme", run=1500),
    Row("flat", "bf16", 1100, 640, 64, 1, 6, "bf16 <2,32> on its own (9 query blocks: an idle slot); k = 1 over tied "
        "rows with implicit ids from a negative base, as the k-means assignment runs", regime="tie", ids="implicit",
        id_base=-5000, run=40),
    Row("flat", "f16", 600, 5000, 64, 1024, 7, "<4,64>: 5 query blocks at CL 4 (3 idle slots); a run of 2600 equal rows "
        "(over the 2048-entry list) straddles k = 1024", cl=4, regime="tie", ids="extreme", run=2600),
    Row("flat", "bf16", 129, 2000, 1024, 33, 8, "bf16 <4,32> at dim 1024, one range forced, every score < 0",
        cl=4, ranges=1, regime="neg"),
    Row("flat", "f16", 1, 256, 768, 256, 9, "<4,32>: one query at CL 4, dim 768, k = n", cl=4),
    Row("flat", "bf16", 128, 300, 128, 1024, 10, "bf16 <4,64>: k = 1024 > n; 32 ranges asked of 3 tiles (ignored)",
        cl=4, ranges=32, ids="extreme"),
    Row("flat", "f16", 256, 20000, 64, 1000, 11, "<2,64> on its own plan (two query blocks, automatic ranges)"),
    Row("flat", "bf16", 1, 9000, 128, 257, 12, "bf16 <1,64> forced: one query over many ranges, a run of 2600 equal "
        "rows", cl=1, regime="tie", ids="extreme", run=2600),
    Row("flat", "split", 129, 4000, 192, 32, 13, "fp32 split over 9 k-blocks (3 * dim / 64) on <__half,2,32>"),
    Row("flat", "split", 5, 1000, 64, 256, 14, "fp32 split over 3 k-blocks, every score < 0", regime="neg",
        ids="extreme"),
    # ---- ivf_search (plain and gather): flat_ip_tc_kernel<T,1,EPL,true> and flat_ip_tc_gather_kernel<T,EPL>
    Row("ivf", "f16", 200, 1239, 64, 31, 21, "empty, one-row, 128-row, 129-row and multi-tile lists; list 3 probed by "
        "all 200 queries (two work items); probes of -1 and >= nlist", ids="extreme",
        lists=(0, 1, 128, 300, 5, 77, 256, 0, 129, 40, 303), nprobe=4),
    Row("ivf", "bf16", 130, 814, 128, 256, 22, "bf16, nprobe = 1 into lists whose next list (or the end of the rows) "
        "outranks them: every score < 0", regime="neg", lists=(60, 70, 1, 90, 128, 20, 0, 30, 200, 215), nprobe=1),
    Row("ivf", "f16", 70, 2792, 64, 257, 23, "a run of 2600 equal rows over three probed lists, 2100 of them in one "
        "list (over the 2048-entry list), straddles k = 257; INT64 edge ids", regime="tie", ids="extreme", run=2600,
        lists=(2100, 300, 203, 128, 1, 0, 60), nprobe=5),
    Row("ivf", "bf16", 3, sum(BIG_LISTS), 64, 1000, 24, "bf16, nprobe = 1024 of 1100 short lists, k = 1000",
        lists=BIG_LISTS, nprobe=1024),
    # ---- ivf_search_residual: flat_ip_tc_residual_kernel<EPL, bits>
    Row("residual", "f16", 40, 309, 64, 32, 31, "1-bit codes at dim 64, every score < 0", regime="neg",
        lists=(50, 60, 129, 40, 0, 30), nprobe=2, bits=1),
    Row("residual", "f16", 20, 1651, 128, 256, 32, "2-bit codes at dim 128; a run of 1400 equal rows over two lists "
        "(1100 in one: over the 1024-entry list) straddles k = 256", regime="tie", ids="extreme", run=1400,
        lists=(1100, 300, 200, 50, 1), nprobe=4, bits=2),
    Row("residual", "f16", 150, 833, 768, 257, 33, "1-bit codes at dim 768, k = 257; list 2 probed by all 150 queries",
        lists=(300, 5, 400, 0, 128), nprobe=3, bits=1),
    Row("residual", "f16", 9, 3631, 64, 1024, 34, "2-bit codes at k = 1024, every score < 0",
        regime="neg", ids="extreme", lists=(700, 800, 1500, 10, 600, 20, 1), nprobe=2, bits=2),
    # ---- e4m3 flat_ip_topk: flat_ip_tc_fp8_kernel<CL, EPL>
    Row("flat", "e4m3", 1, 127, 128, 33, 41, "e4m3 <1,32>: one query against 127 rows, every score < 0 (the zero fill "
        "of the tile's row 127 would win)", regime="neg"),
    Row("flat", "e4m3", 5, 640, 384, 1, 42, "e4m3 <1,32>: k = 1 over tied rows, implicit ids from a negative base",
        regime="tie", ids="implicit", id_base=-3000, run=40),
    Row("flat", "e4m3", 128, 4097, 384, 1024, 43, "e4m3 <1,64>: 32 ranges asked of 33 tiles (17 run), merged in three "
        "groups; INT64 edge ids", ranges=32, ids="extreme"),
    Row("flat", "e4m3", 256, 3000, 128, 256, 44, "e4m3 <2,32>: a run of 1500 equal rows (over the 1024-entry list) "
        "straddles k = 256", regime="tie", ids="extreme", run=1500),
    Row("flat", "e4m3", 129, 256, 1024, 257, 45, "e4m3 <2,64> at dim 1024: k = 257 > n = 256"),
    Row("flat", "e4m3", 300, 2000, 1024, 32, 46, "e4m3 <4,32> forced at dim 1024, one range", cl=4, ranges=1),
    Row("flat", "e4m3", 600, 5000, 128, 1000, 47, "e4m3 <4,64> forced: a run of 2600 equal rows (over the 2048-entry "
        "list) straddles k = 1000", cl=4, regime="tie", ids="extreme", run=2600),
    # ---- e4m3 ivf_search with row_index: flat_ip_tc_gather_fp8_kernel<EPL>
    Row("ivf", "e4m3", 200, 1239, 128, 31, 51, "e4m3 gather: empty, one-row, 128-row and multi-tile lists; probes of -1 "
        "and >= nlist; INT64 edge ids", ids="extreme", lists=(0, 1, 128, 300, 5, 77, 256, 0, 129, 40, 303), nprobe=4),
    Row("ivf", "e4m3", 130, 814, 128, 256, 52, "e4m3 gather, nprobe = 1, every score < 0: the next list and the padding "
        "rows outrank every candidate", regime="neg", lists=(60, 70, 1, 90, 128, 20, 0, 30, 200, 215), nprobe=1),
    Row("ivf", "e4m3", 70, 2792, 256, 257, 53, "e4m3 gather <64>: a run of 2600 equal rows, 2100 in one list, straddles "
        "k = 257", regime="tie", ids="extreme", run=2600, lists=(2100, 300, 203, 128, 1, 0, 60), nprobe=5),
    Row("ivf", "e4m3", 3, sum(BIG_LISTS), 128, 1000, 54, "e4m3 gather, nprobe = 1024 of 1100 short lists, k = 1000",
        lists=BIG_LISTS, nprobe=1024),
)

METAMORPHIC_ROW = MATRIX[6]   # run under CL 1 / 2 / 4 x ranges 1 / auto / 32


# ---------------------------------------------------------------------------------------------------------------------
# features: what the matrix is there for besides the instantiations
# ---------------------------------------------------------------------------------------------------------------------
K_EDGES = (1, 31, 32, 33, 256, 257, 1000, 1024)


def features(row: Row, sm_count: int = SM_COUNT_H100) -> frozenset:
    if row.dtype == "e4m3":
        return _e4m3_features(row, sm_count)
    f = set()
    if row.k in K_EDGES:
        f.add(f"k {row.k}")
    f.add(f"{row.regime} {row.mode}")
    if row.regime == "tie" and row.run > 32 * epl_for_k(row.k):
        f.add(f"tie run over the list capacity, EPL {epl_for_k(row.k)}, {row.mode}")
    if row.ids == "extreme":
        f.add(f"INT64 edge ids, {row.mode}")
    if row.mode == "flat":
        if row.k == row.n:
            f.add("k = n")
        if row.k > row.n:
            f.add("k > n")
        if row.n == 1:
            f.add("n 1")
        elif row.n < BN:
            f.add("n < 128")
        if row.n >= BN - 1:
            f.update({1: {"n 128m + 1"}, 0: {"n 128m"}, BN - 1: {"n 128m - 1"}}.get(row.n % BN, set()))
        if row.nq in (1, 127, 128, 129):
            f.add(f"nq {row.nq}")
        if row.dim in (64, 128, 768, 1024):
            f.add(f"dim {row.dim}")
        pl = row.plan(sm_count)
        if pl["n_qblocks"] % pl["cl"]:
            f.add(f"idle cluster slots at CL {pl['cl']}")
        if row.ranges == 1:
            f.add("ranges 1")
        if row.ranges == MAX_RANGES and pl["n_tiles"] >= MAX_RANGES:
            f.add("ranges 32")
        if row.merge_candidates(sm_count) > MERGE_SEG:
            f.add("multi-pass merge")
        if row.ids == "implicit" and row.id_base < 0:
            f.add("implicit ids, negative id_base")
        if row.k == 1 and row.regime == "tie":
            f.add("k 1 over tied rows")
        if row.dtype == "split":
            f.add("split" if row.dim == 64 else "split over more than 3 k-blocks")
    else:
        L = row.lists
        if 0 in L:
            f.add("empty list")
        if 1 in L:
            f.add("one-row list")
        if any(v and v % BN == 0 for v in L):
            f.add("list of 128m rows")
        if any(v > 2 * BN for v in L):
            f.add("multi-tile list")
        if row.nq > BM and row.regime == "rand":
            f.add("a list probed by more than 128 queries")
        if row.nprobe in (1, 1024):
            f.add(f"nprobe {row.nprobe}")
        if row.mode == "residual":
            f.add(f"residual bits {row.bits}")
            f.add(f"residual dim {row.dim}")
    return frozenset(f)


E4M3_K_EDGES = (1, 32, 33, 256, 257, 1024)


def _e4m3_features(row: Row, sm_count: int = SM_COUNT_H100) -> frozenset:
    """The features of an e4m3 row, named apart from the 16-bit rows' (none is shared with them)."""
    f = {f"e4m3 {row.regime} {row.mode}"}
    if row.regime == "tie" and row.run > 32 * epl_for_k(row.k):
        f.add(f"e4m3 tie run over the list capacity, EPL {epl_for_k(row.k)}, {row.mode}")
    if row.ids == "extreme":
        f.add(f"e4m3 INT64 edge ids, {row.mode}")
    if row.mode == "flat":
        if row.k in E4M3_K_EDGES:
            f.add(f"e4m3 k {row.k}")
        if row.k > row.n:
            f.add("e4m3 k > n")
        f.update({1: {"e4m3 n 128m + 1"}, 0: {"e4m3 n 128m"}, BN - 1: {"e4m3 n 128m - 1"}}.get(row.n % BN, set()))
        if row.dim in (128, 384, 1024):
            f.add(f"e4m3 dim {row.dim}")
        if row.cl is not None or row.ranges is not None:
            f.add("e4m3 forced plan")
        if row.merge_candidates(sm_count) > MERGE_SEG:
            f.add("e4m3 multi-pass merge")
    else:
        L = row.lists
        f.update({"e4m3 empty list"} if 0 in L else set())
        f.update({"e4m3 one-row list"} if 1 in L else set())
        if any(v and v % BN == 0 for v in L):
            f.add("e4m3 list of 128m rows")
        if any(v > 2 * BN for v in L):
            f.add("e4m3 multi-tile list")
        if row.nprobe in (1, 1024):
            f.add(f"e4m3 nprobe {row.nprobe}")
        if row.nprobe > 1 and row.regime != "neg":
            f.add("e4m3 probes of -1 and >= nlist")
        if row.nq > BM and row.regime == "rand":
            f.add("e4m3 a list probed by more than 128 queries")
    return frozenset(f)


E4M3_REQUIRED_FEATURES = frozenset(
    {f"e4m3 k {k}" for k in E4M3_K_EDGES} | {f"e4m3 dim {d}" for d in (128, 384, 1024)}
    | {"e4m3 k > n", "e4m3 n 128m - 1", "e4m3 n 128m", "e4m3 n 128m + 1", "e4m3 forced plan", "e4m3 multi-pass merge"}
    | {f"e4m3 {r} {m}" for r in ("rand", "neg", "tie") for m in ("flat", "ivf")}
    | {f"e4m3 tie run over the list capacity, EPL {e}, flat" for e in (32, 64)}
    | {"e4m3 tie run over the list capacity, EPL 64, ivf", "e4m3 INT64 edge ids, flat", "e4m3 INT64 edge ids, ivf"}
    | {"e4m3 empty list", "e4m3 one-row list", "e4m3 list of 128m rows", "e4m3 multi-tile list", "e4m3 nprobe 1",
       "e4m3 nprobe 1024", "e4m3 probes of -1 and >= nlist", "e4m3 a list probed by more than 128 queries"})


REQUIRED_FEATURES = E4M3_REQUIRED_FEATURES | frozenset(
    {f"k {k}" for k in K_EDGES}
    | {"k = n", "k > n", "n 1", "n < 128", "n 128m - 1", "n 128m", "n 128m + 1"}
    | {f"nq {n}" for n in (1, 127, 128, 129)} | {f"dim {d}" for d in (64, 128, 768, 1024)}
    | {"idle cluster slots at CL 2", "idle cluster slots at CL 4", "ranges 1", "ranges 32", "multi-pass merge"}
    | {"split", "split over more than 3 k-blocks", "implicit ids, negative id_base", "k 1 over tied rows"}
    | {f"neg {m}" for m in ("flat", "ivf", "residual")}
    | {"tie run over the list capacity, EPL 32, flat", "tie run over the list capacity, EPL 64, flat",
       "tie run over the list capacity, EPL 64, ivf", "tie run over the list capacity, EPL 32, residual"}
    | {f"INT64 edge ids, {m}" for m in ("flat", "ivf", "residual")}
    | {"empty list", "one-row list", "list of 128m rows", "multi-tile list", "a list probed by more than 128 queries",
       "nprobe 1", "nprobe 1024"}
    | {f"residual bits {b}" for b in (1, 2)} | {f"residual dim {d}" for d in (64, 128, 768)})


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    q: torch.Tensor                      # [nq, dim] f64 integers
    p: torch.Tensor                      # [n, dim] f64: the passages, or the rows in list order (decoded for residual)
    ids: Optional[torch.Tensor]          # [n] int64 (None: implicit, id_base + position)
    offsets: Optional[torch.Tensor] = None     # [nlist + 1]
    probes: Optional[torch.Tensor] = None      # [nq, nprobe]
    store: Optional[torch.Tensor] = None       # [n_store, dim] f64: list rows in shuffled order, padding rows between
    store_ids: Optional[torch.Tensor] = None   # [n_store]
    row_index: Optional[torch.Tensor] = None   # [n]: store row of list position p
    codes: Optional[np.ndarray] = None         # residual: [n_store, dim * bits / 8] uint8
    base: Optional[np.ndarray] = None          # [nlist, dim] fp16 integers
    weight: Optional[np.ndarray] = None        # [dim, 2^bits] fp16 integers
    store_lists: Optional[np.ndarray] = None   # [n_store] int32 list of every store row


def _randint(g, lo, hi, shape):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _ids(row: Row, g, n: int, run_pos: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """Distinct ids: even numbers from -n / 8 in shuffled order; "extreme" rows put -1, INT64_MIN,
    INT64_MIN + 1, INT64_MAX and INT64_MAX - 1 inside the tie run (or anywhere without one) and INT64_MIN + 2 outside."""
    if row.ids == "implicit":
        return None
    ids = (torch.randperm(n, generator=g) - n // 16) * 2
    if row.ids == "extreme":
        pool = torch.tensor([-1, I64_MIN, I64_MIN + 1, I64_MAX, I64_MAX - 1], dtype=torch.int64)
        where = run_pos if run_pos is not None else torch.arange(n)
        sel = where[torch.randperm(where.numel(), generator=g)[: min(5, n)]]
        ids[sel] = pool[: sel.numel()]
        if run_pos is not None:
            outside = torch.ones(n, dtype=torch.bool)
            outside[run_pos] = False
            o = outside.nonzero().flatten()
            if o.numel():
                ids[o[int(torch.randint(0, o.numel(), (1,), generator=g))]] = I64_MIN + 2
    return ids


def _split_parts(x: torch.Tensor, role: str):
    from matchmaker_b200.interaction import flat_ip_split_f32
    s, scale = flat_ip_split_f32(x.float(), role)
    return s.double(), scale


def _assert_exact(row: Row, q: torch.Tensor, p: torch.Tensor):
    """sum_i |q_i p_i| < 2^24 grains for every (query, row): every fp32 partial sum is an exact integer of grains."""
    if row.dtype == "split":
        qs, sq = _split_parts(q, "queries")
        ps, sp = _split_parts(p, "passages")
        d = row.dim
        assert torch.equal(qs[:, d:2 * d], torch.zeros_like(qs[:, d:2 * d])), "q_lo must be zero"
        assert torch.equal(ps[:, :d] + ps[:, d:], torch.ldexp(p, torch.tensor(sp, dtype=torch.int64))), "hi + lo != p"
        grain = 2.0 ** (sq + sp - 10)
        mass = qs[:, :d].abs() @ (ps[:, :d].abs() + ps[:, d:].abs()).T / grain
        assert torch.equal(p * 1024, (p * 1024).round())
    elif row.dtype == "e4m3":
        E4 = torch.float8_e4m3fn
        assert torch.equal(q.float().to(E4).double(), q) and torch.equal(p.float().to(E4).double(), p)
        assert torch.equal(p, p.round()) and torch.equal(q, q.round())
        assert float((q.abs() @ p.abs().T).max()) < E4M3_EXACT_GRAINS
        return
    else:
        mass = q.abs() @ p.abs().T
        lim = 4 if row.dtype == "bf16" else 8
        assert q.abs().max() <= lim and p.abs().max() <= lim and torch.equal(p, p.round()) and torch.equal(q, q.round())
    assert float(mass.max()) < 2 ** 24


def _flat_rows(row: Row, g, n: int, dim: int):
    """(q, p, run positions) for the regime: "rand" values in [-3, 3]; "neg" queries in [-3, -1] against rows in
    [1, 3]; "tie" positive queries, `run` rows of all 3 at shuffled positions and 3 rows above them (one entry 4).
    e4m3 (sums below 2^11): "rand" queries in [-1, 1] against rows in [-2, 2]; "neg" queries in {-1, 0} against rows in
    [1, 2]; "tie" queries of all 1 against rows in [-1, 1], the run all 1 and the rows above it with one entry 2."""
    if row.dtype == "e4m3":
        if row.regime == "neg":
            q = -(torch.rand(row.nq, dim, generator=g) < 0.5).double()
            q[:, 0] = -1.0
            return q, _randint(g, 1, 2, (n, dim))
        if row.regime == "tie":
            return torch.ones(row.nq, dim, dtype=torch.float64), _randint(g, -1, 1, (n, dim))
        return _randint(g, -1, 1, (row.nq, dim)), _randint(g, -2, 2, (n, dim))
    if row.regime == "neg":
        q, p = _randint(g, -3, -1, (row.nq, dim)), _randint(g, 1, 3, (n, dim))
    elif row.regime == "tie":
        q, p = _randint(g, 1, 3, (row.nq, dim)), _randint(g, -3, 3, (n, dim))
    else:
        q, p = _randint(g, -3, 3, (row.nq, dim)), _randint(g, -3, 3, (n, dim))
    if row.dtype == "split":
        p = p + _randint(g, -255, 255, (n, dim)) / 1024.0
    return q, p


def _place_run(row: Row, g, p: torch.Tensor, pos: torch.Tensor):
    """Rows `pos` become the tie run (all 3; the split adds a common fraction); up to 3 more rows score above it."""
    top = 1.0 if row.dtype == "e4m3" else 3.0
    v = torch.full((p.shape[1],), top, dtype=torch.float64)
    if row.dtype == "split":
        v += 17 / 1024
    p[pos[: row.run]] = v
    for j, r in enumerate(pos[row.run: row.run + 3].tolist()):
        p[r] = v
        p[r, j] = top + 1.0
    return pos[: row.run]


@functools.lru_cache(maxsize=None)
def make_case(row: Row) -> Case:
    g = torch.Generator().manual_seed(9000 + row.seed)
    if row.mode == "flat":
        q, p = _flat_rows(row, g, row.n, row.dim)
        run_pos = None
        if row.regime == "tie":
            run_pos = _place_run(row, g, p, torch.randperm(row.n, generator=g)[: row.run + (3 if row.k > 1 else 0)])
        _assert_exact(row, q, p)
        return Case(q, p, _ids(row, g, row.n, run_pos))
    return _make_ivf_case(row, g)


def _make_ivf_case(row: Row, g) -> Case:
    L = torch.tensor(row.lists, dtype=torch.int64)
    nlist, n, dim = len(row.lists), int(L.sum()), row.dim
    assert n == row.n, f"{row}: lists hold {n} rows"
    offsets = torch.zeros(nlist + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(L, 0)
    list_of = torch.repeat_interleave(torch.arange(nlist), L)
    # probes: "neg" probes only even lists (the next list is odd: bait), "tie" every query probes the run's lists
    probeable = torch.arange(0, nlist, 2) if row.regime == "neg" else torch.arange(nlist)
    probes = torch.empty(row.nq, row.nprobe, dtype=torch.int64)
    for r in range(row.nq):
        probes[r] = probeable[torch.randperm(probeable.numel(), generator=g)[: row.nprobe]]
    run_lists = ()
    if row.regime == "tie":
        run_lists = tuple(range(3 if row.mode == "ivf" else 2))
        probes[:, : len(run_lists)] = torch.tensor(run_lists)
        for r in range(row.nq):
            rest = torch.tensor([l for l in torch.randperm(nlist, generator=g).tolist() if l not in run_lists])
            probes[r, len(run_lists):] = rest[: row.nprobe - len(run_lists)]
    elif row.regime == "rand" and row.nq > BM:
        hot = int(torch.argmax(L))
        for r in range(row.nq):   # the longest list first in every query's probes
            has = (probes[r] == hot).nonzero().flatten()
            if has.numel():
                probes[r, int(has[0])] = probes[r, 0]
            probes[r, 0] = hot
    if row.regime != "neg" and row.nprobe > 1:   # lists that probe nothing: -1 and ids >= nlist
        probes[::3, -1] = -1
        probes[1::3, -1] = nlist + 5
    if row.mode == "residual":
        return _make_residual_case(row, g, offsets, list_of, probes, run_lists)
    q, p = _flat_rows(row, g, n, dim)
    if row.regime == "neg":   # rows of the odd lists outrank every probed row
        odd = (list_of % 2 == 1)
        p[odd] = -p[odd]
    run_pos = None
    if row.regime == "tie":
        in_run = torch.isin(list_of, torch.tensor(run_lists)).nonzero().flatten()
        assert in_run.numel() >= row.run + 3
        run_pos = _place_run(row, g, p, in_run[torch.randperm(in_run.numel(), generator=g)[: row.run + 3]])
    _assert_exact(row, q, p)
    ids = _ids(row, g, n, run_pos)
    store, store_ids, row_index = _gather_store(row, g, p, ids)
    if row.dtype == "e4m3":
        _assert_exact(row, q, store)   # the padding rows too: the gather kernel reads them if it reads wrong
    return Case(q, p, ids, offsets, probes, store, store_ids, row_index)


def _gather_store(row: Row, g, p: torch.Tensor, ids: torch.Tensor):
    """The rows of list position p at store row row_index[p], in shuffled order with padding rows (no list) between,
    which outrank every candidate in the "neg" and "tie" regimes; their ids are distinct from the list rows' ids."""
    n, n_pad = p.shape[0], 37 + p.shape[0] // 10
    pos = torch.randperm(n + n_pad, generator=g)
    row_index = pos[:n]
    store = torch.empty(n + n_pad, p.shape[1], dtype=torch.float64)
    store[row_index] = p
    bait = {"neg": -3.0, "tie": 4.0}.get(row.regime, 3.0)
    store[pos[n:]] = bait
    store_ids = torch.empty(n + n_pad, dtype=torch.int64)
    store_ids[row_index] = ids
    store_ids[pos[n:]] = 10 ** 15 + torch.arange(n_pad)
    return store, store_ids, row_index


def _make_residual_case(row: Row, g, offsets, list_of, probes, run_lists) -> Case:
    """Residual codes over integer tables: "rand" bases in [-1, 1] and weights in [-2, 2]; "neg" even lists' bases in
    [2, 3], odd lists' in [-4, -3], weights in [-1, 1], queries in [-3, -1]; "tie" the run's lists have base 1, the run
    rows the code of each dimension's largest weight (2): the run is all 3, everything else at most 3."""
    nlist, n, dim, bits = len(row.lists), row.n, row.dim, row.bits
    nlev = 1 << bits
    rng = np.random.default_rng(9000 + row.seed)
    if row.regime == "neg":
        base = np.where((np.arange(nlist) % 2 == 0)[:, None], rng.integers(2, 4, (nlist, dim)),
                        rng.integers(-4, -2, (nlist, dim)))
        weight = rng.integers(-1, 2, (dim, nlev))
        q = _randint(g, -3, -1, (row.nq, dim))
    elif row.regime == "tie":
        base = rng.integers(-1, 2, (nlist, dim))
        base[list(run_lists)] = 1
        weight = rng.integers(-2, 2, (dim, nlev))
        top = rng.integers(0, nlev, dim)
        weight[np.arange(dim), top] = 2
        q = _randint(g, 1, 3, (row.nq, dim))
    else:
        base = rng.integers(-1, 2, (nlist, dim))
        weight = rng.integers(-2, 3, (dim, nlev))
        q = _randint(g, -3, 3, (row.nq, dim))
    base, weight = base.astype(np.float16), weight.astype(np.float16)
    n_pad = 29 + n // 10
    pos = torch.randperm(n + n_pad, generator=g).numpy()
    row_index = pos[:n]
    store_lists = np.full(n + n_pad, 1 if (row.regime == "neg" and nlist > 1) else 0, dtype=np.int32)
    store_lists[row_index] = list_of.numpy()
    codes = rng.integers(0, nlev, (n + n_pad, dim))
    run_pos = None
    if row.regime == "tie":
        in_run = np.nonzero(np.isin(list_of.numpy(), run_lists))[0]
        run_pos = torch.from_numpy(in_run[rng.permutation(in_run.size)[: row.run]])
        codes[row_index[run_pos.numpy()]] = top
        codes[pos[n:]] = top   # padding rows tie with the run
    packed = RO.pack(codes.astype(np.uint8), bits)
    dec = torch.from_numpy(RO.decode(packed, store_lists, base, weight, bits).astype(np.float64))
    if row.regime == "tie":
        assert bool((dec[row_index[run_pos.numpy()]] == 3).all())
    p = dec[torch.from_numpy(row_index)]
    _assert_exact(row, q, p)
    ids = _ids(row, g, n, run_pos)
    store_ids = torch.empty(n + n_pad, dtype=torch.int64)
    store_ids[torch.from_numpy(row_index)] = ids
    store_ids[torch.from_numpy(pos[n:])] = 10 ** 15 + torch.arange(n_pad)
    return Case(q, p, ids, offsets, probes, dec, store_ids, torch.from_numpy(row_index), packed, base, weight,
                store_lists)


# ---------------------------------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------------------------------
def rank(q: torch.Tensor, p: torch.Tensor, ids: torch.Tensor, k: int, cand: Optional[torch.Tensor] = None):
    """fp64 top-k of s = q p^T over the candidate rows (cand [nq, n] bool, default all) under (score desc, signed id
    asc), padded with (-3.4028235e38, -1): (scores [nq, k] f32, ids [nq, k] int64)."""
    s = q.double() @ p.double().T
    if cand is not None:
        s = s.masked_fill(~cand, float("-inf"))
    oid = torch.argsort(ids, stable=True)
    order = torch.argsort(s[:, oid], dim=1, descending=True, stable=True)[:, :k]
    sel = oid[order]
    sc, si = torch.gather(s, 1, sel), ids[sel]
    out_s = torch.full((q.shape[0], k), NO_RESULT, dtype=torch.float64)
    out_i = torch.full((q.shape[0], k), -1, dtype=torch.int64)
    kk = sc.shape[1]
    live = sc > float("-inf")
    out_s[:, :kk] = torch.where(live, sc, torch.full_like(sc, NO_RESULT))
    out_i[:, :kk] = torch.where(live, si, torch.full_like(si, -1))
    assert torch.equal(out_s, out_s.float().double()), "an fp64 score is not an fp32 value"
    return out_s.float(), out_i


def candidates(c: Case) -> torch.Tensor:
    """[nq, n] bool: the rows of each query's probed lists (ivf_oracle.union_rows)."""
    cand = torch.zeros(c.q.shape[0], c.p.shape[0], dtype=torch.bool)
    for r in range(c.q.shape[0]):
        cand[r, ivf_oracle.union_rows(c.offsets, c.probes[r])] = True
    return cand


def row_ids(row: Row, c: Case) -> torch.Tensor:
    return c.ids if c.ids is not None else row.id_base + torch.arange(c.p.shape[0])


@functools.lru_cache(maxsize=None)
def expected(row: Row):
    c = make_case(row)
    return rank(c.q, c.p, row_ids(row, c), row.k, None if row.mode == "flat" else candidates(c))
