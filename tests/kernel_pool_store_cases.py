"""Shared cases of the kernel-pooling store-mode envelope tests (no GPU): the shape matrix that runs every compiled
instantiation of the two store-mode kernels, a ragged store built to trip the per-CTA pair loop, and the fp64 reference.

The store mode (``interaction.kernel_pool_store``) picks its kernel and template instantiation from K, Lq, D and
``max_doc_len`` (L):

- tensor-core ``kernel_pool_ts_store_kernel<KB>`` (csrc/kernel_pool_ts.cu:442-447, routing :527-532): K == 11 -> 11,
  K == 21 -> 21, K <= 12 -> 12, K <= 24 -> 24, else 32 (``kernel_pool_cases.tc_kb``).  It takes the shape iff
  Lq <= 128 and D % 4 == 0 (:540); longer queries run one pass per block of 32 query rows and ``kp_combine_query_blocks``.
- FFMA ``kernel_pool_fwd_simt_store<KB, JR>`` (csrc/kernel_pool.cu:578-581): KB 12 / 24 / 32, JR = 2 iff L > 48.  Its
  shared-memory plan (:482-483) must fit the device's opt-in limit, which bounds D.

``impl="auto"`` takes the tensor-core kernel where it accepts the shape, else the FFMA kernel (:569-577).

Every row's store holds the same ragged passage layout, and its pairs make every CTA of both grids walk several pairs of
mixed tile counts (0 to 3 tiles of 128 rows), so the per-pair ring bookkeeping, the stale rows another pair left in the
raw ring, the over-fetch into the next passage and past the end of the store all run (``make_case``)."""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

import kernel_pool_cases as KP

TS_STORE, SIMT_STORE = "kernel_pool_ts_store_kernel", "kernel_pool_fwd_simt_store"
KERNELS = (TS_STORE, SIMT_STORE)
TS_MAX_LQ = 128                 # kernel_pool_ts.cu:539-540
SMEM_OPTIN_H100 = 232448        # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
SM_H100 = 132
MIN_PAIRS = 1200                # >= 9 pairs per CTA on the tensor-core grid, >= 2 on the FFMA grid of a 132-SM H100

# passage lengths of every store (clipped to the row's max_doc_len), then passages longer than max_doc_len
LENGTHS = (0, 1, 7, 8, 9, 31, 32, 33, 127, 128, 129, 255, 256, 257)
POISON_ROWS = 8                 # an unreferenced poisoned passage follows every referenced one of length % 8 != 0
TAIL_ROWS = 8                   # rows of the buffer past the store view
# tile counts of consecutive pairs of one query (0: pair_d -1 or the empty passage, never next to another 0)
TILE_PATTERN = (1, 0, 2, 3, 1, 2, 0, 3, 1, 3, 2)


def inst(kernel: str, *a) -> str:
    return f"{kernel}<{','.join(str(x) for x in a)}>"


def ts_store_kb(K: int) -> int:
    """KB of the tensor-core store kernel: kernel_pool_ts.cu:527-532, the rule of the padded kernel."""
    return KP.tc_kb(K)


def simt_store_inst(K: int, max_doc_len: int) -> Tuple[int, int]:
    """(KB, JR) of the FFMA store kernel: kernel_pool.cu:578-581."""
    return KP.simt_kb(K), 2 if max_doc_len > 48 else 1


def ts_accepts(Lq: int, D: int) -> bool:
    """kernel_pool_fwd_ts (kernel_pool_ts.cu:540) in store mode: no saved state, no cosine output, K <= 32."""
    return Lq <= TS_MAX_LQ and D % 4 == 0


def padded_row_stride(D: int) -> int:
    """device_util.cuh:43-47."""
    dp = (D + 3) & ~3
    return dp + 4 if ((dp >> 2) & 1) == 0 else dp


def simt_smem_bytes(D: int, K: int, max_doc_len: int) -> int:
    """The FFMA forward's dynamic shared memory (kernel_pool.cu:482-483)."""
    KB, JR = simt_store_inst(K, max_doc_len)
    TJ = 32 * JR
    return ((32 + TJ) * padded_row_stride(D) + 32 * (TJ + 1) + 32 * 6 + TJ + 9 * KB * 32) * 4


def simt_accepts(D: int, K: int, max_doc_len: int, smem: int = SMEM_OPTIN_H100) -> bool:
    return simt_smem_bytes(D, K, max_doc_len) <= smem


def simt_d_edge(K: int, max_doc_len: int, smem: int = SMEM_OPTIN_H100) -> int:
    """The largest D (a multiple of 4) the FFMA store kernel serves at this K and max_doc_len."""
    D = 4
    while simt_accepts(D + 4, K, max_doc_len, smem):
        D += 4
    return D


def impls(Lq: int, D: int, K: int, max_doc_len: int, smem: int = SMEM_OPTIN_H100) -> Tuple[str, ...]:
    """The kernels that accept the shape, as ``impl`` names."""
    return tuple(i for i, ok in (("tcgen05", ts_accepts(Lq, D)), ("simt", simt_accepts(D, K, max_doc_len, smem))) if ok)


def auto_impl(Lq: int, D: int) -> str:
    return "tcgen05" if ts_accepts(Lq, D) else "simt"


def instantiation(impl: str, K: int, max_doc_len: int) -> str:
    return inst(TS_STORE, ts_store_kb(K)) if impl == "tcgen05" else inst(SIMT_STORE, *simt_store_inst(K, max_doc_len))


def dispatched(Lq: int, D: int, K: int, max_doc_len: int) -> frozenset:
    return frozenset(instantiation(i, K, max_doc_len) for i in impls(Lq, D, K, max_doc_len))


EVERY = frozenset({inst(TS_STORE, kb) for kb in (11, 12, 21, 24, 32)}
                  | {inst(SIMT_STORE, kb, jr) for kb in (12, 24, 32) for jr in (1, 2)})


@dataclass(frozen=True)
class Row:
    K: int
    Lq: int
    D: int
    L: int           # max_doc_len
    n_q: int
    knrm: bool       # KNRM form: no alpha, log_scale 0.01
    seed: int
    claims: Tuple[str, ...]
    why: str

    @property
    def impls(self):
        return impls(self.Lq, self.D, self.K, self.L)

    def __str__(self):
        return f"K{self.K}-Lq{self.Lq}-D{self.D}-L{self.L}" + ("-knrm" if self.knrm else "")


def _c(*names):
    return tuple(sorted(names))


T, F = True, False
D_EDGE = simt_d_edge(25, 300)   # 484: the last D of the FFMA <32, 2> plan on an H100
MATRIX = (
    Row(1, 1, 4, 1, 4, F, 11, _c(inst(TS_STORE, 12), inst(SIMT_STORE, 12, 1)),
        "one live kernel slot; one query term; 16-byte rows; every passage at most one row (0 or 1 tile)"),
    Row(5, 31, 32, 8, 4, T, 12, _c(inst(TS_STORE, 12), inst(SIMT_STORE, 12, 1)),
        "KNRM form; D = 32: one 32-column chunk per tile, the operand ring under the most pressure"),
    Row(12, 32, 36, 48, 4, F, 13, _c(inst(TS_STORE, 12), inst(SIMT_STORE, 12, 1)),
        "exact <12>; Lq = 32; D = 36: a 4-column last chunk; max_doc_len 48: the last JR = 1 length"),
    Row(13, 33, 300, 49, 4, F, 14, _c(inst(TS_STORE, 24), inst(SIMT_STORE, 24, 2)),
        "Lq = 33: two query-block passes; max_doc_len 49: the first JR = 2 length"),
    Row(22, 96, 384, 300, 3, T, 15, _c(inst(TS_STORE, 24), inst(SIMT_STORE, 24, 2)),
        "KNRM form; Lq = 96: three query-block passes; passages of up to 3 tiles"),
    Row(24, 128, 32, 48, 3, F, 16, _c(inst(TS_STORE, 24), inst(SIMT_STORE, 24, 1)),
        "exact <24>; Lq = 128: four query-block passes at one 32-column chunk"),
    Row(25, 8, D_EDGE, 300, 4, F, 17, _c(inst(TS_STORE, 32), inst(SIMT_STORE, 32, 2)),
        "D at the FFMA <32, 2> kernel's shared-memory edge; 16 k-chunks per tile on the tensor cores"),
    Row(31, 129, 64, 8, 3, F, 18, _c(inst(SIMT_STORE, 32, 1)),
        "Lq = 129: past the tensor-core kernel, auto takes the FFMA kernel"),
    Row(11, 30, 300, 300, 4, F, 19, _c(inst(TS_STORE, 11), inst(SIMT_STORE, 12, 2)),
        "regression: TK / TK-Sparse at K = 11 over passages truncated to 300 rows"),
    Row(21, 30, 128, 256, 4, F, 20, _c(inst(TS_STORE, 21), inst(SIMT_STORE, 24, 2)),
        "regression: TK at K = 21; max_doc_len 256: a passage of exactly two full tiles"),
)

REQUIRED_FEATURES = frozenset(
    {f"K {k}" for k in (1, 5, 12, 13, 22, 24, 25, 31, 11, 21)}
    | {f"max_doc_len {n}" for n in (1, 8, 48, 49, 300)}
    | {f"Lq {n}" for n in (1, 31, 32, 33, 96, 128, 129)}
    | {f"D {n}" for n in (4, 32, 36, 300, 384)} | {"D at the FFMA edge", "KNRM form"})


def features(row: Row) -> frozenset:
    f = {f"K {row.K}", f"max_doc_len {row.L}", f"Lq {row.Lq}", f"D {row.D}"}
    if row.D == simt_d_edge(row.K, row.L):
        f.add("D at the FFMA edge")
    if row.knrm:
        f.add("KNRM form")
    return frozenset(f)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    q: torch.Tensor            # [n_q, Lq, D]; masked query rows hold data
    qm: torch.Tensor           # [n_q, Lq] bool
    buf: torch.Tensor          # [n_rows + TAIL_ROWS, D]; the store is buf[:n_rows], rows past it are NaN
    clean_buf: torch.Tensor    # buf with every poisoned row (unreferenced passages, the tail) replaced by finite rows
    n_rows: int
    off: torch.Tensor          # [n_docs + 1] int64
    gate: Optional[torch.Tensor]         # [n_rows]: >= 0, about a quarter 0; NaN on the poisoned rows
    clean_gate: Optional[torch.Tensor]
    referenced: torch.Tensor   # [n_docs] bool
    pair_q: torch.Tensor       # [P] int32, pairs of one query adjacent
    pair_d: torch.Tensor       # [P] int32, -1 = void
    mu: torch.Tensor
    sigma: torch.Tensor
    alpha: Optional[torch.Tensor]
    weight: torch.Tensor
    log_scale: float
    L: int                     # max_doc_len

    @property
    def store(self):
        return self.buf[:self.n_rows]

    def lengths(self) -> torch.Tensor:
        """Rows of every pair's passage the kernels read (0 for a void pair), [P] int64."""
        n = (self.off[1:] - self.off[:-1]).clamp(max=self.L)
        return torch.where(self.pair_d >= 0, n[self.pair_d.long().clamp(min=0)], torch.zeros_like(self.pair_d).long())

    def tiles(self) -> torch.Tensor:
        return (self.lengths() + 127) // 128

    def void(self) -> torch.Tensor:
        """Pairs that score -inf: pair_d < 0 or a passage without rows."""
        return self.lengths() == 0

    def unique_pairs(self):
        """(unique [U, 2] (query, passage) of the non-void pairs, inverse [P] index into it, -1 for void pairs)."""
        live = ~self.void()
        key = torch.stack([self.pair_q.long(), self.pair_d.long()], 1)
        u, inv = torch.unique(key[live], dim=0, return_inverse=True)
        full = torch.full((len(key),), -1, dtype=torch.int64)
        full[live] = inv
        return u, full


def _poison(n: int, D: int) -> torch.Tensor:
    """NaN, +inf and -inf rows, in turn."""
    vals = torch.tensor([float("nan"), float("inf"), float("-inf")])
    return vals[torch.arange(n) % 3].view(-1, 1).expand(n, D).clone()


def passage_lengths(L: int) -> Tuple[int, ...]:
    """The referenced passages of a store with max_doc_len L: LENGTHS clipped to L, two passages longer than L, and a
    last passage of length 1..7 (mod 8)."""
    last = L if L % 8 else L - 1
    return tuple(min(n, L) for n in LENGTHS) + (L + 1, 2 * L + 3, last)


def make_case(K: int, Lq: int, D: int, L: int, n_q: int, seed: int, *, knrm: bool = False, gate: bool = False,
              min_pairs: int = MIN_PAIRS, normalise: bool = False) -> Case:
    """A ragged store and at least ``min_pairs`` pairs over it:

    - passages of ``passage_lengths(L)`` rows, each row 1 of a passage a scaled copy of a query row (a cosine of 1);
      after every one of length % 8 != 0 an unreferenced passage of NaN / +-inf rows (NaN gates), which the tensor-core
      kernel's over-fetch of up to 7 rows reads; the last passage has length % 8 != 0 and the buffer the store is a view
      of continues with NaN rows;
    - pairs of one query adjacent, their tile counts following TILE_PATTERN (so pair_d -1 and the empty passage sit
      between non-empty pairs), every (query, passage) at several positions;
    - with ``gate``, a gate >= 0 that is exactly 0 on about a quarter of the rows."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(n_q, Lq, D, generator=g) * 0.4
    q_len = torch.randint(1, Lq + 1, (n_q,), generator=g)
    q_len[0] = Lq
    qm = torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)
    lens = passage_lengths(L)
    chunks, clean_chunks, doc_len, referenced = [], [], [], []
    for p, n in enumerate(lens):
        rows = torch.randn(n, D, generator=g) * 0.4
        if n >= 2:
            rows[1] = 2.0 * q[p % n_q, (7 * p) % int(q_len[p % n_q])]
        chunks.append(rows)
        clean_chunks.append(rows)
        doc_len.append(n)
        referenced.append(True)
        if n % 8 and p != len(lens) - 1:
            chunks.append(_poison(POISON_ROWS, D))
            clean_chunks.append(torch.randn(POISON_ROWS, D, generator=g) * 0.4)
            doc_len.append(POISON_ROWS)
            referenced.append(False)
    n_rows = sum(doc_len)
    buf = torch.cat(chunks + [torch.full((TAIL_ROWS, D), float("nan"))])
    clean_buf = torch.cat(clean_chunks + [torch.randn(TAIL_ROWS, D, generator=g) * 0.4])
    if normalise:
        buf, clean_buf = torch.nn.functional.normalize(buf, dim=-1), torch.nn.functional.normalize(clean_buf, dim=-1)
        q = torch.nn.functional.normalize(q, dim=-1)
    off = torch.zeros(len(doc_len) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.tensor(doc_len), 0)
    referenced = torch.tensor(referenced)
    gt = clean_gt = None
    if gate:
        clean_gt = torch.rand(n_rows, generator=g) * 1.5
        clean_gt[torch.rand(n_rows, generator=g) < 0.25] = 0.0
        gt = clean_gt.clone()
        for d in torch.nonzero(~referenced).view(-1).tolist():
            gt[int(off[d]):int(off[d + 1])] = float("nan")
    # pairs: per query, tile counts in TILE_PATTERN order, each bucket walked round-robin from a per-query start
    ids = torch.nonzero(referenced).view(-1).tolist()
    read = (off[1:] - off[:-1]).clamp(max=L)
    buckets: Dict[int, list] = {0: [-1]}
    for d in ids:
        buckets.setdefault(int((read[d] + 127) // 128), []).append(d)
    pattern = [t for t in TILE_PATTERN if t in buckets]
    per_q = math.ceil(min_pairs / n_q)
    pq, pd = [], []
    for qi in range(n_q):
        nxt = {t: qi for t in buckets}
        for i in range(per_q):
            t = pattern[i % len(pattern)]
            pd.append(buckets[t][nxt[t] % len(buckets[t])])
            nxt[t] += 1
            pq.append(qi)
    mu, sigma, alpha, weight = KP.kernel_set(K, g, knrm)
    return Case(q, qm, buf, clean_buf, n_rows, off, gt, clean_gt, referenced, torch.tensor(pq, dtype=torch.int32),
                torch.tensor(pd, dtype=torch.int32), mu, sigma, alpha, weight, 0.01 if knrm else 1.0, L)


def row_case(row: Row, gate: bool) -> Case:
    return make_case(row.K, row.Lq, row.D, row.L, row.n_q, row.seed + (100 if gate else 0), knrm=row.knrm, gate=gate)


def truncated(c: Case) -> Case:
    """The case with every passage physically cut to its first max_doc_len rows (offsets, rows and gates); the rows past
    the store view stay."""
    keep = torch.zeros(c.n_rows, dtype=torch.bool)
    for d in range(len(c.off) - 1):
        a, b = int(c.off[d]), int(c.off[d + 1])
        keep[a:min(b, a + c.L)] = True
    off = torch.zeros_like(c.off)
    off[1:] = torch.cumsum((c.off[1:] - c.off[:-1]).clamp(max=c.L), 0)
    cut = (lambda x: None if x is None else x[keep])
    return dataclasses.replace(c, buf=torch.cat([c.buf[:c.n_rows][keep], c.buf[c.n_rows:]]),
                               clean_buf=torch.cat([c.clean_buf[:c.n_rows][keep], c.clean_buf[c.n_rows:]]),
                               n_rows=int(keep.sum()), off=off, gate=cut(c.gate), clean_gate=cut(c.clean_gate))


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
REF_CHUNK_ELEMENTS = 4_000_000   # [pairs, Lq, Ld, K] fp64 elements per reference chunk (32 MB per intermediate)


def gather(c: Case, pair_q: torch.Tensor, pair_d: torch.Tensor, Ld: int) -> KP.Case:
    """The pairs in the padded layout of kernel_pool_cases (the store's rows in fp32; the gate zeros past a passage)."""
    from tk_store_cases import gather_padded
    d, dm, dg = gather_padded(c.clean_buf[:c.n_rows], c.off, pair_d, Ld, c.clean_gate)
    qi = pair_q.long()
    return KP.Case(c.q[qi], d, c.qm[qi].float(), dm.float(), c.mu, c.sigma, c.alpha, c.weight, dg,
                   torch.zeros(len(qi)), c.log_scale)


def reference(c: Case, clamp_min: float = KP.DEFAULT_FLOOR, bias: float = 0.0) -> Dict[str, torch.Tensor]:
    """``kernel_pool_cases.reference(grads=False)`` once per unique (query, passage), in chunks of at most
    REF_CHUNK_ELEMENTS activations over the referenced rows only (so no poisoned row enters it): score [P] fp64
    (-inf for void pairs), per_kernel [P, K] (0 for void pairs) and aS [U, Lq, K] with qm [U, Lq] of the unique pairs."""
    u, inv = c.unique_pairs()
    U, Lq, K = len(u), c.q.shape[1], c.mu.numel()
    read = (c.off[1:] - c.off[:-1]).clamp(max=c.L)
    ulen = read[u[:, 1]]
    order = torch.argsort(ulen)
    score_u = torch.empty(U, dtype=torch.float64)
    pk_u = torch.empty(U, K, dtype=torch.float64)
    aS_u = torch.empty(U, Lq, K, dtype=torch.float64)
    i = 0
    while i < U:
        j = i + 1
        while j < U and (j + 1 - i) * Lq * int(ulen[order[j]]) * K <= REF_CHUNK_ELEMENTS:
            j += 1
        sel = order[i:j]
        pc = gather(c, u[sel, 0], u[sel, 1], int(ulen[sel].max()))
        r = KP.reference(pc, clamp_min=clamp_min, bias=bias, grads=False)
        score_u[sel], pk_u[sel], aS_u[sel] = r["score"], r["per_kernel"], r["aS"]
        i = j
    live = inv >= 0
    score = torch.full((len(inv),), float("-inf"), dtype=torch.float64)
    pk = torch.zeros(len(inv), K, dtype=torch.float64)
    score[live], pk[live] = score_u[inv[live]], pk_u[inv[live]]
    return {"score": score, "per_kernel": pk, "aS": aS_u, "qm": c.qm[u[:, 0]]}
