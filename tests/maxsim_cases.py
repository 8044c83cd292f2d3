"""Shared cases of the max-sim envelope tests (no GPU): the routing rules of ``maxsim_fwd_device``, the shape matrix that
runs every compiled max-sim instantiation, seeded integer inputs on which every kernel's fp32 arithmetic is exact, and one
fp64 oracle of colbert.py:68-75 with an explicit argmax and the gradient written out from it.

Routing (``csrc/maxsim.cu:476-503``): ``auto`` and ``tcgen05`` first offer the shape to the queries-on-M kernel; outside
its envelope ``tcgen05`` and ``tcgen05_docm`` need ``tc_supported`` and run the documents-on-M kernel, ``simt`` and every
shape ``tc_supported`` refuses run the SIMT kernel, ``auto`` otherwise runs the documents-on-M kernel.  Neither
tensor-core launch falls back to another kernel when its tiles do not fit in shared memory: the call is refused.

- queries-on-M ``maxsim_qm_kernel<T, ARGMAX, STORE>`` (csrc/maxsim_qm.cu:536-584): f16 / bf16, Lq <= 32, dim 64 or 128,
  Ld <= 4096, no argmax in store mode, and at least 4 stages of ``dim * 128 + 1024`` bytes beside two query slots.
- documents-on-M ``maxsim_tc_kernel<T, KBS, NC>``: ``tc_supported`` (csrc/maxsim.cu:377-385) takes f16 / bf16,
  dim % 64 == 0 with 64 <= dim <= 1024, Lq <= 128 and no argmax; ``launch_tc`` (:410-460) sets NC = ceil(Lq / 32),
  KBS = 2 when dim / 64 is even, else 1, and keeps two query slots when they leave room for two document stages of
  ``KBS * 16 KB``, else one; with fewer than two stages beside one slot the call is refused.
- ``maxsim_simt_kernel<T>`` (:462-466): Lq <= 128 and ``(Lq * (dim + 1) + 8 * Lq) * 4`` bytes of shared memory.
- backward ``maxsim_bwd_d_kernel<T>``, ``maxsim_bwd_q_kernel<T>`` (csrc/maxsim_host.cu): any shape.
- e4m3 store ``maxsim_tc_fp8_kernel<KBS, NC>``: ``maxsim_store`` over float8_e4m3fn, auto / tcgen05_docm only, the
  documents-on-M plan over 1-byte elements (kblocks = dim / 128); residual codes ``maxsim_tc_residual_kernel<KBS, NC,
  bits>``: ``maxsim_store_residual``, the 16-bit plan with the [dim][2^bits] fp16 weight table beside the control block.
  Their rows are built by ``make_store_case`` and scored by ``store_oracle``.

Shared memory is the device's opt-in limit per block: 232 448 B on an H100 (``SMEM_OPTIN_H100``); the GPU tests read it
from the device."""
from __future__ import annotations

import functools
from dataclasses import dataclass
from typing import Dict, Optional

import torch

H, BF, F32, E4 = torch.float16, torch.bfloat16, torch.float32, torch.float8_e4m3fn
TNAME = {H: "__half", BF: "__nv_bfloat16", F32: "float"}
SHORT = {H: "f16", BF: "bf16", F32: "f32", E4: "e4m3"}
QM, TC, SIMT, BWD_D, BWD_Q = ("maxsim_qm_kernel", "maxsim_tc_kernel", "maxsim_simt_kernel", "maxsim_bwd_d_kernel",
                              "maxsim_bwd_q_kernel")
TC_FP8, TC_RES = "maxsim_tc_fp8_kernel", "maxsim_tc_residual_kernel"
KERNELS = (QM, TC, SIMT, BWD_D, BWD_Q, TC_FP8, TC_RES)
IMPLS = ("tcgen05", "tcgen05_docm", "simt", "auto")
ARGMAX_IMPLS = ("tcgen05", "simt", "auto")
SMEM_OPTIN_H100 = 232448
SM_COUNT_H100 = 132
FILL = -1000.0   # colbert.py:69

# queries-on-M (maxsim_qm.cu:52-78)
QM_MAX_LQ, QM_MAX_LD, QM_MAX_STAGES = 32, 4096, 32
QM_SHARED = 2 * 32 * 8 + 2 * 2 * 8 + 2 * 2 * 8 * 8 + 2 * 8 * 4 + 2 * 2 * 4   # sizeof(QmShared) = 880
# documents-on-M (maxsim.cu:147-160)
TC_MAX_STAGES, TC_KBLOCK_BYTES = 12, 128 * 128
TC_SHARED = 2 * 12 * 8 + 2 * 2 * 8 + 2 * 8 * 128 * 4                          # sizeof(TcShared) = 8416


def inst(kernel: str, *args) -> str:
    """Canonical instantiation name, e.g. ``maxsim_tc_kernel<__half,2,1>``."""
    return kernel + "<" + ",".join(str(a).lower() if isinstance(a, bool) else str(a) for a in args) + ">"


def qm_handles(dtype, Lq: int, Ld: int, dim: int, argmax: bool, store: bool, smem: int) -> bool:
    """maxsim_qm_launch, maxsim_qm.cu:536-549 (the pointers are 16-byte aligned here)."""
    if dtype not in (H, BF) or Lq > QM_MAX_LQ or dim not in (64, 128) or Ld > QM_MAX_LD or (store and argmax):
        return False
    kblocks = dim // 64
    fixed = 2 * kblocks * 32 * 128 + QM_SHARED + 1024
    stages = min(QM_MAX_STAGES, (smem - fixed) // (kblocks * 64 * 128 + 1024)) & ~1
    return stages >= 4


def tc_supported(dtype, Lq: int, dim: int, argmax: bool) -> bool:
    """maxsim.cu:377-385 (Ld >= 1 and 16-byte alignment always hold here)."""
    return dtype in (H, BF) and dim % 64 == 0 and 64 <= dim <= 1024 and 1 <= Lq <= 128 and not argmax


def plan_tc(Lq: int, dim: int, smem: int, esize: int = 2, extra: int = 0) -> Optional[Dict[str, int]]:
    """plan_tc, maxsim.cu:529-552, over elements of ``esize`` bytes with ``extra`` bytes of shared memory after the
    control block: KBS, NC, query slots and stages; None where the query tile does not fit (MMB200_ERR_UNSUPPORTED)."""
    npad = (Lq + 31) // 32 * 32
    kblocks = dim * esize // 128
    kbs = 2 if kblocks % 2 == 0 else 1
    qslot = kblocks * npad * 128
    for qslots in (2, 1):
        fixed = qslots * qslot + TC_SHARED + extra + 1024
        stages = min(TC_MAX_STAGES, int((smem - fixed) / (kbs * TC_KBLOCK_BYTES)))   # C++ division truncates
        if stages >= 2:
            return {"kbs": kbs, "nc": npad // 32, "qslots": qslots, "stages": stages}
    return None


def tc_launch(Lq: int, dim: int, smem: int) -> Optional[Dict[str, int]]:
    """launch_tc over 16-bit elements (maxsim.cu:565-597)."""
    return plan_tc(Lq, dim, smem)


def residual_extra(dim: int, bits: int) -> int:
    """The shared-memory weight table of the residual max-sim: [dim][2^bits] fp16 (maxsim.cu:742)."""
    return (dim << bits) * 2


def route_e4m3(Lq: int, dim: int, impl: str, smem: int = SMEM_OPTIN_H100) -> Optional[str]:
    """maxsim_store_fp8, maxsim.cu:646-661: only auto and tcgen05_docm, on maxsim_tc_fp8_kernel<KBS, NC> with
    kblocks = dim / 128; dim % 128 == 0, 128 <= dim <= 1024, Lq <= 128; None where the call is refused."""
    if impl not in ("auto", "tcgen05_docm") or dim % 128 or not 128 <= dim <= 1024 or not 1 <= Lq <= 128:
        return None
    L = plan_tc(Lq, dim, smem, 1, 0)
    return None if L is None else inst(TC_FP8, L["kbs"], L["nc"])


def route_residual(Lq: int, dim: int, bits: int, smem: int = SMEM_OPTIN_H100) -> Optional[str]:
    """mmb200_maxsim_store_residual_fwd, maxsim.cu:718-753: maxsim_tc_residual_kernel<KBS, NC, bits> over 16-bit
    k-blocks with the weight table beside the control block; None where the call is refused."""
    if bits not in (1, 2) or dim % 64 or not 64 <= dim <= 1024 or not 1 <= Lq <= 128:
        return None
    L = plan_tc(Lq, dim, smem, 2, residual_extra(dim, bits))
    return None if L is None else inst(TC_RES, L["kbs"], L["nc"], bits)


def last_lq_e4m3(dim: int, smem: int = SMEM_OPTIN_H100) -> int:
    return max([lq for lq in range(1, 130) if route_e4m3(lq, dim, "auto", smem)] or [0])


def last_lq_residual(dim: int, bits: int, smem: int = SMEM_OPTIN_H100) -> int:
    return max([lq for lq in range(1, 130) if route_residual(lq, dim, bits, smem)] or [0])


def simt_fits(Lq: int, dim: int, smem: int) -> bool:
    """launch_simt, maxsim.cu:462-466."""
    return Lq <= 128 and (Lq * (dim + 1) + 8 * Lq) * 4 <= smem


def route(dtype, Lq: int, Ld: int, dim: int, impl: str, argmax: bool = False, store: bool = False,
          smem: int = SMEM_OPTIN_H100) -> Optional[str]:
    """The instantiation maxsim_fwd_device runs for one call (maxsim.cu:476-503), or None where the host refuses it."""
    T = TNAME[dtype]
    if impl in ("auto", "tcgen05") and qm_handles(dtype, Lq, Ld, dim, argmax, store, smem):
        return inst(QM, T, argmax, store)
    ok = tc_supported(dtype, Lq, dim, argmax)
    if impl in ("tcgen05", "tcgen05_docm") and not ok:
        return None
    if impl == "simt" or not ok:
        return inst(SIMT, T) if simt_fits(Lq, dim, smem) else None
    L = tc_launch(Lq, dim, smem)
    return None if L is None else inst(TC, T, L["kbs"], L["nc"])


def last_lq(dtype, dim: int, argmax: bool, smem: int = SMEM_OPTIN_H100) -> int:
    """The largest Lq that ``auto`` runs at this dim (with the argmax: the training forward); 0 if none."""
    return max([lq for lq in range(1, 130) if route(dtype, lq, 64, dim, "auto", argmax, smem=smem)] or [0])


@dataclass(frozen=True)
class Row:
    dtype: torch.dtype
    n_q: int
    dpq: int            # docs_per_query (pairs and store mode)
    n_d: int
    Lq: int
    Ld: int             # max_doc_len in store mode
    dim: int
    mode: str           # "pairs" (docs_per_query), "inbatch" (maxsim_allpairs, reference mask indexing), "store",
                        # "residual" (maxsim_store_residual over both code widths); an E4 store row is the e4m3 store
    seed: int
    claims: tuple
    why: str
    regime: str = "rand"   # e4m3 / residual store rows: "rand", or "neg" (every product a window holds is < 0)
    pairs: int = 0         # e4m3 / residual store rows: the number of pairs

    @property
    def n_pairs(self) -> int:
        if self.pairs:
            return self.pairs
        return self.n_q * self.n_d if self.mode == "inbatch" else self.n_d

    @property
    def coded(self) -> bool:
        """An e4m3 or residual store row (make_store_case, store_oracle)."""
        return self.dtype == E4 or self.mode == "residual"

    def __str__(self):
        if self.coded:
            return (f"{'e4m3-store' if self.dtype == E4 else 'residual'}-nq{self.n_q}-nd{self.n_d}-p{self.pairs}"
                    f"-Lq{self.Lq}-Ld{self.Ld}-d{self.dim}-{self.regime}")
        return f"{SHORT[self.dtype]}-{self.mode}-nq{self.n_q}x{self.dpq}-nd{self.n_d}-Lq{self.Lq}-Ld{self.Ld}-d{self.dim}"


def runs(row: Row, smem: int = SMEM_OPTIN_H100) -> Dict[tuple, Optional[str]]:
    """What the envelope test calls for a row: ("score", impl) and, outside store mode, ("argmax", impl), each mapped to
    the instantiation it runs or None (refused); ("bwd",) in pairs mode maps to the two backward kernels.  An e4m3
    store row: ("score", impl) through maxsim_store; a residual row: ("residual", bits) for 1- and 2-bit codes."""
    if row.dtype == E4:
        return {("score", impl): route_e4m3(row.Lq, row.dim, impl, smem) for impl in IMPLS}
    if row.mode == "residual":
        return {("residual", b): route_residual(row.Lq, row.dim, b, smem) for b in RESIDUAL_BITS}
    store = row.mode == "store"
    out = {("score", impl): route(row.dtype, row.Lq, row.Ld, row.dim, impl, False, store, smem) for impl in IMPLS}
    if not store:
        out.update({("argmax", impl): route(row.dtype, row.Lq, row.Ld, row.dim, impl, True, False, smem)
                    for impl in ARGMAX_IMPLS})
    if row.mode == "pairs":
        out[("bwd",)] = inst(BWD_D, TNAME[row.dtype]) + " " + inst(BWD_Q, TNAME[row.dtype])
    return out


def dispatched(row: Row, smem: int = SMEM_OPTIN_H100) -> frozenset:
    """The set of instantiations the envelope test runs for a row."""
    names = set()
    for v in runs(row, smem).values():
        if v is not None:
            names.update(v.split(" "))
    return frozenset(names)


def features(row: Row, smem: int = SMEM_OPTIN_H100) -> frozenset:
    """Launch configurations and cases the matrix must hold, derived from the row's shape."""
    if row.coded:
        return _coded_features(row, smem)
    f = set()
    T = SHORT[row.dtype]
    r = runs(row, smem)
    if (row.dtype, row.Lq, row.Ld, row.dim) == (H, 30, 200, 768):
        f.add({"pairs": "reference configuration", "inbatch": "reference in-batch scoring"}.get(row.mode, ""))
    if row.Ld in (127, 128, 129, 256, 257, 4097):
        f.add(f"Ld {row.Ld}")
    if r[("score", "tcgen05_docm")] is not None:
        L = tc_launch(row.Lq, row.dim, smem)
        if L["qslots"] == 1:
            f.add(f"one query slot {T}")
        if L["stages"] == 2:
            f.add(f"two-stage ring {T}")
        if row.dim == 1024:
            f.add(f"documents-on-M at dim 1024 {T}")
        if row.mode == "store" and row.dtype == BF and row.Lq > 32:
            f.add("bf16 store mode on the documents-on-M kernel, Lq > 32")
    if r.get(("argmax", "simt")) is not None:
        if 33 <= row.Lq <= 96:
            f.add("SIMT argmax, Lq 33-96")
        if row.Lq > 96:
            f.add("SIMT argmax, Lq 97-128 (four tokens per lane)")
        if row.dim == 768:
            f.add("SIMT argmax at dim 768")
        if row.Lq == last_lq(row.dtype, row.dim, True) < 128:
            f.add("SIMT argmax at the last Lq of its dim")
    if row.mode == "pairs" and row.dim in (64, 100, 128, 768):
        f.add(f"backward {T} dim {row.dim}")
    if row.mode == "pairs" and row.dpq > 1 and row.n_d % row.dpq:
        f.add("partial last query")
    if row.Lq == 1 and row.Ld == 1:
        f.add("Lq 1, Ld 1")
    if row.n_pairs > SM_COUNT_H100:
        f.add("more pairs than SMs")
    f.discard("")
    return frozenset(f)


RESIDUAL_BITS = (1, 2)
# passage lengths of every e4m3 / residual store row: empty, one row, and both sides of the 64-row chunk and 128-row tile
LAYOUT = (0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257)
LQ_EDGES = (1, 32, 33, 64, 65, 96, 97, 128)


def _coded_features(row: Row, smem: int = SMEM_OPTIN_H100) -> frozenset:
    """The features of an e4m3 or residual store row, named by its kernel family (none is shared with the 16-bit rows)."""
    fam = "e4m3" if row.dtype == E4 else "residual"
    f = {f"{fam} {row.regime}"}
    if row.pairs == 1:
        f.add(f"{fam} single pair")
    else:
        f.update(f"{fam} passage of {n} rows" for n in LAYOUT if n <= row.Ld)
        if row.Ld % 128:   # make_store_case draws lengths up to Ld + 40: some passages are longer (asserted)
            f.add(f"{fam} max_doc_len not a multiple of 128, longer passages truncated")
        f.update({f"{fam} passage ends at the last store row", f"{fam} pair_d -1", f"{fam} one passage, many queries"})
        if row.n_q >= 3:
            f.add(f"{fam} unsorted pair_q returning to earlier queries")
    if row.n_pairs > SM_COUNT_H100:
        f.add(f"{fam} more pairs than SMs")
    if row.Lq in LQ_EDGES:
        f.add(f"{fam} Lq {row.Lq}")
    if row.dtype == E4:
        L = plan_tc(row.Lq, row.dim, smem, 1, 0)
        if L["kbs"] == 1:
            f.add("e4m3 KBS 1 at dim 128" if row.dim == 128 else "e4m3 KBS 1 over several k-blocks")
        if row.dim == 1024 and row.Lq == 128:
            f.add("e4m3 Lq 128 at dim 1024")
        if row.regime == "rand" and row.pairs != 1:
            f.add("e4m3 subnormal passage")
        plans = [L]
    else:
        plans = [plan_tc(row.Lq, row.dim, smem, 2, residual_extra(row.dim, b)) for b in RESIDUAL_BITS]
        if row.dim == 1024 and row.Lq == last_lq_residual(1024, 2, smem):
            f.add("residual dim 1024 at its last Lq")
    if any(L["qslots"] == 1 for L in plans):
        f.add(f"{fam} one query slot")
    if any(L["stages"] == 2 for L in plans):
        f.add(f"{fam} two-stage ring")
    return frozenset(f)


CODED_REQUIRED_FEATURES = frozenset(
    {f"{fam} {x}" for fam in ("e4m3", "residual") for x in
     ("rand", "neg", "single pair", "max_doc_len not a multiple of 128, longer passages truncated",
      "passage ends at the last store row", "pair_d -1", "one passage, many queries",
      "unsorted pair_q returning to earlier queries", "more pairs than SMs", "one query slot", "two-stage ring")}
    | {f"{fam} passage of {n} rows" for fam in ("e4m3", "residual") for n in LAYOUT}
    | {f"e4m3 Lq {n}" for n in LQ_EDGES} | {f"residual Lq {n}" for n in (1, 32, 64, 96, 128)}
    | {"e4m3 KBS 1 at dim 128", "e4m3 KBS 1 over several k-blocks", "e4m3 Lq 128 at dim 1024", "e4m3 subnormal passage",
       "residual dim 1024 at its last Lq"})


REQUIRED_FEATURES = CODED_REQUIRED_FEATURES | frozenset(
    {"reference configuration", "reference in-batch scoring", "bf16 store mode on the documents-on-M kernel, Lq > 32",
     "SIMT argmax, Lq 33-96", "SIMT argmax, Lq 97-128 (four tokens per lane)", "SIMT argmax at dim 768",
     "SIMT argmax at the last Lq of its dim", "partial last query", "more pairs than SMs", "Lq 1, Ld 1"}
    | {f"documents-on-M at dim 1024 {t}" for t in ("f16", "bf16")}
    | {f"Ld {n}" for n in (127, 128, 129, 256, 257, 4097)}
    | {f"{k} {t}" for k in ("one query slot", "two-stage ring") for t in ("f16", "bf16")}
    | {f"backward {t} dim {n}" for t in ("f32", "f16", "bf16") for n in (64, 100, 128, 768)})


def _c(*names):
    return tuple(sorted(names))


def _tc(dt, kbs, nc):
    return inst(TC, TNAME[dt], kbs, nc)


def _qm(dt, argmax, store):
    return inst(QM, TNAME[dt], argmax, store)


def _simt(dt):
    return inst(SIMT, TNAME[dt])


def _bwd(dt):
    return (inst(BWD_D, TNAME[dt]), inst(BWD_Q, TNAME[dt]))


def _f8(kbs, nc):
    return inst(TC_FP8, kbs, nc)


def _res(kbs, nc):
    return tuple(inst(TC_RES, kbs, nc, b) for b in RESIDUAL_BITS)


MATRIX = (
    Row(H, 4, 3, 11, 30, 200, 768, "pairs", 1, _c(_tc(H, 2, 1), _simt(H), *_bwd(H)),
        "the reference configuration (colbert.yaml: dim 768, Lq 30, Ld 200): <__half,2,1>, 2 query slots, 3 stages; "
        "training on the SIMT argmax; the last query has 2 of its 3 documents"),
    Row(H, 6, 1, 6, 30, 200, 768, "inbatch", 2, _c(_tc(H, 2, 1), _simt(H)),
        "in-batch teacher scoring at the reference configuration (colbert.py:154-162, pair_dmask indirection)"),
    Row(H, 3, 5, 14, 32, 127, 64, "pairs", 3, _c(_qm(H, False, False), _qm(H, True, False), _tc(H, 1, 1), _simt(H), *_bwd(H)),
        "queries-on-M at Lq 32, dim 64 and both argmax producers; Ld 127 one row short of a 128-row tile"),
    Row(BF, 70, 4, 279, 17, 129, 128, "pairs", 4,
        _c(_qm(BF, False, False), _qm(BF, True, False), _tc(BF, 2, 1), _simt(BF), *_bwd(BF)),
        "bf16 queries-on-M with argmax over 279 pairs (every CTA walks several, the query changes every 4); Ld 129"),
    Row(BF, 3, 2, 6, 1, 1, 64, "pairs", 5, _c(_qm(BF, False, False), _qm(BF, True, False), _tc(BF, 1, 1), _simt(BF), *_bwd(BF)),
        "one query token, one document row: <__nv_bfloat16,1,1>"),
    Row(H, 2, 3, 5, 64, 256, 192, "pairs", 6, _c(_tc(H, 1, 2), _simt(H), *_bwd(H)),
        "<__half,1,2>: three k-blocks, two query chunks; Ld 256 = two full tiles"),
    Row(BF, 2, 3, 6, 40, 257, 64, "pairs", 7, _c(_tc(BF, 1, 2), _simt(BF), *_bwd(BF)),
        "<__nv_bfloat16,1,2>; Ld 257: one row into a third tile"),
    Row(H, 3, 2, 5, 96, 128, 128, "pairs", 8, _c(_tc(H, 2, 3), _simt(H), *_bwd(H)),
        "<__half,2,3> at Lq 96, the last three-chunk length; Ld 128 = one full tile"),
    Row(H, 3, 2, 5, 65, 100, 320, "pairs", 9, _c(_tc(H, 1, 3), _simt(H), *_bwd(H)),
        "<__half,1,3> at Lq 65, the first three-chunk length; five k-blocks"),
    Row(BF, 3, 2, 5, 80, 150, 256, "pairs", 10, _c(_tc(BF, 2, 3), _simt(BF), *_bwd(BF)),
        "<__nv_bfloat16,2,3>"),
    Row(BF, 3, 2, 5, 70, 60, 192, "pairs", 11, _c(_tc(BF, 1, 3), _simt(BF), *_bwd(BF)),
        "<__nv_bfloat16,1,3>; a document shorter than one tile"),
    Row(H, 3, 2, 5, 128, 129, 64, "pairs", 12, _c(_tc(H, 1, 4), _simt(H), *_bwd(H)),
        "<__half,1,4>: Lq 128; the SIMT argmax of tokens 97-127 (four tokens per lane)"),
    Row(BF, 2, 3, 5, 128, 70, 256, "pairs", 13, _c(_tc(BF, 2, 4), _simt(BF), *_bwd(BF)),
        "<__nv_bfloat16,2,4> at Lq 128"),
    Row(H, 3, 2, 5, 113, 90, 128, "pairs", 14, _c(_tc(H, 2, 4), _simt(H), *_bwd(H)),
        "<__half,2,4>: a ragged fourth query chunk"),
    Row(BF, 3, 2, 5, 100, 80, 448, "pairs", 15, _c(_tc(BF, 1, 4), _simt(BF), *_bwd(BF)),
        "<__nv_bfloat16,1,4>: seven k-blocks, one query slot"),
    Row(BF, 2, 3, 5, 40, 100, 768, "pairs", 17, _c(_tc(BF, 2, 2), _simt(BF), *_bwd(BF)),
        "bf16 one query slot at dim 768; the bf16 backward at dim 768"),
    Row(H, 3, 2, 5, 74, 200, 768, "pairs", 18, _c(_tc(H, 2, 3), _simt(H), *_bwd(H)),
        "f16 one query slot and two stages (dim 768, Lq 65-96); Lq 74 is the last the SIMT argmax takes at dim 768"),
    Row(BF, 2, 2, 4, 20, 130, 1024, "pairs", 19, _c(_tc(BF, 2, 1), _simt(BF), *_bwd(BF)),
        "bf16 two-stage ring with two query slots (dim 1024)"),
    Row(H, 2, 2, 4, 64, 64, 1024, "pairs", 20, _c(_tc(H, 2, 2), *_bwd(H)),
        "dim 1024, Lq 64: the documents-on-M kernel's last Lq there (one slot, two stages); the SIMT kernel and so "
        "the training forward refuse it"),
    Row(H, 1, 2, 2, 32, 4097, 128, "pairs", 21, _c(_tc(H, 2, 1), _simt(H), *_bwd(H)),
        "Ld 4097: beyond the queries-on-M kernel, so tcgen05 and auto take the documents-on-M kernel"),
    Row(H, 3, 4, 12, 32, 180, 128, "store", 22, _c(_qm(H, False, True), _tc(H, 2, 1), _simt(H)),
        "f16 store mode on the queries-on-M kernel; passages longer than max_doc_len"),
    Row(BF, 3, 4, 10, 20, 90, 64, "store", 23, _c(_qm(BF, False, True), _tc(BF, 1, 1), _simt(BF)),
        "bf16 store mode on the queries-on-M kernel"),
    Row(BF, 2, 3, 6, 48, 150, 128, "store", 24, _c(_tc(BF, 2, 2), _simt(BF)),
        "bf16 store mode on the documents-on-M kernel with Lq > 32"),
    Row(F32, 3, 2, 5, 16, 40, 64, "pairs", 25, _c(_simt(F32), *_bwd(F32)), "f32, dim 64"),
    Row(F32, 3, 2, 5, 33, 50, 100, "pairs", 26, _c(_simt(F32), *_bwd(F32)), "f32, dim 100"),
    Row(F32, 3, 2, 5, 32, 60, 128, "pairs", 27, _c(_simt(F32), *_bwd(F32)), "f32, dim 128"),
    Row(F32, 2, 2, 4, 30, 200, 768, "pairs", 28, _c(_simt(F32), *_bwd(F32)), "f32 at the reference configuration"),
    Row(H, 3, 2, 5, 30, 50, 100, "pairs", 29, _c(_simt(H), *_bwd(H)),
        "dim 100 (not a multiple of 64): only the SIMT kernel; the tensor-core names are refused"),
    Row(BF, 3, 2, 5, 30, 50, 100, "pairs", 30, _c(_simt(BF), *_bwd(BF)), "bf16 at dim 100"),
    # ---- e4m3 store (maxsim_store over float8_e4m3fn): maxsim_tc_fp8_kernel<KBS, NC>, kblocks = dim / 128
    Row(E4, 4, 1, 20, 1, 300, 128, "store", 40, _c(_f8(1, 1)),
        "<1,1>: one query token at dim 128 (one k-block); 400 pairs over 4 queries", pairs=400),
    Row(E4, 5, 1, 18, 33, 260, 384, "store", 41, _c(_f8(1, 2)),
        "<1,2>: three k-blocks through KBS 1, the first two-chunk Lq; every product a window holds < 0", regime="neg",
        pairs=300),
    Row(E4, 4, 1, 16, 65, 300, 640, "store", 42, _c(_f8(1, 3)), "<1,3>: five k-blocks, the first three-chunk Lq",
        pairs=280),
    Row(E4, 4, 1, 14, 97, 270, 896, "store", 43, _c(_f8(1, 4)),
        "<1,4>: seven k-blocks, the first four-chunk Lq, one query slot", regime="neg", pairs=200),
    Row(E4, 6, 1, 20, 32, 333, 256, "store", 44, _c(_f8(2, 1)), "<2,1>: 600 pairs over 6 queries", pairs=600),
    Row(E4, 4, 1, 16, 64, 290, 512, "store", 45, _c(_f8(2, 2)), "<2,2> at the last two-chunk Lq", regime="neg",
        pairs=300),
    Row(E4, 4, 1, 14, 96, 300, 768, "store", 46, _c(_f8(2, 3)), "<2,3> at the last three-chunk Lq", pairs=200),
    Row(E4, 4, 1, 14, 128, 300, 1024, "store", 47, _c(_f8(2, 4)),
        "<2,4>: Lq 128 at dim 1024 (where the fp16 kernel stops at 64): one query slot, two stages", regime="neg",
        pairs=160),
    Row(E4, 1, 1, 12, 1, 300, 1024, "store", 48, _c(_f8(2, 1)), "a single pair at dim 1024", pairs=1),
    # ---- residual codes (maxsim_store_residual, 1- and 2-bit codes): maxsim_tc_residual_kernel<KBS, NC, bits>
    Row(H, 4, 1, 16, 1, 300, 64, "residual", 50, _c(*_res(1, 1)), "<1,1,b>: one token, dim 64", pairs=400),
    Row(H, 4, 1, 16, 40, 260, 192, "residual", 51, _c(*_res(1, 2)), "<1,2,b>: three k-blocks", regime="neg",
        pairs=300),
    Row(H, 4, 1, 16, 70, 300, 320, "residual", 52, _c(*_res(1, 3)), "<1,3,b>: five k-blocks", pairs=250),
    Row(H, 4, 1, 14, 128, 270, 704, "residual", 53, _c(*_res(1, 4)),
        "<1,4,b>: Lq 128 at dim 704, past 640 and 768 where the envelope stops at 96", regime="neg", pairs=200),
    Row(H, 5, 1, 20, 32, 333, 128, "residual", 54, _c(*_res(2, 1)), "<2,1,b>: 600 pairs over 5 queries", pairs=600),
    Row(H, 4, 1, 14, 64, 300, 1024, "residual", 55, _c(*_res(2, 2)),
        "<2,2,b>: dim 1024 at its last Lq, one query slot, two stages", regime="neg", pairs=200),
    Row(H, 4, 1, 16, 96, 290, 256, "residual", 56, _c(*_res(2, 3)), "<2,3,b>", pairs=250),
    Row(H, 4, 1, 14, 128, 300, 512, "residual", 57, _c(*_res(2, 4)), "<2,4,b> at Lq 128", pairs=200),
    Row(H, 1, 1, 12, 30, 300, 64, "residual", 58, _c(*_res(1, 1)), "a single pair", pairs=1),
)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
# documents with a constructed purpose (index into the batch), where the batch has room for them
FULL_DOC, FILL_DOC, TIE1000_DOC, REALTIE_DOC, MASKED_DOC = 0, 1, 2, 3, 4
TIE1000_MASKED, TIE1000_REAL = 2, 6            # j and j' = j + 4: the same row stride of the SIMT kernel's warp 2
REALTIE_ROWS = (3, 4, 7, 67)                   # equal real rows across warps, inside one warp's stride, across chunks
POISON = (float("nan"), float("inf"), float("-inf"))


@dataclass
class Case:
    q: torch.Tensor          # [n_q, Lq, dim] f32 holding small integers (representable in f16 and bf16)
    d: torch.Tensor          # [n_d, Ld, dim] f32; store mode: each passage's first min(len, Ld) rows, zero padded
    qm: torch.Tensor         # [n_q, Lq] int64 (all ones in store mode)
    dm: torch.Tensor         # [n_d, Ld] int64 (store mode: rows < len)
    pair_q: torch.Tensor     # [n_pairs] int64
    pair_d: torch.Tensor
    pair_dm: torch.Tensor    # the document-mask row of each pair
    gout: torch.Tensor       # [n_pairs] f32 integers
    lens: Optional[torch.Tensor] = None    # store mode: passage lengths (some beyond Ld)
    store: Optional[torch.Tensor] = None   # store mode: [n_rows, dim] f32, rows past max_doc_len and a tail poisoned
    offsets: Optional[torch.Tensor] = None


def row_with_dot(u: torch.Tensor, target: int) -> torch.Tensor:
    """A document row with entries in [-8, 3] whose dot product with u = [1, 3, 3, ...] is exactly ``target``
    (-8 * sum(u) <= target <= -8 * sum(u) + 11 * sum(u))."""
    dim = u.numel()
    r = torch.full((dim,), -8.0)
    delta = target - int((u * r).sum())
    assert delta >= 0, "target below the reach of the row"
    r[0] += delta % 3
    steps = delta // 3
    for k in range(1, dim):
        if steps == 0:
            break
        s = min(11, steps)
        r[k] += s
        steps -= s
    assert steps == 0 and int((u * r).sum()) == target
    return r


@functools.lru_cache(maxsize=None)
def make_case(row: Row) -> Case:
    """Seeded integers in [-3, 3]: every dot product, score and gradient sum is an integer below 2^24, so exact in fp32
    whatever the order.  Query masks with holes, a fully masked query (3 or more queries); document masks with holes
    and ragged lengths, document 0 fully live.  Where the batch has room: a document whose real rows all score below
    -1000 against one token (the fill wins), one where a real row scores exactly -1000 four rows after a masked row, one
    with equal real rows that hold the maximum, and a fully masked document."""
    assert not row.coded, f"{row}: e4m3 and residual store rows are built by make_store_case"
    g = torch.Generator().manual_seed(1000 + row.seed)
    n_q, n_d, Lq, Ld, dim = row.n_q, row.n_d, row.Lq, row.Ld, row.dim
    q = torch.randint(-3, 4, (n_q, Lq, dim), generator=g).float()
    store = row.mode == "store"
    Lgen = Ld + 9 if store else Ld
    d = torch.randint(-3, 4, (n_d, Lgen, dim), generator=g).float()
    qm = (torch.rand(n_q, Lq, generator=g) > 0.15).long()
    qm[0] = 1
    if row.mode == "pairs" and n_q >= 3 and n_q - 1 > REALTIE_DOC // row.dpq:
        qm[n_q - 1] = 0                  # a query with no live token (none of the constructed documents is its)
    if not store and Lq >= 3:
        qm[n_q - 1, Lq - 1] = 0
    if store:
        qm[:] = 1
    lens = torch.randint(max(1, Ld // 2), Lgen + 1, (n_d,), generator=g)
    lens[0], lens[-1] = Ld, Lgen
    dm = (torch.arange(Lgen).unsqueeze(0) < lens.unsqueeze(1)).long()
    if not store:
        dm &= (torch.rand(n_d, Lgen, generator=g) > 0.1).long()
        dm[0] = 1
    if row.mode == "inbatch":
        dm[:, -3:] = 0   # a tail masked in every document: the rows the reference mask indexing never reads
    pair_q = torch.arange(row.n_pairs) // (n_d if row.mode == "inbatch" else row.dpq)
    pair_d = torch.arange(row.n_pairs) % n_d if row.mode == "inbatch" else torch.arange(n_d)
    pair_dm = pair_q.clone() if row.mode == "inbatch" else pair_d.clone()
    special = row.mode != "inbatch" and Ld >= 8
    if special:
        # token 0 of the query of FILL_DOC and TIE1000_DOC is u = [1, 3, 3, ...]; -8 * sum(u) < -1000 from dim 64 on
        u = torch.full((dim,), 3.0)
        u[0] = 1.0
        for p in (FILL_DOC, TIE1000_DOC):
            if p >= n_d:
                continue
            qi = int(pair_q[p])
            q[qi, 0] = u
            qm[qi, 0] = 1
            lo = -8 * int(u.sum())
            for j in range(Lgen):
                d[p, j] = row_with_dot(u, int(torch.randint(lo, -1000, (1,), generator=g)))
            if not store:
                dm[p, :Ld] = 1
                dm[p, Ld - 1] = 0        # a masked row: the fill exists
                if p == TIE1000_DOC:
                    dm[p, TIE1000_MASKED] = 0
                    d[p, TIE1000_REAL] = row_with_dot(u, -1000)
                    dm[p, TIE1000_REAL] = 1
    if special and n_d > REALTIE_DOC and Lq >= 2:
        qi = int(pair_q[REALTIE_DOC])
        qm[qi, 1] = 1
        w = torch.where(q[qi, 1] >= 0, 3.0, -3.0)    # the largest dot any row in [-3, 3] reaches with token 1
        for j in REALTIE_ROWS:
            if j < Ld:
                d[REALTIE_DOC, j] = w
                dm[REALTIE_DOC, j] = 1
    if n_d > MASKED_DOC and not store and row.mode != "inbatch":
        dm[MASKED_DOC] = 0

    gout = torch.randint(-3, 4, (row.n_pairs,), generator=g).float()
    gout[gout == 0] = 2.0
    if not store:
        return Case(q, d, qm, dm, pair_q, pair_d, pair_dm, gout)
    # store mode: passage p is rows [off[p], off[p] + lens[p]); only the first Ld (max_doc_len) are read
    rows = [d[p, :int(lens[p])].clone() for p in range(n_d)]
    for p in range(n_d):
        rows[p][Ld:] = POISON[p % 3]
    tail = torch.full((3, dim), float("nan"))
    store_t = torch.cat(rows + [tail])
    offsets = torch.zeros(n_d + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(lens, 0)
    live = torch.minimum(lens, torch.tensor(Ld))
    dm = (torch.arange(Ld).unsqueeze(0) < live.unsqueeze(1)).long()
    dd = d[:, :Ld].clone() * dm.unsqueeze(-1)
    return Case(q, dd, qm, dm, pair_q, pair_d, pair_dm, gout, lens, store_t, offsets)


def poisoned(c: Case, row: Row):
    """q and d with NaN / +inf / -inf in every masked query token and in every document row no pair reads (masked rows;
    in-batch scoring with the reference mask indexing: rows masked in every document)."""
    q, d = c.q.clone(), c.d.clone()
    for i, (a, b) in enumerate((~c.qm.bool()).nonzero().tolist()):
        q[a, b] = POISON[i % 3]
    dead = ~c.dm.bool()
    if row.mode == "inbatch":
        dead = dead.all(0, keepdim=True).expand_as(dead)
    for i, (a, b) in enumerate(dead.nonzero().tolist()):
        d[a, b] = POISON[i % 3]
    return q, d


# ---------------------------------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------------------------------
def oracle(c: Case, fill: bool = True):
    """fp64 colbert.py:68-75 per pair with an explicit argmax: score [n_pairs], argmax [n_pairs, Lq] (int64).

    The max of token i over the document is taken over its real rows and, when the document has a masked position, the
    -1000 fill.  The argmax is the first maximal real row; a real row wins an exact tie against the fill; -1 when the
    fill wins or the query token is masked.  ``fill=False``: store mode, where rows past a passage's length are not
    candidates at all."""
    Q = c.q.double()[c.pair_q]
    D = c.d.double()[c.pair_d]
    S = torch.bmm(Q, D.transpose(1, 2))                           # colbert.py:68
    real = c.dm.bool()[c.pair_dm]                                 # [P, Ld]
    has_fill = (~real).any(-1, keepdim=True) & fill               # [P, 1]
    V = S.masked_fill(~real.unsqueeze(1), float("-inf"))
    best = V.max(-1).values
    j = torch.arange(V.shape[-1])
    first = torch.where(V == best.unsqueeze(-1), j, V.shape[-1]).min(-1).values
    fill_wins = has_fill & (best < FILL)
    m = torch.where(fill_wins, torch.full_like(best, FILL), best)  # colbert.py:69-71
    arg = torch.where(fill_wins | torch.isinf(best), torch.full_like(first, -1), first)
    live = c.qm.bool()[c.pair_q]
    score = torch.where(live, m, torch.zeros_like(m)).sum(-1)    # colbert.py:73-75
    return score, arg.masked_fill(~live, -1)


def oracle_grads(c: Case, arg: torch.Tensor, dpq: int):
    """The gradient of sum_p gout[p] * score[p] with respect to q and d, written out from the argmax (pairs mode:
    pair p is query p // dpq against document p)."""
    gq = torch.zeros(c.q.shape, dtype=torch.float64)
    gd = torch.zeros(c.d.shape, dtype=torch.float64)
    p, i = (arg >= 0).nonzero(as_tuple=True)
    a = arg[p, i]
    qi = p // dpq
    g = c.gout.double()[p].unsqueeze(-1)
    gq.index_put_((qi, i), g * c.d.double()[p, a], accumulate=True)
    gd.index_put_((p, a), g * c.q.double()[qi, i], accumulate=True)
    return gq, gd


def reference_autograd(q, d, qm, dm, dpq: int, gout):
    """fp64 torch autograd of the reference expression colbert.py:68-75 (queries repeated over their documents)."""
    q = q.double().detach().requires_grad_(True)
    d = d.double().detach().requires_grad_(True)
    qe = q.repeat_interleave(dpq, dim=0)[: d.shape[0]]
    s = torch.bmm(qe, d.transpose(2, 1))
    s = s.masked_fill(~dm.bool().unsqueeze(1).expand(-1, s.shape[1], -1), FILL)
    s = s.max(-1).values
    s = s.masked_fill(~qm.bool().repeat_interleave(dpq, dim=0)[: d.shape[0]], 0.0)
    s = s.sum(-1)
    s.backward(gout.double())
    return s.detach(), q.grad, d.grad


# ---------------------------------------------------------------------------------------------------------------------
# e4m3 and residual store rows: inputs and oracle
# ---------------------------------------------------------------------------------------------------------------------
E4M3_MIN_NORMAL = 2.0 ** -6
E4M3_SUBNORMAL = 2.0 ** -9     # e4m3 subnormals are m * 2^-9, 1 <= m <= 7
E4M3_EXACT_GRAINS = 2 ** 11    # premise of the exact e4m3 rows (test_maxsim_envelope_gpu.py::test_fp8_mma_accumulates_exactly)


@dataclass
class StoreCase:
    q: torch.Tensor              # [n_q, Lq, dim] f64 integers
    store: torch.Tensor          # [n_rows, dim] f64: the e4m3 values, or the decoded residual rows; NaN where no pair reads
    offsets: torch.Tensor        # [n_d + 1] int64; the last passage ends at the last store row
    pair_q: torch.Tensor         # [n_pairs] int64, the query changing every pair
    pair_d: torch.Tensor         # [n_pairs] int64, -1 for some
    poison_doc: int = -1         # a passage no pair reads (rand regime), every row NaN
    subnormal_doc: int = -1      # e4m3 rand regime: a passage of subnormal values only
    codes: Optional[torch.Tensor] = None      # residual: [n_rows, dim * bits / 8] uint8
    list_ids: Optional[torch.Tensor] = None   # [n_rows] int32; the last list is the poison list (base row NaN)
    base: Optional[torch.Tensor] = None       # [nlist, dim] fp16 integers (NaN in the poison list)
    weight: Optional[torch.Tensor] = None     # [dim, 2^bits] fp16 integers

    def window(self, d: int, Ld: int):
        """Store rows [a, b) that pair_d = d reads (a == b: none)."""
        if d < 0:
            return 0, 0
        a = int(self.offsets[d])
        return a, a + min(int(self.offsets[d + 1]) - a, Ld)


@functools.lru_cache(maxsize=None)
def make_store_case(row: Row, bits: int = 0) -> StoreCase:
    """Passages of every LAYOUT length, then seeded lengths up to max_doc_len + 40 (longer ones truncated), the last
    one ending at the last store row.  Pairs: every passage once, then seeded ones, the query changing every pair and
    coming back to earlier queries, every fifth the 257-row passage, every 17th pair_d = -1.

    "rand": e4m3 queries in [-1, 1] against rows in [-2, 2] and one passage of subnormals m * 2^-9 (|m| <= 7, in the
    first 64 dimensions); residual
    queries in [-3, 3], bases in [-1, 1], weights in [-2, 2].  Rows past max_doc_len and a passage no pair reads are NaN
    (e4m3 0x7F; residual: rows of the poison list, whose base row is NaN).
    "neg": passages alternate between positive and negative rows (counting non-empty ones), each query reads passages
    of one sign with entries of the other sign, and rows past max_doc_len take the other sign: every product a window
    holds is < 0, and the row just past it (a truncated row, the next passage, the TMA zero fill past the store) is not."""
    g = torch.Generator().manual_seed(5000 + row.seed + 100 * bits)
    n_d, Lq, Ld, dim, n_q = row.n_d, row.Lq, row.Ld, row.dim, row.n_q
    neg, e4 = row.regime == "neg", row.dtype == E4
    lens = torch.randint(1, Ld + 41, (n_d,), generator=g)
    lens[: len(LAYOUT)] = torch.tensor(LAYOUT)
    if n_d > len(LAYOUT) + 2:
        lens[len(LAYOUT) + 1] = Ld + 17
    lens[-1] = Ld // 2 + 1
    poison_doc = len(LAYOUT) if not neg and n_d > len(LAYOUT) + 1 else -1
    offsets = torch.zeros(n_d + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(lens, 0)
    n_rows = int(offsets[-1])
    sign = torch.zeros(n_d, dtype=torch.int64)
    nonempty = (lens > 0).nonzero().flatten()
    sign[nonempty] = 1 - 2 * (torch.arange(nonempty.numel()) % 2)
    qsign = 1 - 2 * (torch.arange(n_q) % 2)
    hot = LAYOUT.index(257)
    if row.n_pairs == 1:
        qsign[0] = sign[hot]
    # per store row: the sign its products must take (+1: the row scores below zero for the pairs that read it)
    row_sign = torch.zeros(n_rows, dtype=torch.int64)
    for d in range(n_d):
        a, b = int(offsets[d]), int(offsets[d + 1])
        row_sign[a:b] = sign[d]
        row_sign[a + min(b - a, Ld):b] = -sign[d]

    def ints(lo, hi, shape):
        return torch.randint(lo, hi + 1, shape, generator=g).double()

    if neg:
        mag = (torch.rand(n_q, Lq, dim, generator=g) < 0.5).double()
        mag[..., 0] = 1.0
        q = -(qsign.view(-1, 1, 1).double()) * mag * (1.0 if e4 else ints(1, 3, (n_q, Lq, dim)))
    else:
        q = ints(-1, 1, (n_q, Lq, dim)) if e4 else ints(-3, 3, (n_q, Lq, dim))

    # pairs
    def pick(qi):
        while True:
            d = int(torch.randint(0, n_d, (1,), generator=g))
            if d != poison_doc and (not neg or lens[d] == 0 or sign[d] == qsign[qi]):
                return d
    pq, pd = [], []
    prev = -1
    order = [d for d in range(n_d) if d != poison_doc]
    for p in range(row.n_pairs):
        if row.n_pairs == 1:
            qi, d = 0, hot
        else:
            want = order[p] if p < len(order) else (hot if p % 5 == 0 else None)
            cands = [i for i in range(n_q) if i != prev and (want is None or not neg or lens[want] == 0
                                                               or qsign[i] == sign[want])]
            qi = cands[int(torch.randint(0, len(cands), (1,), generator=g))]
            d = pick(qi) if want is None else want
            if p >= len(order) and p % 17 == 5:
                d = -1
        pq.append(qi)
        pd.append(d)
        prev = qi
    pair_q, pair_d = torch.tensor(pq, dtype=torch.int64), torch.tensor(pd, dtype=torch.int64)
    read = torch.zeros(n_rows, dtype=torch.bool)   # the rows some pair reads
    for d in set(pd):
        if d >= 0:
            read[int(offsets[d]):int(offsets[d]) + min(int(lens[d]), Ld)] = True

    if e4:
        if neg:
            store = row_sign.view(-1, 1).double() * ints(1, 2, (n_rows, dim))
        else:
            store = ints(-2, 2, (n_rows, dim))
        subnormal_doc = -1
        if not neg and row.n_pairs > 1:
            subnormal_doc = LAYOUT.index(65)
            a, b = int(offsets[subnormal_doc]), int(offsets[subnormal_doc + 1])
            m = torch.zeros(b - a, dim, dtype=torch.float64)
            m[:, :64] = ints(-7, 7, (b - a, 64))
            m[:, 0] = torch.where(m[:, 0] == 0, 3.0, m[:, 0])
            store[a:b] = m * E4M3_SUBNORMAL
        if not neg:
            store[~read] = float("nan")
        return StoreCase(q, store, offsets, pair_q, pair_d, poison_doc, subnormal_doc)

    # residual codes: lists 0 .. nl - 1 real (neg: even lists positive rows, odd lists negative), list nl the poison list
    nl = 6
    if neg:
        base = torch.where((torch.arange(nl) % 2 == 0).view(-1, 1), ints(2, 3, (nl, dim)), ints(-4, -3, (nl, dim)))
        weight = ints(-1, 1, (dim, 1 << bits))
    else:
        base, weight = ints(-1, 1, (nl, dim)), ints(-2, 2, (dim, 1 << bits))
    base = torch.cat([base, torch.full((1, dim), float("nan"), dtype=torch.float64)])
    lid = torch.randint(0, nl // 2, (n_rows,), generator=g) * 2
    if neg:
        lid += (row_sign < 0).long()          # positive rows on even lists, negative rows on odd ones
    else:
        lid += torch.randint(0, 2, (n_rows,), generator=g)
        lid[~read] = nl
    import colbert_residual_oracle as RO
    raw = torch.randint(0, 1 << bits, (n_rows, dim), generator=g)
    packed = RO.pack(raw.numpy().astype("uint8"), bits)
    base16, weight16 = base.half(), weight.half()
    dec = RO.decode(packed, lid.numpy().astype("int32"), base16.numpy(), weight16.numpy(), bits)
    store = torch.from_numpy(dec.astype("float64"))
    return StoreCase(q, store, offsets, pair_q, pair_d, poison_doc, -1, torch.from_numpy(packed),
                     lid.to(torch.int32), base16, weight16)


def store_oracle(c: StoreCase, Ld: int, extra: int = 0, flush: bool = False) -> torch.Tensor:
    """fp64 scores [n_pairs] of colbert.py:100-112 over the store: per live query token the max over the rows of the
    passage's window, summed; -inf for pair_d < 0 and empty passages.  ``extra`` > 0 reads that many rows past every
    window (zero rows past the end of the store, as a TMA load fills them); ``flush`` sets e4m3 subnormals to zero."""
    st = c.store
    if flush:
        st = torch.where(st.abs() < E4M3_MIN_NORMAL, torch.zeros_like(st), st)
    st = torch.cat([st, torch.zeros(extra, st.shape[1], dtype=st.dtype)])
    ts = torch.einsum("qld,rd->qlr", c.q, st)
    out = torch.full((c.pair_q.numel(),), float("-inf"), dtype=torch.float64)
    for p, (qi, d) in enumerate(zip(c.pair_q.tolist(), c.pair_d.tolist())):
        a, b = c.window(d, Ld)
        if b > a:
            out[p] = ts[qi, :, a:b + extra].max(-1).values.sum()
    return out


def assert_exact_e4m3(c: StoreCase, Ld: int):
    """Every value is an e4m3 value, and for every (query token, row a pair reads) sum_k |q_k d_k| < 2^11 grains, the
    grain being 2^-9 for subnormal rows and 1 otherwise: the premise under which the FP8 MMA sums exactly."""
    live = ~torch.isnan(c.store)
    assert torch.equal(c.store[live].to(E4).double(), c.store[live]) and torch.equal(c.q.to(E4).double(), c.q)
    assert torch.equal(c.q, c.q.round())
    rows = torch.zeros(c.store.shape[0], dtype=torch.bool)
    for d in set(c.pair_d.tolist()):
        a, b = c.window(d, Ld)
        rows[a:b] = True
    s = c.store[rows]
    sub = (s != s.round()).any(1, keepdim=True)
    grains = torch.where(sub, s / E4M3_SUBNORMAL, s)
    assert torch.equal(grains, grains.round())
    mass = torch.einsum("qld,rd->qlr", c.q.abs(), grains.abs())
    assert float(mass.max()) < E4M3_EXACT_GRAINS, float(mass.max())
