"""Cases of the TKL forward envelope tests: the routing of the window-score entries restated (which kernel, which plan
path, how the FFMA kernel splits its work), the instantiations the library holds, a matrix whose rows between them run all
of them, one ragged corpus builder for both entries with a cheap fp64 reference, a float32 restatement of the hill
selection, and a float32 restatement of the plan kernel's cover test."""
import dataclasses
from typing import Optional

import numpy as np
import torch

from matchmaker_b200 import interaction
from oracle import interaction_oracle as O
from tkl_oracle import covering_params, sat_args
from tkl_store_cases import ffma_fits, tc_fits

CHUNK, WINDOW = 40, 30
TILE_SLOTS = 3        # tkl_ts.cu: kTileSlots, chunk slots per tile
SM_H100 = 132         # SMs of an H100 SXM, the routing the CPU tests assume
PREFIX_SMEM_MAX = 1024   # tkl_ts.cu: tkl_plan_body keeps the prefix arrays in shared memory up to this many documents
BALLOT_MAX_C = 64        # ... and takes the two-ballot path up to this many chunk slots (and Lq <= 64)


def n_windows(C: int) -> int:
    return (C * CHUNK - WINDOW) // 2 + 1


def kb(K: int) -> int:
    """Kernel-count instantiation of the FFMA kernel (tkl.cu: tkl_window_scores_run)."""
    return 12 if K <= 12 else 16


def plan_path(B: int, C: int, Lq: int):
    """(prefix, pass) of the plan kernel for B documents: the prefix arrays in shared memory or in the global plan, and
    the per-document pass with two ballots or the general loop."""
    return ("smem" if B <= PREFIX_SMEM_MAX else "global"), ("ballot" if C <= BALLOT_MAX_C and Lq <= 64 else "general")


def sm_count() -> int:
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(0).multi_processor_count
    return SM_H100


def ffma_split(B: int, C: int, sms: Optional[int] = None):
    """(segs, grid) of the FFMA kernel: documents split into segments of chunk slots when there are fewer documents than
    SMs, and a grid of at most two CTAs per SM walking the (document, segment) items."""
    sms = sm_count() if sms is None else sms
    segs = 1
    if B < sms:
        segs = min(C, max(1, -(-2 * sms // B)))
    per = -(-C // segs)
    segs = -(-C // per)
    return segs, min(B * segs, 2 * sms)


def inst(kernel: str, *args) -> str:
    return f"{kernel}<{', '.join(str(a) for a in args)}>" if args else kernel


def _b(x: bool) -> str:
    return "true" if x else "false"


# every TKL forward kernel the library holds (tkl.cu, tkl_ts.cu); tkl_window_kernel<KB, true, ...> is the profiling
# instantiation that only a -DMMB200_ENABLE_PROF build compiles
EVERY = frozenset({inst("tkl_window_kernel", k, "false", _b(s)) for k in (12, 16) for s in (False, True)}
                  | {inst("tkl_ts_kernel", sat, _b(s)) for sat in (0, 1) for s in (False, True)}
                  | {"tkl_plan_kernel", "tkl_plan_store_kernel", "tkl_hills_kernel", "tkl_slot_map_kernel"})
PLAN_CLAIMS = frozenset(f"{k}/{p}/{w}" for k in ("tkl_plan_kernel", "tkl_plan_store_kernel")
                        for p in ("smem", "global") for w in ("ballot", "general"))
FFMA_CLAIMS = frozenset({"ffma/segs>1", "ffma/docs-per-cta>1"})
REQUIRED = {"K": {1, 11, 12, 13, 16}, "Lq": {1, 40}, "LqK": {512}, "D": {4, 44, 300, 356}, "C": {1, 3, 64, 65, 130}}


@dataclasses.dataclass(frozen=True)
class Row:
    entry: str   # "padded" (tkl_window_scores) or "store" (tkl_store_window_scores)
    impl: str    # "tcgen05" (tkl_ts.cu) or "simt" (the FFMA kernel, tkl.cu)
    sat: str
    K: int
    Lq: int
    D: int
    C: int
    n: int       # documents (padded) or pairs (store)
    claims: tuple

    def __str__(self):
        return f"{self.entry}-{self.impl}-{self.sat}-K{self.K}-Lq{self.Lq}-D{self.D}-C{self.C}-n{self.n}"


def routed_claims(entry, impl, sat, K, Lq, D, C, n, sms=SM_H100):
    """What a call of this shape runs: its instantiations, the plan path and the FFMA work split."""
    store = entry == "store"
    out = {"tkl_hills_kernel"}   # the selection runs on every row's windows
    if not store:
        out.add("tkl_slot_map_kernel")
    if impl == "tcgen05":
        assert tc_fits(Lq, K)
        plan = "tkl_plan_store_kernel" if store else "tkl_plan_kernel"
        out |= {inst("tkl_ts_kernel", 0 if sat == "embedding" else 1, _b(store)), plan, "%s/%s/%s" % ((plan,) + plan_path(n, C, Lq))}
    else:
        assert ffma_fits(D, K)
        out.add(inst("tkl_window_kernel", kb(K), "false", _b(store)))
        segs, grid = ffma_split(n, C, sms)
        if segs > 1:
            out.add("ffma/segs>1")
        if n * segs >= 2 * grid:
            out.add("ffma/docs-per-cta>1")
    return tuple(sorted(out))


def _row(*a):
    return Row(*a, claims=routed_claims(*a))


MATRIX = [
    _row("padded", "tcgen05", "embedding", 16, 32, 44, 65, 40),
    _row("padded", "tcgen05", "log", 11, 40, 32, 3, 1100),
    _row("padded", "tcgen05", "embedding", 1, 1, 4, 130, 1030),
    _row("padded", "tcgen05", "log", 12, 40, 356, 64, 100),
    _row("padded", "simt", "log", 13, 40, 44, 4, 5),
    _row("padded", "simt", "embedding", 12, 5, 300, 65, 600),
    _row("store", "tcgen05", "log", 12, 40, 4, 66, 1100),
    _row("store", "tcgen05", "embedding", 11, 30, 300, 50, 1100),
    _row("store", "tcgen05", "log", 16, 32, 356, 1, 300),
    _row("store", "tcgen05", "embedding", 13, 1, 44, 130, 200),
    _row("store", "simt", "embedding", 16, 40, 32, 3, 1100),
    _row("store", "simt", "log", 1, 1, 300, 65, 7),
]


def seed(row: Row) -> int:
    return row.K * 100000 + row.Lq * 1000 + row.C * 10 + row.D % 7 + row.n


def features(row: Row) -> set:
    return {("K", row.K), ("Lq", row.Lq), ("LqK", row.Lq * row.K), ("D", row.D), ("C", row.C)}


REQUIRED_FEATURES = {(k, v) for k, vs in REQUIRED.items() for v in vs}


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
N_Q, N_DOCS = 4, 16     # at most 64 distinct (query, passage) combinations, whatever the pair count


def slot_patterns(C: int, g: torch.Generator):
    """Chunk slots of the 16 passages: empty ones, all C slots, the last packed slot at C - 1, C - 2 and C - 3 with
    dropped slots before it, single chunks, and random subsets."""
    def subset(last, k):
        before = torch.randperm(last, generator=g)[:k].tolist() if last > 0 else []
        return sorted(set(before) | {last})

    pats = [list(range(C)), [], [0]]
    for r in range(1, 4):   # last packed slot C - r: every residue mod 3 when C >= 3
        if C - r >= 0:
            pats.append(subset(C - r, max(0, (C - r) // 2)))
    pats.append([int(torch.randint(0, C, (1,), generator=g))])
    while len(pats) < N_DOCS - 1:
        n = int(torch.randint(1, C + 1, (1,), generator=g))
        pats.append(sorted(torch.randperm(C, generator=g)[:n].tolist()))
    pats.append([])
    return pats


@dataclasses.dataclass
class Case:
    q: torch.Tensor           # [N_Q, Lq, D]
    q_mask: torch.Tensor      # [N_Q, Lq]
    store_base: torch.Tensor  # [n_chunks + 2, 40, D]: the store, then NaN chunks
    chunk_mask: torch.Tensor  # [n_chunks, 40]
    doc_slots: torch.Tensor   # [N_DOCS, C] int32
    poison: list              # store indices of the chunks no slot references
    pair_q: torch.Tensor      # [n] int32
    pair_d: torch.Tensor      # [n] int32, -1 = void pair
    params: dict
    C: int

    @property
    def chunks(self):
        return self.store_base[:self.chunk_mask.shape[0]]

    def unique(self):
        """(distinct live (pair_q, pair_d) in first-seen order, index of every pair into them or -1 for void pairs)."""
        seen, inv = {}, []
        for qv, dv in zip(self.pair_q.tolist(), self.pair_d.tolist()):
            if dv < 0:
                inv.append(-1)
                continue
            inv.append(seen.setdefault((qv, dv), len(seen)))
        return list(seen), torch.tensor(inv)


def build(Lq: int, D: int, C: int, K: int, n: int, seed: int, q: Optional[torch.Tensor] = None,
          q_mask: Optional[torch.Tensor] = None) -> Case:
    """One ragged corpus and n pairs over it.

    16 passages (slot_patterns); every third non-empty passage has a partly masked last chunk.  After every second
    passage the store holds a chunk of NaN / +inf / -inf rows that no slot references, and the store is a view whose
    buffer continues with NaN chunks.  The n pairs repeat at most 64 distinct (query, passage) combinations, with
    void pairs (pair_d = -1) among them, shuffled; the padded layout of the same pairs is ``gathered``."""
    g = torch.Generator().manual_seed(seed)
    rows, masks, poison = [], [], []
    doc_slots = torch.full((N_DOCS, C), -1, dtype=torch.int32)
    for d, slots in enumerate(slot_patterns(C, g)):
        for j, s in enumerate(slots):
            m = torch.ones(CHUNK)
            if d % 3 == 0 and j == len(slots) - 1:
                m[int(torch.randint(1, CHUNK, (1,), generator=g)):] = 0
            doc_slots[d, s] = len(rows)
            rows.append(torch.randn(CHUNK, D, generator=g) * 0.4 * m[:, None])
            masks.append(m)
        if d % 2 == 1:
            bad = torch.full((CHUNK, D), float("nan"))
            bad[1::3], bad[2::3] = float("inf"), float("-inf")
            poison.append(len(rows))
            rows.append(bad)
            masks.append(torch.ones(CHUNK))
    base = torch.full((len(rows) + 2, CHUNK, D), float("nan"))
    base[:len(rows)] = torch.stack(rows)
    if q is None:
        q_len = torch.randint(1, Lq + 1, (N_Q,), generator=g)
        q_len[0] = Lq
        q_mask = (torch.arange(Lq)[None] < q_len[:, None]).float()
        q = torch.randn(N_Q, Lq, D, generator=g) * 0.4 * q_mask[..., None]
    # distinct combinations, the longest passage first so that short pair lists still hold a full document
    combos = [(qi, d) for d in range(N_DOCS) for qi in range(q.shape[0])]
    n_void = max(1, n // 16) if n >= 4 else 0
    n_live = n - n_void
    uniq = combos[:max(1, min(len(combos), (n_live + 1) // 2))]
    live = [uniq[i % len(uniq)] for i in range(n_live)]
    pq = torch.tensor([c[0] for c in live] + torch.randint(0, q.shape[0], (n_void,), generator=g).tolist(), dtype=torch.int32)
    pd = torch.tensor([c[1] for c in live] + [-1] * n_void, dtype=torch.int32)
    perm = torch.randperm(n, generator=g)
    params = covering_params(K, D, g)
    if K == 1:   # one kernel covers [-1, 1] only around 0
        params["mu"] = torch.zeros(1)
    return Case(q, q_mask, base, torch.stack(masks), doc_slots, poison, pq[perm], pd[perm], params, C)


def gathered(case: Case, pair_q=None, pair_d=None):
    """The padded layout of the pairs: q[pair_q], q_mask[pair_q], the referenced chunks and masks in slot order, the
    packing mask [n * C] (what tkl_window_scores takes)."""
    pq = (case.pair_q if pair_q is None else pair_q).long()
    pd = (case.pair_d if pair_d is None else pair_d).long()
    slots = torch.where(pd[:, None] >= 0, case.doc_slots[pd.clamp(min=0)], -1)
    packed = (slots >= 0).reshape(-1)
    idx = slots.reshape(-1)[packed].long()
    return case.q[pq], case.q_mask[pq], case.chunks[idx].contiguous(), case.chunk_mask[idx].contiguous(), packed


def windows(case: Case, entry: str, sat: str, impl: str, dev="cuda", q_mask="case", chunk_mask="case", mask_dtype=None):
    """Window scores [n, W] of one entry.  The store entry reads the store as a device view whose buffer continues with
    NaN chunks; q_mask / chunk_mask = None drop the mask (store entry), mask_dtype recasts both."""
    p = case.params
    sp, red = sat_args(p, sat)
    args = (p["mu"].to(dev), p["sigma"].to(dev), p["dense_weight"].to(dev), sat, sp.to(dev),
            None if red is None else red.to(dev))

    def cast(m):
        return None if m is None else (m.to(dev) if mask_dtype is None else m.to(mask_dtype).to(dev))

    if entry == "store":
        qm = case.q_mask if q_mask == "case" else q_mask
        cm = case.chunk_mask if chunk_mask == "case" else chunk_mask
        chunks = case.store_base.to(dev)[:case.chunk_mask.shape[0]]
        return interaction.tkl_store_window_scores(case.q.to(dev), cast(qm), chunks, cast(cm), case.doc_slots.to(dev),
                                                   case.pair_q.to(dev), case.pair_d.to(dev), *args[:5],
                                                   sat_red_weight=args[5], impl=impl)
    q, qm, ch, cm, packed = gathered(case)
    return interaction.tkl_window_scores(q.to(dev), cast(qm), ch.to(dev), cast(cm), packed.to(dev), case.C, *args[:5],
                                         sat_red_weight=args[5], impl=impl)


def reference(case: Case, sat: str, per_call: int = 8):
    """fp64 window scores of the distinct live pairs (oracle.interaction_oracle.tkl_interaction, per_call pairs per call:
    it materialises [Lq, C * 40, K] per pair), with its top-3 windows and its secondary outputs concatenated."""
    uniq, _ = case.unique()
    p64 = {k: v.double() for k, v in case.params.items()}
    outs = []
    for lo in range(0, len(uniq), per_call):
        part = uniq[lo:lo + per_call]
        pq = torch.tensor([u[0] for u in part])
        pd = torch.tensor([u[1] for u in part])
        q, qm, ch, cm, packed = gathered(case, pq, pd)
        _, sec = O.tkl_interaction(q.double(), qm.double(), ch.double(), cm.double(), packed, case.C, p64, sat)
        outs.append(sec)
    keys = ["orig_score", "top_non_overlapping_idx", "lengths"] + (["sat_influencer"] if sat == "embedding" else [])
    return {k: torch.cat([o[k] for o in outs]) for k in keys}


# ---------------------------------------------------------------------------------------------------------------------
# the embedding saturation's continuous region
# ---------------------------------------------------------------------------------------------------------------------
RED_SCALE = 64.0                                        # sat_emb_reduce1_weight = RED_SCALE * e_RED_COL
RED_COL = 1
RED_OFFSETS = (0.0, 2.0 ** -10, -2.0 ** -10, 2.0 ** -6, -2.0 ** -6, 0.5, -0.5)


def continuous_case(Lq: int, D: int, C: int, K: int, seed: int) -> Case:
    """``build`` with sat_emb_reduce1 · q_i = len + offset exactly in fp32 for every query row i: the weight is 64 times
    a basis vector and q_i holds (len + offset) / 64 there.  Query 0 aims every row at full windows (len 30), queries
    1-3 at the lengths 1-29 that passage tails and dropped slots produce; the offsets cycle through RED_OFFSETS, so
    LayerNorm((red, len)) is evaluated inside its continuous region (|red - len| within a few sqrt(1e-5)) on a fixed
    share of the live (query row, window) cells, and at +-0.5 just outside it."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(N_Q, Lq, D, generator=g) * 0.4
    for qi in range(N_Q):
        for i in range(Lq):
            target = 30 if qi == 0 else 1 + (i * 7 + qi * 11) % 29
            q[qi, i, RED_COL] = (target + RED_OFFSETS[(i + qi) % len(RED_OFFSETS)]) / RED_SCALE
    q_mask = torch.ones(N_Q, Lq)
    q_mask[3, Lq // 2:] = 0
    q = q * q_mask[..., None]
    case = build(Lq, D, C, K, 4 * N_Q * N_DOCS // 2, seed, q=q, q_mask=q_mask)
    w = torch.zeros(D)
    w[RED_COL] = RED_SCALE
    case.params["sat_emb_reduce1_weight"] = w
    return case


def continuous_share(case: Case, ref: dict) -> float:
    """Share of the live (query row, window) cells whose LayerNorm output lies strictly inside (-0.99, 0.99)."""
    uniq, _ = case.unique()
    qm = case.q_mask[torch.tensor([u[0] for u in uniq])]
    p = case.params
    v = (ref["sat_influencer"][..., 0] - p["sat_normer_bias"][0].double()) / p["sat_normer_weight"][0].double()
    live = (qm[:, :, None] != 0) & (ref["lengths"] > 0)
    inside = (v.abs() < 0.99) & live
    return float(inside.sum()) / max(1, int(live.sum()))


# ---------------------------------------------------------------------------------------------------------------------
# hill selection, float32
# ---------------------------------------------------------------------------------------------------------------------
def top_hills_f32(window_score: np.ndarray, chunk_scoring: np.ndarray):
    """sigir20_tkl.py:254-286 in float32, as tkl_hills_kernel evaluates it: exact zeros become -9900, three times the
    first maximum with |r - best| < 15 suppressed to -10001 - c, the +-1 / +-2 neighbours clamped to [0, W), values
    <= -9900 read as 0, and the score summed in slot order from the float32 products.
    Returns (score [B], orig_score [B, W], top_idx [B, 3] int64, top15 [B, 15])."""
    ws = np.asarray(window_score, dtype=np.float32)
    cs = np.asarray(chunk_scoring, dtype=np.float32).reshape(-1)
    B, W = ws.shape
    orig = np.where(ws == 0, np.float32(-9900), ws).astype(np.float32)
    work = orig.copy()
    r = np.arange(W)
    top = np.zeros((B, 3), dtype=np.int64)
    for c in range(3):
        best = np.argmax(work, axis=1)   # the first maximum
        top[:, c] = best
        work[np.abs(r[None, :] - best[:, None]) < WINDOW // 2] = np.float32(-10001 - c)
    nb = np.clip(np.concatenate([top + o for o in (0, -1, 1, -2, 2)], axis=1), 0, W - 1)
    top15 = np.take_along_axis(orig, nb, axis=1)
    top15 = np.where(top15 <= -9900, np.float32(0), top15).astype(np.float32)
    score = np.zeros(B, dtype=np.float32)
    for l in range(15):
        score = (score + (top15[:, l] * cs[l]).astype(np.float32)).astype(np.float32)
    orig_out = np.where(orig <= -9900, np.float32(0), orig).astype(np.float32)
    return score, orig_out, top, top15


def hill_rows(B: int, W: int, seed: int) -> np.ndarray:
    """[B, W] float32 window scores cycling through the rows the selection must get right: ties at several positions,
    all zeros, all negative, genuine scores <= -9900 among the others, the maximum at 0 and at W - 1, exact zeros among
    positive scores, and a few levels only (ties everywhere)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, W)).astype(np.float32)
    for b in range(B):
        k = b % 8
        if k == 0:     # ties at several positions
            m = np.float32(x[b].max() + 1)
            x[b, rng.choice(W, size=min(W, 4), replace=False)] = m
        elif k == 1:
            x[b] = 0
        elif k == 2:
            x[b] = -np.abs(x[b]) - np.float32(0.01)
        elif k == 3:   # real scores at and below the sentinel
            x[b, rng.choice(W, size=max(1, W // 3), replace=False)] = rng.choice(
                np.array([-9900, -9899.5, -9950, -10001, -10002.5, -3e4], dtype=np.float32), size=max(1, W // 3))
        elif k == 4:
            x[b, 0] = np.float32(x[b].max() + 1)
        elif k == 5:
            x[b, W - 1] = np.float32(x[b].max() + 1)
        elif k == 6:   # exact zeros among the scores
            x[b, rng.random(W) < 0.5] = 0
        else:          # three levels: ties everywhere
            x[b] = rng.integers(-1, 2, W).astype(np.float32) * np.float32(0.5)
    return x


# ---------------------------------------------------------------------------------------------------------------------
# cover
# ---------------------------------------------------------------------------------------------------------------------
def plan_cover_f32(mu, sigma) -> bool:
    """tkl_ts.cu: tkl_plan_body's cover test restated in float32: h = 11 sigma / rbf_scale(1), the intervals
    [mu - h, mu + h), and every end point of [-1.01, 1.01) (the left end and each right end inside it) inside an
    interval that extends past it."""
    mu = np.asarray(mu, dtype=np.float32).reshape(-1)
    sg = np.asarray(sigma, dtype=np.float32).reshape(-1)
    r = np.sqrt(np.float32(0.5) * np.float32(1.4426950408889634))
    h = (np.float32(11.0) * sg) / r
    klo, khi = mu - h, mu + h
    ends = np.concatenate([np.array([-1.01], dtype=np.float32), khi])
    check = (ends >= np.float32(-1.01)) & (ends < np.float32(1.01))
    inside = ((klo[None, :] <= ends[:, None]) & (khi[None, :] > ends[:, None])).any(axis=1)
    return bool((inside | ~check).all())


def cover_sweep_f64(mu, sigma) -> bool:
    """The cover test as a sweep in doubles: what interaction.tkl_kernel_set_covers computed before it restated the
    plan kernel's float32 test."""
    x, ok = -1.01, True
    m, sg = [float(v) for v in mu], [float(v) for v in sigma]
    while x < 1.01:
        reach = x
        for mk, sk in zip(m, sg):
            h = 11.0 * sk / (0.5 * 1.4426950408889634) ** 0.5
            if mk - h <= x and mk + h > reach:
                reach = mk + h
        if reach <= x:
            ok = False
            break
        x = reach
    return ok


# a kernel set whose neighbouring intervals overlap in doubles and miss each other by one float32 ulp
# (khi[1] = -0.17645362, klo[2] = -0.1764536)
ULP_GAP_SET = ([-0.9349996447563171, -0.5611380338668823, 0.20823080837726593, 0.2675345540046692, 0.8191457390785217,
                0.875964879989624],
               [0.014433128759264946, 0.029701897874474525, 0.029701897874474525, 0.021295243874192238,
                0.021295247599482536, 0.010348997078835964])


def near_touching_sets(n: int, K: int, seed: int):
    """n float32 kernel sets whose K intervals [mu - h, mu + h] tile [-1.05, 1.05] end to end (neighbours meet), with
    every sigma then jittered by up to +-3e-7 relative: about half of the meeting points open a gap."""
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.uniform(-1.0, 1.0, (n, K - 1)), axis=1)
    edges = np.concatenate([np.full((n, 1), -1.05), cuts, np.full((n, 1), 1.05)], axis=1)
    mu = (edges[:, 1:] + edges[:, :-1]) / 2
    h = (edges[:, 1:] - edges[:, :-1]) / 2
    sigma = h * (0.5 * 1.4426950408889634) ** 0.5 / 11.0
    sigma = sigma * (1 + rng.uniform(-3e-7, 3e-7, sigma.shape))
    return mu.astype(np.float32), sigma.astype(np.float32)
