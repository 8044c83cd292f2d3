"""Cases of the TKL store mode (interaction.tkl_store_window_scores): the routing envelope restated, a ragged store
builder with poison around the referenced chunks, and the padded layout the store mode must reproduce bit for bit."""
import torch

from matchmaker_b200 import interaction
from tkl_oracle import covering_params, sat_args

CHUNK = 40
IMPLS = ("simt", "tcgen05")   # the FFMA kernel (tkl.cu) and the TMA + wgmma kernel (tkl_ts.cu)


def ffma_fits(D: int, K: int, smem_optin: int = 227 * 1024) -> bool:
    """The FFMA kernel's shared-memory plan (tkl.cu: tkl_window_scores_run)."""
    kb = 12 if K <= 12 else 16
    dp = (D + 3) & ~3
    if ((dp >> 2) & 1) == 0:
        dp += 4
    need = (2 * 40 * dp + 40 * 41 + 40 * (40 * kb + 1) + 40 * 41 + 3 * 40 + 4 * kb + 16 + 20 * kb + 20 * 40 * kb) * 4
    return need <= smem_optin


def tc_fits(Lq: int, K: int) -> bool:
    """The tensor-core kernel's envelope (tkl_ts.cu: tkl_window_ts_launch); the kernel sets here all have cover."""
    return Lq <= 40 and K <= 16 and Lq * K <= 512


# (impl, saturation, K, Lq, D, C, many pairs): each row inside its kernel's envelope.  Together they cover both kernels and
# saturations, K 1/11/12/13/16 (both FFMA kernel-count instantiations), Lq 1/5/30/40 with Lq * K on both sides of 512,
# D 4/32/300/356, C 1/2/3/4/50/65 (65 > 64: the plan kernel's general path), more than 1024 pairs (the plan kernel's
# global prefix path) and fewer pairs than SMs (the FFMA kernel's segment split).
MATRIX = [
    ("tcgen05", "log", 11, 30, 300, 50, False),
    ("tcgen05", "embedding", 12, 40, 32, 4, True),
    ("tcgen05", "log", 13, 5, 356, 3, False),
    ("tcgen05", "embedding", 16, 30, 4, 65, False),
    ("tcgen05", "log", 1, 1, 4, 1, True),
    ("tcgen05", "embedding", 11, 40, 300, 2, False),
    ("simt", "embedding", 16, 40, 32, 50, False),
    ("simt", "log", 13, 30, 32, 65, False),
    ("simt", "log", 11, 30, 300, 4, True),
    ("simt", "embedding", 12, 5, 4, 1, False),
    ("simt", "log", 1, 40, 300, 3, False),
    ("simt", "embedding", 11, 1, 300, 2, False),
]


def row_id(row):
    impl, sat, K, Lq, D, C, many = row
    return f"{impl}-{sat}-K{K}-Lq{Lq}-D{D}-C{C}" + ("-many" if many else "")


def build(Lq: int, D: int, C: int, K: int, seed: int, many: bool = False):
    """A ragged store and a pair list.

    Passages hold 0, 1, 2, 3, 4, 7 or C packed chunks (at most C) on random slots, so middle slots are dropped; every
    third passage has a partly masked last chunk, and the last passage of the table is empty.  An unreferenced chunk of
    NaN / +inf / -inf rows follows every second passage, and the store is a view whose buffer continues with NaN rows.
    Pairs: every (query, passage) twice, void pairs (-1) between them, shuffled.  Returns a dict of CPU tensors."""
    g = torch.Generator().manual_seed(seed)
    n_q, n_docs = (5, 220) if many else (3, 12)
    counts = [min(C, [0, 1, 2, 3, 4, 7, C][d % 7]) for d in range(n_docs)]
    counts[-1] = 0
    rows, masks, slot_rows = [], [], []
    doc_slots = torch.full((n_docs, C), -1, dtype=torch.int32)
    for d, n in enumerate(counts):
        slots = torch.sort(torch.randperm(C, generator=g)[:n]).values
        for j, s in enumerate(slots.tolist()):
            m = torch.ones(CHUNK)
            if d % 3 == 0 and j == n - 1:
                m[int(torch.randint(1, CHUNK, (1,), generator=g)):] = 0
            doc_slots[d, s] = len(rows)
            rows.append(torch.randn(CHUNK, D, generator=g) * 0.4 * m[:, None])
            masks.append(m)
        if d % 2 == 1:   # poison that no slot references
            bad = torch.full((CHUNK, D), float("nan"))
            bad[1::3], bad[2::3] = float("inf"), float("-inf")
            rows.append(bad)
            masks.append(torch.ones(CHUNK))
    n_chunks = len(rows)
    base = torch.full((n_chunks + 2, CHUNK, D), float("nan"))
    base[:n_chunks] = torch.stack(rows)
    q_len = torch.randint(1, Lq + 1, (n_q,), generator=g)
    q_len[0] = Lq
    qm = (torch.arange(Lq)[None] < q_len[:, None]).float()
    q = torch.randn(n_q, Lq, D, generator=g) * 0.4 * qm[..., None]
    pq, pd = torch.meshgrid(torch.arange(n_q), torch.arange(n_docs), indexing="ij")
    pq, pd = pq.reshape(-1).repeat(2), pd.reshape(-1).repeat(2)
    n_void = max(3, len(pq) // 8)
    pq = torch.cat([pq, torch.randint(0, n_q, (n_void,), generator=g)])
    pd = torch.cat([pd, torch.full((n_void,), -1)])
    perm = torch.randperm(len(pq), generator=g)
    params = covering_params(K, D, g)
    if K == 1:   # one kernel covers [-1, 1] only around 0 (linspace puts it at -0.9)
        params["mu"] = torch.zeros(1)
    return {"q": q, "q_mask": qm, "store_base": base, "chunks": base[:n_chunks], "chunk_mask": torch.stack(masks),
            "doc_slots": doc_slots, "pair_q": pq[perm].int(), "pair_d": pd[perm].int(), "params": params, "C": C}


def gathered(case):
    """The padded layout of the pairs: q[pair_q], q_mask[pair_q], the referenced chunks and masks in slot order, the
    packing mask [n_pairs * C] and C (what tkl_window_scores takes)."""
    pq, pd = case["pair_q"].long(), case["pair_d"].long()
    slots = torch.where(pd[:, None] >= 0, case["doc_slots"][pd.clamp(min=0)], -1)
    packed = (slots >= 0).reshape(-1)
    idx = slots.reshape(-1)[packed].long()
    return (case["q"][pq], case["q_mask"][pq], case["chunks"][idx].contiguous(), case["chunk_mask"][idx].contiguous(),
            packed, case["C"])


def store_windows(case, sat, impl, dev="cuda"):
    """Window scores of the store mode; the chunks are a device view whose buffer continues with the NaN rows."""
    p = case["params"]
    sp, red = sat_args(p, sat)
    chunks = case["store_base"].to(dev)[:case["chunks"].shape[0]]
    return interaction.tkl_store_window_scores(
        case["q"].to(dev), case["q_mask"].to(dev), chunks,
        case["chunk_mask"].to(dev), case["doc_slots"].to(dev), case["pair_q"].to(dev), case["pair_d"].to(dev),
        p["mu"].to(dev), p["sigma"].to(dev), p["dense_weight"].to(dev), sat, sp.to(dev),
        None if red is None else red.to(dev), impl=impl)


def padded_windows(case, sat, impl, dev="cuda"):
    p = case["params"]
    sp, red = sat_args(p, sat)
    q, qm, ch, cm, packed, C = gathered(case)
    return interaction.tkl_window_scores(q.to(dev), qm.to(dev), ch.to(dev), cm.to(dev), packed.to(dev), C,
                                         p["mu"].to(dev), p["sigma"].to(dev), p["dense_weight"].to(dev), sat, sp.to(dev),
                                         None if red is None else red.to(dev), impl=impl)
