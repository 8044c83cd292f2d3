"""The max-sim tensor-core kernel takes each document's live-row count, fill flag and row bits from a per-document record
that scout warps fill ahead of the TMA producer, in a ring of record slots whose depth (up to 48) and stride follow from
Ld and dim.  Every CTA takes a contiguous share of the pairs, so each case here runs enough pairs (through pair_q /
pair_d over a few distinct queries and documents) that every CTA's share is several times the deepest ring: every slot
of every CTA is filled and reused many times, at every Ld.  Inputs are small integers, so every dot product and every
sum over query tokens is exact in fp32: the kernel, the SIMT kernel and an fp64 oracle must agree bit for bit, scores
and argmax."""
import pytest
import torch

from matchmaker_b200 import interaction

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
MAX_RECORDS = 48
PER_CTA = 5 * MAX_RECORDS   # pairs per CTA: the deepest record ring wraps five times


def n_pairs(per_cta=PER_CTA):
    return torch.cuda.get_device_properties(DEV).multi_processor_count * per_cta


def ints(shape, g, lo=-3, hi=3):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def oracle_table(q, d, qm, dm):
    """fp64 ColBERT max-sim of every (query, document), with the reference's -1000 fill and the kernel's argmax
    convention (first row on ties; -1 when the fill wins or the query token is masked): [n_q, n_d] and [n_q, n_d, Lq]."""
    m = dm.bool()
    df = torch.where(m[:, :, None], d.double(), torch.zeros((), dtype=torch.float64))
    sim = torch.einsum("qik,djk->qdij", q.double(), df)
    sim = torch.where(m[None, :, None, :], sim, torch.full_like(sim, -float("inf")))
    best = sim.max(dim=-1).values
    arg = torch.argmax(sim, dim=-1)
    fill = (~m).any(dim=-1)[None, :, None] & (best < -1000)
    best = torch.where(fill, torch.full_like(best, -1000.0), best)
    tok = qm.bool()[:, None, :]
    arg = torch.where(fill | ~tok | torch.isinf(best), torch.full_like(arg, -1), arg)
    return torch.where(tok, best, torch.zeros_like(best)).sum(dim=-1).float(), arg.int()


def run(impl, q, d, qm, dm, pq, pd):
    args = [t.to(DEV) for t in (q, d, qm, dm)]
    kw = dict(pair_q=pq.to(DEV), pair_d=pd.to(DEV))
    s, a = interaction.maxsim(*args, impl=impl, return_argmax=True, **kw)
    s2 = interaction.maxsim(*args, impl=impl, **kw)
    assert torch.equal(s, s2)   # the training and the inference instantiation agree
    return s.cpu(), a.cpu()


def docs(lengths, ld, dim, dtype, g, holes=True):
    """One document per entry of `lengths`, live up to that row (with holes before the last live row when asked); rows
    past it hold small integers like the rest."""
    n = len(lengths)
    d = ints((n, ld, dim), g)
    dm = torch.zeros(n, ld, dtype=torch.bool)
    for i, live in enumerate(lengths):
        dm[i, :live] = True
        if holes and live > 2:
            dm[i, torch.randint(0, live - 1, (max(1, live // 8),), generator=g)] = False
    return d.to(dtype), dm


def queries(n_q, dim, dtype, g):
    q = ints((n_q, 32, dim), g).to(dtype)
    qm = torch.ones(n_q, 32, dtype=torch.bool)
    qm[::2, 27:] = False
    return q, qm


def check(q, d, qm, dm, pq, pd, mask_dtype=torch.bool):
    """tcgen05 == SIMT == fp64 oracle, bit for bit; and NaN / inf past each document's last live row change nothing."""
    ts, ta = oracle_table(q, d, qm, dm)
    want_s, want_a = ts[pq, pd], ta[pq, pd]
    s, a = run("tcgen05", q, d, qm.to(mask_dtype), dm.to(mask_dtype), pq, pd)
    assert torch.equal(s, want_s) and torch.equal(a, want_a)
    ws, wa = run("simt", q, d, qm, dm, pq, pd)
    assert torch.equal(ws, want_s) and torch.equal(wa, want_a)
    idx = torch.arange(1, d.shape[1] + 1)
    past = idx[None, :] > (dm.long() * idx).amax(dim=1)[:, None]
    for bad in (float("nan"), float("inf")):
        s2, a2 = run("tcgen05", q, d.masked_fill(past[:, :, None], bad), qm, dm, pq, pd)
        assert torch.equal(s2, want_s) and torch.equal(a2, want_a), bad


@pytest.mark.parametrize("ld,dim", [(255, 128), (256, 128), (257, 128), (1000, 128), (4096, 128), (4096, 64)])
def test_record_stride_and_depth(ld, dim):
    """Ld values where the record stride (2 + 2 * ceil(Ld / 64) words) and the ring depth change: 48 slots up to Ld
    256, fewer past it, 30 at Ld 4096 and dim 128, 48 at dim 64.  The documents' lengths cover every chunk boundary,
    0 (fully masked) and Ld; pairs pick them in random order."""
    g = torch.Generator().manual_seed(ld + dim)
    edges = sorted({x for b in range(0, ld + 64, 64) for x in (b - 1, b, b + 1) if 0 <= x <= ld} | {ld})
    lengths = edges if len(edges) <= 40 else edges[:: len(edges) // 40] + [ld]
    d, dm = docs(lengths, ld, dim, torch.float16, g)
    q, qm = queries(3, dim, torch.float16, g)
    n = n_pairs()
    check(q, d, qm, dm, torch.randint(0, 3, (n,), generator=g), torch.randint(0, len(lengths), (n,), generator=g))


@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.int32, torch.int64, torch.float32])
def test_mask_dtypes(mask_dtype):
    g = torch.Generator().manual_seed(11)
    lengths = torch.randint(0, 181, (60,), generator=g).tolist() + [0, 180]
    d, dm = docs(lengths, 180, 64, torch.bfloat16, g)
    q, qm = queries(3, 64, torch.bfloat16, g)
    n = n_pairs()
    check(q, d, qm, dm, torch.randint(0, 3, (n,), generator=g), torch.randint(0, len(lengths), (n,), generator=g),
          mask_dtype=mask_dtype)


@pytest.mark.parametrize("order", ["short_then_long", "long_then_short", "alternating", "fully_masked_runs"])
def test_adversarial_length_orders(order):
    """Length orders that flood and drain the record and stage rings inside every CTA's share: runs of 100 one-row
    documents against runs of 100 Ld-row ones, either first, alternating ones, and runs of 50 fully masked documents
    between runs of 10 full ones.  Each CTA's share holds several of these runs, so each CTA sees every transition."""
    ld, dim = 300, 128
    g = torch.Generator().manual_seed(len(order))
    pools = {"short": [1] * 4, "long": [ld] * 4, "empty": [0] * 4}
    lengths = pools["short"] + pools["long"] + pools["empty"]
    base = {"short": 0, "long": 4, "empty": 8}
    period = {"short_then_long": ["short"] * 100 + ["long"] * 100,
              "long_then_short": ["long"] * 100 + ["short"] * 100,
              "alternating": ["short", "long"],
              "fully_masked_runs": ["empty"] * 50 + ["long"] * 10}[order]
    n = n_pairs(4 * len(period) if len(period) > 2 else PER_CTA)
    kinds = [period[i % len(period)] for i in range(n)]
    pd = torch.tensor([base[k] + i % 4 for i, k in enumerate(kinds)])
    d, dm = docs(lengths, ld, dim, torch.float16, g, holes=order == "alternating")
    q, qm = queries(2, dim, torch.float16, g)
    pq = torch.arange(n) // 37 % 2      # the query changes every 37 pairs, inside and across batches of 32
    check(q, d, qm, dm, pq, pd)


def test_ring_wraps_many_times():
    """40 000 distinct documents (about 300 per CTA) with random lengths and holes, one query per document."""
    g = torch.Generator().manual_seed(40000)
    n = 40000
    lengths = torch.randint(0, 131, (n,), generator=g)
    d = ints((n, 130, 64), g).to(torch.float16)
    dm = torch.arange(130)[None, :] < lengths[:, None]
    dm &= torch.rand(n, 130, generator=g) > 0.1
    q, qm = queries(n, 64, torch.float16, g)
    args = [t.to(DEV) for t in (q, d, qm, dm)]
    s, a = interaction.maxsim(*args, impl="tcgen05", return_argmax=True)
    ws, wa = interaction.maxsim(*args, impl="simt", return_argmax=True)
    assert torch.equal(s, ws) and torch.equal(a, wa)
    for i in torch.randperm(n, generator=g)[:50].tolist():   # fp64 oracle on a sample
        ts, ta = oracle_table(q[i:i + 1], d[i:i + 1], qm[i:i + 1], dm[i:i + 1])
        assert torch.equal(s[i:i + 1].cpu(), ts[0]) and torch.equal(a[i:i + 1].cpu(), ta[0])
