"""The max-sim tensor-core kernel streams only each document's live rows (up to its last unmasked one) through a ring of
64-row chunks.  Inputs here are small integers, so every dot product and every sum over query tokens is exact in fp32:
the kernel, the SIMT kernel and an fp64 oracle must then agree bit for bit, scores and argmax.  This checks the chunk
boundaries, the -1000 fill of the reference (now a per-document flag), that rows past the last live one are never used,
the pair-indirection modes and store mode."""
import pytest
import torch

from matchmaker_b200 import interaction

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
LIVE = (0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129)


def ints(shape, g, lo=-3, hi=3):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def oracle(q, d, qm, dm, pair_q, pair_d, pair_dm):
    """fp64 ColBERT max-sim with the reference's -1000 fill and the kernel's argmax convention (first row on ties; -1
    when the fill wins or the query token is masked)."""
    qf, df, m = q.double()[pair_q], d.double()[pair_d], dm.bool()[pair_dm]
    sim = torch.einsum("pik,pjk->pij", qf, torch.where(m[:, :, None], df, torch.zeros_like(df)))
    sim = torch.where(m[:, None, :], sim, torch.full_like(sim, -float("inf")))
    best = sim.max(dim=-1).values
    arg = torch.argmax(sim, dim=-1)   # first maximal row
    fill = (~m).any(dim=-1)[:, None] & (best < -1000)
    best = torch.where(fill, torch.full_like(best, -1000.0), best)
    tok = qm.bool()[pair_q]
    arg = torch.where(fill | ~tok | torch.isinf(best), torch.full_like(arg, -1), arg)
    score = torch.where(tok, best, torch.zeros_like(best)).sum(dim=-1)
    return score.float(), arg.int()


def run(impl, q, d, qm, dm, dpq=None, pair_q=None, pair_d=None, pair_dm=None):
    args = [t.to(DEV) if t is not None else None for t in (q, d, qm, dm)]
    kw = dict(pair_q=None if pair_q is None else pair_q.to(DEV), pair_d=None if pair_d is None else pair_d.to(DEV),
              pair_dmask=None if pair_dm is None else pair_dm.to(DEV))
    s, a = interaction.maxsim(*args, docs_per_query=dpq or 1, impl=impl, return_argmax=True, **kw)
    s2 = interaction.maxsim(*args, docs_per_query=dpq or 1, impl=impl, **kw)
    assert torch.equal(s, s2)   # the training and the inference instantiation agree
    return s.cpu(), a.cpu()


def docs_with_lengths(lengths, ld, dim, dtype, g, holes=False, pad=0.0):
    n = len(lengths)
    d = ints((n, ld, dim), g)
    dm = torch.zeros(n, ld, dtype=torch.bool)
    for i, live in enumerate(lengths):
        dm[i, :live] = True
        if holes and live > 2:
            dm[i, torch.randint(0, live - 1, (max(1, live // 8),), generator=g)] = False   # never the last live row
        d[i, live:] = pad
    return d.to(dtype), dm


@pytest.mark.parametrize("ld", [7, 64, 180, 181, 255, 256, 300])
@pytest.mark.parametrize("dim,dtype", [(128, torch.float16), (64, torch.bfloat16), (64, torch.float16)])
def test_live_lengths_exact(ld, dim, dtype):
    g = torch.Generator().manual_seed(1000 + ld + dim)
    lengths = sorted({min(x, ld) for x in LIVE + (ld,)}) * 4
    n_q = 3
    lengths += [ld] * (-len(lengths) % n_q)
    n = len(lengths)
    dpq = n // n_q                               # the query changes inside a batch of 32 pairs
    q = ints((n_q, 32, dim), g).to(dtype)
    qm = torch.ones(n_q, 32, dtype=torch.bool)
    qm[1, 29:] = False
    d, dm = docs_with_lengths(lengths, ld, dim, dtype, g, holes=True)
    pq = torch.arange(n) // dpq
    want_s, want_a = oracle(q, d, qm, dm, pq, torch.arange(n), torch.arange(n))
    for impl in ("tcgen05", "tcgen05_ragged", "simt"):
        s, a = run(impl, q, d, qm, dm, dpq=dpq)
        assert torch.equal(s, want_s), impl
        assert torch.equal(a, want_a), impl
    # rows past each document's last live row are never used: NaN / inf there change nothing
    for bad in (float("nan"), float("inf"), -float("inf")):
        d2 = d.clone()
        for i, live in enumerate(lengths):
            last = int(dm[i].nonzero().max()) + 1 if dm[i].any() else 0
            d2[i, last:] = bad
        s, a = run("tcgen05", q, d2, qm, dm, dpq=dpq)
        assert torch.equal(s, want_s) and torch.equal(a, want_a), bad


@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.int32, torch.int64, torch.float32])
def test_fill_flag(mask_dtype):
    """Documents whose real scores lie below -1000: the fill wins exactly when a masked position exists anywhere in the
    document -- trailing padding that is never visited, or holes only."""
    g = torch.Generator().manual_seed(7)
    ld, dim = 181, 128
    q = torch.full((1, 32, dim), 3.0)
    q[0, :, 0] = 1.0
    cases = [(70, False), (181, False), (181, True), (0, False), (64, False), (128, True), (129, False)]
    n = len(cases)
    d = -3.0 - ints((n, ld, dim), g, 0, 0)     # every dot product is -3 * (3 * 127 + 1) = -1146 < -1000
    d[:, :, 0] = ints((n, ld), g, -3, 3)       # ... give or take a few, so the argmax is not a tie everywhere
    dm = torch.zeros(n, ld, dtype=torch.bool)
    for i, (live, hole) in enumerate(cases):
        dm[i, :live] = True
        if hole:
            dm[i, 5] = False
        d[i, live:] = float("nan")
    qm = torch.ones(1, 32, dtype=torch.bool)
    want_s, want_a = oracle(q, d, qm, dm, torch.zeros(n, dtype=torch.long), torch.arange(n), torch.arange(n))
    # the full-length document without holes keeps its real score; every other one takes the fill
    assert want_s[1] < -1000 * 32 and all(want_s[i] == -1000 * 32 for i in (0, 2, 3, 4, 5, 6))
    dmt = dm.to(mask_dtype)
    for impl, dd in (("tcgen05", d), ("simt", torch.nan_to_num(d, nan=0.0))):
        s, a = run(impl, q.half(), dd.half(), qm, dmt, dpq=n)
        assert torch.equal(s, want_s), impl
        assert torch.equal(a, want_a), impl


def test_pair_indirection():
    g = torch.Generator().manual_seed(11)
    ld, dim, n_q, n_d, n_pairs = 200, 128, 5, 90, 700
    q = ints((n_q, 32, dim), g).half()
    qm = torch.rand(n_q, 32, generator=g) < 0.9
    lengths = [int(x) for x in torch.randint(0, ld + 1, (n_d,), generator=g)]
    d, dm = docs_with_lengths(lengths, ld, dim, torch.float16, g, holes=True, pad=float("nan"))
    d = torch.nan_to_num(d, nan=0.0)   # pair_dmask may pair a document with another document's mask
    pq = torch.randint(0, n_q, (n_pairs,), generator=g)
    pd = torch.randint(0, n_d, (n_pairs,), generator=g)
    pdm = torch.randint(0, n_d, (n_pairs,), generator=g)
    want_s, want_a = oracle(q, d, qm, dm, pq, pd, pdm)
    for impl in ("tcgen05", "tcgen05_ragged", "simt"):
        s, a = run(impl, q, d, qm, dm, pair_q=pq.int(), pair_d=pd.int(), pair_dm=pdm.int())
        assert torch.equal(s, want_s), impl
        assert torch.equal(a, want_a), impl
    want_s, want_a = oracle(q, d, qm, dm, pq, pd, pd)
    s, a = run("tcgen05", q, d, qm, dm, pair_q=pq.int(), pair_d=pd.int())
    assert torch.equal(s, want_s) and torch.equal(a, want_a)


@pytest.mark.parametrize("dim", [64, 128])
def test_store_mode_chunk_boundaries(dim):
    g = torch.Generator().manual_seed(13 + dim)
    max_len = 200
    lengths = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 191, 192, 193, 200, 230, 0, 40]
    offs = torch.tensor([0] + lengths).cumsum(0)
    store = ints((int(offs[-1]) + 5, dim), g).half()
    n_q = 2
    q = ints((n_q, 32, dim), g).half()
    n = len(lengths)
    pq = torch.arange(2 * n) % n_q
    pd = torch.cat([torch.arange(n), torch.arange(n).flip(0)])
    pd[3] = -1
    got = interaction.maxsim_store(q.to(DEV), store.to(DEV), offs.to(DEV), pq.int().to(DEV), pd.int().to(DEV), max_len,
                                   impl="tcgen05").cpu()
    # the same passages padded to max_len with masks
    d = torch.zeros(n, max_len, dim, dtype=torch.float16)
    dm = torch.zeros(n, max_len, dtype=torch.bool)
    for i, ln in enumerate(lengths):
        ln = min(ln, max_len)
        d[i, :ln] = store[offs[i]:offs[i] + ln]
        dm[i, :ln] = True
    want, _ = oracle(q, d, torch.ones(n_q, 32, dtype=torch.bool), dm, pq, pd.clamp(min=0), pd.clamp(min=0))
    empty = torch.tensor([pd[p] < 0 or lengths[pd[p]] == 0 for p in range(2 * n)])
    assert torch.isinf(got[empty]).all() and (got[empty] < 0).all()
    assert torch.equal(got[~empty], want[~empty])


@pytest.mark.parametrize("ld", [4096, 4097])
def test_longest_documents(ld):
    """Up to 4096 rows a document runs on the live-row kernel (its writers keep 4096 rows of mask ballots); longer ones
    on the documents-on-M kernel.  Both sides of the boundary give exact results."""
    g = torch.Generator().manual_seed(17)
    lengths = [0, 1, 300, 4000, 4095, min(4096, ld), ld]
    q = ints((1, 32, 64), g).half()
    qm = torch.ones(1, 32, dtype=torch.bool)
    d, dm = docs_with_lengths(lengths, ld, 64, torch.float16, g, holes=True)
    n = len(lengths)
    want_s, want_a = oracle(q, d, qm, dm, torch.zeros(n, dtype=torch.long), torch.arange(n), torch.arange(n))
    s = interaction.maxsim(q.to(DEV), d.to(DEV), qm.to(DEV), dm.to(DEV), docs_per_query=n, impl="tcgen05").cpu()
    assert torch.equal(s, want_s)
    if ld <= 4096:
        s, a = run("tcgen05", q, d, qm, dm, dpq=n)
        assert torch.equal(s, want_s) and torch.equal(a, want_a)
