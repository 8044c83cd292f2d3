"""The headline max-sim kernel with document rows on the MMA's M side: each thread keeps running maxima of 8 query
tokens over its 2 rows of every chunk, and the rows of a document meet only once, after its last chunk (lane shuffles,
then the four warps through shared memory).  What that combine can get wrong is pinned here, bit for bit against the
fp64 oracle of `maxsim_cases` and the SIMT kernel, scores and training argmax:

- equal maxima in rows of different warps, of different quads of one warp, in rows r and r + 8 of one thread, and in
  different chunks of one document, where a later chunk's row sits in a lower warp: the first row must win;
- the -1000 fill winning, and a real row at exactly -1000 tying with it (the real row wins);
- Lq 1, 7, 31 and 32 (tokens >= Lq are zero rows of the query tile and must not count);
- live mod 64 = 0, 1 and 63, empty documents, an end-aligned first chunk (starting below row 0) with holes;
- NaN / inf in every masked or padding row and in masked query tokens;
- dim 64 and 128, f16 and bf16, store mode, and pair_q with a different query at every pair.

Inputs are small integers, so every dot product and every sum is exact in fp32 whatever the order."""
import pytest
import torch

from matchmaker_b200 import interaction

from maxsim_cases import Case, oracle, row_with_dot

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
BAD = (float("nan"), float("inf"), -float("inf"))
LD = 200

# documents: (live rows, masked rows below live - 1)
TIE_A, TIE_B, FILL_WINS, FILL_TIE = 0, 1, 2, 3
DOCS = [(128, ()), (100, ()), (199, ()), (200, (2,)), (64, ()), (1, ()), (63, ()), (0, ()), (65, (0, 1)), (129, ()),
        (200, ()), (191, (0, 3, 64)), (2, ()), (37, (0, 1, 2, 3)), (127, (126 - 64,))]
# equal maxima (document, rows), each on a query token of its own; the first row must win
TIES = [
    (TIE_A, (5, 21)),        # warp 0 and warp 1
    (TIE_A, (1, 2)),         # two quads of warp 0
    (TIE_A, (3, 11)),        # rows r and r + 8 of one thread
    (TIE_A, (50, 65)),       # chunk 0 in warp 3, then chunk 1 in warp 0
    (TIE_B, (30, 40)),       # end-aligned: chunk 0 starts at row -28 (row 30 is its row 58, warp 3), chunk 1 at row 36
    (TIE_A, (9, 17)),        # warp 0's second row against warp 1's first
    (TIE_A, (63, 64, 127)),  # across the chunk boundary
]
FILL_TOKEN_QUERY = 1         # token 0 of query 1 scores every row of FILL_WINS / FILL_TIE below -1000, one row at -1000
FILL_TIE_ROW, FILL_TIE_MASKED = 6, 2


def ints(shape, g):
    return torch.randint(-3, 4, shape, generator=g).float()


def make(Lq, dim, seed):
    g = torch.Generator().manual_seed(seed)
    tie_q0 = 2
    n_q = tie_q0 + (len(TIES) + Lq - 1) // Lq
    q = ints((n_q, Lq, dim), g)
    qm = (torch.rand(n_q, Lq, generator=g) > 0.2).long()
    n_d = len(DOCS)
    d = ints((n_d, LD, dim), g)
    dm = torch.zeros(n_d, LD, dtype=torch.long)
    for i, (live, holes) in enumerate(DOCS):
        dm[i, :live] = 1
        for r in holes:
            dm[i, r] = 0
    # the fill: every row of FILL_WINS below -1000 against u; FILL_TIE has one row at exactly -1000 after a masked row
    u = torch.full((dim,), 3.0)
    u[0] = 1.0
    q[FILL_TOKEN_QUERY, 0] = u
    qm[FILL_TOKEN_QUERY, 0] = 1
    lo = -8 * int(u.sum())
    for p in (FILL_WINS, FILL_TIE):
        for j in range(LD):
            d[p, j] = row_with_dot(u, int(torch.randint(lo, -1000, (1,), generator=g)))
    d[FILL_TIE, FILL_TIE_ROW] = row_with_dot(u, -1000)
    assert dm[FILL_TIE, FILL_TIE_ROW] == 1 and dm[FILL_TIE, FILL_TIE_MASKED] == 0
    # the ties: rows holding the sign pattern of their token reach its largest dot product
    for k, (doc, rows) in enumerate(TIES):
        qi, t = tie_q0 + k // Lq, k % Lq
        qm[qi, t] = 1
        w = torch.where(q[qi, t] >= 0, 3.0, -3.0)
        for r in rows:
            assert dm[doc, r] == 1
            d[doc, r] = w
    # poison: NaN / inf in every masked document row and masked query token
    for k, (i, r) in enumerate((dm == 0).nonzero().tolist()):
        d[i, r] = BAD[k % 3]
    for k, (i, t) in enumerate((qm == 0).nonzero().tolist()):
        q[i, t] = BAD[k % 3]
    # every document against every query, the query changing at every pair, three times over (several documents per
    # CTA, both consumer warpgroups and both buffers of the cross-warp combine)
    pair_d = torch.arange(n_d).repeat_interleave(n_q).repeat(3)
    pair_q = torch.arange(n_q).repeat(n_d * 3)
    return q, d, qm, dm, pair_q, pair_d


def clean(x):
    return torch.nan_to_num(x, nan=0.0, posinf=0.0, neginf=0.0)


@pytest.mark.parametrize("Lq", [1, 7, 31, 32])
@pytest.mark.parametrize("dim,dtype", [(64, torch.float16), (64, torch.bfloat16), (128, torch.float16),
                                       (128, torch.bfloat16)])
def test_docs_on_m_combine(Lq, dim, dtype):
    q, d, qm, dm, pair_q, pair_d = make(Lq, dim, 100 * Lq + dim + (dtype == torch.bfloat16))
    n = pair_d.numel()
    want_s, want_a = oracle(Case(clean(q), clean(d), qm, dm, pair_q, pair_d, pair_d, torch.ones(n)))
    # the constructed cases are what the oracle says they are
    for k, (doc, rows) in enumerate(TIES):
        qi, t = 2 + k // Lq, k % Lq
        sel = ((pair_q == qi) & (pair_d == doc)).nonzero()[0, 0]
        assert want_a[sel, t] == rows[0]
    sel = ((pair_q == FILL_TOKEN_QUERY) & (pair_d == FILL_WINS)).nonzero()[0, 0]
    assert want_a[sel, 0] == -1
    sel = ((pair_q == FILL_TOKEN_QUERY) & (pair_d == FILL_TIE)).nonzero()[0, 0]
    assert want_a[sel, 0] == FILL_TIE_ROW

    args = (q.to(dtype).to(DEV), d.to(dtype).to(DEV), qm.to(DEV), dm.to(DEV))
    kw = dict(pair_q=pair_q.int().to(DEV), pair_d=pair_d.int().to(DEV))
    s, a = interaction.maxsim(*args, impl="tcgen05", return_argmax=True, **kw)
    s2 = interaction.maxsim(*args, impl="tcgen05", **kw)
    assert torch.equal(s.cpu(), want_s.float())
    assert torch.equal(a.cpu().long(), want_a)
    assert torch.equal(s2, s)
    args_simt = (clean(q).to(dtype).to(DEV), clean(d).to(dtype).to(DEV), args[2], args[3])
    s3, a3 = interaction.maxsim(*args_simt, impl="simt", return_argmax=True, **kw)
    assert torch.equal(s3, s) and torch.equal(a3, a)


@pytest.mark.parametrize("dim,dtype", [(64, torch.bfloat16), (128, torch.float16)])
@pytest.mark.parametrize("Lq", [7, 32])
def test_docs_on_m_store_mode(Lq, dim, dtype):
    """Store mode (start-aligned chunks, no fill): the scores of passages read from the store equal the oracle's over
    the same passages padded with masks, with NaN / inf in the rows around each passage and a query change at every
    pair."""
    g = torch.Generator().manual_seed(7 * Lq + dim)
    max_len = 150
    lengths = [1, 63, 64, 65, 128, 129, 150, 170, 2, 100]
    pieces, offs = [], [0]
    for k, ln in enumerate(lengths):
        for rows in (torch.full((3, dim), BAD[k % 3]), ints((ln, dim), g)):
            pieces.append(rows)
            offs.append(offs[-1] + rows.shape[0])
    pieces.append(torch.full((3, dim), float("nan")))
    offs.append(offs[-1] + 3)
    store, offs = torch.cat(pieces), torch.tensor(offs)
    n, n_q = len(lengths), 3
    q = ints((n_q, Lq, dim), g)
    pd = torch.arange(n).repeat_interleave(n_q).repeat(4)
    pq = torch.arange(n_q).repeat(n * 4)
    got = interaction.maxsim_store(q.to(dtype).to(DEV), store.to(dtype).to(DEV), offs.to(DEV), pq.int().to(DEV),
                                   (2 * pd + 1).int().to(DEV), max_len, impl="tcgen05").cpu()
    d = torch.zeros(n, max_len, dim)
    dm = torch.zeros(n, max_len, dtype=torch.long)
    for i, ln in enumerate(lengths):
        ln = min(ln, max_len)
        d[i, :ln] = store[offs[2 * i + 1]:offs[2 * i + 1] + ln]
        dm[i, :ln] = 1
    want, _ = oracle(Case(q, d, torch.ones(n_q, Lq, dtype=torch.long), dm, pq, pd, pd, torch.ones(pd.numel())),
                     fill=False)
    assert torch.equal(got, want.float())
