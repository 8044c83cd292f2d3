"""End-aligned chunks of the max-sim tensor-core kernel: a document with `live` rows (1 + its last unmasked row) and
nch = max(1, ceil(live / 64)) chunks reads rows [live - 64 nch, live), so its first chunk can start below row 0.  Those
rows are zero-filled by TMA and carry a -inf penalty; the argmax maps column j of a chunk to row start + j.

Inputs are small integers, so every dot product and every sum over query tokens is exact in fp32: scores and the
training argmax must equal the fp64 oracle of `maxsim_cases` and the SIMT kernel bit for bit.  Store mode stays
start-aligned and is checked against the same passages padded with masks."""
import pytest
import torch

from matchmaker_b200 import interaction

from maxsim_cases import Case, oracle

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
BAD = (float("nan"), float("inf"), -float("inf"))


def ints(shape, g):
    return torch.randint(-3, 4, shape, generator=g).float()


def padded_docs(lengths, ld, dim, g, holes=()):
    """Documents with `live` rows each (row live - 1 unmasked), masked rows in `holes` (a list of (doc, row)), and every
    masked or padding row holding NaN / inf, so that the document's own padding and the previous document's padding
    both sit next to rows an end-aligned chunk reads."""
    n = len(lengths)
    d = ints((n, ld, dim), g)
    dm = torch.zeros(n, ld, dtype=torch.long)
    for i, live in enumerate(lengths):
        dm[i, :live] = 1
    for i, r in holes:
        assert r < lengths[i] - 1
        dm[i, r] = 0
    dead = (dm == 0).nonzero().tolist()
    for k, (i, r) in enumerate(dead):
        d[i, r] = BAD[k % 3]
    return d, dm


def check(q, d, qm, dm, pair_d, dtype, dpq=None):
    """Scores and argmax of the tensor-core kernel (training and inference instantiations) against the oracle and the
    SIMT kernel."""
    n_pairs = pair_d.numel()
    dpq = dpq or n_pairs
    pair_q = torch.arange(n_pairs) // dpq
    want_s, want_a = oracle(Case(q, torch.nan_to_num(d, nan=0.0, posinf=0.0, neginf=0.0), qm, dm, pair_q, pair_d,
                                 pair_d, torch.ones(n_pairs)))
    args = (q.to(dtype).to(DEV), d.to(dtype).to(DEV), qm.to(DEV), dm.to(DEV))
    kw = dict(docs_per_query=dpq, pair_d=pair_d.int().to(DEV), pair_q=pair_q.int().to(DEV))
    s, a = interaction.maxsim(*args, impl="tcgen05", return_argmax=True, **kw)
    s2 = interaction.maxsim(*args, impl="tcgen05", **kw)
    assert torch.equal(s.cpu(), want_s.float())
    assert torch.equal(a.cpu().long(), want_a)
    assert torch.equal(s2, s)
    # the SIMT kernel reads every row it multiplies, so it gets the padding zeroed
    args_simt = (args[0], torch.nan_to_num(args[1], nan=0.0, posinf=0.0, neginf=0.0), args[2], args[3])
    s3, a3 = interaction.maxsim(*args_simt, impl="simt", return_argmax=True, **kw)
    assert torch.equal(s3, s) and torch.equal(a3, a)


@pytest.mark.parametrize("ld", [40, 63, 64, 180, 256])
@pytest.mark.parametrize("dim,dtype", [(128, torch.float16), (128, torch.bfloat16), (64, torch.float16),
                                       (64, torch.bfloat16)])
def test_end_aligned_edges(ld, dim, dtype):
    g = torch.Generator().manual_seed(ld * 7 + dim)
    # live mod 64 = 0, 1 and 63, no live row, short documents; document 0 is short, so its first chunk starts below
    # row 0 of the whole tensor
    lengths = [5, 0, 1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 2, 33, ld, ld - 1]
    lengths = [min(x, ld) for x in lengths]
    n = len(lengths)
    # holes in rows that land in a partly out-of-bounds first chunk
    holes = [(i, r) for i, live in enumerate(lengths) if live > 3 for r in (0, (live - 1) % 64 // 2) if r < live - 1]
    d, dm = padded_docs(lengths, ld, dim, g, sorted(set(holes)))
    q = ints((2, 32, dim), g)
    qm = torch.ones(2, 32, dtype=torch.long)
    qm[1, 30:] = 0
    pair_d = torch.arange(n)
    check(q, d, qm, dm, torch.cat([pair_d, pair_d.flip(0)]), dtype, dpq=n)   # forward and reversed pair_d


def test_end_aligned_ld_4096():
    g = torch.Generator().manual_seed(4096)
    ld, dim = 4096, 64
    lengths = [4096, 1, 4033, 4095, 64, 0, 4000]
    d, dm = padded_docs(lengths, ld, dim, g, [(2, 0), (2, 10), (3, 30)])
    q = ints((1, 32, dim), g)
    qm = torch.ones(1, 32, dtype=torch.long)
    check(q, d, qm, dm, torch.arange(len(lengths)), torch.float16)


@pytest.mark.parametrize("dim", [64, 128])
def test_store_mode_start_aligned(dim):
    """Store mode reads each passage from its first row: its scores equal those of the same passages padded with
    masks, bit for bit, also when the rows just before and after a passage hold NaN / inf (passages no pair reads)."""
    g = torch.Generator().manual_seed(31 + dim)
    max_len = 150
    lengths = [1, 63, 64, 65, 129, 150, 170, 7]
    pieces, offs = [], [0]
    for k, ln in enumerate(lengths):
        for rows in (torch.full((3, dim), BAD[k % 3]), ints((ln, dim), g)):
            pieces.append(rows)
            offs.append(offs[-1] + rows.shape[0])
    pieces.append(torch.full((3, dim), float("nan")))
    offs.append(offs[-1] + 3)
    store, offs = torch.cat(pieces), torch.tensor(offs)
    n = len(lengths)
    q = ints((2, 32, dim), g)
    pq = torch.arange(2 * n) % 2
    pd = torch.cat([torch.arange(n), torch.arange(n).flip(0)])
    got = interaction.maxsim_store(q.half().to(DEV), store.half().to(DEV), offs.to(DEV), pq.int().to(DEV),
                                   (2 * pd + 1).int().to(DEV), max_len, impl="tcgen05").cpu()
    d = torch.zeros(n, max_len, dim)
    dm = torch.zeros(n, max_len, dtype=torch.long)
    for i, ln in enumerate(lengths):
        ln = min(ln, max_len)
        d[i, :ln] = store[offs[2 * i + 1]:offs[2 * i + 1] + ln]
        dm[i, :ln] = 1
    want, _ = oracle(Case(q, d, torch.ones(2, 32, dtype=torch.long), dm, pq, pd, pd, torch.ones(2 * n)), fill=False)
    assert torch.equal(got, want.float())
