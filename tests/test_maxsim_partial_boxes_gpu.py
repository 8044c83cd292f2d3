"""A padded document's end-aligned first chunk whose lower half lies below row 0 loads only its upper half (a 32-row
box per k-block); the lower half of the stage keeps what an earlier chunk left there.  Here the documents alternate
between long ones whose masked holes hold NaN / inf in every row of a chunk and short ones of 1 to 64 live rows, so
stale NaN / inf rows sit under every half box, and both box kinds are taken.  Inputs are small integers, so the
kernel and an fp64 oracle must agree bit for bit, scores and argmax."""
import pytest
import torch

from matchmaker_b200 import interaction

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None


def oracle(q, d, qm, dm, pq, pd):
    """fp64 max-sim of pair p = (pq[p], pd[p]) with the reference's -1000 fill; argmax: first row on ties, -1 when the
    fill wins or the query token is masked."""
    m = dm.bool()
    dd = torch.where(m[:, :, None], d.double(), torch.zeros((), dtype=torch.float64))
    sim = torch.einsum("qik,djk->qdij", q.double(), dd)
    sim = torch.where(m[None, :, None, :], sim, torch.full_like(sim, -float("inf")))
    best, arg = sim.max(dim=-1).values, torch.argmax(sim, dim=-1)
    fill = (~m).any(dim=-1)[None, :, None] & (best < -1000)
    best = torch.where(fill, torch.full_like(best, -1000.0), best)
    tok = qm.bool()[:, None, :]
    arg = torch.where(fill | ~tok | torch.isinf(best), torch.full_like(arg, -1), arg)
    return torch.where(tok, best, torch.zeros_like(best)).sum(dim=-1).float()[pq, pd], arg.int()[pq, pd]


@pytest.mark.parametrize("dim,dtype", [(128, torch.float16), (64, torch.bfloat16)])
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_stale_rows_under_partial_boxes(dim, dtype, bad):
    ld = 192
    g = torch.Generator().manual_seed(dim)
    short = list(range(1, 65))                       # every first-chunk height: 1..64 rows at or above row 0
    n_long = 8
    lengths = [ld] * n_long + short
    n_d = len(lengths)
    d = torch.randint(-2, 3, (n_d, ld, dim), generator=g).to(torch.float32)
    dm = torch.arange(ld)[None, :] < torch.tensor(lengths)[:, None]
    # long documents: every row but the last one of each 64-row chunk masked and holding NaN / inf
    hole = torch.ones(ld, dtype=torch.bool)
    hole[63::64] = False
    dm[:n_long] &= ~hole
    d[:n_long][:, hole] = bad
    d[n_long:][~dm[n_long:]] = bad                  # short documents' padding too
    d = d.to(dtype)
    q = torch.randint(-2, 3, (2, 32, dim), generator=g).to(dtype)
    qm = torch.ones(2, 32, dtype=torch.bool)
    qm[1, 25:] = False
    n = torch.cuda.get_device_properties(DEV).multi_processor_count * 64
    i = torch.arange(n)
    # long, short, long, short, ...: both consumer warpgroups' stages see long chunks, then partial boxes
    pd = torch.where(i % 4 < 2, i // 4 % n_long, n_long + (i * 7) % len(short))
    pq = i // 3 % 2
    want_s, want_a = oracle(q, d.float().nan_to_num(0.0, 0.0, 0.0), qm, dm, pq, pd)
    args = [t.to(DEV) for t in (q, d, qm, dm)]
    kw = dict(pair_q=pq.to(DEV), pair_d=pd.to(DEV), impl="tcgen05")
    s, a = interaction.maxsim(*args, return_argmax=True, **kw)
    assert torch.equal(s.cpu(), want_s) and torch.equal(a.cpu(), want_a)
    assert torch.equal(interaction.maxsim(*args, **kw).cpu(), want_s)
