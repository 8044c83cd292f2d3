"""The max-sim tensor-core kernel's mask scouts keep each document-mask word as loaded and test it when they scan the
document (nonzero = live row; a float32 word by its value).  These masks carry words a narrower test would get wrong:
int64 words whose only set bits are in the upper half, and float32 words of -0.0 (masked) next to tiny nonzero ones
(live).  Every CTA takes many documents, so every prefetch buffer of every scout is reused.  Inputs are small integers,
so the kernel and an fp64 oracle must agree bit for bit, scores and argmax."""
import pytest
import torch

from matchmaker_b200 import interaction

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None


def oracle(q, d, qm, dm, pq, pd):
    """fp64 max-sim of pair p = (pq[p], pd[p]) with the reference's -1000 fill; argmax: first row on ties, -1 when the
    fill wins or the query token is masked."""
    m = dm.bool()
    sim = torch.einsum("qik,djk->qdij", q.double(), d.double())
    sim = torch.where(m[None, :, None, :], sim, torch.full_like(sim, -float("inf")))
    best, arg = sim.max(dim=-1).values, torch.argmax(sim, dim=-1)
    fill = (~m).any(dim=-1)[None, :, None] & (best < -1000)
    best = torch.where(fill, torch.full_like(best, -1000.0), best)
    tok = qm.bool()[:, None, :]
    arg = torch.where(fill | ~tok | torch.isinf(best), torch.full_like(arg, -1), arg)
    return torch.where(tok, best, torch.zeros_like(best)).sum(dim=-1).float()[pq, pd], arg.int()[pq, pd]


@pytest.mark.parametrize("kind", ["int64_high_bits", "float32_signed_zero"])
@pytest.mark.parametrize("ld", [180, 300])
def test_mask_words_tested_whole(kind, ld):
    g = torch.Generator().manual_seed(ld + len(kind))
    n_d, n_q, dim = 40, 3, 64
    d = torch.randint(-2, 3, (n_d, ld, dim), generator=g).to(torch.float16)
    q = torch.randint(-2, 3, (n_q, 32, dim), generator=g).to(torch.float16)
    qm = torch.ones(n_q, 32, dtype=torch.bool)
    qm[1, 20:] = False
    live = torch.rand(n_d, ld, generator=g) > 0.3
    live &= torch.arange(ld)[None, :] < torch.randint(0, ld + 1, (n_d, 1), generator=g)
    if kind == "int64_high_bits":
        # live words have only upper-half bits (or only the sign bit) set; dead words are 0
        hi = torch.where(torch.rand(n_d, ld, generator=g) > 0.5, torch.tensor(1 << 40), torch.tensor(-(1 << 63)))
        dm = torch.where(live, hi, torch.zeros((), dtype=torch.int64))
    else:
        # live words are tiny nonzero values; dead words are +0.0 or -0.0
        dead = torch.where(torch.rand(n_d, ld, generator=g) > 0.5, torch.tensor(-0.0), torch.tensor(0.0))
        dm = torch.where(live, torch.tensor(1e-30), dead)
    n = torch.cuda.get_device_properties(DEV).multi_processor_count * 50
    pq = torch.arange(n) % n_q
    pd = torch.randint(0, n_d, (n,), generator=g)
    want_s, want_a = oracle(q, d, qm, live, pq, pd)
    args = [t.to(DEV) for t in (q, d, qm.to(dm.dtype), dm)]   # one mask dtype, or both would become bool
    s, a = interaction.maxsim(*args, pair_q=pq.to(DEV), pair_d=pd.to(DEV), impl="tcgen05", return_argmax=True)
    assert torch.equal(s.cpu(), want_s) and torch.equal(a.cpu(), want_a)
