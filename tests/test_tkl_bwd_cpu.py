"""The conditional fp64 reference of the TKL backward (tests/tkl_oracle.py), checked against the unmodified oracle: with the
oracle's own top-3 windows as the given choice it must be the oracle's score exactly, and its gradients must be autograd's
gradients through oracle.interaction_oracle.tkl_interaction."""
import pytest
import torch

import tkl_oracle as T
from oracle import interaction_oracle as O


def _case(B, Lq, Ld, D, K, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    q_len = torch.randint(1, Lq + 1, (B,), generator=g)
    d_len = torch.randint(1, Ld + 1, (B,), generator=g)
    q_len[0], d_len[0] = Lq, Ld
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    for b in range(B):
        d[b, int(d_len[b]) // 2] = q[b, 0]
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    chunks = cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    cmask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    return q, qm, chunks, cmask, packed, pieces, T.covering_params(K, D, g), torch.randn(B, generator=g)


@pytest.mark.parametrize("sat", ["embedding", "log"])
@pytest.mark.parametrize("shape", [(5, 14, 420, 32, 11), (3, 1, 20, 4, 11), (4, 9, 250, 44, 16), (6, 33, 160, 12, 13)])
def test_conditional_reference_is_the_oracle_at_its_own_windows(shape, sat):
    q, qm, chunks, cmask, packed, pieces, params, gout = _case(*shape, seed=sum(shape))
    # unmodified oracle, fp64 autograd
    leaf = {k: v.double().clone().requires_grad_(True) for k, v in params.items() if k not in ("mu", "sigma")}
    p64 = dict(leaf, mu=params["mu"].double(), sigma=params["sigma"].double())
    q64 = q.double().clone().requires_grad_(True)
    c64 = chunks.double().clone().requires_grad_(True)
    s64, sec64 = O.tkl_interaction(q64, qm.double(), c64, cmask.double(), packed, pieces, p64, sat)
    s64.backward(gout.double())
    # conditional reference at the oracle's own choice
    score, sec, grads = T.reference_grads(q, qm, chunks, cmask, packed, pieces, params, sat, gout)
    assert torch.equal(sec["top_non_overlapping_idx"], sec64["top_non_overlapping_idx"])
    assert torch.equal(score, s64.detach()), "the conditional score must be the oracle's score bit for bit"
    sat_keys = T.SAT_EMBEDDING_KEYS if sat == "embedding" else ("kernel_mult0",)
    ref_sat = torch.cat([leaf[k].grad.reshape(-1) for k in sat_keys])
    pairs = [("q", q64.grad), ("chunks", c64.grad), ("dense_weight", leaf["dense_weight"].grad),
             ("chunk_scoring", leaf["chunk_scoring"].grad), ("sat", ref_sat)]
    if sat == "embedding":
        pairs.append(("sat_red", leaf["sat_emb_reduce1_weight"].grad))
    else:
        assert grads["sat_red"] is None
    for name, ref in pairs:
        torch.testing.assert_close(grads[name], ref, rtol=1e-12, atol=1e-15, msg=lambda m: f"grad {name}: {m}")
    assert grads["q"].abs().max() > 0 and grads["chunks"].abs().max() > 0


def test_gathered_windows_clamp_and_covered_rows():
    """The 15 gathered windows follow sigir20_tkl.py:274-278 (slot 3 * j + c, offsets 0, -1, +1, -2, +2, clamped), and the
    covered rows are exactly the positions of those windows, mapped through the packing."""
    W = 6   # one chunk of 40 positions
    nb = T.gathered_windows(torch.tensor([[0, 5, 3]]), W)
    assert nb.tolist() == [[0, 5, 3, 0, 4, 2, 1, 5, 4, 0, 3, 1, 2, 5, 5]]
    # two documents of 3 chunk slots; document 0's middle chunk is dropped by the packing
    packed = torch.tensor([True, False, True, True, True, True])
    top_idx = torch.tensor([[2, 45, 45], [0, 0, 0]])
    cov = T.covered_rows(top_idx, packed, 3)
    assert cov.shape == (5, 40)
    # document 0: windows 0..4 cover positions 0..37 and windows 43..45 cover 86..119 (chunk slot 2 = packed row 1)
    assert cov[0].tolist() == [True] * 38 + [False] * 2
    assert cov[1].tolist() == [False] * 6 + [True] * 34
    # document 1: windows 0..2 cover positions 0..33
    assert cov[2].tolist() == [True] * 34 + [False] * 6 and not cov[3:].any()
