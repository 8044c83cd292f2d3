"""Host-side pieces of the AH (faiss_index_type "scann") index: the config mapping, the anisotropic weight, nibble
packing, the workspace envelope and the training steps on small CPU tensors."""
import ctypes

import pytest
import torch

import ah_oracle as A
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import scann_index as S


def _cfg(**qs):
    return {"token_dim": 64, "faiss_use_gpu": False, "token_dtype": "float16",
            "query_sets": {"first": dict(qs), "second": {"top_n": 7}}}


def test_leaves_probes_and_shortlist_follow_the_reference_config():
    assert S.leaf_count(1_100_000) == 1048 and S.leaf_count(10) == 3 and S.leaf_count(1) == 1
    assert S.probe_count(1048) == 100 and S.probe_count(30) == 30
    assert S.build_top_n(_cfg(top_n=100, index_hit_top_n=1000)) == 1000    # index_hit_top_n wins
    assert S.build_top_n(_cfg(top_n=100)) == 100
    assert S.shortlist_size(100, 10) == 100 and S.shortlist_size(100, 300) == 300
    with pytest.raises(_lib.MatchmakerB200Error, match="index_hit_top_n"):
        S.shortlist_size(2000, 10)
    with pytest.raises(_lib.MatchmakerB200Error, match="top_n"):
        S.shortlist_size(10, 1025)


def test_eta_is_the_anisotropic_weight():
    for dim in (64, 128, 768):
        assert S.anisotropic_eta(dim) == pytest.approx(A.eta(dim), rel=1e-15)
    assert S.anisotropic_eta(768) == pytest.approx(767 * 0.04 / 0.96)


def test_nibble_packing_round_trips():
    g = torch.Generator().manual_seed(0)
    codes = torch.randint(0, 16, (37, 384), generator=g)
    packed = S.pack_codes(codes)
    assert packed.dtype == torch.uint8 and packed.shape == (37, 192)
    assert torch.equal(packed, A.pack(codes))
    assert torch.equal(S.unpack_codes(packed), codes) and torch.equal(A.unpack(packed), codes)
    assert int(S.pack_codes(torch.tensor([[3, 12]]))[0, 0]) == 3 + 16 * 12


def test_workspace_query_is_zero_outside_the_envelope():
    ws = _lib.load().mmb200_ah_workspace_bytes
    assert ws(10, 8, 100, 50, 96, 100) == 0          # dim not a multiple of 64
    assert ws(10, 8, 100, 50, 32, 100) == 0
    assert ws(10, 8, 100, 50, 3648, 100) == 0        # the lookup table and the code ring leave shared memory
    assert ws(10, 8, 100, 50, 128, 0) == 0 and ws(10, 8, 100, 50, 128, 1025) == 0
    assert ws(10, 0, 100, 50, 128, 100) == 0 and ws(10, 1025, 100, 50, 128, 100) == 0
    assert ws(0, 8, 100, 50, 128, 100) == 0
    assert ws(1 << 30, 8, 100, 50, 128, 100) == 0    # nq * nprobe past 2^31
    if not torch.cuda.is_available():
        assert ws(10, 8, 100, 50, 768, 1024) == -1   # inside the envelope, but no device to size the grid


def test_ah_symbols_are_bound():
    for name in ("mmb200_ah_workspace_bytes", "mmb200_ah_search", "mmb200_ah_reorder"):
        assert name in _lib.SIGNATURES and hasattr(ctypes.CDLL(_lib.LIB_PATH), name)


def test_cpu_tensors_are_rejected():
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.ah_reorder(torch.zeros(1, 64), torch.zeros(4, 64), torch.arange(4), torch.zeros(1, 2, dtype=torch.int64), 1)


def _residuals(n, dim, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, dim, generator=g) + 0.5 * torch.randn(1, dim, generator=g)
    x[0] = 0.0                                         # a zero row: plain loss
    r = x - 0.8 * torch.nn.functional.normalize(x.sum(0, keepdim=True), dim=1)
    return x, r


def test_loss_and_coordinate_descent_match_the_oracle():
    x, r = _residuals(300, 64, 1)
    e = A.eta(64)
    cb = S.block_kmeans(r)
    codes = S.nearest_codes(r, cb)
    assert torch.allclose(S.ah_loss(r, S.unit_rows(x), cb, codes, e), A.loss(r, x, cb, codes, e), rtol=1e-12)
    cd = S.coordinate_descent(r, S.unit_rows(x), cb, codes, e, 2)
    before, after = A.loss(r, x, cb, codes, e), A.loss(r, x, cb, cd, e)
    assert torch.all(after <= before * (1 + 1e-12))
    # the last block of a sweep holds its best codeword given all the others
    final = A.loss(r, x, cb, cd, e)
    for j in range(16):
        alt = cd.clone()
        alt[:, 31] = j
        assert torch.all(A.loss(r, x, cb, alt, e) >= final * (1 - 1e-12))


def test_least_squares_update_minimises_the_loss_and_keeps_unused_codewords():
    x, r = _residuals(400, 64, 2)
    e = A.eta(64)
    cb = S.block_kmeans(r)
    codes = S.nearest_codes(r, cb)
    codes[:, 3] = torch.where(codes[:, 3] == 5, torch.tensor(4), codes[:, 3])     # codeword 5 of block 3 unused
    new = S.least_squares_codebook(r, S.unit_rows(x), codes, cb, e)
    assert torch.equal(new[3, 5], cb[3, 5].double())
    base = A.loss(r, x, new, codes, e).sum()
    assert base <= A.loss(r, x, cb, codes, e).sum() * (1 + 1e-12)
    g = torch.Generator().manual_seed(3)
    for _ in range(5):                                 # any perturbation of the solution raises the loss
        moved = new + 1e-3 * torch.randn(new.shape, generator=g, dtype=torch.float64)
        moved[3, 5] = new[3, 5]
        assert A.loss(r, x, moved, codes, e).sum() > base


def test_training_loss_never_rises_on_cpu():
    x, r = _residuals(500, 64, 4)
    _, _, _, losses = S.train_codebook(r, S.unit_rows(x), A.eta(64), rounds=3)
    assert len(losses) == 4
    assert all(b <= a * (1 + 1e-12) for a, b in zip(losses, losses[1:])), losses
