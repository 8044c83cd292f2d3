"""Host-side pieces of ColBERT end-to-end retrieval: the oracle's de-duplication against the reference's maxP loop,
the passage-aligned shard split, the offsets built from id_mapping, and the exported symbols."""
import numpy as np
import pytest
import torch

import colbert_e2e_oracle as E
from matchmaker_b200 import _lib, interaction, sharding
from matchmaker_b200.retrieval.colbert_e2e import doc_offsets_from_id_mapping


@pytest.mark.parametrize("seed", range(5))
def test_oracle_topk_unique_agrees_with_maxp_loop(seed):
    rng = np.random.default_rng(seed)
    nq, hits, top_n = 4, 200, 30
    scores = np.round(rng.normal(size=(nq, hits)) * 3) / 3         # exact ties between different passages
    ids = rng.integers(0, 40 if seed % 2 else 400, size=(nq, hits))
    # hit lists as an index returns them: (score desc, id asc)
    order = np.lexsort((ids, -scores), axis=1)
    scores = np.take_along_axis(scores, order, 1).astype(np.float32)
    ids = np.take_along_axis(ids, order, 1)
    s, i = E.topk_unique(torch.from_numpy(scores), torch.from_numpy(ids), top_n)
    loop = E.maxp_loop(scores, ids, top_n)
    for a in range(nq):
        n = len(loop[a])
        assert i[a, :n].tolist() == [x for x, _ in loop[a]]
        assert s[a, :n].tolist() == [v for _, v in loop[a]]
        assert (i[a, n:] == -1).all() and (s[a, n:] == np.float32(-E.FLT_MAX)).all()


@pytest.mark.parametrize("lengths,world", [([3, 0, 5, 2, 7, 1, 0, 4], 3), ([10, 1, 1], 4), ([0, 0, 6], 2),
                                           (list(np.random.default_rng(1).integers(0, 180, 1001)), 8), ([5], 3)])
def test_passage_shard_bounds(lengths, world):
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    n_docs, n_rows = len(lengths), int(off[-1])
    spans = [sharding.passage_shard_bounds(off, r, world) for r in range(world)]
    assert spans[0][0] == 0 and spans[0][2] == 0 and spans[-1][1] == n_docs and spans[-1][3] == n_rows
    for r in range(world - 1):
        assert spans[r][1] == spans[r + 1][0] and spans[r][3] == spans[r + 1][2]
    for d_lo, d_hi, r_lo, r_hi in spans:
        assert d_lo <= d_hi and r_lo == off[d_lo] and r_hi == off[d_hi]
    owner = [r for r, (a, b, _, _) in enumerate(spans) for _ in range(a, b)]
    assert len(owner) == n_docs                     # every passage on exactly one rank
    # balanced up to one passage: rank r starts at the first passage at or after its even row share
    for r, (d_lo, _, r_lo, _) in enumerate(spans):
        target = sharding.shard_bounds(n_rows, r, world)[0]
        assert r_lo >= target and (d_lo == 0 or off[d_lo - 1] < target)


def test_passage_shard_bounds_empty_rank():
    off = np.array([0, 100], dtype=np.int64)       # one passage, three ranks
    spans = [sharding.passage_shard_bounds(off, r, 3) for r in range(3)]
    assert spans[0] == (0, 1, 0, 100) and spans[1] == (1, 1, 100, 100) and spans[2] == (1, 1, 100, 100)


def test_doc_offsets_from_id_mapping():
    off = doc_offsets_from_id_mapping([np.array([0, 0, 0, 2]), np.array([], dtype=np.int64), np.array([2, 3, 5, 5])])
    assert off.tolist() == [0, 3, 3, 5, 6, 6, 8]
    with pytest.raises(_lib.MatchmakerB200Error):
        doc_offsets_from_id_mapping([np.array([0, 1]), np.array([0, 2])])


def test_new_symbols_are_bound():
    assert "mmb200_topk_unique" in _lib.SIGNATURES and "mmb200_maxsim_store_fwd" in _lib.SIGNATURES
    lib = _lib.load()
    assert hasattr(lib, "mmb200_topk_unique") and hasattr(lib, "mmb200_maxsim_store_fwd")
    from matchmaker_b200 import retrieval
    assert hasattr(retrieval, "ColBERTEndToEndIndexer")
    assert callable(interaction.topk_unique) and callable(interaction.maxsim_store)


def test_topk_unique_rejects_large_k_without_a_device():
    """k > 4096 is refused before any device work (a pass would not shrink the candidate list)."""
    lib = _lib.load()
    assert lib.mmb200_topk_unique(1, 1, 1, 1, 1, 10000, 4097, None) == _lib.ERR_UNSUPPORTED
