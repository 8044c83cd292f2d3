"""Host-side pieces of PLAID centroid-interaction search (retrieval.colbert_plaid): the oracle against a plain loop,
the passage lists built from a layout, the config checks that need no device, and the compiled kernels' SASS."""
import math
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import colbert_plaid_oracle as P
from matchmaker_b200 import _lib
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer, ColBERTResidualIndexer, colbert_plaid

CPU = torch.device("cpu")


def _cfg(dim=64, nlist=8, nprobe=2, **extra):
    return {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": nlist,
            "faiss_ivf_search_probe_count": nprobe, **extra}


# ----------------------------------------------------------------------------------------------------------------------
# the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,lq,prune", [(1, 5, True), (2, 33, True), (3, 7, False)])
def test_interaction_oracle_matches_a_plain_loop(seed, lq, prune):
    g = torch.Generator().manual_seed(seed)
    nlist, nq, dim = 11, 3, 64
    lengths = [0, 1, 5, 40, 3, 0, 17]
    off = np.concatenate([[0], np.cumsum(lengths)])
    list_ids = torch.randint(0, nlist, (int(off[-1]),), generator=g)
    q = torch.randint(-2, 3, (nq, lq, dim), generator=g).float() / 4
    q[1, lq // 2:] = 0
    cents = torch.randint(-2, 3, (nlist, dim), generator=g).float() / 8
    s, keep = P.centroid_scores(q, cents, 0.5)
    cand = torch.tensor([[2, 3, -1, 0, 6, 1], [4, 5, 6, 7, -1, 3], [1, 2, 3, 4, 5, 6]]) + 10
    cand[cand == 9] = -1
    got = P.interaction(s, keep if prune else None, list_ids, off, cand, lq, first_doc=10)
    ref = P.interaction_loop(s, keep if prune else None, list_ids, off, cand, lq, first_doc=10)
    assert got.tolist() == ref
    assert any(math.isinf(v) for row in ref for v in row) and any(not math.isinf(v) for row in ref for v in row)


def test_centroid_scores_oracle_dead_tokens_and_thresholds():
    q = torch.zeros(2, 3, 64)
    q[0, 0, 0], q[0, 1, 1] = 1.0, -0.5
    cents = torch.eye(64)[:4]
    s, keep = P.centroid_scores(q, cents, -math.inf)
    assert s.shape == (2, 4, 32) and bool((s[:, :, 3:] == 0).all())
    assert keep[0].all() and not keep[1].any()                   # an all-dead query keeps nothing, even at -inf
    _, keep = P.centroid_scores(q, cents, 0.0)
    assert keep[0].tolist() == [True, True, True, True]          # the dead token's 0 does not count, the live ones do
    _, keep = P.centroid_scores(q, cents, 0.5)
    assert keep[0].tolist() == [True, False, False, False]
    w = P.keep_words(torch.tensor([[True] + [False] * 30 + [True, True]]))
    assert w.tolist() == [[-(1 << 31) + 1, 1]]


# ----------------------------------------------------------------------------------------------------------------------
# passage lists from a layout
# ----------------------------------------------------------------------------------------------------------------------
def test_passage_lists_from_a_layout():
    # passages 0..5 over 7 lists: list 3 empty, list 5 a single row, passage 2 spread over lists 0, 1, 4 and 6
    rows_of = [[0, 1], [1, 4], [], [0, 4, 6], [2], [1, 6], [4, 1, 0]]    # list per row, passage by passage
    row_pid = torch.tensor([d for d, ls in enumerate(rows_of) for _ in ls])
    assign = torch.tensor([l for ls in rows_of for l in ls])
    nlist = 7
    row_index = torch.sort(assign, stable=True).indices
    off = torch.zeros(nlist + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.bincount(assign, minlength=nlist), 0)
    p_off, p_pids, longest = colbert_plaid.passage_lists(row_index, off, row_pid)
    ref = P.passage_lists(row_index, off, row_pid)
    r_off, r_pids = P.flatten_lists(ref)
    assert torch.equal(p_off, r_off) and torch.equal(p_pids, r_pids) and p_pids.dtype == torch.int32
    assert ref[3] == [] and ref[5] == [] and ref[2] == [4] and [l for l in range(nlist) if 3 in ref[l]] == [0, 4, 6]
    assert ref[0] == [0, 3, 6] and longest == max(len(p) for p in ref)
    lid = colbert_plaid.row_list_ids(row_index, off, len(assign))
    assert torch.equal(lid, assign.to(torch.int32))


def test_passage_lists_of_an_empty_layout():
    p_off, p_pids, longest = colbert_plaid.passage_lists(torch.zeros(0, dtype=torch.int64), torch.zeros(5, dtype=torch.int64),
                                                         torch.zeros(0, dtype=torch.int64))
    assert p_off.tolist() == [0] * 5 and p_pids.numel() == 0 and longest == 0


def test_candidate_oracle_is_the_ascending_union():
    plists = [[0, 3], [], [3, 5, 9], [1]]
    probes = torch.tensor([[2, 0, -1, 2, 7], [-1, -1, -1, -1, -1], [1, 1, 3, 1, 1]])
    c = P.candidates(probes, plists, 6, first_doc=100)
    assert c.tolist() == [[100, 103, 105, 109, -1, -1], [-1] * 6, [101, -1, -1, -1, -1, -1]]


# ----------------------------------------------------------------------------------------------------------------------
# config checks
# ----------------------------------------------------------------------------------------------------------------------
def test_config_keys():
    assert colbert_plaid.config_keys({}) is None
    assert colbert_plaid.config_keys({"colbert_plaid_ndocs": 256}) == (256, 0.45)
    assert colbert_plaid.config_keys({"colbert_plaid_ndocs": 4, "colbert_plaid_centroid_score_threshold": -math.inf}) \
        == (4, -math.inf)
    for bad in ({"colbert_plaid_ndocs": 3}, {"colbert_plaid_ndocs": 4097},
                {"colbert_plaid_ndocs": 64, "colbert_plaid_centroid_score_threshold": float("nan")},
                {"colbert_plaid_centroid_score_threshold": 0.5}):
        with pytest.raises(_lib.MatchmakerB200Error):
            colbert_plaid.config_keys(bad)


def test_indexers_accept_or_refuse_the_keys():
    idx = ColBERTIVFIndexer(_cfg(colbert_plaid_ndocs=64), device=CPU)
    assert idx.plaid.ndocs == 64 and idx.plaid.threshold == 0.45
    assert ColBERTIVFIndexer(_cfg(), device=CPU).plaid is None
    res = ColBERTResidualIndexer(_cfg(colbert_residual_bits=2, colbert_plaid_ndocs=128,
                                      colbert_plaid_centroid_score_threshold=0.4), device=CPU)
    assert res.plaid.ndocs == 128 and res.plaid.threshold == 0.4
    fp8 = ColBERTIVFIndexer(_cfg(dim=128, colbert_store_dtype="float8_e4m3", colbert_plaid_ndocs=64), device=CPU)
    assert fp8.fp8 and fp8.plaid is not None
    with pytest.raises(_lib.MatchmakerB200Error, match="IVF token index"):
        ColBERTEndToEndIndexer({"token_dim": 64, "faiss_use_gpu": True, "token_dtype": "float16",
                                "colbert_plaid_ndocs": 64}, device=CPU)
    with pytest.raises(_lib.MatchmakerB200Error, match="nlist"):
        ColBERTIVFIndexer(_cfg(nlist=(1 << 18) + 1, colbert_plaid_ndocs=64), device=CPU)
    for dim in (32, 96, 1088):
        with pytest.raises(_lib.MatchmakerB200Error, match="token_dim"):
            ColBERTIVFIndexer(_cfg(dim=dim, colbert_plaid_ndocs=64), device=CPU)


def test_plaid_symbols_are_bound():
    lib = _lib.load()
    for name in ("mmb200_plaid_centroid_scores", "mmb200_plaid_candidates", "mmb200_plaid_interaction"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES


# ----------------------------------------------------------------------------------------------------------------------
# SASS
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def plaid_sass():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        out = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump unavailable: {e}")
    funcs, name = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items() if "plaid_" in k}


def test_plaid_kernels_compiled_scores_on_the_tensor_cores_without_spills(plaid_sass):
    counts = {n: sum(n in k for k in plaid_sass) for n in ("plaid_scores_kernel", "plaid_mark_kernel",
                                                         "plaid_compact_kernel", "plaid_interaction_kernel")}
    assert counts == {"plaid_scores_kernel": 3, "plaid_mark_kernel": 1, "plaid_compact_kernel": 1,
                     "plaid_interaction_kernel": 8}
    for k, text in plaid_sass.items():
        if "plaid_scores_kernel" in k:
            assert any("HGMMA" in l and "gdesc[URZ]" not in l for l in text.splitlines()), f"{k}: no wgmma"
        assert "STL" not in text and "LDL" not in text, f"{k}: local-memory spill"
