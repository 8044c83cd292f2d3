"""PLAID centroid-interaction search (retrieval.colbert_plaid) on the H100: each kernel against the fp64 oracle on grid
inputs (every fp32 sum exact, every centroid score an fp16 number), the whole search against brute force and against
the oracle, sharding, persistence, CUDA-graph replay, recall and the search-time checks.  Exact comparisons only."""
import math

import numpy as np
import pytest
import torch

import colbert_plaid_oracle as P
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer, ColBERTResidualIndexer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _grid_queries(nq, lq, dim, seed):
    """Entries in {-1, 0, 1} / 4 with dead (all-zero) tokens; against centroids in {-2..2} / 8 every dot product is a
    multiple of 1 / 32 below 2^6 in magnitude for dim <= 1024: exact in fp32 sums and in fp16."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(-1, 2, (nq, lq, dim), generator=g).float() / 4
    q[0, lq - max(1, lq // 4):] = 0
    if nq > 2:
        q[2, ::3] = 0
    return q


def _grid_centroids(nlist, dim, seed):
    return torch.randint(-2, 3, (nlist, dim), generator=torch.Generator().manual_seed(seed)).float() / 8


def _f64(t):
    return t.double().cpu()


# ----------------------------------------------------------------------------------------------------------------------
# 1. centroid scores and keep mask
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lq,dim,nlist", [(1, 64, 37), (31, 128, 4099), (32, 768, 37), (33, 64, 1), (64, 128, 37),
                                          (100, 768, 4099), (128, 64, 4099), (128, 128, 1)])
def test_centroid_scores_and_keep_equal_oracle(lq, dim, nlist):
    q, c = _grid_queries(3, lq, dim, seed=lq + dim), _grid_centroids(nlist, dim, seed=nlist)
    qd, cd = q.half().to(DEV), c.half().to(DEV)
    s_ref, _ = P.centroid_scores(q, c, 0.0)
    mid = float(s_ref[1, :, :lq].max(-1).values.median())     # query 1 has no dead token
    for t in (-math.inf, 0.0, mid):
        s, keep = interaction.plaid_centroid_scores(qd, cd, t)
        _, k_ref = P.centroid_scores(q, c, t)
        assert s.shape == (3, nlist, P.lqp(lq)) and torch.equal(_f64(s), s_ref)
        assert torch.equal(keep.cpu(), P.keep_words(k_ref)), f"keep mask at t_cs {t}"
    assert k_ref.any()


def test_all_dead_query_keeps_nothing():
    q = torch.zeros(2, 40, 64, dtype=torch.float16, device=DEV)
    q[1, 3, 5] = 0.25
    s, keep = interaction.plaid_centroid_scores(q, _grid_centroids(70, 64, 1).half().to(DEV), -math.inf)
    assert bool((s[0] == 0).all()) and int(keep[0].abs().sum()) == 0
    assert keep[1].cpu().tolist() == [-1, -1, (1 << 6) - 1]


# ----------------------------------------------------------------------------------------------------------------------
# 2. candidates
# ----------------------------------------------------------------------------------------------------------------------
def test_candidates_equal_the_oracle_union():
    g = torch.Generator().manual_seed(4)
    n_docs, nlist = 3000, 50
    plists = [sorted(torch.randperm(n_docs, generator=g)[:int(torch.randint(0, 120, (1,), generator=g))].tolist())
              for _ in range(nlist)]
    plists[7] = []
    plists[8] = [n_docs - 1]
    off, pids = P.flatten_lists(plists)
    probes = torch.randint(-1, nlist, (5, 64), generator=g)
    probes[0, :32] = 7                                  # duplicate probes and an empty list
    probes[1] = -1                                      # an all-dead query
    probes[2, 10:] = probes[2, :10].repeat(6)[:54]      # duplicates across tokens
    cap = min(n_docs, 64 * max(len(p) for p in plists))
    got = interaction.plaid_candidates(probes.to(DEV), off.to(DEV), pids.to(DEV), n_docs, cap, first_doc=12345)
    ref = P.candidates(probes, plists, cap, first_doc=12345)
    assert torch.equal(got.cpu(), ref) and bool((got[1] == -1).all())


@pytest.mark.parametrize("whole", [True, False])
def test_candidates_reaching_cap_exactly(whole):
    # whole: the union is every passage (cap = n_docs); else disjoint lists of equal length, union = n_probes * length
    n_docs, nlist, length = 4000, 40, 100
    plists = [list(range(l * length, (l + 1) * length)) for l in range(nlist)]
    off, pids = P.flatten_lists(plists)
    probes = torch.arange(nlist).view(1, nlist) if whole else torch.tensor([[3, 9, 27, 31]])
    cap = min(n_docs, probes.shape[1] * length)
    got = interaction.plaid_candidates(probes.to(DEV), off.to(DEV), pids.to(DEV), n_docs, cap)
    ref = P.candidates(probes, plists, cap)
    assert torch.equal(got.cpu(), ref) and bool((got >= 0).all())


# ----------------------------------------------------------------------------------------------------------------------
# 3. pruned and full interaction
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lq", [20, 64, 90, 128])
def test_interaction_equals_oracle(lq):
    dim, nlist, nq = 64, 300, 3
    lengths = [0, 1, 64, 65, 333, 7, 0, 128, 129, 40]
    off = np.concatenate([[0], np.cumsum(lengths)])
    g = torch.Generator().manual_seed(lq)
    list_ids = torch.randint(0, nlist, (int(off[-1]),), generator=g)
    list_ids[int(off[3]):int(off[4])] = 17              # one passage on a single list (pruned for the strict query)
    q, c = _grid_queries(nq, lq, dim, seed=lq), _grid_centroids(nlist, dim, seed=lq + 1)
    s_ref, _ = P.centroid_scores(q, c, 0.0)
    top = s_ref[1, :, :lq].max(-1).values
    t = float(top.sort().values[nlist * 3 // 4])
    s, keep = interaction.plaid_centroid_scores(q.half().to(DEV), c.half().to(DEV), t)
    _, k_ref = P.centroid_scores(q, c, t)
    assert torch.equal(_f64(s), s_ref) and torch.equal(keep.cpu(), P.keep_words(k_ref))
    first = 500
    cand = torch.tensor([list(range(10)) + [-1, 10, 9999, first - 1]] * nq) + first
    cand[:, 10] = -1
    cand_d = cand.to(DEV)
    for prune in (True, False):
        got = interaction.plaid_interaction(s, keep if prune else None, list_ids.to(DEV), torch.from_numpy(off).to(DEV),
                                            cand_d, lq, first_doc=first)
        ref = P.interaction(s_ref, k_ref if prune else None, list_ids, off, cand, lq, first_doc=first)
        assert torch.equal(_f64(got), ref), f"prune={prune}"
        assert bool(torch.isinf(ref[:, [0, 6, 10, 11, 12, 13]]).all())        # empty passages and void ids
    assert bool(torch.isfinite(ref[:, [1, 2, 3, 4]]).all())


def test_interaction_all_rows_pruned_is_void():
    q, c = _grid_queries(2, 32, 64, seed=3), _grid_centroids(20, 64, seed=4)
    s, keep = interaction.plaid_centroid_scores(q.half().to(DEV), c.half().to(DEV), 1e30)
    assert int(keep.abs().sum()) == 0
    off = torch.tensor([0, 5, 9])
    got = interaction.plaid_interaction(s, keep, torch.arange(9, dtype=torch.int32).to(DEV) % 20, off.to(DEV),
                                        torch.tensor([[0, 1], [1, 0]]).to(DEV), 32)
    assert bool(torch.isinf(got).all() & (got < 0).all())


# ----------------------------------------------------------------------------------------------------------------------
# shared stores
# ----------------------------------------------------------------------------------------------------------------------
def _cfg(dim, nlist, nprobe, dtype="float16", **extra):
    return {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": dtype, "faiss_ivf_list_count": nlist,
            "faiss_ivf_search_probe_count": nprobe, **extra}


def _clustered_store(n_pass, dim, n_centres, seed, max_len=40):
    g = torch.Generator().manual_seed(seed)
    lengths = np.random.default_rng(seed).integers(1, max_len, n_pass)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    c = torch.nn.functional.normalize(torch.randn(n_centres, dim, generator=g), dim=1)
    which = torch.randint(0, n_centres, (int(off[-1]),), generator=g)
    store = (c[which] + 0.25 * torch.randn(int(off[-1]), dim, generator=g) / dim ** 0.5).half()
    return store, off, c


def _pid(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def _queries(cent, nq, lq, seed):
    g = torch.Generator().manual_seed(seed)
    dim = cent.shape[1]
    q = (cent[torch.randint(0, cent.shape[0], (nq, lq), generator=g)] + 0.3 * torch.randn(nq, lq, dim, generator=g) /
         dim ** 0.5)
    q[0, lq - 5:] = 0
    return q


def _build(cls, store, off, cfg, dtype="float16"):
    blocks = [store.numpy().astype(np.float16 if dtype == "float16" else np.float32)]
    idx = cls(cfg, device=DEV)
    idx.prepare(blocks)
    idx.index([_pid(off)], blocks)
    return idx


def _brute_force(idx, q, top_n):
    """The store's own max-sim over every (query, passage) pair, ranked, unscaled: what the indexer's last stage
    computes when every passage reaches it."""
    qs, sq = idx.tokens.queries(q.to(DEV, idx.store_dtype).contiguous())
    nq, n = q.shape[0], idx.d_hi - idx.d_lo
    pair_d = torch.arange(n, device=DEV, dtype=torch.int32).repeat(nq)
    pair_q = torch.arange(nq, device=DEV, dtype=torch.int32).repeat_interleave(n)
    if idx.residual:   # over the rows the codes decode to
        sc = interaction.maxsim_store(qs.half(), idx.decoded_store(), idx.offsets, pair_q, pair_d, idx.max_doc_len,
                                      impl="tcgen05_docm")
    else:
        sc = idx.tokens.maxsim(qs, idx.offsets, pair_q, pair_d, idx.max_doc_len)
    sc = sc.view(nq, n)
    s, i = interaction.topk_merge(sc, torch.arange(idx.d_lo, idx.d_hi, device=DEV).repeat(nq, 1), top_n)
    return idx.tokens.unscale(s, sq), i


# ----------------------------------------------------------------------------------------------------------------------
# 4. exact end to end: every list probed, nothing pruned, every passage survives
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("store_kind", ["fp16", "fp32", "e4m3", "residual1", "residual2"])
def test_exhaustive_search_equals_brute_force(store_kind):
    dim, nlist, top_n = 128, 16, 100
    store, off, cent = _clustered_store(700, dim, 24, seed=31)
    q = _queries(cent, 4, 32, seed=32)
    extra = {"colbert_plaid_ndocs": 4096, "colbert_plaid_centroid_score_threshold": -math.inf}
    dtype, cls = "float16", ColBERTIVFIndexer
    if store_kind == "fp32":
        dtype = "float32"
    elif store_kind == "e4m3":
        extra["colbert_store_dtype"] = "float8_e4m3"
    elif store_kind.startswith("residual"):
        extra["colbert_residual_bits"] = int(store_kind[-1])
        cls = ColBERTResidualIndexer
    idx = _build(cls, store, off, _cfg(dim, nlist, nlist, dtype, **extra), dtype)
    s, i = idx.search_device(q.to(DEV), top_n)
    rs, ri = _brute_force(idx, q, top_n)
    assert torch.equal(i, ri) and torch.equal(s, rs)


# ----------------------------------------------------------------------------------------------------------------------
# 5. pruning active on grid inputs, 6. two halves
# ----------------------------------------------------------------------------------------------------------------------
def _grid_store(n_pass, dim, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = np.random.default_rng(seed).integers(1, 30, n_pass)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    store = (torch.randint(-2, 3, (int(off[-1]), dim), generator=g).float() / 8).half()
    return store, off


def _grid_index(store, off, cents, nprobe, ndocs, t_cs, first_doc=0):
    dim, nlist = store.shape[1], cents.shape[0]
    idx = ColBERTIVFIndexer(_cfg(dim, nlist, nprobe, colbert_plaid_ndocs=ndocs,
                                 colbert_plaid_centroid_score_threshold=t_cs), device=DEV)
    idx.ivf.set_centroids(cents)
    idx.index_device(store.to(DEV), off, first_doc)
    return idx


def _oracle_search(idx, q, store, off, top_n, first_doc=0):
    qd = q.half().to(DEV)
    lq, dim = q.shape[1], q.shape[2]
    toks = qd.reshape(-1, dim)
    probes = idx.ivf.coarse(toks).masked_fill((toks == 0).all(1, keepdim=True), -1).view(q.shape[0], -1).cpu()
    row_pid = torch.from_numpy(_pid(off))
    plists = P.passage_lists(idx.row_index.cpu(), idx.list_offsets.cpu(), row_pid)
    list_ids = idx.plaid.list_ids.cpu()
    return P.search(q.half().float(), idx.ivf.centroids.cpu(), probes, store, off, list_ids, plists, idx.plaid.ndocs,
                    idx.plaid.threshold, top_n, first_doc)


def test_pruned_search_equals_oracle():
    dim, nlist, n_pass = 64, 24, 400
    store, off = _grid_store(n_pass, dim, seed=41)
    cents = _grid_centroids(nlist, dim, seed=42)
    q = _grid_queries(3, 32, dim, seed=43)
    s_tab, _ = P.centroid_scores(q, cents, 0.0)
    t = float(s_tab[1, :, :32].max(-1).values.median())
    idx = _grid_index(store, off, cents, 3, 16, t)
    s, i = idx.search_device(q.half().to(DEV), 4)
    rs, ri = _oracle_search(idx, q, store, off, 4)
    assert torch.equal(i.cpu(), ri) and torch.equal(_f64(s), rs)
    cand = idx.plaid.candidates(idx, idx.plaid.centroid_scores(idx, q.half().to(DEV))[2], 32)
    assert int((cand[1] >= 0).sum()) > 16                                   # more candidates than ndocs


def test_two_halves_merged_equal_the_oracle_per_half():
    dim, nlist, n_pass, top_n = 64, 24, 300, 8
    store, off = _grid_store(n_pass, dim, seed=51)
    cents = _grid_centroids(nlist, dim, seed=52)
    q = _grid_queries(3, 40, dim, seed=53)
    h = n_pass // 2
    parts, refs = [], []
    for lo, hi in ((0, h), (h, n_pass)):
        o = off[lo:hi + 1] - off[lo]
        st = store[int(off[lo]):int(off[hi])]
        idx = _grid_index(st, o, cents, 4, 32, 0.25, first_doc=lo)
        parts.append(idx.search_device(q.half().to(DEV), top_n))
        refs.append(_oracle_search(idx, q, st, o, top_n, first_doc=lo))
    s, i = interaction.topk_merge(torch.cat([parts[0][0], parts[1][0]], 1), torch.cat([parts[0][1], parts[1][1]], 1),
                                  top_n)
    rs, ri = P.topk(torch.cat([refs[0][0], refs[1][0]], 1), torch.cat([refs[0][1], refs[1][1]], 1), top_n)
    assert torch.equal(i.cpu(), ri) and torch.equal(_f64(s), rs)
    assert bool((i < h).any() & (i >= h).any())


# ----------------------------------------------------------------------------------------------------------------------
# 7. save / load, 8. CUDA graph
# ----------------------------------------------------------------------------------------------------------------------
def test_save_load_same_results(tmp_path):
    dim, nlist = 128, 32
    store, off, cent = _clustered_store(500, dim, 40, seed=61)
    q = _queries(cent, 4, 32, seed=62).to(DEV).half()
    blocks = [store.numpy()]
    cfg = _cfg(dim, nlist, 4, colbert_plaid_ndocs=256)
    idx = _build(ColBERTIVFIndexer, store, off, cfg)
    ref = idx.search_device(q, 50)
    idx.save(str(tmp_path / "ivf"))
    re_ = ColBERTIVFIndexer(cfg, device=DEV)
    re_.load(str(tmp_path / "ivf"))
    re_.index([_pid(off)], blocks)
    got = re_.search_device(q, 50)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])

    rcfg = _cfg(dim, nlist, 4, colbert_plaid_ndocs=256, colbert_residual_bits=2)
    res = _build(ColBERTResidualIndexer, store, off, rcfg)
    ref = res.search_device(q, 50)
    res.save(str(tmp_path / "res"))
    re_ = ColBERTResidualIndexer(rcfg, device=DEV)
    re_.load(str(tmp_path / "res"))
    got = re_.search_device(q, 50)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    assert re_.plaid.list_ids is re_.tokens.list_ids                        # the codes' list ids, not a copy


@pytest.mark.parametrize("residual", [False, True])
def test_search_device_replays_in_cuda_graph(residual):
    dim = 128
    store, off, cent = _clustered_store(800, dim, 30, seed=71)
    extra = {"colbert_plaid_ndocs": 128, "colbert_plaid_centroid_score_threshold": 0.3}
    if residual:
        extra["colbert_residual_bits"] = 1
    idx = _build(ColBERTResidualIndexer if residual else ColBERTIVFIndexer, store, off, _cfg(dim, 32, 4, **extra))
    q = _queries(cent, 4, 32, seed=72).half().to(DEV)
    ref_s, ref_i = idx.search_device(q, 32)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gs, gi = idx.search_device(q, 32)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gs, ref_s) and torch.equal(gi, ref_i)


# ----------------------------------------------------------------------------------------------------------------------
# 9. recall against the exact indexer
# ----------------------------------------------------------------------------------------------------------------------
RECALL_FLOOR = 0.80   # first H100 measurement: 0.8156


def test_recall_at_100_against_exact_indexer():
    dim, nlist, top_n = 128, 128, 100
    store, off, cent = _clustered_store(5000, dim, 160, seed=81)
    q = _queries(cent, 16, 32, seed=82).half()
    blocks = [store.numpy()]
    exact = ColBERTEndToEndIndexer({"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16"}, device=DEV)
    exact.index([_pid(off)], blocks)
    _, ri = exact.search_device(q.to(DEV), top_n)
    idx = _build(ColBERTIVFIndexer, store, off, _cfg(dim, nlist, 4, colbert_plaid_ndocs=1024))
    _, i = idx.search_device(q.to(DEV), top_n)
    i, ri = i.cpu(), ri.cpu()
    rec = float(np.mean([len(set(i[a].tolist()) & set(ri[a].tolist())) / top_n for a in range(q.shape[0])]))
    print(f"PLAID recall@100 against the exact indexer: {rec:.4f}")
    assert rec >= RECALL_FLOOR, rec


# ----------------------------------------------------------------------------------------------------------------------
# 10. search-time checks
# ----------------------------------------------------------------------------------------------------------------------
def test_search_checks():
    dim = 64
    store, off = _grid_store(100, dim, seed=91)
    idx = _grid_index(store, off, _grid_centroids(8, dim, 92), 2, 64, 0.0)
    q = _grid_queries(2, 32, dim, 93).half().to(DEV)
    idx.search_device(q, 16)
    with pytest.raises(_lib.MatchmakerB200Error, match="ndocs // 4"):
        idx.search_device(q, 17)
    with pytest.raises(_lib.MatchmakerB200Error, match="token_top_k"):
        idx.search_device(q, 10, token_top_k=8)
    with pytest.raises(_lib.MatchmakerB200Error, match="Lq"):
        idx.search_device(_grid_queries(2, 129, dim, 94).half().to(DEV), 10)
    with pytest.raises(_lib.MatchmakerB200Error, match="NaN"):
        interaction.plaid_centroid_scores(q, _grid_centroids(8, dim, 92).half().to(DEV), float("nan"))
