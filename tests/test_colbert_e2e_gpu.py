"""ColBERT end-to-end retrieval on the GPU: store-mode max-sim, per-query de-duplication, the indexer, maxP."""
import numpy as np
import pytest
import torch

import colbert_e2e_oracle as E
from conftest import assert_close_rel
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, FlatIPIndexer
from matchmaker_b200.retrieval.colbert_e2e import doc_offsets_from_id_mapping
from matchmaker_b200.retrieval.token_storage import TokenStorageWriter, load_token_storage

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FLT_MAX = 3.4028234663852886e38


def _config(dim, dtype="float16"):
    return {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": dtype}


def _store(lengths, dim, seed, dtype=torch.float16, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    lengths = [int(x) for x in lengths]
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    store = (torch.randn(int(off[-1]), dim, generator=g) * scale).to(dtype)
    return store, off


def _padded(store, off, max_len):
    n = len(off) - 1
    d = torch.zeros((n, max_len, store.shape[1]), dtype=store.dtype)
    m = torch.zeros((n, max_len), dtype=torch.bool)
    for i in range(n):
        L = int(off[i + 1] - off[i])
        d[i, :L] = store[off[i]:off[i + 1]]
        m[i, :L] = True
    return d, m


def _index(store, off, dim, dtype="float16"):
    idx = ColBERTEndToEndIndexer(_config(dim, dtype), device=DEV)
    pid = np.repeat(np.arange(len(off) - 1), np.diff(off))
    idx.index([pid], [store.float().numpy().astype(np.float16 if dtype == "float16" else np.float32)])
    return idx


# ----------------------------------------------------------------------------------------------------------------------
# 1. store max-sim == padded max-sim (bit-exact, per kernel) and the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl,dim,lq,dtype", [("tcgen05", 64, 32, torch.float16), ("tcgen05", 128, 32, torch.float16),
                                               ("tcgen05", 128, 20, torch.bfloat16),
                                               ("tcgen05_docm", 768, 40, torch.float16), ("simt", 128, 32, torch.float32)])
def test_store_maxsim_matches_padded(impl, dim, lq, dtype):
    rng = np.random.default_rng(11)
    n_docs = 120
    lengths = rng.integers(1, 301, n_docs)
    lengths[[7, 50]] = 0                      # passages without rows
    lengths[-1] = 300                         # the last passage ends at row T-1 and needs two tiles
    store, off = _store(lengths, dim, seed=12, dtype=dtype)
    max_len = int(lengths.max())
    g = torch.Generator().manual_seed(13)
    n_q = 5
    q = (torch.randn(n_q, lq, dim, generator=g) * 0.3).to(dtype)
    n_pairs = 1001                            # not a multiple of the grid
    pq = torch.from_numpy(rng.integers(0, n_q, n_pairs)).to(torch.int32)
    live = np.flatnonzero(lengths > 0)
    pd = torch.from_numpy(rng.choice(live, n_pairs)).to(torch.int32)
    got = interaction.maxsim_store(q.to(DEV), store.to(DEV), torch.from_numpy(off).to(DEV), pq.to(DEV), pd.to(DEV),
                                   max_len, impl=impl)
    d, m = _padded(store, off, max_len)
    ref = interaction.maxsim(q.to(DEV), d.to(DEV), None, m.to(DEV), pair_q=pq.to(DEV), pair_d=pd.to(DEV), impl=impl)
    assert torch.equal(got.cpu(), ref.cpu()), f"{impl}: store mode differs from the padded layout"
    full = E.maxsim_store(q.float(), store.float(), off)
    assert_close_rel(got.cpu(), full[pq.long(), pd.long()], rel=1e-3, what=f"{impl} vs oracle")

    # skipped pairs and passages without rows score -inf (the padded path has no equivalent)
    pd2 = torch.tensor([-1, 7, 50, -5, int(live[0])], dtype=torch.int32)
    pq2 = torch.tensor([0, 1, 2, 3, 4], dtype=torch.int32)
    s2 = interaction.maxsim_store(q.to(DEV), store.to(DEV), torch.from_numpy(off).to(DEV), pq2.to(DEV), pd2.to(DEV),
                                  max_len, impl=impl).cpu()
    assert torch.isneginf(s2[:4]).all() and torch.isfinite(s2[4])


# ----------------------------------------------------------------------------------------------------------------------
# 2. topk_unique == oracle, bit-exact
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nq,L,id_range,k", [(3, 500, 60, 40), (2, 20000, 3000, 1000), (2, 20000, 9000, 4096),
                                             (4, 300, 10, 50), (1, 8193, 5000, 4096)])
def test_topk_unique_matches_oracle(nq, L, id_range, k):
    rng = np.random.default_rng(L + k)
    scores = np.round(rng.normal(size=(nq, L)) * 4) / 4        # many exact ties
    ids = rng.integers(-5, id_range, size=(nq, L))             # duplicates, negative ids
    void = rng.random((nq, L))
    scores[void < 0.03] = np.nan
    scores[(void >= 0.03) & (void < 0.06)] = -np.inf
    scores[(void >= 0.06) & (void < 0.09)] = -FLT_MAX
    s = torch.from_numpy(scores).float()
    i = torch.from_numpy(ids).long()
    gs, gi = interaction.topk_unique(s.to(DEV), i.to(DEV), k)
    rs, ri = E.topk_unique(s, i, k)
    assert torch.equal(gi.cpu(), ri)
    assert torch.equal(gs.cpu(), rs)


# ----------------------------------------------------------------------------------------------------------------------
# 3. exhaustive k': the index equals max-sim over every passage + topk_merge
# ----------------------------------------------------------------------------------------------------------------------
def test_exhaustive_matches_maxsim_over_all_passages():
    rng = np.random.default_rng(21)
    lengths = rng.integers(1, 26, 70)
    lengths[[3, 40]] = 0
    dim, lq, top_n = 128, 32, 50
    store, off = _store(lengths, dim, seed=22)
    assert off[-1] <= 1024
    idx = _index(store, off, dim)
    q = (torch.randn(4, lq, dim, generator=torch.Generator().manual_seed(23)) * 0.3).half()
    s, i = idx.search_device(q.to(DEV), top_n, token_top_k=1024)
    max_len = int(lengths.max())
    d, m = _padded(store, off, max_len)
    live = torch.from_numpy(np.flatnonzero(lengths > 0))
    n = len(live)
    pq = torch.arange(4).repeat_interleave(n).to(torch.int32)
    pd = live.repeat(4).to(torch.int32)
    all_s = interaction.maxsim(q.to(DEV), d.to(DEV), None, m.to(DEV), pair_q=pq.to(DEV), pair_d=pd.to(DEV)).view(4, n)
    rs, ri = interaction.topk_merge(all_s, live.to(DEV).unsqueeze(0).expand(4, -1), top_n)
    assert torch.equal(i, ri) and torch.equal(s, rs)
    os_, oi = E.colbert_e2e_search(q.float(), store.float(), off, top_n)
    assert_close_rel(s.cpu(), os_.float(), rel=1e-3, what="exhaustive vs oracle")


# ----------------------------------------------------------------------------------------------------------------------
# 4. bounded k' against the fp64 oracle
# ----------------------------------------------------------------------------------------------------------------------
def _token_hits64(q, store, off, kp):
    """Per (query, live token): fp64 scores and tolerances of all rows, plus the k'-th / (k'+1)-th best score."""
    s64 = E.token_scores(q, store, torch.float64)
    tol = E.accumulation_tol(q, store)
    live = (q != 0).any(-1)
    srt = s64.sort(-1, descending=True).values
    return s64, tol, live, srt


def test_bounded_token_top_k_candidates_and_ranking():
    rng = np.random.default_rng(31)
    lengths = rng.integers(5, 40, 2000)
    dim, lq, kp, top_n = 128, 32, 16, 20
    store, off = _store(lengths, dim, seed=32)
    q = (torch.randn(3, lq, dim, generator=torch.Generator().manual_seed(33)) * 0.3).half()
    q[2, 25:] = 0
    idx = _index(store, off, dim)
    cs, ci = idx.candidates_device(q.to(DEV), kp)
    ci = ci.cpu()
    pid = E.row_passages(off)
    s64, tol, live, srt = _token_hits64(q, store, off, kp)
    for a in range(q.shape[0]):
        got = set(int(x) for x in ci[a] if x >= 0)
        must, may = set(), set()
        for t in range(lq):
            if not live[a, t]:
                continue
            tmax = float(tol[a, t].max())
            hi_cut, lo_cut = float(srt[a, t, kp]) + 2 * tmax, float(srt[a, t, kp - 1]) - 2 * tmax
            must |= set(pid[s64[a, t] > hi_cut].tolist())
            may |= set(pid[s64[a, t] >= lo_cut].tolist())
        assert must <= got, f"query {a}: decided candidates missing: {sorted(must - got)[:10]}"
        assert got <= may, f"query {a}: passages outside every token's top-k': {sorted(got - may)[:10]}"
    # final ranking over the candidates, checked against fp64 wherever fp64 separates neighbouring ranks
    s, i = idx.search_device(q.to(DEV), top_n, token_top_k=kp)
    s, i = s.cpu().double(), i.cpu()
    for a in range(q.shape[0]):
        cands = sorted(int(x) for x in ci[a] if x >= 0)
        sc, tl = [], []
        for dd in cands:
            blk = s64[a, :, off[dd]:off[dd + 1]]
            j = blk.argmax(-1)
            sc.append(float(blk.max(-1).values[live[a]].sum()))
            tl.append(float(tol[a, :, off[dd]:off[dd + 1]].gather(-1, j.unsqueeze(-1)).squeeze(-1).sum()) + lq * 2 ** -23 * abs(sc[-1]))
        order = sorted(range(len(cands)), key=lambda x: (-sc[x], cands[x]))
        for r in range(top_n):
            o = order[r]
            left = r == 0 or sc[order[r - 1]] - sc[o] > 2 * max(tl[o], tl[order[r - 1]])
            right = sc[o] - sc[order[r + 1]] > 2 * max(tl[o], tl[order[r + 1]])
            if left and right:
                assert int(i[a, r]) == cands[o], f"query {a} rank {r}"
            assert abs(s[a, r] - sc[order[r]]) <= 1e-3 * abs(sc[order[r]]) + 1e-3


def test_candidate_cap_keeps_best_distinct_passages():
    rng = np.random.default_rng(41)
    lengths = rng.integers(1, 8, 20000)
    dim, lq, kp = 128, 32, 256                 # Lq * k' = 8192 > 4096
    store, off = _store(lengths, dim, seed=42)
    q = (torch.randn(2, lq, dim, generator=torch.Generator().manual_seed(43)) * 0.3).half()
    idx = _index(store, off, dim)
    cs, ci = idx.candidates_device(q.to(DEV), kp)
    assert ci.shape[1] == 4096
    ci = ci.cpu()
    pid = E.row_passages(off)
    s64, tol, live, srt = _token_hits64(q, store, off, kp)
    for a in range(q.shape[0]):
        best = {}
        tmax = float(tol[a].max())
        for t in range(lq):
            top = torch.topk(s64[a, t], kp)
            for v, r in zip(top.values.tolist(), top.indices.tolist()):
                p = int(pid[r])
                best[p] = max(best.get(p, -1e300), v)
        assert len(best) > 4096
        ranked = sorted(best.values(), reverse=True)
        hi_cut, lo_cut = ranked[4096] + 2 * tmax, ranked[4095] - 2 * tmax
        got = set(int(x) for x in ci[a])
        must = {p for p, v in best.items() if v > hi_cut}
        never = {p for p, v in best.items() if v < lo_cut}
        assert must <= got and not (got & never)


# ----------------------------------------------------------------------------------------------------------------------
# 5. planted passages come first
# ----------------------------------------------------------------------------------------------------------------------
def test_planted_passages_rank_first():
    rng = np.random.default_rng(51)
    lengths = rng.integers(10, 120, 3000)
    dim, lq = 128, 32
    store, off = _store(lengths, dim, seed=52)
    g = torch.Generator().manual_seed(53)
    q = torch.randn(4, lq, dim, generator=g) * 0.3
    planted = [17, 900, 1500, 2999]
    for a, p in enumerate(planted):
        n = int(off[p + 1] - off[p])
        rows = q[a, torch.arange(n) % lq] + torch.randn(n, dim, generator=g) * 0.02
        store[off[p]:off[p + 1]] = rows.half()
    idx = _index(store, off, dim)
    s, i = idx.search(q.half().numpy(), 10, token_top_k=32)
    assert i[:, 0].tolist() == planted


# ----------------------------------------------------------------------------------------------------------------------
# 6. storage round trip
# ----------------------------------------------------------------------------------------------------------------------
def test_storage_round_trip(tmp_path):
    rng = np.random.default_rng(61)
    dim = 128
    w = TokenStorageWriter(str(tmp_path), dim, 256, "float16")
    mats = []
    for n in range(40):
        L = int(rng.integers(3, 25))              # at most 40 * 24 rows: token_top_k = 1024 is exhaustive
        m = (rng.normal(size=(L, dim)) * 0.3).astype(np.float16)
        if n == 23:
            m[:] = 0                              # all rows stripped: the passage has no stored rows
        mats.append(m)
        w.add(f"doc{n}", m)
    w.close()
    storage, id_mapping, seq_ids, doc_infos = load_token_storage(str(tmp_path))
    assert len(storage) > 2 and doc_infos["doc23"][1] == doc_infos["doc23"][2]
    idx = ColBERTEndToEndIndexer(_config(dim), device=DEV)
    idx.index(id_mapping, storage)
    q = np.zeros((3, 20, dim), dtype=np.float16)
    for j, k in enumerate((5, 30, 39)):
        n = min(20, len(mats[k]))
        q[j, :n] = mats[k][:n]
    s, i = idx.search(q, 50, token_top_k=1024)
    assert 23 not in set(i.flatten().tolist())
    assert [seq_ids[x] for x in i[:, 0]] == ["doc5", "doc30", "doc39"]
    off = doc_offsets_from_id_mapping(id_mapping)
    rows = torch.from_numpy(np.concatenate(storage)).float()
    os_, oi = E.colbert_e2e_search(torch.from_numpy(q).float(), rows, off, 50)
    assert (i[:, 39:] == -1).all() and (oi[:, 39:] == -1).all()      # 39 passages have rows
    assert_close_rel(torch.from_numpy(s[:, :39]), os_[:, :39].float(), rel=1e-3, what="round trip")


# ----------------------------------------------------------------------------------------------------------------------
# 7. two shards in one process
# ----------------------------------------------------------------------------------------------------------------------
def test_two_shards_merge_to_single_index(monkeypatch):
    rng = np.random.default_rng(71)
    lengths = rng.integers(1, 25, 60)
    dim, top_n = 128, 40
    store, off = _store(lengths, dim, seed=72)
    q = (torch.randn(3, 32, dim, generator=torch.Generator().manual_seed(73)) * 0.3).half().to(DEV)
    single = _index(store, off, dim)
    s_ref, i_ref = single.search_device(q, top_n, token_top_k=1024)
    parts = []
    for r in range(2):
        idx = ColBERTEndToEndIndexer(_config(dim), device=DEV)
        monkeypatch.setattr(idx, "_world", lambda r=r: (r, 2))
        pid = np.repeat(np.arange(len(off) - 1), np.diff(off))
        idx.index([pid], [store.numpy()])
        assert 0 < idx.d_hi - idx.d_lo < len(off) - 1
        parts.append(idx.search_device(q, top_n, token_top_k=1024))
    s, i = interaction.topk_merge(torch.cat([parts[0][0], parts[1][0]], 1), torch.cat([parts[0][1], parts[1][1]], 1), top_n)
    assert torch.equal(i, i_ref) and torch.equal(s, s_ref)


# ----------------------------------------------------------------------------------------------------------------------
# 8. query padding
# ----------------------------------------------------------------------------------------------------------------------
def test_query_padding_adds_nothing():
    rng = np.random.default_rng(81)
    lengths = rng.integers(1, 60, 500)
    dim = 128
    store, off = _store(lengths, dim, seed=82)
    idx = _index(store, off, dim)
    q = (torch.randn(3, 32, dim, generator=torch.Generator().manual_seed(83)) * 0.3).half()
    q[:, 20:] = 0
    q[2] = 0                                    # a query made only of padding
    s_pad, i_pad = idx.search_device(q.to(DEV), 30, token_top_k=8)
    s_trim, i_trim = idx.search_device(q[:, :20].contiguous().to(DEV), 30, token_top_k=8)
    assert torch.equal(i_pad, i_trim) and torch.equal(s_pad, s_trim)
    assert (i_pad[2] == -1).all() and (s_pad[2] == -FLT_MAX).all()
    cs, ci = idx.candidates_device(q.to(DEV), 8)
    cs2, ci2 = idx.candidates_device(q[:, :20].contiguous().to(DEV), 8)
    assert torch.equal(ci[:, :ci2.shape[1]], ci2) and (ci[:, ci2.shape[1]:] == -1).all()


# ----------------------------------------------------------------------------------------------------------------------
# 9. maxP de-duplication
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_pass,vec_per,hits,top_n", [(400, 6, 256, 50), (10, 20, 64, 30)])
def test_search_unique_matches_maxp_loop(n_pass, vec_per, hits, top_n):
    from oracle import interaction_oracle as O
    g = torch.Generator().manual_seed(91)
    dim = 128
    vecs = (torch.randn(n_pass * vec_per, dim, generator=g) * 0.3).half()
    pid = np.repeat(np.arange(n_pass), vec_per)
    idx = FlatIPIndexer(_config(dim), device=DEV)
    idx.index([pid], [vecs.numpy()])
    q = (torch.randn(5, dim, generator=g) * 0.3).half()
    raw_s, raw_i = idx.search(q.numpy(), hits)
    ref_s, _ = O.flat_ip_search(q.float(), vecs, torch.from_numpy(pid), hits)
    assert_close_rel(torch.from_numpy(raw_s), ref_s, rel=1e-3, what="vector hits")
    s, i = idx.search_unique(q.numpy(), top_n, hits)
    ref = E.maxp_loop(raw_s, raw_i, top_n)
    for a in range(5):
        n = len(ref[a])
        assert i[a, :n].tolist() == [x for x, _ in ref[a]]
        assert s[a, :n].tolist() == [np.float32(v).item() for _, v in ref[a]]
        assert (i[a, n:] == -1).all() and (s[a, n:] == -FLT_MAX).all()
    if n_pass < top_n:
        assert (i[:, n_pass:] == -1).all()


# ----------------------------------------------------------------------------------------------------------------------
# 10. bad input
# ----------------------------------------------------------------------------------------------------------------------
def test_bad_input_raises():
    dim = 128
    store, off = _store([5, 7, 3], dim, seed=101)
    idx = ColBERTEndToEndIndexer(_config(dim), device=DEV)
    with pytest.raises(_lib.MatchmakerB200Error):
        idx.index([np.array([0, 0, 2, 2, 1])], [store[:5].numpy()])
    idx = _index(store, off, dim)
    with pytest.raises(_lib.MatchmakerB200Error):
        idx.search(np.zeros((1, 32, 64), dtype=np.float16), 10)
    with pytest.raises(_lib.MatchmakerB200Error):
        idx.search(np.ones((1, 32, dim), dtype=np.float16), 10, token_top_k=2000)
    s = torch.zeros(2, 6000, device=DEV)
    ids = torch.arange(6000, device=DEV).repeat(2, 1)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.topk_unique(s, ids, 5000)
