"""Graph index on the GPU.  With integer-valued vectors (|x| <= 8) every dot product is exact in fp32, so the pruning, the
built graph and the search must equal the CPU oracle bit for bit; on Gaussian data the results are checked against exact
search with the flat-IP tolerances.  Also the drop-in behaviour of retrieval.GraphIndexer."""
import functools

import numpy as np
import pytest
import torch

import colbert_e2e_oracle as E
import graph_oracle as G
import ivf_oracle as V
from matchmaker_b200 import _lib, interaction, sharding
from matchmaker_b200.retrieval import FlatIPIndexer, GraphIndexer
from matchmaker_b200.retrieval.graph_index import graph_degrees, search_list_size
from oracle import interaction_oracle as O
from test_graph_cpu import HAND_KNN, HAND_PRUNED

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cfg(dtype="float16", M=8, efc=32, efs=32, dim=64, use_gpu=True):
    return {"token_dim": dim, "faiss_use_gpu": use_gpu, "token_dtype": dtype, "faiss_hnsw_graph_neighbors": M,
            "faiss_hnsw_efConstruction": efc, "faiss_hnsw_efSearch": efs}


def _index(x, ids, cfg):
    idx = GraphIndexer(cfg)
    idx.index([np.asarray(ids, dtype=np.int64)], [x.numpy()])
    return idx


@functools.lru_cache(maxsize=None)
def _knn_case(K):
    """Integer rows in [-2, 2] over 16 dims (heavy ties) with 10 % duplicate rows; their oracle k-NN lists and counts."""
    n = {32: 400, 256: 600, 1023: 1100}[K]
    x = G.integer_rows(n, 16, seed=K, dup=n // 10, lim=2)
    knn = G.knn(x, K)
    return knn, G.detour_counts(knn)


@pytest.mark.parametrize("R", [16, 64, 1024])
@pytest.mark.parametrize("K", [32, 256, 1023])
def test_prune_matches_oracle(K, R):
    knn, counts = _knn_case(K)
    got = interaction.graph_prune(torch.from_numpy(knn).to(DEV), R).cpu().numpy()
    assert np.array_equal(got, G.prune(knn, R, counts))


def test_prune_hand_built_graph():
    got = interaction.graph_prune(torch.from_numpy(HAND_KNN).to(DEV), 2).cpu().numpy()
    assert np.array_equal(got, HAND_PRUNED)


@pytest.mark.parametrize("dtype", ["float16", "float32"])
@pytest.mark.parametrize("dim, n, M, efc", [(64, 20, 16, 16), (128, 1500, 8, 40), (768, 700, 32, 64), (64, 1100, 4, 24),
                                            (64, 900, 12, 40)])
def test_built_graph_matches_oracle(dtype, dim, n, M, efc):
    x = G.integer_rows(n, dim, seed=n + dim, dup=n // 20)
    idx = _index(x, np.arange(n), _cfg(dtype, M, efc, 64, dim))
    R, K = graph_degrees(M, efc)
    assert np.array_equal(idx.graph.cpu().numpy(), G.build(x, R, K))
    assert np.array_equal(idx.entry_pos.cpu().numpy(), G.entry_positions(n))


def _search_case(dtype, n, M, efs, top_n, nq, dim=64, seed=0):
    x = G.integer_rows(n, dim, seed=n + seed, dup=n // 50)
    q = G.integer_rows(nq, dim, seed=n + seed + 1)
    ids = np.arange(n, dtype=np.int64) * 3 - n           # negative user ids too
    idx = _index(x, ids, _cfg(dtype, M, 32, efs, dim))
    s, i = idx.search(q.numpy(), top_n)
    L = search_list_size(efs, top_n)
    rs, ri, visited = G.search(q, x, idx.graph.cpu().numpy(), G.entry_positions(n), L, top_n, ids=ids)
    return (s, i), (rs.numpy(), ri.numpy()), visited, L, idx


@pytest.mark.parametrize("dtype", ["float16", "float32"])
@pytest.mark.parametrize("n, M, efs, top_n, nq", [(3000, 8, 32, 1, 16), (3000, 8, 64, 10, 16), (3000, 16, 128, 100, 8),
                                                  (2000, 16, 1024, 1000, 3), (50, 8, 128, 10, 8), (1, 8, 32, 10, 4),
                                                  (3000, 8, 150, 100, 8), (3000, 12, 64, 10, 16)])
def test_search_matches_oracle(dtype, n, M, efs, top_n, nq):
    (s, i), (rs, ri), _, _, _ = _search_case(dtype, n, M, efs, top_n, nq)
    assert np.array_equal(i, ri) and np.array_equal(s, rs)
    if n < top_n:
        assert np.all(i[:, n:] == -1) and np.all(s[:, n:] == np.float32(G.NO_RESULT))


def test_search_visiting_more_rows_than_the_hash_holds_is_unchanged():
    (s, i), (rs, ri), visited, L, idx = _search_case("float16", 6000, 8, 32, 10, 16, seed=5)
    slots = interaction.graph_hash_slots(L, idx.R)
    assert visited.max() > slots, (visited, slots)
    assert np.array_equal(i, ri) and np.array_equal(s, rs)


def test_empty_shard_and_two_shards(monkeypatch):
    n, dim = 3000, 64
    x = G.integer_rows(n, dim, seed=7, dup=30)
    q = G.integer_rows(12, dim, seed=8)
    ids = np.arange(n, dtype=np.int64) * 5 - 7000
    parts, ref_s, ref_i = [], [], []
    for rank in (0, 1):
        monkeypatch.setattr(GraphIndexer, "_world", lambda self, r=rank: (r, 2))
        idx = GraphIndexer(_cfg(M=8, efs=64))
        idx.index([ids[:1000], ids[1000:]], [x[:1000].numpy(), x[1000:].numpy()])
        monkeypatch.setattr(GraphIndexer, "_world", lambda self: (0, 1))
        lo, hi = sharding.shard_bounds(n, rank, 2)
        assert (idx.lo, idx.hi) == (lo, hi) and torch.equal(idx.ids.cpu(), torch.from_numpy(ids[lo:hi]))
        parts.append(idx.search_device(q.to(DEV).half(), 100))
        rs, ri, _ = G.search(q, x[lo:hi], idx.graph.cpu().numpy(), G.entry_positions(hi - lo), 128, 100, ids=ids[lo:hi])
        ref_s.append(rs)
        ref_i.append(ri)
    s, i = interaction.topk_merge(torch.cat([parts[0][0], parts[1][0]], 1), torch.cat([parts[0][1], parts[1][1]], 1), 100)
    ms, mi = sharding.rank_topk(torch.cat(ref_s, 1), torch.cat(ref_i, 1), 100)
    assert torch.equal(i.cpu(), mi) and torch.equal(s.cpu(), ms)
    # a rank without rows answers with the tail only
    monkeypatch.setattr(GraphIndexer, "_world", lambda self: (1, 2))
    empty = GraphIndexer(_cfg(M=8))
    empty.index([ids[:1]], [x[:1].numpy()])
    monkeypatch.setattr(GraphIndexer, "_world", lambda self: (0, 1))
    es, ei = empty.search(q.numpy(), 10)
    assert np.all(ei == -1) and np.all(es == np.float32(G.NO_RESULT))


def _clusters(n, dim, seed, nq=64, n_clusters=50, spread=1.0):
    """Gaussian clusters around unit centres, noise of length `spread`: (rows, queries, row labels, query labels)."""
    g = torch.Generator().manual_seed(seed)
    centers = torch.nn.functional.normalize(torch.randn(n_clusters, dim, generator=g), dim=1)
    lx = torch.randint(0, n_clusters, (n,), generator=g)
    x = centers[lx] + spread * torch.randn(n, dim, generator=g) / dim ** 0.5
    lq = torch.randint(0, n_clusters, (nq,), generator=g)
    q = centers[lq] + spread * torch.randn(nq, dim, generator=g) / dim ** 0.5
    return x, q, lx, lq


def _gauss(n, dim, seed, nq=64):
    return _clusters(n, dim, seed, nq)[:2]


def test_two_runs_are_bit_identical():
    x, q = _gauss(4000, 128, seed=1)
    a = _index(x, np.arange(4000), _cfg(M=16, efc=64, efs=64, dim=128))
    b = _index(x, np.arange(4000), _cfg(M=16, efc=64, efs=64, dim=128))
    assert torch.equal(a.graph, b.graph)
    qd = q.to(DEV).half()
    s1, i1 = a.search_device(qd, 50)
    s2, i2 = b.search_device(qd, 50)
    assert torch.equal(s1, s2) and torch.equal(i1, i2)


@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_every_row_an_entry_equals_flat_search(dtype):
    n = 1000                                        # E = min(n, max(1024, n // 128)) = n
    x, q = _gauss(n, 128, seed=2)
    ids = np.arange(n, dtype=np.int64) * 7 - 3000
    graph = _index(x, ids, _cfg(dtype, M=16, efc=64, efs=128, dim=128))
    assert graph.entry_pos.numel() == n
    flat = FlatIPIndexer(_cfg(dtype, dim=128))
    flat.index([ids], [x.numpy()])
    s, i = graph.search(q.numpy(), 100)
    fs, fi = flat.search(q.numpy(), 100)
    tids = torch.from_numpy(ids)
    if dtype == "float16":
        O.flat_ip_check_exact(q.half().float(), x.half().float(), tids, torch.from_numpy(s), torch.from_numpy(i), 100)
    else:
        whole, probes = torch.tensor([0, n]), torch.zeros(q.shape[0], 1, dtype=torch.int64)
        V.ivf_check_split(q, x, tids, whole, probes, torch.from_numpy(s), torch.from_numpy(i), 100)
    assert (i == fi).mean() > 0.99


def test_recall_on_overlapping_clusters():
    """Noise twice as long as the centres: at spread 1 in 128 dimensions the exact k-NN graph keeps almost every edge
    inside its cluster and falls into one component per cluster, so the entry sample alone would find each query's
    cluster and recall would say nothing about the graph."""
    x, q, lx, lq = _clusters(20000, 128, seed=3, nq=128, spread=2.0)
    ids = np.arange(20000, dtype=np.int64)
    graph = _index(x, ids, _cfg(M=32, efc=128, efs=128, dim=128))
    flat = FlatIPIndexer(_cfg(dim=128))
    flat.index([ids], [x.numpy()])
    _, i = graph.search(q.numpy(), 100)
    _, fi = flat.search(q.numpy(), 100)

    def recall(got):
        return np.mean([len(set(a) & set(b)) / 100 for a, b in zip(got.tolist(), fi.tolist())])
    # the clusters overlap: a quarter or more of a query's exact top-100 lies outside its own cluster, and the entry
    # scan alone (the 100 best of the 1024 entry rows) finds few of them
    same = (lx[torch.from_numpy(fi)] == lq.unsqueeze(1)).float().mean().item()
    assert same < 0.85, same
    entry_only = graph.entries(q.to(DEV).half(), 128)[:, :100].cpu().numpy()
    assert recall(entry_only) < 0.2, recall(entry_only)
    assert recall(i) >= 0.95, recall(i)


def test_drop_in_behaviour(tmp_path):
    x, q = _gauss(5000, 64, seed=4)
    ids = np.arange(5000, dtype=np.int64) * 2 - 3000
    idx = GraphIndexer(_cfg(M=8, efc=32, efs=32, use_gpu=False))     # the reference's example config sets False
    idx.prepare([x.numpy()])
    idx.index([ids[:2500], ids[2500:]], [x[:2500].numpy(), x[2500:].numpy()])
    s, i = idx.search(q.numpy().astype(np.float16), 10)
    assert isinstance(s, np.ndarray) and s.dtype == np.float32 and i.dtype == np.int64 and s.shape == (64, 10)
    s1, i1 = idx.search(q[3].numpy(), 10)                 # 1-D query
    assert np.array_equal(i1[0], i[3])
    path = str(tmp_path / "faiss.index")
    idx.save(path)
    back = GraphIndexer(_cfg(M=8, efc=32, efs=32))
    back.load(path)
    s2, i2 = back.search(q.numpy(), 10)
    assert np.array_equal(s2, s) and np.array_equal(i2, i)
    wide = GraphIndexer(_cfg(M=8, efc=32, efs=32))
    wide.load(path, {"faiss_hnsw_efSearch": 256})
    assert wide.ef_search == 256
    s3, i3 = wide.search(q.numpy(), 10)
    flat = FlatIPIndexer(_cfg())
    flat.index([ids], [x.numpy()])
    _, fi = flat.search(q.numpy(), 10)
    hits = lambda got: np.mean([len(set(a) & set(b)) for a, b in zip(got.tolist(), fi.tolist())])  # noqa: E731
    assert hits(i3) >= hits(i)
    with pytest.raises(_lib.MatchmakerB200Error):
        GraphIndexer(_cfg("float32", M=8)).load(path)
    blob = torch.load(path)
    blob["world"] = 2
    torch.save(blob, path)
    with pytest.raises(_lib.MatchmakerB200Error):
        GraphIndexer(_cfg(M=8)).load(path)


def test_search_unique_matches_the_maxp_loop():
    x, q = _gauss(4000, 64, seed=5, nq=8)
    ids = (np.arange(4000) // 4).astype(np.int64)        # four vectors per passage
    idx = _index(x, ids, _cfg(M=8, efs=64))
    s, i = idx.search_unique(q.numpy(), 10, 200)
    hs, hi = idx.search(q.numpy(), 200)
    loop = E.maxp_loop(hs, hi, 10)
    for a in range(8):
        assert [int(v) for v in i[a, :len(loop[a])]] == [int(p) for p, _ in loop[a]]
        assert [float(v) for v in s[a, :len(loop[a])]] == [sc for _, sc in loop[a]]


def test_search_device_replays_in_a_cuda_graph():
    x, q = _gauss(6000, 64, seed=6)
    idx = _index(x, np.arange(6000), _cfg(M=8, efs=64))
    qd = q.to(DEV).half()
    ref_s, ref_i = idx.search_device(qd, 100)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gs, gi = idx.search_device(qd, 100)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gs, ref_s) and torch.equal(gi, ref_i)


def test_search_rejects_sizes_outside_the_envelope():
    rows = torch.zeros(10, 64, dtype=torch.float16, device=DEV)
    q = torch.zeros(2, 64, dtype=torch.float16, device=DEV)
    ids, graph = torch.arange(10, device=DEV), torch.full((10, 4), -1, dtype=torch.int32, device=DEV)
    ent = torch.zeros(2, 1, dtype=torch.int64, device=DEV)
    for L, k in ((48, 1), (1056, 1), (32, 33)):
        with pytest.raises(_lib.MatchmakerB200Error):
            interaction.graph_search(q, rows, ids, graph, ent, k, L)
    with pytest.raises(_lib.MatchmakerB200Error):         # queries wider than the rows
        interaction.graph_search(torch.zeros(2, 128, dtype=torch.float16, device=DEV), rows, ids, graph, ent, 1, 32)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.graph_prune(torch.zeros(4, 1024, dtype=torch.int32, device=DEV), 4)
