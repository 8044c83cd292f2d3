"""Host-side pieces of the graph index: the oracle on hand-built graphs, the parameter mapping and its limits, the oracle's
search against the flat search, the bound symbols, and ptxas's report for the graph kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import graph_oracle as G
from matchmaker_b200 import _lib, build, interaction
from matchmaker_b200.retrieval import graph_index
from oracle import interaction_oracle as O

# N(0) = [1, 2, 3]: edge 0 -> 2 (rank 1) has a detour through 1 (2 is N(1)[0]); edge 0 -> 3 (rank 2) has none, since 3
# sits at rank 2 in N(1) and N(2).  N(3) = [2, 1, 0]: 3 -> 1 through 2, 3 -> 0 through 2 and through 1.
HAND_KNN = np.array([[1, 2, 3], [2, 0, 3], [1, 0, 3], [2, 1, 0]], dtype=np.int32)
HAND_COUNTS = np.array([[0, 1, 0], [0, 0, 0], [0, 0, 0], [0, 1, 2]])
HAND_PRUNED = np.array([[1, 3], [2, 0], [1, 0], [2, 1]], dtype=np.int32)
# head = first edge; reverse edges: 1 <- {0, 2}, 2 <- {1, 3} (all at rank 0, so ordered by w); then the rest
HAND_MERGED = np.array([[1, 3], [2, 0], [1, 3], [2, 1]], dtype=np.int32)


def test_hand_built_detour_counts_and_pruning():
    assert np.array_equal(G.detour_counts(HAND_KNN), HAND_COUNTS)
    assert np.array_equal(G.prune(HAND_KNN, 2), HAND_PRUNED)
    assert np.array_equal(G.prune(HAND_KNN, 3), HAND_KNN)           # R >= K keeps every edge in rank order
    assert np.array_equal(G.prune(HAND_KNN, 1), HAND_KNN[:, :1])


def test_hand_built_reverse_merge():
    assert np.array_equal(G.reverse_merge(HAND_PRUNED), HAND_MERGED)
    # R = 3, head of 2: u = 0 keeps [1, 2], gains 3 (0 is in the head of N(3) = [0, 1, 2]), duplicates skipped
    pruned = np.array([[1, 2, -1], [0, 2, -1], [0, 1, -1], [0, 1, 2]], dtype=np.int32)
    assert np.array_equal(G.reverse_merge(pruned), [[1, 2, 3], [0, 2, 3], [0, 1, -1], [0, 1, 2]])


def test_hand_built_graph_with_fewer_rows_than_edges_is_padded():
    x = torch.tensor([[3.0, 0.0], [2.0, 1.0], [0.0, 3.0]])
    k = G.knn(x, 4)
    assert np.array_equal(k, [[1, 2, -1, -1], [0, 2, -1, -1], [1, 0, -1, -1]])
    g = G.reverse_merge(G.prune(k, 4))
    assert np.array_equal(g, [[1, 2, -1, -1], [0, 2, -1, -1], [1, 0, -1, -1]])


def test_knn_drops_the_row_itself_among_duplicates():
    x = torch.tensor([[1.0, 0.0]] * 5 + [[0.0, 1.0]])
    k = G.knn(x, 3)
    for u in range(5):   # four tied copies: the lowest positions other than u
        assert list(k[u]) == [p for p in range(5) if p != u][:3]


def test_parameter_mapping():
    assert graph_index.graph_degrees(32, 128) == (64, 128)
    assert graph_index.graph_degrees(64, 40) == (128, 128)
    assert graph_index.graph_degrees(1, 1) == (2, 2)
    assert graph_index.search_list_size(128, 100) == 128
    assert graph_index.search_list_size(64, 100) == 128
    assert graph_index.search_list_size(1, 1) == 32
    assert graph_index.search_list_size(1000, 10) == 1024
    assert graph_index.search_list_size(16, 1000) == 1024
    assert len(graph_index.entry_positions(500)) == 500
    assert len(graph_index.entry_positions(200_000)) == 1562
    assert np.array_equal(graph_index.entry_positions(3000), G.entry_positions(3000))
    assert len(set(graph_index.entry_positions(3000).tolist())) == 1024


@pytest.mark.parametrize("M, efc, efs, key", [(1024, 128, 128, "faiss_hnsw_graph_neighbors"),
                                              (512, 128, 128, "faiss_hnsw_graph_neighbors"),
                                              (0, 128, 128, "faiss_hnsw_graph_neighbors"),
                                              (32, 1024, 128, "faiss_hnsw_efConstruction"),
                                              (32, 128, 1025, "faiss_hnsw_efSearch")])
def test_limits_name_the_key(M, efc, efs, key):
    cfg = {"token_dim": 64, "faiss_use_gpu": False, "token_dtype": "float16", "faiss_hnsw_graph_neighbors": M,
           "faiss_hnsw_efConstruction": efc, "faiss_hnsw_efSearch": efs}
    with pytest.raises(_lib.MatchmakerB200Error, match=key):
        graph_index.GraphIndexer(cfg, device="cuda:0")


def test_top_n_past_the_list_limit_names_it():
    with pytest.raises(_lib.MatchmakerB200Error, match="top_n"):
        graph_index.search_list_size(16, 1025)


def test_limits_inside_are_accepted():
    cfg = {"token_dim": 64, "faiss_use_gpu": False, "token_dtype": "float32", "faiss_hnsw_graph_neighbors": 511,
           "faiss_hnsw_efConstruction": 1023, "faiss_hnsw_efSearch": 1024}
    idx = graph_index.GraphIndexer(cfg, device="cuda:0")   # faiss_use_gpu False is accepted, and ignored
    assert (idx.R, idx.K) == (1022, 1023)


def test_oracle_search_with_every_row_an_entry_is_flat_search():
    g = torch.Generator().manual_seed(0)
    x, q = torch.randn(300, 16, generator=g), torch.randn(6, 16, generator=g)
    ids = torch.randperm(300, generator=g) * 3 - 400
    graph = np.full((300, 4), -1, dtype=np.int32)           # no edges at all: the entries alone
    s, i, visited = G.search(q, x, graph, np.arange(300), 320, 50, ids=ids.numpy())
    rs, ri = O.flat_ip_search(q.double(), x.double(), torch.arange(300), 50)
    assert torch.equal(i, ids[ri]) and torch.allclose(s, rs.float(), rtol=1e-6)
    assert np.all(visited == 300)


def test_oracle_search_tail_and_visited_count():
    x = G.integer_rows(40, 8, seed=1)
    q = G.integer_rows(3, 8, seed=2)
    graph = G.build(x, 4, 6)
    s, i, visited = G.search(q, x, graph, np.arange(5), 32, 60)
    assert torch.all(i[:, 40:] == -1) and torch.all(s[:, 40:] == G.NO_RESULT)
    assert np.all(visited <= 40) and np.all(visited >= 5)


def test_hash_size_formula():
    assert interaction.graph_hash_slots(32, 16) == 256
    assert interaction.graph_hash_slots(128, 64) == 1024
    assert interaction.graph_hash_slots(1024, 1024) == 8192
    assert interaction.graph_hash_slots(0, 16) == 0


def test_graph_symbols_are_bound():
    for name in ("mmb200_graph_prune", "mmb200_graph_search", "mmb200_graph_hash_slots"):
        assert name in _lib.SIGNATURES
        assert hasattr(_lib.load(), name)


def test_graph_kernels_do_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "graph.cu")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True,
                       text=True, check=True)
    reports = re.findall(r"Compiling entry function '(\S+)'.*?\n(.*?spill.*?)\n", r.stderr, re.S)
    names = [n for n, _ in reports]
    assert sum("graph_search_kernel" in n for n in names) == 2 and any("graph_prune_kernel" in n for n in names), names
    for name, line in reports:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
