"""Host-side pieces of the IVF index: the oracle against direct restatements, the query batching under the workspace cap,
and the GPU-only constructor."""
import numpy as np
import pytest
import torch

import ivf_oracle as V
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import IVFIndexer
from oracle import interaction_oracle as O


def _lists(sizes):
    off = torch.zeros(len(sizes) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.tensor(sizes), 0)
    return off


def test_oracle_search_with_every_list_probed_is_flat_search():
    g = torch.Generator().manual_seed(0)
    rows, q = torch.randn(300, 16, generator=g), torch.randn(5, 16, generator=g)
    ids = torch.randperm(300, generator=g) - 150
    off = _lists([0, 1, 150, 49, 100])
    probes = torch.tensor([[0, 1, 2, 3, 4]] * 5)
    s, i = V.ivf_search(q, rows, ids, off, probes, 20)
    rs, ri = O.flat_ip_search(q, rows, ids, 20)
    assert torch.equal(i, ri) and torch.allclose(s, rs, rtol=1e-5)   # per-query products: another fp32 sum order


def test_oracle_search_is_restricted_to_the_probed_lists_and_pads_the_tail():
    g = torch.Generator().manual_seed(1)
    rows, q = torch.randn(40, 8, generator=g), torch.randn(3, 8, generator=g)
    ids = torch.arange(40) * 10
    off = _lists([10, 0, 5, 25])
    probes = torch.tensor([[1, 2], [0, -1], [1, 1 + 10]])   # empty list, a -1 filler and an out-of-range id
    s, i = V.ivf_search(q, rows, ids, off, probes, 8)
    assert set(i[0, :5].tolist()) == set(range(100, 150, 10)) and torch.all(i[0, 5:] == -1)
    assert torch.all(s[0, 5:] == V.NO_RESULT)
    assert set(i[1].tolist()) <= set(range(0, 100, 10)) and torch.all(i[1] >= 0)
    assert torch.all(i[2] == -1) and torch.all(s[2] == V.NO_RESULT)


def test_oracle_kmeans_step_matches_a_loop():
    g = torch.Generator().manual_seed(2)
    x, c = torch.randn(200, 6, generator=g), torch.nn.functional.normalize(torch.randn(7, 6, generator=g), dim=1)
    c[6] = c[5]                       # an exact tie: the lower list wins, list 6 stays empty
    assign, new, gap = V.kmeans_step(x, c)
    for r in range(200):
        best = max(range(7), key=lambda l: (float(x[r].double() @ c[l].double()), -l))
        assert assign[r] == best
    assert torch.all(new[6] == 0)
    for l in range(6):
        m = x[assign == l].double().sum(0)
        assert torch.allclose(new[l], m / m.norm())
    assert torch.all(gap >= 0)


def test_query_batches_fit_the_cap():
    def ws(b):
        return 1000 + 300 * b
    assert interaction.ivf_query_batch(100, ws, 10 ** 9) == 100
    b = interaction.ivf_query_batch(100, ws, 5000)
    assert ws(b) <= 5000 and b >= 1
    assert interaction.ivf_query_batch(100, ws, 10) == 1      # never fewer than one query
    assert interaction.ivf_query_batch(0, ws, 10) == 1

    def ws_envelope(b):            # 0: nq * nprobe past the kernel's envelope -> must be halved, not taken as fitting
        return 0 if b > 1000 else 10 * b
    b = interaction.ivf_query_batch(4000, ws_envelope, 10 ** 9)
    assert 0 < ws_envelope(b) and b == 1000


def test_ivf_indexer_is_gpu_only():
    cfg = {"token_dim": 64, "faiss_use_gpu": False, "token_dtype": "float16", "faiss_ivf_list_count": 4,
           "faiss_ivf_search_probe_count": 2}
    with pytest.raises(_lib.MatchmakerB200Error):
        IVFIndexer(cfg)


def test_ivf_symbols_are_bound():
    for name in ("mmb200_ivf_search", "mmb200_ivf_workspace_bytes", "mmb200_ivf_list_means"):
        assert name in _lib.SIGNATURES
    assert np.int64(interaction.IVF_MAX_PROBE) == 1024
