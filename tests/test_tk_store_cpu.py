"""TK / TK-Sparse store scoring without a GPU: the store restatement against the pinned oracles, dropping gate-zero rows,
the gated encode folder, the passage-aligned shards and the rank merge under gloo, and the wrapper's envelope."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import tk_store_cases as C
from matchmaker_b200 import _lib, interaction, sharding
from matchmaker_b200.retrieval.colbert_e2e import doc_offsets_from_id_mapping
from matchmaker_b200.retrieval.tk_store import TKStoreWriter, load_gates, local_pairs, merge
from matchmaker_b200.retrieval.token_storage import TokenStorageWriter, load_token_storage
from oracle import interaction_oracle as O

LENGTHS = [5, 1, 0, 9, 3]


def _inputs(seed, gate_zeros=False):
    store, off, gate = C.make_store(LENGTHS, 16, seed, gate_zeros)
    g = torch.Generator().manual_seed(seed + 1)
    q = torch.randn(2, 4, 16, generator=g)
    qm = torch.tensor([[1, 1, 1, 0], [1, 1, 1, 1]], dtype=torch.float64)
    mu, sigma = C.kernels(11)
    w = torch.rand(11, generator=g) - 0.5
    alpha = torch.rand(11, generator=g) + 0.5
    pq = torch.tensor([0, 0, 0, 1, 1, 1, 1], dtype=torch.int32)
    pd = torch.tensor([0, 2, 3, 1, -1, 4, 3], dtype=torch.int32)
    return store, off, gate, q, qm, mu, sigma, w, alpha, pq, pd


@pytest.mark.parametrize("gated", [False, True])
def test_store_restatement_matches_padded_oracle(gated):
    store, off, gate, q, qm, mu, sigma, w, alpha, pq, pd = _inputs(3)
    g = gate if gated else None
    got = C.store_oracle(q, qm, store, off, pq, pd, mu, sigma, alpha, w, g)
    d, dm, dg = C.gather_padded(store.double(), off, pd, 12, None if g is None else g.double())
    qq, qmm = q[pq.long()].double(), qm[pq.long()]
    if gated:
        ref, _ = O.kernel_pool_tk_sparse(qq, d, qmm, dm.double(), dg, mu.double(), sigma.double(), alpha.double(),
                                         w.double())
    else:
        ref, _ = O.kernel_pool_tk(qq, d, qmm, dm.double(), mu.double(), sigma.double(), alpha.double(), w.double())
    empty = (pd < 0) | torch.tensor([LENGTHS[i] == 0 if i >= 0 else True for i in pd.tolist()])
    assert torch.isneginf(got[empty]).all()
    torch.testing.assert_close(got[~empty], ref[~empty], rtol=1e-12, atol=1e-12)


def test_dropping_gate_zero_rows_keeps_tk_sparse_score():
    store, off, gate, q, qm, mu, sigma, w, alpha, pq, pd = _inputs(5, gate_zeros=True)
    full = C.store_oracle(q, qm, store, off, pq, pd, mu, sigma, alpha, w, gate)
    keep = gate != 0
    kept_len = [int(keep[int(off[i]):int(off[i + 1])].sum()) for i in range(len(LENGTHS))]
    off2 = torch.zeros_like(off)
    off2[1:] = torch.cumsum(torch.tensor(kept_len), 0)
    dropped = C.store_oracle(q, qm, store[keep], off2, pq, pd, mu, sigma, alpha, w, gate[keep])
    both = torch.isfinite(dropped)
    assert torch.equal(torch.isneginf(dropped), torch.isneginf(full) | torch.tensor(
        [pd_ >= 0 and kept_len[pd_] == 0 for pd_ in pd.tolist()]))
    torch.testing.assert_close(dropped[both], full[both], rtol=1e-13, atol=1e-13)


def test_gated_encode_folder_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    w = TKStoreWriter(str(tmp_path), 8, 10, gated=True)
    docs, gates = [], []
    for i, n in enumerate([4, 7, 3, 0, 5]):
        v = rng.standard_normal((n, 8)).astype(np.float32)
        g = rng.random(n).astype(np.float32) + 0.1
        if n >= 3:
            v[1] = 0.0    # an all-zero row is dropped with its gate
        w.add(str(i), v, g)
        keep = np.abs(v).sum(-1) > 0
        docs.append(v[keep])
        gates.append(g[keep])
    w.close()
    storage, idm, seq_ids, infos = load_token_storage(str(tmp_path), 8, 10, "float32")
    gl = load_gates(str(tmp_path), 10, storage)
    assert len(storage) > 1   # the passages span several blocks
    rows, gg = np.concatenate(storage), np.concatenate(gl)
    np.testing.assert_array_equal(rows, np.concatenate(docs))
    np.testing.assert_array_equal(gg, np.concatenate(gates))
    off = doc_offsets_from_id_mapping(idm)
    assert np.diff(off).tolist() == [len(x) for x in docs]
    # without gates the folder is exactly TokenStorageWriter's
    a, b = tmp_path / "a", tmp_path / "b"
    wa, wb = TKStoreWriter(str(a), 8, 10), TokenStorageWriter(str(b), 8, 10, "float32")
    for i, v in enumerate(docs):
        wa.add(str(i), v)
        wb.add(str(i), v)
    wa.close()
    wb.close()
    assert sorted(os.listdir(a)) == sorted(os.listdir(b))
    for f in os.listdir(a):
        assert open(a / f, "rb").read() == open(b / f, "rb").read(), f
    with pytest.raises(_lib.MatchmakerB200Error):
        load_gates(str(a), 10, load_token_storage(str(a), 8, 10, "float32")[0])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, off, cand, full_scores, k, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        d_lo, d_hi, _, _ = sharding.passage_shard_bounds(off, rank, world)
        pair_d, ids = local_pairs(cand, d_lo, d_hi)
        # what the store kernel returns for this rank: the score where the rank owns the passage, else -inf
        local = torch.where(pair_d.view(cand.shape) >= 0, full_scores, torch.full_like(full_scores, float("-inf")))
        s, i = merge(local, ids, k)
        out[rank] = (s, i, (d_lo, d_hi))
    finally:
        dist.destroy_process_group()


def test_passage_shards_and_merge_under_gloo():
    off = np.array([0, 3, 3, 10, 12, 20, 21, 30], dtype=np.int64)   # passage 1 is empty
    world = 2
    bounds = [sharding.passage_shard_bounds(off, r, world) for r in range(world)]
    assert bounds[0][0] == 0 and bounds[-1][1] == len(off) - 1
    assert all(bounds[r][1] == bounds[r + 1][0] and bounds[r][3] == bounds[r + 1][2] for r in range(world - 1))
    cand = torch.tensor([[6, 0, -1, 3, 1, 5], [2, 2, -1, -1, 4, 0]], dtype=torch.int64)
    g = torch.Generator().manual_seed(0)
    full = torch.randn(cand.shape, generator=g)
    full[1, 0] = full[1, 1] = 0.25                     # one passage twice: a tie broken by id
    full[0, 4] = float("-inf")                         # the empty passage
    full = full.masked_fill(cand < 0, float("-inf"))
    k = 5
    with mp.Manager() as mgr:
        out = mgr.dict()
        mp.spawn(_rank_main, args=(world, _free_port(), off, cand, full, k, out), nprocs=world, join=True)
        res = dict(out)
    # expected: every owned candidate with its score, the rest -inf / -1, under (score desc, id asc)
    for r in range(cand.shape[0]):
        items = [(float(full[r, j]), int(cand[r, j])) for j in range(cand.shape[1]) if cand[r, j] >= 0]
        items += [(float("-inf"), -1)] * (world * cand.shape[1])
        items.sort(key=lambda x: (-x[0], x[1]))
        exp = items[:k]
        for rank in range(world):
            s, i, _ = res[rank]
            assert [(float(a), int(b)) for a, b in zip(s[r], i[r])] == exp, (rank, r)


def test_kernel_pool_store_envelope_raises_before_launch():
    q = torch.zeros(2, 4, 16)
    store = torch.zeros(10, 16)
    off = torch.tensor([0, 4, 10])
    pq = pd = torch.zeros(2, dtype=torch.int32)
    mu, sigma, w = torch.zeros(11), torch.ones(11), torch.zeros(11)

    def call(**kw):
        a = dict(q=q, q_mask=None, store=store, doc_offsets=off, pair_q=pq, pair_d=pd, mu=mu, sigma=sigma, weight=w)
        a.update(kw)
        return interaction.kernel_pool_store(**a)

    for kw, msg in [(dict(q=torch.zeros(2, 4, 18), store=torch.zeros(10, 18)), "multiple of 4"),
                    (dict(store=torch.zeros(10, 12)), "expected q"),
                    (dict(mu=torch.zeros(33), sigma=torch.ones(33), weight=torch.zeros(33)), "K <="),
                    (dict(sigma=torch.ones(10)), "K <="),
                    (dict(store=torch.zeros(0, 16)), "n_rows"),
                    (dict(doc_offsets=torch.tensor([0])), "doc_offsets"),
                    (dict(q_mask=torch.ones(2, 5)), "q_mask"),
                    (dict(gate=torch.ones(9)), "gate")]:
        with pytest.raises(_lib.MatchmakerB200Error, match=msg):
            call(**kw)
    with pytest.raises(_lib.MatchmakerB200Error, match="CUDA"):   # in the envelope: no CPU fallback
        call()
