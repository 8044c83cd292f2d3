"""Store mode of the kernel-pooling kernels and TK / TK-Sparse re-ranking over an encoded store, on the GPU.

The store mode must give the bits of ``interaction.kernel_pool`` on the same rows gathered into the padded layout with
masks, on the tensor-core and the FFMA kernel; the end-to-end store must agree with the rankers' ``forward``."""
import pytest
import torch

import tk_store_cases as C
from matchmaker_b200 import interaction
from matchmaker_b200.rankers.tk import ECAI20_TK
from matchmaker_b200.rankers.tk_sparse import CIKM20_TK_Sparse
from matchmaker_b200.retrieval import TKDocumentStore
from matchmaker_b200.retrieval.tk_store import TKStoreWriter, load_gates
from matchmaker_b200.retrieval.token_storage import load_token_storage

pytestmark = pytest.mark.gpu

LENGTHS = [1, 63, 64, 65, 127, 128, 129, 300, 0, 40]   # 300 = max_doc_len; 0 = a passage without rows
MAX_LEN = 300


def _pairs(n_q, n_docs, seed, shuffle=False):
    g = torch.Generator().manual_seed(seed)
    pq = torch.arange(n_q).repeat_interleave(n_docs)
    pd = torch.arange(n_docs).repeat(n_q)
    pd[3] = -1                                   # a void candidate
    if shuffle:
        perm = torch.randperm(len(pq), generator=g)
        pq, pd = pq[perm], pd[perm]
    return pq.to(torch.int32), pd.to(torch.int32)


def _case(K, Lq, D, seed, gate_zeros=False, shuffle=False):
    g = torch.Generator().manual_seed(seed)
    store, off, gate = C.make_store(LENGTHS, D, seed, gate_zeros)
    n_q = 3
    q = torch.randn(n_q, Lq, D, generator=g)
    qm = torch.ones(n_q, Lq, dtype=torch.bool)
    if Lq > 4:
        qm[1, Lq - 3:] = False
    mu, sigma = C.kernels(K)
    w = torch.rand(K, generator=g) * 0.02 - 0.01
    alpha = torch.rand(K, generator=g) + 0.5
    pq, pd = _pairs(n_q, len(LENGTHS), seed, shuffle)
    dev = "cuda"
    return dict(q=q.to(dev), qm=qm.to(dev), store=store.to(dev), off=off.to(dev), gate=gate.to(dev), pq=pq.to(dev),
                pd=pd.to(dev), mu=mu.to(dev), sigma=sigma.to(dev), w=w.to(dev), alpha=alpha.to(dev))


def _both(c, impl, gated):
    gate = c["gate"] if gated else None
    s = interaction.kernel_pool_store(c["q"], c["qm"], c["store"], c["off"], c["pq"], c["pd"], c["mu"], c["sigma"],
                                      c["w"], c["alpha"], max_doc_len=MAX_LEN, impl=impl, gate=gate)
    d, dm, dg = C.gather_padded(c["store"], c["off"].cpu(), c["pd"].cpu(), MAX_LEN, gate)
    pq = c["pq"].long()
    ref = interaction.kernel_pool(c["q"][pq], d, c["qm"][pq], dm, c["mu"], c["sigma"], c["w"], c["alpha"], impl=impl,
                                  doc_gate=dg)["score"]
    return s, ref


def _empty(c):
    pd = c["pd"].cpu()
    lens = (c["off"][1:] - c["off"][:-1]).cpu()
    return (pd < 0) | (lens[pd.clamp(min=0).long()] == 0)


@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
@pytest.mark.parametrize("D", [128, 300, 384])
@pytest.mark.parametrize("Lq", [1, 8, 30, 32, 33, 64])
@pytest.mark.parametrize("K", [11, 21, 32])
def test_store_mode_bit_identical_to_padded(K, Lq, D, impl):
    c = _case(K, Lq, D, seed=K * 1000 + Lq * 10 + D)
    s, ref = _both(c, impl, gated=False)
    empty = _empty(c)
    assert torch.isneginf(s.cpu()[empty]).all()
    assert torch.equal(s.cpu()[~empty], ref.cpu()[~empty])


@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
@pytest.mark.parametrize("K", [11, 21])
def test_store_mode_gate_with_zeros(K, impl):
    c = _case(K, 30, 300, seed=7 + K, gate_zeros=True)
    s, ref = _both(c, impl, gated=True)
    empty = _empty(c)
    assert torch.isneginf(s.cpu()[empty]).all()
    assert torch.equal(s.cpu()[~empty], ref.cpu()[~empty])
    o = C.store_oracle(c["q"].cpu(), c["qm"].cpu(), c["store"].cpu(), c["off"].cpu(), c["pq"].cpu(), c["pd"].cpu(),
                       c["mu"].cpu(), c["sigma"].cpu(), c["alpha"].cpu(), c["w"].cpu(), c["gate"].cpu())
    torch.testing.assert_close(s.cpu().double()[~empty], o[~empty], rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
def test_store_mode_shuffled_pairs(impl):
    c = _case(21, 30, 300, seed=11, shuffle=True)
    s, ref = _both(c, impl, gated=False)
    empty = _empty(c)
    assert torch.isneginf(s.cpu()[empty]).all()
    assert torch.equal(s.cpu()[~empty], ref.cpu()[~empty])
    o = C.store_oracle(c["q"].cpu(), c["qm"].cpu(), c["store"].cpu(), c["off"].cpu(), c["pq"].cpu(), c["pd"].cpu(),
                       c["mu"].cpu(), c["sigma"].cpu(), c["alpha"].cpu(), c["w"].cpu())
    torch.testing.assert_close(s.cpu().double()[~empty], o[~empty], rtol=2e-3, atol=2e-3)


def _tk(sparse, D=64, K=11):
    torch.manual_seed(5)
    mu, sigma = C.kernels(K)
    if sparse:
        m = CIKM20_TK_Sparse(D, mu.tolist(), sigma.tolist(), att_heads=4, att_layer=2, att_proj_dim=32, att_ff_dim=96,
                             max_length=200, use_diff_posencoding=True)
        m.stop_word_reducer2.bias.data.fill_(0.0)   # a gate that is 0 on a good share of the terms
    else:
        m = ECAI20_TK(D, mu.tolist(), sigma.tolist(), att_heads=4, att_layer=2, att_ff_dim=96, max_length=200,
                      use_diff_posencoding=True, mix_hybrid_context=True)
    with torch.no_grad():
        m.kernel_bin_weights.weight.uniform_(-0.05, 0.05)
    return m.cuda().eval()


def _docs(n, Ld, D, seed):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(n, Ld, D, generator=g)
    lens = torch.randint(1, Ld + 1, (n,), generator=g)
    lens[0] = Ld
    dm = torch.arange(Ld).unsqueeze(0) < lens.unsqueeze(1)
    return d.cuda(), dm.float().cuda()


def _build_store(model, d, dm, folder, sparse, batch=7):
    D = d.shape[-1]
    w = TKStoreWriter(str(folder), D, 4096, gated=sparse)
    for b0 in range(0, d.shape[0], batch):
        enc = model.encode_documents(d[b0:b0 + batch], dm[b0:b0 + batch])
        rows, lens = enc[0].cpu().numpy(), enc[1].cpu().tolist()
        gate = enc[2].cpu().numpy() if sparse else None
        r0 = 0
        for i, L in enumerate(lens):
            w.add(str(b0 + i), rows[r0:r0 + L], None if gate is None else gate[r0:r0 + L])
            r0 += L
    w.close()
    storage, idm, _, _ = load_token_storage(str(folder), D, 4096, "float32")
    gates = load_gates(str(folder), 4096, storage) if sparse else None
    cfg = {"token_dim": D, "faiss_use_gpu": True, "token_dtype": "float32"}
    st = TKDocumentStore(cfg, model)
    st.index(idm, storage, gates)
    return st, cfg, (idm, storage, gates)


@pytest.mark.parametrize("sparse", [False, True])
def test_rerank_matches_forward(sparse, tmp_path):
    D, Ld, n_docs, nq, Lq = 64, 90, 40, 3, 12
    model = _tk(sparse, D)
    d, dm = _docs(n_docs, Ld, D, seed=1)
    st, cfg, raw = _build_store(model, d, dm, tmp_path / "enc", sparse)
    g = torch.Generator().manual_seed(2)
    q = torch.randn(nq, Lq, D, generator=g).cuda()
    qm = torch.ones(nq, Lq, device="cuda")
    qm[2, 9:] = 0
    cand = torch.stack([torch.randperm(n_docs, generator=g)[:25] for _ in range(nq)]).cuda()
    cand[1, 4] = -1
    with torch.no_grad():
        pos = model.positional_features_q[:, :Lq, :]
        qctx = model.forward_representation(q, qm, pos)
        qctx = qctx[0] if sparse else qctx
        s, ids = st.rerank(qctx, qm, cand, top_n=10)
        # the reference path: forward on every (query, candidate) pair
        flat = cand.clamp(min=0).reshape(-1)
        qi = torch.arange(nq, device="cuda").repeat_interleave(cand.shape[1])
        fs = model(q[qi], d[flat], qm[qi], dm[flat])
        fs = (fs[0] if sparse else fs).view(nq, -1).masked_fill(cand < 0, float("-inf"))
    assert s.shape == (nq, 10) and ids.shape == (nq, 10)
    for r in range(nq):
        ref = {int(c): float(v) for c, v in zip(cand[r].tolist(), fs[r].tolist()) if c >= 0}
        for v, i in zip(s[r].tolist(), ids[r].tolist()):
            assert i in ref
            assert abs(v - ref[i]) <= 1e-3 * max(1.0, abs(ref[i])), (r, i, v, ref[i])
        # ranking: the forward's order under (score desc, id asc), wherever neighbours differ by more than the bound
        order = sorted(ref.items(), key=lambda kv: (-kv[1], kv[0]))
        for j, (i_ref, v_ref) in enumerate(order[:10]):
            nxt = [abs(v_ref - order[j + o][1]) for o in (-1, 1) if 0 <= j + o < len(order)]
            if all(x > 2e-3 * max(1.0, abs(v_ref)) for x in nxt):
                assert ids[r, j].item() == i_ref
    # save / load round trip
    st.save(str(tmp_path / "tk.store"))
    st2 = TKDocumentStore(cfg, model)
    st2.load(str(tmp_path / "tk.store"))
    s2, ids2 = st2.rerank(qctx, qm, cand, top_n=10)
    assert torch.equal(s, s2) and torch.equal(ids, ids2)


def test_tk_sparse_store_drops_gate_zero_rows(tmp_path):
    model = _tk(True)
    d, dm = _docs(12, 60, 64, seed=4)
    with torch.no_grad():
        model.stop_word_reducer2.bias.data.fill_(-100.0)   # every gate 0: each passage keeps exactly one row
        rows, lens, gate = model.encode_documents(d, dm)
    assert lens.tolist() == [1] * 12 and (gate == 0).all()
    model.stop_word_reducer2.bias.data.fill_(0.0)
    rows, lens, gate = model.encode_documents(d, dm)
    assert int(lens.sum()) == rows.shape[0] == gate.shape[0]
    assert (lens >= 1).all()                  # a passage whose terms are all gated 0 keeps one row of gate 0
    assert int((gate == 0).sum()) <= len(lens)
    assert int(lens.sum()) < int(dm.sum())    # the test model gates a share of the terms to exactly 0
