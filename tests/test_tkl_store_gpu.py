"""TKL store mode on the GPU: bit identity with the padded window-score path over the routing matrix, fp64 window scores,
pair order / repeats / void pairs / poison, and TKLDocumentStore end to end against TKL_sigir20.forward."""
import numpy as np
import pytest
import torch

import tkl_store_cases as C
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.rankers.tkl import TKL_sigir20
from matchmaker_b200.retrieval import TKLDocumentStore
from matchmaker_b200.retrieval.tkl_store import TKLStoreWriter, load_chunk_meta
from matchmaker_b200.retrieval.token_storage import load_token_storage
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("row", C.MATRIX, ids=C.row_id)
def test_store_windows_bit_identical_to_padded(row):
    impl, sat, K, Lq, D, Cs, many = row
    assert (C.tc_fits(Lq, K) if impl == "tcgen05" else C.ffma_fits(D, K)), "matrix row outside its kernel's envelope"
    case = C.build(Lq, D, Cs, K, seed=K * 1000 + Lq * 10 + Cs, many=many)
    # a kernel set without cover would send the shape to the FFMA kernel (a forced tensor-core call writes zeros)
    assert interaction.tkl_kernel_set_covers(case["params"]["mu"], case["params"]["sigma"])
    n_pairs = case["pair_q"].numel()
    assert (n_pairs > 1024) if many else (n_pairs <= 1024)
    got = C.store_windows(case, sat, impl)
    ref = C.padded_windows(case, sat, impl)
    assert got.shape == ref.shape == (n_pairs, (Cs * 40 - 30) // 2 + 1)
    assert torch.isfinite(got).all(), "poison reached a window"
    assert (got != 0).sum() > got.shape[0], "hardly any window scored"
    assert torch.equal(got, ref), f"max diff {(got - ref).abs().max().item()}"
    void = case["pair_d"].to(DEV) < 0
    assert (got[void] == 0).all()
    # the selection on top: bit-identical too
    cs = case["params"]["chunk_scoring"].to(DEV)
    for a, b in zip(interaction.tkl_top_hills(got, cs), interaction.tkl_top_hills(ref, cs)):
        assert torch.equal(a, b)
    # pair order: a permutation of the pairs permutes the rows, bit for bit; a second run gives the same bits
    perm = torch.randperm(n_pairs, generator=torch.Generator().manual_seed(1))
    case2 = dict(case, pair_q=case["pair_q"][perm], pair_d=case["pair_d"][perm])
    assert torch.equal(C.store_windows(case2, sat, impl), got[perm.to(DEV)])
    assert torch.equal(C.store_windows(case, sat, impl), got)
    # every (query, passage) is there twice: both copies equal
    key = case["pair_q"].long() * 100000 + case["pair_d"].long()
    first = {}
    for i, k in enumerate(key.tolist()):
        if k in first:
            assert torch.equal(got[i], got[first[k]])
        else:
            first[k] = i
    # auto routes to the same kernel where only one kernel takes the shape
    if impl == "tcgen05" or not C.tc_fits(Lq, K):
        assert torch.equal(C.store_windows(case, sat, "auto"), got)


@pytest.mark.parametrize("impl", C.IMPLS)
@pytest.mark.parametrize("sat", ["embedding", "log"])
@pytest.mark.parametrize("Cs", [3, 50])
def test_store_windows_against_fp64(impl, sat, Cs):
    K, Lq, D = 11, 30, 32
    case = C.build(Lq, D, Cs, K, seed=7 + Cs)
    got = C.store_windows(case, sat, impl).double().cpu()
    # the oracle once per distinct live pair
    pq, pd = case["pair_q"].long(), case["pair_d"].long()
    live = [i for i in range(len(pq)) if pd[i] >= 0]
    uniq = sorted({(int(pq[i]), int(pd[i])): i for i in live}.values())[:24]
    sub = dict(case, pair_q=case["pair_q"][uniq], pair_d=case["pair_d"][uniq])
    q, qm, ch, cm, packed, _ = C.gathered(sub)
    p64 = {k: v.double() for k, v in case["params"].items()}
    _, sec = O.tkl_interaction(q.double(), qm.double(), ch.double(), cm.double(), packed, Cs, p64, sat)
    ref = sec["orig_score"]   # window scores with exact zeros where the reference's sentinel applies
    g = got[uniq]
    assert ((g == 0) == (ref == 0)).all(), "exact-zero windows must stay exactly zero"
    # 1e-3 of the magnitude summed: the window's terms are bounded by the largest window of the pair
    scale = ref.abs().amax(dim=1, keepdim=True).clamp(min=1e-30)
    err = ((g - ref).abs() / scale).max().item()
    assert err <= 1e-3, err
    # top-3 windows: exact, except between windows tied within the tolerance
    _, _, top_idx, _ = interaction.tkl_top_hills(got[uniq].float().to(DEV), case["params"]["chunk_scoring"].to(DEV))
    ti, ri = top_idx.cpu(), sec["top_non_overlapping_idx"]
    for b in range(len(uniq)):
        for c in range(3):
            if ti[b, c] != ri[b, c]:
                a, r = ref[b, ti[b, c]], ref[b, ri[b, c]]
                assert abs(a - r) <= 1e-3 * scale[b, 0], (b, c, ti[b].tolist(), ri[b].tolist())


def test_empty_pair_list_and_bad_shapes():
    case = C.build(5, 32, 3, 11, seed=3)
    empty = dict(case, pair_q=case["pair_q"][:0], pair_d=case["pair_d"][:0])
    assert C.store_windows(empty, "log", "auto").shape == (0, (3 * 40 - 30) // 2 + 1)
    with pytest.raises(_lib.MatchmakerB200Error, match="tensor-core"):
        C.store_windows(dict(case, q=torch.randn(3, 40, 32), q_mask=torch.ones(3, 40), params=C.covering_params(
            16, 32, torch.Generator().manual_seed(0))), "log", "tcgen05")   # Lq * K = 640 > 512


# ---------------------------------------------------------------------------------------------------------------------
# end to end: encode_documents -> writer -> load_token_storage -> TKLDocumentStore.rerank against forward
EMB, MAXLEN = 32, 400


def _model(sat, seed=0):
    torch.manual_seed(seed)
    mu = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
    m = TKL_sigir20(EMB, mu, [0.1] * 11, 2, 1, 64, MAXLEN, True, True, sat).to(DEV).eval()
    with torch.no_grad():
        m.dense.weight.normal_(0, 0.1)
        m.dense.weight[0, 0] = 1.0
        m.kernel_mult.uniform_(0.5, 1.5)
        m.chunk_scoring.uniform_(0.5, 1.5)
        m.saturation_linear.bias.fill_(3.0)
        m.saturation_linear2.bias.fill_(2.0)
        m.saturation_linear3.bias.fill_(1.0)
    return m


def _documents(g):
    """Passages of 0-400 tokens: one with an all-OOV middle span (a dropped chunk slot), two identical ones (an exact
    tie), and an empty last one."""
    lens = [400, 1, 57, 121, 399, 0, 200, 200, 333, 40, 0]
    emb = torch.randn(len(lens), MAXLEN, EMB, generator=g) * 0.4
    mask = (torch.arange(MAXLEN)[None] < torch.tensor(lens)[:, None]).float()
    mask[4, 90:170] = 0     # slots 2 and 3 hold no token: dropped by the packing
    emb[7] = emb[6]         # passage 7 is passage 6 again
    return emb * mask[..., None], mask


def _encode(model, emb, mask, folder):
    w = TKLStoreWriter(str(folder), EMB, 800)
    # two batches padded to different lengths: a chunk is contextualised alone, so batching does not matter
    for lo, hi in ((0, 5), (5, len(emb))):
        L = int((mask[lo:hi].sum(dim=0) > 0).nonzero().max()) + 1   # the batch's last token: 400, then 333
        e, m = emb[lo:hi, :L].to(DEV), mask[lo:hi, :L].to(DEV)
        chunks, cmask, slots, counts = model.encode_documents(e, m)
        r = 0
        for i, n in enumerate(counts.tolist()):
            w.add(str(lo + i), chunks[r:r + n].cpu().numpy(), cmask[r:r + n].cpu().numpy(), slots[r:r + n].cpu().numpy())
            r += n
    w.close()
    storage, idm, seq_ids, _ = load_token_storage(str(folder), EMB, 800, "float32")
    assert seq_ids == [str(i) for i in range(len(emb))]
    return storage, idm, load_chunk_meta(str(folder), 800, storage)


CONFIG = {"token_dim": EMB, "faiss_use_gpu": True, "token_dtype": "float32"}


@pytest.mark.parametrize("sat", ["embedding", "log"])
def test_rerank_matches_forward(tmp_path, sat):
    g = torch.Generator().manual_seed(11)
    model = _model(sat)
    emb, mask = _documents(g)
    storage, idm, meta = _encode(model, emb, mask, tmp_path / "enc")
    store = TKLDocumentStore(CONFIG, model)
    store.index(idm, storage, meta)
    assert store.C == 10
    nq, Lq = 4, 12
    q_emb = torch.randn(nq, Lq, EMB, generator=g) * 0.4
    q_mask = (torch.arange(Lq)[None] < torch.tensor([12, 3, 7, 1])[:, None]).float()
    q_emb = q_emb * q_mask[..., None]
    cand = torch.tensor([[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10],
                         [6, 7, 4, -1, 2, -1, -1, -1, -1, -1, -1],        # short list; 6 and 7 tie exactly
                         [5, 10, -1, 10, -1, -1, -1, -1, -1, -1, -1],     # empty passages only: all void
                         [9, 8, 3, 0, 4, 1, 7, 6, 2, -1, 5]])
    with torch.no_grad():
        q_ctx = model.forward_representation(q_emb.to(DEV), q_mask.to(DEV), model.positional_features_q[:, :Lq, :])[0]
        scores, ids = store.rerank(q_ctx, q_mask.to(DEV), cand, top_n=8)
        # forward over every (query, live candidate) with the documents padded to max_doc_length
        pairs = [(i, int(d)) for i in range(nq) for d in cand[i].tolist() if d >= 0 and mask[d].sum() > 0]
        pq, pd = torch.tensor([p[0] for p in pairs]), torch.tensor([p[1] for p in pairs])
        ref, sec = model(q_emb[pq].to(DEV), emb[pd].to(DEV), q_mask[pq].to(DEV), mask[pd].to(DEV),
                         output_secondary_output=True)
        s2, sec2 = model.score_store(q_ctx, q_mask.to(DEV), store.chunks, store.chunk_mask, store.doc_slots,
                                     pq.int().to(DEV), pd.int().to(DEV), output_secondary_output=True)
    ref, s2 = ref.cpu().double(), s2.cpu().double()
    tiny = 1e-6
    assert ((s2 - ref).abs() <= 1e-3 * ref.abs().clamp(min=tiny)).all(), (s2 - ref).abs().max()
    # secondary outputs: the selected regions
    orig, orig_ref = sec2["orig_score"].cpu().double(), sec["orig_score"].cpu().double()
    assert orig.shape == orig_ref.shape
    sc = orig_ref.abs().amax(dim=1, keepdim=True).clamp(min=tiny)
    assert ((orig - orig_ref).abs() <= 1e-3 * sc).all()
    assert torch.equal(sec2["top_non_overlapping_idx"].cpu(), sec["top_non_overlapping_idx"].cpu())
    top_sc = sec["top_k_non_overlapping"].abs().amax(dim=1, keepdim=True).clamp(min=tiny).cpu()
    assert ((sec2["top_k_non_overlapping"].cpu() - sec["top_k_non_overlapping"].cpu()).abs() <= 1e-3 * top_sc).all()
    # the ranking: live candidates with their forward score, sorted by (score desc, id asc), then (-inf, -1)
    want = {(i, d): float(r) for (i, d), r in zip(pairs, ref.tolist())}
    scores, ids = scores.cpu(), ids.cpu()
    assert scores.shape == ids.shape == (nq, 8)
    for i in range(nq):
        live = sorted({d for d in cand[i].tolist() if (i, d) in want})
        got = [(float(s), int(d)) for s, d in zip(scores[i], ids[i])]
        n_live = min(8, len([d for d in cand[i].tolist() if (i, d) in want]))
        for s, d in got[:n_live]:
            assert d in live and abs(s - want[(i, d)]) <= 1e-3 * max(abs(want[(i, d)]), tiny)
        assert all(s == float("-inf") and d == -1 for s, d in got[n_live:]), got
        assert all((a[0], -a[1]) >= (b[0], -b[1]) for a, b in zip(got[:n_live], got[1:n_live]))
    assert (ids[2] == -1).all() and torch.isneginf(scores[2]).all()
    row = [int(d) for d in ids[1].tolist()]
    assert row.index(6) < row.index(7) and scores[1, row.index(6)] == scores[1, row.index(7)]   # exact tie, id order

    # save / load: the same ranking; refused for another max_doc_length or another passage range
    store.save(str(tmp_path / "s.pt"))
    other = TKLDocumentStore(CONFIG, model)
    other.load(str(tmp_path / "s.pt"))
    s3, i3 = other.rerank(q_ctx, q_mask.to(DEV), cand, top_n=8)
    assert torch.equal(s3.cpu(), scores) and torch.equal(i3.cpu(), ids)
    short = _model(sat)
    short.max_length = 200
    with pytest.raises(_lib.MatchmakerB200Error, match="chunk slots"):
        TKLDocumentStore(CONFIG, short).load(str(tmp_path / "s.pt"))
    blob = torch.load(str(tmp_path / "s.pt"))
    blob["d_hi"] -= 1
    torch.save(blob, str(tmp_path / "t.pt"))
    with pytest.raises(_lib.MatchmakerB200Error, match="passages"):
        TKLDocumentStore(CONFIG, model).load(str(tmp_path / "t.pt"))
    with pytest.raises(_lib.MatchmakerB200Error, match="float32"):
        TKLDocumentStore(dict(CONFIG, token_dtype="float16"), model)


def test_index_refuses_passages_longer_than_max_doc_length(tmp_path):
    model = _model("log")
    g = torch.Generator().manual_seed(2)
    emb = torch.randn(1, 520, EMB, generator=g) * 0.4
    mask = torch.ones(1, 520)
    w = TKLStoreWriter(str(tmp_path), EMB, 800)
    chunks, cmask, slots, counts = model.encode_documents(emb.to(DEV), mask.to(DEV))
    w.add("0", chunks.cpu().numpy(), cmask.cpu().numpy(), slots.cpu().numpy())
    w.close()
    storage, idm, _, _ = load_token_storage(str(tmp_path), EMB, 800, "float32")
    with pytest.raises(_lib.MatchmakerB200Error, match="below C"):
        TKLDocumentStore(CONFIG, model).index(idm, storage, load_chunk_meta(str(tmp_path), 800, storage))
    assert np.array_equal(counts.cpu().numpy(), [13])
