"""Residual token codes on the GPU: the encode / decode kernels against the numpy format (bit for bit), the residual
list scan and max-sim against the existing kernels over the decoded store (bit for bit), and
retrieval.ColBERTResidualIndexer end to end, streamed, saved and loaded, and its recall against the uncompressed
ColBERTIVFIndexer."""
import numpy as np
import pytest
import torch

import colbert_residual_oracle as R
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import ColBERTIVFIndexer, ColBERTResidualIndexer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _cfg(dim, nlist, nprobe, bits=None):
    c = {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": nlist,
         "faiss_ivf_search_probe_count": nprobe}
    if bits is not None:
        c["colbert_residual_bits"] = bits
    return c


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16 if a.dtype == torch.float16 else torch.int32),
                       b.contiguous().view(torch.int16 if b.dtype == torch.float16 else torch.int32))


# ----------------------------------------------------------------------------------------------------------------------
# 1. encode / decode kernels == numpy format
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 2])
@pytest.mark.parametrize("dim", [64, 128, 768])
def test_encode_decode_kernels_equal_the_format(bits, dim):
    rows, lids, base, cutoff, weight = R.synth(3000, dim, 9, bits, seed=dim * bits)
    codes = interaction.residual_encode(_t(rows), _t(lids), _t(base), _t(cutoff), bits)
    ref = R.encode(rows, lids, base, cutoff, bits)
    assert np.array_equal(codes.cpu().numpy(), ref)
    dec = interaction.residual_decode(codes, _t(lids), _t(base), _t(weight), bits)
    assert np.array_equal(dec.cpu().numpy().view(np.int16), R.decode(ref, lids, base, weight, bits).view(np.int16))
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.residual_encode(_t(rows), _t(lids + 9), _t(base), _t(cutoff), bits)   # list ids out of range


# ----------------------------------------------------------------------------------------------------------------------
# 2. residual scan == gather scan over the decoded rows
# ----------------------------------------------------------------------------------------------------------------------
def _sizes(n, nlist, seed):
    """List sizes with an empty list 0, a one-row list 1, a list of several tiles (2) and random others."""
    rng = np.random.default_rng(seed)
    sizes = np.zeros(nlist, dtype=np.int64)
    sizes[1], sizes[2] = 1, n // 3
    sizes[3:] = rng.multinomial(n - int(sizes.sum()), np.ones(nlist - 3) / (nlist - 3))
    return sizes


def _coded_lists(n, dim, nlist, bits, seed):
    """(codes, list ids, base, weight, row_index, list_offsets, max list length, decoded rows) on the device."""
    g = torch.Generator().manual_seed(seed)
    sizes = _sizes(n, nlist, seed)
    lids = torch.from_numpy(np.repeat(np.arange(nlist), sizes))[torch.randperm(n, generator=g)].numpy().astype(np.int32)
    rng = np.random.default_rng(seed)
    base = (rng.standard_normal((nlist, dim)) * 0.3).astype(np.float16)
    base[0] = 0
    rows = (base[lids].astype(np.float32) + rng.standard_normal((n, dim)) * 0.1).astype(np.float16)
    cutoff, weight = R.quantile_tables(R.residuals(rows, lids, base), bits)
    codes = interaction.residual_encode(_t(rows), _t(lids), _t(base), _t(cutoff), bits)
    row_index = torch.sort(torch.from_numpy(lids.astype(np.int64)), stable=True).indices
    off = torch.zeros(nlist + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.from_numpy(sizes), 0)
    dec = interaction.residual_decode(codes, _t(lids), _t(base), _t(weight), bits)
    return codes, _t(lids), _t(base), _t(weight), row_index.to(DEV), off.to(DEV), int(sizes.max()), dec


@pytest.mark.parametrize("bits", [1, 2])
@pytest.mark.parametrize("dim,k,nprobe,nlist", [(128, 64, 8, 40), (64, 300, 4, 12), (128, 32, 6, 40),
                                                (128, 1000, 2, 5), (768, 100, 5, 12)])
def test_residual_scan_equals_gather_scan_over_decoded_rows(bits, dim, k, nprobe, nlist):
    n, nq = 5000, 40
    codes, lids, base, weight, ri, off, max_len, dec = _coded_lists(n, dim, nlist, bits, seed=dim + k + bits)
    g = torch.Generator().manual_seed(k)
    q = torch.randn(nq, dim, generator=g).half().to(DEV)
    row_ids = torch.sort(torch.randint(0, n // 4, (n,), generator=g)).values.to(DEV)
    probes = torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(nq)])
    probes[0] = torch.arange(nprobe)                       # the empty, one-row and long lists
    probes[1, nprobe // 2:] = -1
    probes = probes.to(DEV)
    s_r, i_r = interaction.ivf_search_residual(q, codes, base, weight, bits, row_ids, ri, off, probes, k, max_len)
    s_g, i_g = interaction.ivf_search(q, dec, row_ids, off, probes, k, max_len, row_index=ri)
    assert torch.equal(i_r, i_g)
    assert _same_bits(s_r, s_g)
    assert bool((i_r[1] >= 0).any()) and int((i_r[0] >= 0).sum()) == min(k, int((off[1:nprobe + 1] - off[:nprobe]).sum()))


# ----------------------------------------------------------------------------------------------------------------------
# 3. residual max-sim == documents-on-M max-sim over the decoded store
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 2])
@pytest.mark.parametrize("dim,lq", [(128, 32), (128, 64), (768, 32), (64, 64)])
def test_residual_maxsim_equals_docm_maxsim_over_decoded_store(bits, dim, lq):
    nlist = 11
    lengths = np.array([0, 1, 64, 65, 180, 3, 0, 127, 128, 129] + list(np.random.default_rng(dim).integers(1, 90, 40)))
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    n = int(off[-1])
    rows, lids, base, cutoff, weight = R.synth(n, dim, nlist, bits, seed=dim + lq + bits)
    codes = interaction.residual_encode(_t(rows), _t(lids), _t(base), _t(cutoff), bits)
    dec = interaction.residual_decode(codes, _t(lids), _t(base), _t(weight), bits)
    g = torch.Generator().manual_seed(lq)
    nq = 6
    q = torch.randn(nq, lq, dim, generator=g).half().to(DEV)
    q[2, lq // 2:] = 0
    pair_q = torch.arange(nq, dtype=torch.int32).repeat_interleave(len(lengths)).to(DEV)
    pair_d = torch.arange(len(lengths), dtype=torch.int32).repeat(nq)
    pair_d[::7] = -1                                       # void pairs
    pair_d = pair_d.to(DEV)
    offd = _t(off)
    got = interaction.maxsim_store_residual(q, codes, _t(lids), _t(base), _t(weight), bits, offd, pair_q, pair_d,
                                            int(lengths.max()))
    ref = interaction.maxsim_store(q, dec, offd, pair_q, pair_d, int(lengths.max()), impl="tcgen05_docm")
    assert _same_bits(got, ref)
    assert torch.isneginf(got[(pair_d < 0) | (pair_d == 0) | (pair_d == 6)]).all()   # void pairs, empty passages


# ----------------------------------------------------------------------------------------------------------------------
# shared store and indexers
# ----------------------------------------------------------------------------------------------------------------------
def _clustered_store(n_pass, dim, n_centres, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, 40, n_pass)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    g = torch.Generator().manual_seed(seed)
    c = torch.nn.functional.normalize(torch.randn(n_centres, dim, generator=g), dim=1)
    which = torch.randint(0, n_centres, (int(off[-1]),), generator=g)
    store = (c[which] + 0.25 * torch.randn(int(off[-1]), dim, generator=g) / dim ** 0.5).half()
    return store, off


def _pid(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def _queries(store, nq, lq, seed):
    g = torch.Generator().manual_seed(seed)
    q = store[torch.randint(0, store.shape[0], (nq * lq,), generator=g)].float()
    q = (q + 0.05 * torch.randn(q.shape, generator=g) / q.shape[1] ** 0.5).half().view(nq, lq, -1)
    q[1, lq // 2:] = 0
    return q


def _residual(store, off, dim, nlist, nprobe, bits, slab=None):
    idx = ColBERTResidualIndexer(_cfg(dim, nlist, nprobe, bits), device=DEV)
    blocks = [store.numpy()]
    idx.prepare(blocks)
    if slab is not None:
        idx.slab_rows = slab
    idx.index([_pid(off)], blocks)
    return idx


# ----------------------------------------------------------------------------------------------------------------------
# 4. end to end == the uncompressed indexer over the decoded store (same centroids and layout)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 2])
def test_end_to_end_equals_ivf_indexer_over_decoded_store(bits):
    dim, nlist, nprobe, kp, top_n = 128, 32, 4, 64, 50
    store, off = _clustered_store(1500, dim, 40, seed=5)
    res = _residual(store, off, dim, nlist, nprobe, bits)
    q = _queries(store, 6, 32, seed=6).to(DEV)
    ivf = ColBERTIVFIndexer(_cfg(dim, nlist, nprobe), device=DEV)
    ivf.ivf.set_centroids(res.ivf.centroids)
    dec = res.decoded_store()
    ivf.index_device(dec, off)
    ivf._set_layout(res.row_index, res.list_offsets)
    cs, ci = res.candidates_device(q, kp)
    rs, ri = ivf.candidates_device(q, kp)
    assert torch.equal(ci, ri) and _same_bits(cs, rs)
    s, i = res.search_device(q, top_n, token_top_k=kp)
    c = ci.shape[1]
    pair_d = torch.where(ci >= 0, ci, torch.full_like(ci, -1))
    pair_q = torch.arange(q.shape[0], device=DEV, dtype=torch.int32).repeat_interleave(c)
    scores = interaction.maxsim_store(q, dec, res.offsets, pair_q, pair_d, res.max_doc_len, impl="tcgen05_docm")
    es, ei = interaction.topk_merge(scores.view(q.shape[0], c), ci, top_n)
    assert torch.equal(i, ei) and _same_bits(s, es)
    assert int((i[0] >= 0).sum()) == top_n


# ----------------------------------------------------------------------------------------------------------------------
# 5. streaming and determinism
# ----------------------------------------------------------------------------------------------------------------------
def test_streamed_index_equals_one_shot_and_prepare_is_deterministic():
    dim, nlist, bits = 128, 16, 2
    store, off = _clustered_store(400, dim, 20, seed=8)
    a = _residual(store, off, dim, nlist, 4, bits, slab=777)
    b = ColBERTResidualIndexer(_cfg(dim, nlist, 4, bits), device=DEV)
    b.prepare([store.numpy()])
    for name in ("base", "weight", "cutoff"):
        assert _same_bits(getattr(a, name), getattr(b, name)), name
    assert torch.equal(a.ivf.centroids.view(torch.int32), b.ivf.centroids.view(torch.int32))
    b.index_device(store.to(DEV), off)
    assert torch.equal(a.store, b.store) and torch.equal(a.list_ids, b.list_ids)
    assert torch.equal(a.row_index, b.row_index) and torch.equal(a.list_offsets, b.list_offsets)
    assert a.store.dtype == torch.uint8 and a.store.shape == (store.shape[0], dim * bits // 8)


# ----------------------------------------------------------------------------------------------------------------------
# 6. save / load
# ----------------------------------------------------------------------------------------------------------------------
def test_save_load_round_trip(tmp_path):
    dim, nlist, bits = 128, 16, 1
    store, off = _clustered_store(300, dim, 20, seed=9)
    a = _residual(store, off, dim, nlist, 4, bits)
    q = _queries(store, 3, 32, seed=10).to(DEV)
    s0, i0 = a.search_device(q, 20, token_top_k=32)
    path = str(tmp_path / "res.pt")
    a.save(path)
    b = ColBERTResidualIndexer(_cfg(dim, nlist, 4, bits), device=DEV)
    b.load(path)
    s1, i1 = b.search_device(q, 20, token_top_k=32)
    assert torch.equal(i0, i1) and _same_bits(s0, s1)
    for cfg in (_cfg(dim, nlist, 4, 2), _cfg(256, nlist, 4, bits)):
        with pytest.raises(_lib.MatchmakerB200Error):
            ColBERTResidualIndexer(cfg, device=DEV).load(path)


# ----------------------------------------------------------------------------------------------------------------------
# 7. recall at nprobe = nlist against the uncompressed indexer
# ----------------------------------------------------------------------------------------------------------------------
def test_recall_against_uncompressed_indexer():
    dim, nlist, top_n, kp = 128, 64, 100, 100
    store, off = _clustered_store(4000, dim, 200, seed=11)
    q = _queries(store, 16, 32, seed=12).to(DEV)
    ivf = ColBERTIVFIndexer(_cfg(dim, nlist, nlist), device=DEV)
    ivf.prepare([store.numpy()])
    ivf.index([_pid(off)], [store.numpy()])
    _, ref = ivf.search_device(q, top_n, token_top_k=kp)
    recall = {}
    for bits in (1, 2):
        res = _residual(store, off, dim, nlist, nlist, bits)
        _, got = res.search_device(q, top_n, token_top_k=kp)
        hits = sum(len(set(got[r].tolist()) & set(ref[r].tolist()) - {-1}) for r in range(q.shape[0]))
        recall[bits] = hits / float((ref >= 0).sum())
    # first measured on an H100: 0.688 (1 bit), 0.8225 (2 bits); the floors leave a margin of 0.05 (synthetic clusters)
    assert recall[1] >= 0.63 and recall[2] >= 0.77, recall
    assert recall[2] > recall[1]


# ----------------------------------------------------------------------------------------------------------------------
# 8. training: bases and level tables == their definition, on a store larger than the samples and ordered by cluster
# ----------------------------------------------------------------------------------------------------------------------
def test_prepare_trains_the_documented_tables_on_a_cluster_ordered_store(monkeypatch):
    from matchmaker_b200.retrieval import colbert_residual
    monkeypatch.setattr(colbert_residual, "TABLE_SAMPLE_ROWS", 1000)   # below the k-means sample (256 * nlist rows)
    dim, nlist, bits = 128, 16, 2
    store, off = _clustered_store(1500, dim, 40, seed=13)
    g = torch.Generator().manual_seed(14)
    centre = torch.randint(0, 40, (store.shape[0],), generator=g)
    store = store[torch.sort(centre, stable=True).indices]     # rows ordered by cluster, 30 k rows > 4096 sampled
    assert store.shape[0] > 256 * nlist
    idx = ColBERTResidualIndexer(_cfg(dim, nlist, 4, bits), device=DEV)
    blocks = [store.numpy()]
    idx.prepare(blocks)
    x, _ = idx.ivf._training_points(blocks)                    # the k-means sample prepare() trained on
    a = idx.assign(x).cpu().numpy()
    xn = x.cpu().numpy()
    base = np.zeros((nlist, dim), dtype=np.float16)
    for l in range(nlist):
        rows = np.nonzero(a == l)[0]
        s = np.zeros(dim, dtype=np.float64)
        for r in rows:
            s += xn[r].astype(np.float64)
        base[l] = (s / max(1, len(rows))).astype(np.float16)
    assert np.array_equal(idx.base.cpu().numpy().view(np.int16), base.view(np.int16))
    # every list has sample rows across the whole store, so none is left with a zero base
    assert np.bincount(a, minlength=nlist).min() > 0 and (np.abs(base.astype(np.float32)).sum(1) > 0).all()
    pick = torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(colbert_residual.TABLE_SEED))[:1000]
    pick = pick.numpy()
    cutoff, weight = R.quantile_tables(R.residuals(xn[pick], a[pick], base), bits)
    assert np.array_equal(idx.cutoff.cpu().numpy().view(np.int32), cutoff.view(np.int32))
    assert np.array_equal(idx.weight.cpu().numpy().view(np.int16), weight.view(np.int16))
