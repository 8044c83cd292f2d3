"""The E4M3 token store on the GPU: the e4m3 max-sim against the fp64 oracle over the stored values and against the
fp16 kernel on the same values, the e4m3 top-k scans against the oracle and against each other, and the fp8 ColBERT
indexers against the oracle pipeline and the fp16 indexers (layout, streaming, persistence, memory, recall)."""
import numpy as np
import pytest
import torch

import colbert_e2e_oracle as E
import colbert_fp8_oracle as F
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

# Accumulation error of the FP8 MMA per token product, as a fraction of sum_k |q_k d_k| (its internal accumulation
# precision is not documented).  Measured worst case 2^-12.7 over the max-sim grid below (H100 SXM, DESIGN 3.4i);
# pinned with 3x headroom.
C_MMA = 2.0 ** -11


def _fp16_docm_fits(dim, lq):
    """The fp16 documents-on-M kernel's envelope on an H100 (DESIGN 3.1)."""
    return not ((dim >= 896 and lq > 64) or (dim >= 640 and lq > 96))


# ----------------------------------------------------------------------------------------------------------------------
# 1. max-sim over the store
# ----------------------------------------------------------------------------------------------------------------------
def _ragged_store(dim, seed, n_docs=160):
    """Passages of 0, 1, 127, 128, 129 and random lengths, rows of mixed magnitude, quantized with the store scale."""
    rng = np.random.default_rng(seed)
    lens = np.concatenate([[0, 1, 127, 128, 129, 0, 200], rng.integers(1, 60, n_docs - 7)])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    g = torch.Generator().manual_seed(seed)
    rows = (torch.randn(int(off[-1]), dim, generator=g) * torch.rand(int(off[-1]), 1, generator=g) * 3).half()
    sd = F.scale_log2(float(rows.float().abs().max()))
    return F.quantize(rows, sd), off


@pytest.mark.parametrize("dim", [128, 256, 768, 1024])
@pytest.mark.parametrize("lq", [1, 32, 33, 64, 96, 128])
def test_maxsim_store_matches_fp64_oracle_and_fp16_kernel(dim, lq):
    store8, off = _ragged_store(dim, seed=dim + lq)
    n_docs, nq, max_doc_len = len(off) - 1, 3, 128            # the passages of 129 and 200 rows are truncated
    g = torch.Generator().manual_seed(lq)
    q = torch.randn(nq, lq, dim, generator=g).half()
    q[0, lq // 2:] = 0                                        # padding rows of a query are plain zero rows here
    q8, _ = F.quantize_queries(q)
    pair_q = torch.arange(nq, dtype=torch.int32).repeat_interleave(n_docs + 2)
    pair_d = torch.cat([torch.arange(n_docs), torch.tensor([-1, 3])]).repeat(nq).to(torch.int32)
    args = (torch.from_numpy(off).to(DEV), pair_q.to(DEV), pair_d.to(DEV), max_doc_len)
    got = interaction.maxsim_store(q8.to(DEV), store8.to(DEV), *args).cpu().double()
    ref, tol = F.maxsim_store(q8, store8, off, max_doc_len, C_MMA)
    want = torch.stack([ref[int(a), int(d)] if d >= 0 else torch.tensor(-np.inf, dtype=torch.float64)
                        for a, d in zip(pair_q, pair_d)])
    bound = torch.stack([tol[int(a), int(d)] if d >= 0 else torch.tensor(0.0, dtype=torch.float64)
                         for a, d in zip(pair_q, pair_d)])
    void = torch.isinf(want)
    assert torch.equal(torch.isinf(got), void) and bool((got[void] < 0).all())
    err = (got - want)[~void].abs()
    assert bool((err <= bound[~void]).all()), f"worst error / bound {float((err / bound[~void]).max())}"
    if _fp16_docm_fits(dim, lq):
        # every e4m3 value is an fp16 value: the 16-bit kernel scores the same numbers
        h = interaction.maxsim_store(q8.half().to(DEV), store8.half().to(DEV), *args, impl="tcgen05_docm").cpu().double()
        assert torch.equal(torch.isinf(h), void)
        assert bool(((got - h)[~void].abs() <= 2 * bound[~void]).all())


def test_maxsim_store_refuses_mixed_operands():
    store8, off = _ragged_store(128, seed=1, n_docs=10)
    q = torch.zeros(1, 4, 128, dtype=torch.float16, device=DEV)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.maxsim_store(q, store8.to(DEV), torch.from_numpy(off).to(DEV), torch.zeros(1, dtype=torch.int32,
                                 device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV), 8)


# ----------------------------------------------------------------------------------------------------------------------
# 2. stage 1: top-k scans
# ----------------------------------------------------------------------------------------------------------------------
def _dense8(nq, n, dim, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(nq, dim, generator=g)
    p = torch.randn(n, dim, generator=g) * torch.rand(n, 1, generator=g)
    q8 = torch.stack([F.quantize(q[i], F.scale_log2(float(q[i].abs().max()))) for i in range(nq)])
    return q8, F.quantize(p, F.scale_log2(float(p.abs().max())))


@pytest.mark.parametrize("nq,dim,k", [(100, 128, 10), (256, 128, 300), (40, 768, 64), (300, 1024, 16)])
def test_flat_ip_topk_fp8_matches_oracle(nq, dim, k):
    n = 5000
    q8, p8 = _dense8(nq, n, dim, seed=nq + dim + k)
    ids = torch.arange(n) * 7 - 1000
    s, i = interaction.flat_ip_topk(q8.to(DEV), p8.to(DEV), k, ids=ids.to(DEV))
    s, i = s.cpu().double(), i.cpu()
    ref = q8.double() @ p8.double().T
    bound = C_MMA * (q8.double().abs() @ p8.double().abs().T).max(dim=1).values + 2.0 ** -24 * ref.abs().max(1).values
    pos = {int(v): r for r, v in enumerate(ids)}
    for a in range(nq):
        rows = torch.tensor([pos[int(v)] for v in i[a]])
        assert bool(((s[a] - ref[a, rows]).abs() <= bound[a]).all())           # scores of the returned ids
        kth = ref[a].sort(descending=True).values[k - 1]
        assert bool((ref[a, rows] >= kth - 2 * bound[a]).all())                 # nothing clearly outside the top k
        sure = (ref[a] > kth + 2 * bound[a]).nonzero().view(-1)
        assert set(ids[sure].tolist()) <= set(i[a].tolist())                    # nothing clearly inside it missing
        srt = ref[a, rows]
        gaps = (srt[:-1] - srt[1:]) > 2 * bound[a]                              # order wherever the gap decides it
        assert bool((s[a][:-1][gaps] > s[a][1:][gaps]).all())


@pytest.mark.parametrize("dim,k,nlist", [(128, 32, 24), (256, 300, 9), (768, 10, 16)])
def test_gather_scan_at_full_probe_equals_flat_scan(dim, k, nlist):
    n, nq = 4000, 150
    q8, p8 = _dense8(nq, n, dim, seed=dim + k)
    g = torch.Generator().manual_seed(k)
    ids = torch.sort(torch.randint(0, n // 3, (n,), generator=g)).values
    assign = torch.randint(0, nlist, (n,), generator=g)
    assign[assign == 1] = 0                                                     # an empty list
    row_index = torch.sort(assign, stable=True).indices
    off = torch.zeros(nlist + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.bincount(assign, minlength=nlist), 0)
    probes = torch.stack([torch.randperm(nlist, generator=g) for _ in range(nq)])
    max_len = int((off[1:] - off[:-1]).max())
    s_g, i_g = interaction.ivf_search(q8.to(DEV), p8.to(DEV), ids.to(DEV), off.to(DEV), probes.to(DEV), k, max_len,
                                      row_index=row_index.to(DEV))
    s_f, i_f = interaction.flat_ip_topk(q8.to(DEV), p8.to(DEV), k, ids=ids.to(DEV))
    assert torch.equal(i_g, i_f)
    assert torch.equal(s_g.view(torch.int32), s_f.view(torch.int32))


# ----------------------------------------------------------------------------------------------------------------------
# 3. indexers
# ----------------------------------------------------------------------------------------------------------------------
def _cfg(dim, fp8=True, nlist=16, nprobe=4):
    c = {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": nlist,
         "faiss_ivf_search_probe_count": nprobe}
    if fp8:
        c["colbert_store_dtype"] = "float8_e4m3"
    return c


def _lengths(n_pass, seed):
    return np.random.default_rng(seed).integers(1, 40, n_pass)


def _pid(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def _integer_store(n_pass, dim, seed):
    """Entries in {-2..2}: e4m3 holds them (times any power of two) exactly and every sum is exact, so the fp8
    pipeline computes the same numbers as fp64."""
    off = np.concatenate([[0], np.cumsum(_lengths(n_pass, seed))]).astype(np.int64)
    store = torch.randint(-2, 3, (int(off[-1]), dim), generator=torch.Generator().manual_seed(seed)).half()
    return store, off


def _clustered_store(n_pass, dim, n_centres, seed):
    g = torch.Generator().manual_seed(seed)
    off = np.concatenate([[0], np.cumsum(_lengths(n_pass, seed))]).astype(np.int64)
    c = torch.nn.functional.normalize(torch.randn(n_centres, dim, generator=g), dim=1)
    which = torch.randint(0, n_centres, (int(off[-1]),), generator=g)
    store = (c[which] + 0.25 * torch.randn(int(off[-1]), dim, generator=g) / dim ** 0.5).half()
    return store, off, c


def _queries(nq, lq, dim, seed, integer=True):
    g = torch.Generator().manual_seed(seed)
    q = torch.randint(-2, 3, (nq, lq, dim), generator=g).half() if integer else \
        (torch.randn(nq, lq, dim, generator=g) * 0.3).half()
    q[1, lq - 7:] = 0
    q[2] = q[2] * 0.5 if integer else q[2]                                      # another per-query scale
    return q


def _build(cls, store, off, cfg):
    blocks = [store.numpy()]
    idx = cls(cfg, device=DEV)
    if cls is ColBERTIVFIndexer:
        idx.prepare(blocks)
    idx.index([_pid(off)], blocks)
    return idx


@pytest.mark.parametrize("kp,top_n", [(16, 20), (200, 100)])
def test_exact_fp8_indexer_matches_oracle_pipeline(kp, top_n):
    dim = 128
    store, off = _integer_store(600, dim, seed=3)
    q = _queries(4, 32, dim, seed=4)
    idx = _build(ColBERTEndToEndIndexer, store, off, _cfg(dim))
    assert idx.store.dtype == torch.float8_e4m3fn and idx.store_scale == F.scale_log2(2.0)
    assert torch.equal(idx.store.cpu().view(torch.uint8), F.quantize(store, idx.store_scale).view(torch.uint8))
    s, i = idx.search_device(q.to(DEV), top_n, token_top_k=kp)
    rs, ri = E.colbert_e2e_search(q.double(), store.double(), off, top_n, kp, dtype=torch.float64)
    assert torch.equal(i.cpu(), ri)
    assert torch.equal(s.cpu().double(), rs)


def test_ivf_fp8_indexer_keeps_the_fp16_layout_and_results():
    dim, nlist, nprobe = 256, 24, 6
    store, off = _integer_store(700, dim, seed=5)
    q = _queries(3, 32, dim, seed=6)
    ref = _build(ColBERTIVFIndexer, store, off, _cfg(dim, fp8=False, nlist=nlist, nprobe=nprobe))
    idx = ColBERTIVFIndexer(_cfg(dim, nlist=nlist, nprobe=nprobe), device=DEV)
    idx.ivf.set_centroids(ref.ivf.centroids)
    idx.chunk_rows = 1000                                                       # several chunks
    idx.index([_pid(off)], [store.numpy()])
    assert torch.equal(idx.row_index, ref.row_index) and torch.equal(idx.list_offsets, ref.list_offsets)
    for kp, top_n in ((16, 20), (100, 60)):
        s, i = idx.search_device(q.to(DEV), top_n, token_top_k=kp)
        rs, ri = ref.search_device(q.to(DEV), top_n, token_top_k=kp)
        assert torch.equal(i, ri) and torch.equal(s, rs)


def test_streamed_index_equals_one_shot_index():
    dim = 768
    store, off, _ = _clustered_store(500, dim, 30, seed=7)
    a = ColBERTEndToEndIndexer(_cfg(dim), device=DEV)
    a.chunk_rows = 777
    a.index([_pid(off)], [store.numpy()])
    b = ColBERTEndToEndIndexer(_cfg(dim), device=DEV)
    b.index([_pid(off)], [store.numpy()])
    c = ColBERTEndToEndIndexer(_cfg(dim), device=DEV)
    c.index_device(store.to(DEV), off)
    sd = F.scale_log2(float(store.float().abs().max()))
    for x in (a, b, c):
        assert x.store_scale == sd
        assert torch.equal(x.store.cpu().view(torch.uint8), F.quantize(store, sd).view(torch.uint8))
        assert torch.equal(x.offsets, b.offsets) and torch.equal(x.row_ids, b.row_ids)


def test_save_load_round_trip(tmp_path):
    dim, nlist, nprobe = 128, 16, 4
    store, off = _integer_store(400, dim, seed=8)
    q = _queries(3, 32, dim, seed=9)
    idx = _build(ColBERTIVFIndexer, store, off, _cfg(dim, nlist=nlist, nprobe=nprobe))
    s0, i0 = idx.search_device(q.to(DEV), 30, token_top_k=32)
    path = str(tmp_path / "fp8.ivf")
    idx.save(path)
    back = ColBERTIVFIndexer(_cfg(dim, nlist=nlist, nprobe=nprobe), device=DEV)
    back.load(path)
    back.index([_pid(off)], [store.numpy()])
    assert back.store_scale == idx.store_scale
    assert torch.equal(back.row_index, idx.row_index)
    s1, i1 = back.search_device(q.to(DEV), 30, token_top_k=32)
    assert torch.equal(i0, i1) and torch.equal(s0, s1)
    with pytest.raises(_lib.MatchmakerB200Error):      # an fp16 indexer does not take an fp8 file
        ColBERTIVFIndexer(_cfg(dim, fp8=False, nlist=nlist, nprobe=nprobe), device=DEV).load(path)
    other = ColBERTIVFIndexer(_cfg(dim, nlist=nlist, nprobe=nprobe), device=DEV)
    other.load(path)
    with pytest.raises(_lib.MatchmakerB200Error):      # rows of another magnitude give another store scale
        other.index([_pid(off)], [(store.float() * 8).half().numpy()])


def test_index_peak_memory_is_the_store_plus_one_chunk():
    dim, chunk = 128, 4096
    store, off, _ = _clustered_store(20000, dim, 50, seed=10)
    n = store.shape[0]
    idx = ColBERTEndToEndIndexer(_cfg(dim), device=DEV)
    idx.chunk_rows = chunk
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    idx.index([_pid(off)], [store.numpy()])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    kept = n * dim + n * 8 + (len(off) + 1) * 8           # fp8 store, row ids, offsets
    one_chunk = chunk * dim * (2 + 4 + 1)                  # a chunk as given, its fp32 copy and its e4m3 image
    assert peak <= kept + one_chunk + (2 << 20), (peak, kept, one_chunk)
    assert kept + one_chunk + (2 << 20) < n * dim * 2     # below the fp16 store alone: it is never materialised


# Recall@100 of the fp8 indexer against the fp16 indexer on this clustered store: 0.926 measured (H100 SXM), pinned
# with headroom.
RECALL_FLOOR = 0.85


def test_fp8_recall_against_fp16_indexer():
    dim, top_n, kp = 128, 100, 64
    store, off, cent = _clustered_store(3000, dim, 60, seed=11)
    g = torch.Generator().manual_seed(12)
    q = (cent[torch.randint(0, 60, (16, 32), generator=g)] + 0.3 * torch.randn(16, 32, dim, generator=g) / dim ** 0.5)
    q = q.half().to(DEV)
    ref = _build(ColBERTEndToEndIndexer, store, off, _cfg(dim, fp8=False))
    idx = _build(ColBERTEndToEndIndexer, store, off, _cfg(dim))
    _, ri = ref.search_device(q, top_n, token_top_k=kp)
    _, i = idx.search_device(q, top_n, token_top_k=kp)
    rec = np.mean([len(set(i[a].tolist()) & set(ri[a].tolist())) / top_n for a in range(q.shape[0])])
    assert rec >= RECALL_FLOOR, rec
