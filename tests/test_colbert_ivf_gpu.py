"""IVF token index for ColBERT retrieval on the GPU: the gather mode of the probed-list scan against the scan over a
list-ordered copy (bit for bit), and retrieval.ColBERTIVFIndexer against the exact ColBERTEndToEndIndexer and the fp64
stage-1 oracle restricted to each token's probed lists."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import colbert_e2e_oracle as E
import colbert_ivf_oracle as CV
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _cfg(dim, nlist, nprobe, dtype="float16"):
    return {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": dtype, "faiss_ivf_list_count": nlist,
            "faiss_ivf_search_probe_count": nprobe}


# ----------------------------------------------------------------------------------------------------------------------
# 1. gather scan == scan over the list-ordered copy, bit for bit
# ----------------------------------------------------------------------------------------------------------------------
def _sizes(n, nlist, seed):
    """List sizes with an empty list 0, a one-row list 1, a list of several tiles (2) and random others."""
    rng = np.random.default_rng(seed)
    sizes = np.zeros(nlist, dtype=np.int64)
    sizes[1], sizes[2] = 1, n // 3
    sizes[3:] = rng.multinomial(n - int(sizes.sum()), np.ones(nlist - 3) / (nlist - 3))
    return sizes


@pytest.mark.parametrize("fp32,dim,k,nprobe,nlist", [(False, 128, 64, 8, 40), (False, 64, 300, 4, 12),
                                                     (True, 128, 32, 6, 40), (False, 128, 1000, 2, 5),
                                                     (True, 64, 100, 12, 12)])
def test_gather_scan_equals_scan_over_list_ordered_copy(fp32, dim, k, nprobe, nlist):
    n, nq = 5000, 40
    dt = torch.float32 if fp32 else torch.float16
    q, rows = O.synth_dense_inputs(nq, n, dim, seed=dim + k, dtype=dt)
    g = torch.Generator().manual_seed(k)
    row_ids = torch.sort(torch.randint(0, n // 4, (n,), generator=g)).values     # passage ids: runs of equal ids
    sizes = _sizes(n, nlist, seed=nprobe)
    assign = torch.from_numpy(np.repeat(np.arange(nlist), sizes))[torch.randperm(n, generator=g)]
    row_index = torch.sort(assign, stable=True).indices
    off = torch.zeros(nlist + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.from_numpy(sizes), 0)
    probes = torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(nq)])
    probes[0] = torch.arange(nprobe)                       # the empty, one-row and long lists
    probes[1, nprobe // 2:] = -1
    max_len = int(sizes.max())
    qd, rd, ri, od, pd = q.to(DEV), rows.to(DEV), row_index.to(DEV), off.to(DEV), probes.to(DEV)
    scale = None
    if fp32:
        rd, scale = interaction.flat_ip_split_f32(rd.float(), "passages")
    s_g, i_g = interaction.ivf_search(qd, rd, row_ids.to(DEV), od, pd, k, max_len, split_scale=scale, row_index=ri)
    s_c, i_c = interaction.ivf_search(qd, rd[ri].contiguous(), row_ids.to(DEV)[ri].contiguous(), od, pd, k, max_len,
                                      split_scale=scale)
    assert torch.equal(i_g, i_c)
    assert torch.equal(s_g.view(torch.int32), s_c.view(torch.int32))
    assert bool((i_g[1] >= 0).any()) and int((i_g[0] >= 0).sum()) == min(k, int(sizes[:nprobe].sum()))


# ----------------------------------------------------------------------------------------------------------------------
# shared stores
# ----------------------------------------------------------------------------------------------------------------------
def _lengths(n_pass, seed):
    return np.random.default_rng(seed).integers(1, 40, n_pass)


def _integer_store(lengths, dim, seed):
    """Rows and queries with small integer entries: every inner product is exact in fp16 products and fp32 sums."""
    g = torch.Generator().manual_seed(seed)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    store = torch.randint(-2, 3, (int(off[-1]), dim), generator=g).half()
    return store, off


def _clustered_store(lengths, dim, n_centres, seed):
    g = torch.Generator().manual_seed(seed)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    c = torch.nn.functional.normalize(torch.randn(n_centres, dim, generator=g), dim=1)
    which = torch.randint(0, n_centres, (int(off[-1]),), generator=g)
    store = (c[which] + 0.25 * torch.randn(int(off[-1]), dim, generator=g) / dim ** 0.5).half()
    return store, off, c


def _pid(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def _build(store, off, dim, nlist, nprobe, dtype="float16", exact=False):
    blocks = [store.numpy().astype(np.float16 if dtype == "float16" else np.float32)]
    if exact:
        idx = ColBERTEndToEndIndexer({"token_dim": dim, "faiss_use_gpu": True, "token_dtype": dtype}, device=DEV)
    else:
        idx = ColBERTIVFIndexer(_cfg(dim, nlist, nprobe, dtype), device=DEV)
        idx.prepare(blocks)
    idx.index([_pid(off)], blocks)
    return idx


# ----------------------------------------------------------------------------------------------------------------------
# 2. nprobe = nlist on exact data == the exact indexer
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kp,top_n", [(16, 20), (64, 100), (300, 50)])
def test_full_probe_equals_exact_indexer(kp, top_n):
    dim, nlist = 128, 24
    store, off = _integer_store(_lengths(1500, 1), dim, seed=2)
    q = torch.randint(-2, 3, (4, 32, dim), generator=torch.Generator().manual_seed(3)).half()
    q[1, 20:] = 0
    ivf = _build(store, off, dim, nlist, nlist)
    exact = _build(store, off, dim, nlist, nlist, exact=True)
    s, i = ivf.search_device(q.to(DEV), top_n, token_top_k=kp)
    rs, ri = exact.search_device(q.to(DEV), top_n, token_top_k=kp)
    assert torch.equal(i, ri) and torch.equal(s, rs)
    cs, ci = ivf.candidates_device(q.to(DEV), kp)
    rcs, rci = exact.candidates_device(q.to(DEV), kp)
    assert torch.equal(ci, rci) and torch.equal(cs, rcs)


# ----------------------------------------------------------------------------------------------------------------------
# 3. nprobe < nlist: must / may bounds over each token's probed lists
# ----------------------------------------------------------------------------------------------------------------------
def test_probed_candidates_within_fp64_bounds():
    dim, nlist, nprobe, lq, kp = 128, 32, 4, 32, 16
    store, off, _ = _clustered_store(_lengths(2000, 4), dim, 40, seed=5)
    q = (torch.randn(3, lq, dim, generator=torch.Generator().manual_seed(6)) * 0.3).half()
    q[2, 25:] = 0
    idx = _build(store, off, dim, nlist, nprobe)
    _, ci = idx.candidates_device(q.to(DEV), kp)
    ci = ci.cpu()
    probes = idx.ivf.coarse(q.reshape(-1, dim).to(DEV)).cpu().view(3, lq, -1)
    assign = torch.empty(store.shape[0], dtype=torch.int64)
    assign[idx.row_index.cpu()] = torch.repeat_interleave(torch.arange(nlist), (idx.list_offsets[1:] - idx.list_offsets[:-1]).cpu())
    pid = E.row_passages(off)
    s64, tol = E.token_scores(q, store, torch.float64), E.accumulation_tol(q, store)
    live = (q != 0).any(-1)
    for a in range(q.shape[0]):
        got = set(int(x) for x in ci[a] if x >= 0)
        must, may = set(), set()
        for t in range(lq):
            if not live[a, t]:
                continue
            m = CV.probed_rows(assign, probes[a, t])
            s, p, tmax = s64[a, t][m], pid[m], float(tol[a, t].max())
            srt = s.sort(descending=True).values
            hi_cut = float(srt[kp]) + 2 * tmax if len(srt) > kp else -float("inf")
            lo_cut = float(srt[kp - 1]) - 2 * tmax if len(srt) >= kp else -float("inf")
            must |= set(p[s > hi_cut].tolist())
            may |= set(p[s >= lo_cut].tolist())
        assert must <= got, f"query {a}: decided candidates missing: {sorted(must - got)[:10]}"
        assert got <= may, f"query {a}: passages outside every token's probed top-k': {sorted(got - may)[:10]}"
        assert len(must) > 0


# ----------------------------------------------------------------------------------------------------------------------
# 4. recall rises with nprobe, 1.0 at nprobe = nlist
# ----------------------------------------------------------------------------------------------------------------------
def test_recall_does_not_decrease_with_nprobe():
    dim, nlist, top_n, kp = 128, 64, 50, 32
    store, off, cent = _clustered_store(_lengths(4000, 7), dim, 80, seed=8)
    g = torch.Generator().manual_seed(9)
    q = (cent[torch.randint(0, 80, (8, 32), generator=g)] + 0.3 * torch.randn(8, 32, dim, generator=g) / dim ** 0.5).half()
    exact = _build(store, off, dim, nlist, nlist, exact=True)
    _, ri = exact.search_device(q.to(DEV), top_n, token_top_k=kp)
    ri = ri.cpu()
    idx = _build(store, off, dim, nlist, 1)
    rec = []
    for nprobe in (1, 4, 16, nlist):
        idx.ivf.nprobe = nprobe
        _, i = idx.search_device(q.to(DEV), top_n, token_top_k=kp)
        i = i.cpu()
        rec.append(np.mean([len(set(i[a].tolist()) & set(ri[a].tolist())) / top_n for a in range(q.shape[0])]))
    assert all(b >= a - 1e-9 for a, b in zip(rec, rec[1:])), rec
    assert rec[-1] == 1.0, rec


# ----------------------------------------------------------------------------------------------------------------------
# 5. two shards sharing centroids == one index
# ----------------------------------------------------------------------------------------------------------------------
def test_two_shards_merge_to_single_index(monkeypatch):
    dim, nlist, nprobe, top_n = 128, 16, 4, 40
    store, off, _ = _clustered_store(_lengths(300, 10), dim, 20, seed=11)
    q = (torch.randn(3, 32, dim, generator=torch.Generator().manual_seed(12)) * 0.3).half().to(DEV)
    single = _build(store, off, dim, nlist, nprobe)
    s_ref, i_ref = single.search_device(q, top_n, token_top_k=64)
    parts = []
    for r in range(2):
        idx = ColBERTIVFIndexer(_cfg(dim, nlist, nprobe), device=DEV)
        monkeypatch.setattr(idx, "_world", lambda r=r: (r, 2))
        idx.ivf.set_centroids(single.ivf.centroids)
        idx.index([_pid(off)], [store.numpy()])
        assert 0 < idx.d_hi - idx.d_lo < len(off) - 1
        parts.append(idx.search_device(q, top_n, token_top_k=64))
    s, i = interaction.topk_merge(torch.cat([parts[0][0], parts[1][0]], 1), torch.cat([parts[0][1], parts[1][1]], 1), top_n)
    assert torch.equal(i, i_ref) and torch.equal(s, s_ref)


# ----------------------------------------------------------------------------------------------------------------------
# 6. save / load
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_save_load_round_trip(tmp_path, monkeypatch, dtype):
    dim, nlist, nprobe = 128, 16, 3
    store, off, _ = _clustered_store(_lengths(400, 13), dim, 20, seed=14)
    q = (torch.randn(3, 32, dim, generator=torch.Generator().manual_seed(15)) * 0.3).to(DEV)
    idx = _build(store, off, dim, nlist, nprobe, dtype=dtype)
    s_ref, i_ref = idx.search_device(q, 30, token_top_k=32)
    path = str(tmp_path / "tok.ivf")
    idx.save(path)
    blocks = [store.numpy().astype(np.float16 if dtype == "float16" else np.float32)]
    re_ = ColBERTIVFIndexer(_cfg(dim, nlist, 1, dtype), device=DEV)
    re_.load(path, {"faiss_ivf_search_probe_count": nprobe})
    monkeypatch.setattr(re_, "assign", lambda rows: pytest.fail("index() after load() re-assigned the rows"))
    re_.index([_pid(off)], blocks)
    s, i = re_.search_device(q, 30, token_top_k=32)
    assert torch.equal(i, i_ref) and torch.equal(s, s_ref)
    other = ColBERTIVFIndexer(_cfg(dim, nlist, nprobe, dtype), device=DEV)
    other.load(path)
    with pytest.raises(_lib.MatchmakerB200Error, match="re-index"):
        other.index([_pid(off)[:-5]], [blocks[0][:-5]])              # another store
    two = ColBERTIVFIndexer(_cfg(dim, nlist, nprobe, dtype), device=DEV)
    monkeypatch.setattr(two, "_world", lambda: (0, 2))
    with pytest.raises(_lib.MatchmakerB200Error, match="world size"):
        two.load(path)


# ----------------------------------------------------------------------------------------------------------------------
# 7. device memory budget, 8. CUDA graph
# ----------------------------------------------------------------------------------------------------------------------
def test_device_memory_within_budget_of_exact_indexer():
    dim, nlist = 128, 256
    store, off, _ = _clustered_store(_lengths(20000, 16), dim, 300, seed=17)
    n = store.shape[0]

    def resident(make):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated(DEV)
        idx = make()
        torch.cuda.synchronize()
        return idx, torch.cuda.memory_allocated(DEV) - base

    exact, m_exact = resident(lambda: _build(store, off, dim, nlist, 8, exact=True))
    del exact
    ivf, m_ivf = resident(lambda: _build(store, off, dim, nlist, 8))
    budget = 8 * n + 8 * (nlist + 1) + nlist * dim * (4 + 2) + (4 << 20)   # + allocator rounding
    assert m_ivf - m_exact <= budget, (m_ivf, m_exact, budget)
    assert ivf.row_index.numel() == n


def test_search_device_replays_in_cuda_graph():
    dim = 128
    store, off, _ = _clustered_store(_lengths(800, 18), dim, 30, seed=19)
    idx = _build(store, off, dim, 32, 4)
    q = (torch.randn(4, 32, dim, generator=torch.Generator().manual_seed(20)) * 0.3).half().to(DEV)
    ref_s, ref_i = idx.search_device(q, 50, token_top_k=64)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gs, gi = idx.search_device(q, 50, token_top_k=64)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gs, ref_s) and torch.equal(gi, ref_i)


# ----------------------------------------------------------------------------------------------------------------------
# 9. SASS of the gather instantiations
# ----------------------------------------------------------------------------------------------------------------------
def test_gather_kernel_sass_uses_wgmma_and_cp_async():
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = {f.split("\n", 1)[0]: f for f in re.split(r"\n\s+Function : ", txt)}
    gather = {k: v for k, v in funcs.items() if "flat_ip_tc_gather_kernel" in k}
    assert len(gather) == 4, list(gather)
    for name, f in gather.items():
        assert [l for l in f.splitlines() if "HGMMA" in l and "gdesc[URZ]" not in l], f"{name}: no wgmma"
        assert "LDGSTS" in f, f"{name}: no cp.async"
        assert "UTMALDG" in f, f"{name}: no TMA load of the queries"
