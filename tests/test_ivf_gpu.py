"""IVF index on the GPU: the probed-list scan against the CPU oracle (exact top-k over the union of the probed lists),
the coarse stage, k-means, sharding and the drop-in behaviour of retrieval.IVFIndexer."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import colbert_e2e_oracle as E
import ivf_oracle as V
from conftest import assert_close_rel
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import FlatIPIndexer, IVFIndexer
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cfg(dtype="float16", nlist=16, nprobe=4, dim=64):
    return {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": dtype, "faiss_ivf_list_count": nlist,
            "faiss_ivf_search_probe_count": nprobe}


def _layout(n, nlist, seed, skew=True):
    """List offsets with an empty list 0, a one-row list 1 and (skew) list 2 holding half the rows; the rest random."""
    rng = np.random.default_rng(seed)
    sizes = np.zeros(nlist, dtype=np.int64)
    sizes[1] = 1
    if skew:
        sizes[2] = n // 2
    free = np.arange(3 if skew else 2, nlist)
    sizes[free] = rng.multinomial(n - int(sizes.sum()), np.ones(len(free)) / len(free))
    off = np.zeros(nlist + 1, dtype=np.int64)
    off[1:] = np.cumsum(sizes)
    return torch.from_numpy(off)


def _probes(nq, nlist, nprobe, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(nq)])
    p[0] = torch.arange(nprobe)                 # the empty, one-row and half lists
    if nq > 3:
        p[1] = p[0]                             # heavy overlap
        p[2] = p[0].flip(0)
    return p


def _run(q, rows, ids, off, probes, k, fp32, max_len=None):
    if max_len is None:
        max_len = int((off[1:] - off[:-1]).max())
    if fp32:
        split, scale = interaction.flat_ip_split_f32(rows.float().to(DEV), "passages")
        return interaction.ivf_search(q.float().to(DEV), split, ids.to(DEV), off.to(DEV), probes.to(DEV), k, max_len,
                                      split_scale=scale)
    return interaction.ivf_search(q.to(DEV), rows.to(DEV), ids.to(DEV), off.to(DEV), probes.to(DEV), k, max_len)


def _check(q, rows, ids, off, probes, k, got_s, got_i):
    if q.dtype == torch.float32:
        st = V.ivf_check_split(q, rows, ids, off, probes, got_s, got_i, k)
        assert st["decided"] >= 0.95 * max(1, st["decided"] + st["undecided"]), st
        return
    ref_s, ref_i = V.ivf_search(q.float(), rows.float(), ids, off, probes, k)
    assert_close_rel(got_s.cpu(), ref_s, what="scores")
    st = V.ivf_check_exact(q.float(), rows.float(), ids, off, probes, got_s, got_i, k)
    assert st["decided"] >= 0.95 * max(1, st["decided"] + st["undecided"]), st


@pytest.mark.parametrize("case", [(64, 10, 8, 600), (128, 100, 8, 64), (768, 10, 1, 64), (64, 1000, 500, 1000),
                                  (128, 1, 500, 1000), (64, 100, 1, 64), (768, 100, 8, 64)])
@pytest.mark.parametrize("fp32", [False, True])
def test_scan_matches_oracle(case, fp32):
    dim, k, nprobe, nlist = case
    n = 12000 if nlist >= 600 else 6000
    nq = 24
    q, rows = O.synth_dense_inputs(nq, n, dim, seed=dim + k + nprobe, dtype=torch.float32 if fp32 else torch.float16)
    ids = torch.randperm(n, generator=torch.Generator().manual_seed(3)) * 3 - n     # negative user ids too
    off = _layout(n, nlist, seed=k)
    probes = _probes(nq, nlist, nprobe, seed=nprobe)
    s, i = _run(q, rows, ids, off, probes, k, fp32)
    _check(q, rows, ids, off, probes, k, s, i)


def test_scan_small_unions_give_the_empty_tail_and_disjoint_queries():
    dim, n, nlist, k = 64, 2000, 500, 100
    q, rows = O.synth_dense_inputs(6, n, dim, seed=11)
    ids = torch.arange(n) - 1000
    off = _layout(n, nlist, seed=2, skew=False)
    probes = torch.tensor([[0, 1, 3, 4, 5, 6, 7, 8], [9, 10, 11, 12, 13, 14, 15, 16], [0, -1, -1, -1, -1, -1, -1, -1],
                           [20, 21, 22, 23, 24, 25, 26, 27], [0, 1, 3, 4, 5, 6, 7, 8], [100, 200, 300, 400, 1, 2, 3, 4]])
    s, i = _run(q, rows, ids, off, probes, k, False)
    _check(q, rows, ids, off, probes, k, s, i)
    assert torch.all(i[2].cpu() == -1) and torch.all(s[2].cpu() == V.NO_RESULT)


@pytest.mark.parametrize("fp32", [False, True])
def test_scan_exact_ties_resolved_by_id(fp32):
    """300 identical rows whose score is the k-th best of every query: 20 rows score above them, so the run of exact ties
    covers rank k - 1 and goes on past k.  The copies sit at random positions in every list, with ids that do not follow
    the positions, so the per-list compaction, the threshold shared across lists and the merge of the slots all have to
    break the ties by id."""
    dim, n, nlist, k = 64, 3000, 10, 50
    dt = torch.float32 if fp32 else torch.float16
    q, rows = O.synth_dense_inputs(4, n, dim, seed=3, dtype=dt)
    d = torch.nn.functional.normalize(q.float().sum(0), dim=0)
    assert bool((q.float() @ d > 0).all())
    g = torch.Generator().manual_seed(4)
    pos = torch.randperm(n, generator=g)
    tied, above = pos[:300], pos[300:320]
    rows[tied] = (10.0 * d).to(dt)
    rows[above] = ((13.0 + 0.5 * torch.arange(20.0)).unsqueeze(1) * d).to(dt)   # 20 distinct scores well above the tie
    ids = torch.randperm(n, generator=g) * 7 - 10000
    off = torch.arange(0, n + 1, n // nlist)
    lists = torch.randperm(nlist, generator=g)
    probes = torch.stack([torch.arange(nlist), torch.arange(nlist).flip(0), lists, lists.roll(3)])
    probes[2:, 6:] = -1                       # two queries probe 6 of the 10 lists
    s64 = q.double() @ rows.double().T
    tie = s64[:, tied[0]]
    for r in range(4):
        u = V.union_rows(off, probes[r])
        in_u = torch.zeros(n, dtype=torch.bool)
        in_u[u] = True
        n_above = int(((s64[r] > tie[r]) & in_u).sum())
        n_tied = int(((s64[r] == tie[r]) & in_u).sum())
        assert n_above <= k - 1 < k < n_above + n_tied, (r, n_above, n_tied)   # the tie run spans rank k - 1 and k
        assert len(set((tied[in_u[tied]] // (n // nlist)).tolist())) >= 2     # spread over several probed lists
    s, i = _run(q, rows, ids, off, probes, k, fp32)
    # the ranking is taken in fp64, where identical rows tie exactly; the fp32 CPU product does not promise one value
    # for identical rows at different positions, so it cannot be the arbiter of a tie
    for r in range(4):
        u = V.union_rows(off, probes[r])
        ref_s, ref_i = O.rank_desc_stable(s64[r, u], ids[u], k)
        assert torch.equal(i[r].cpu(), ref_i), r
        assert torch.allclose(s[r].cpu().double(), ref_s, rtol=1e-5), r
    assert torch.equal(s.cpu()[:, k - 1], s.cpu()[:, k - 2])


def test_scan_query_batching_is_exact(monkeypatch):
    dim, n, nlist, k, nprobe, nq = 64, 8000, 200, 10, 20, 300
    q, rows = O.synth_dense_inputs(nq, n, dim, seed=5)
    ids = torch.arange(n)
    off = _layout(n, nlist, seed=5)
    probes = _probes(nq, nlist, nprobe, seed=5)
    s0, i0 = _run(q, rows, ids, off, probes, k, False)
    lib = _lib.load()
    one = lib.mmb200_ivf_workspace_bytes(1, nprobe, nlist, int((off[1:] - off[:-1]).max()), dim, k, _lib.F16)
    full = lib.mmb200_ivf_workspace_bytes(nq, nprobe, nlist, int((off[1:] - off[:-1]).max()), dim, k, _lib.F16)
    monkeypatch.setattr(interaction, "IVF_WORKSPACE_CAP", one + (full - one) // 7)   # about 8 batches
    s1, i1 = _run(q, rows, ids, off, probes, k, False)
    assert torch.equal(i0, i1) and torch.equal(s0, s1)
    _check(q[:40], rows, ids, off, probes[:40], k, s1[:40], i1[:40])


def test_scan_rejects_sizes_outside_the_envelope():
    q = torch.zeros(2, 64, dtype=torch.float16, device=DEV)
    rows = torch.zeros(10, 64, dtype=torch.float16, device=DEV)
    ids, off = torch.arange(10, device=DEV), torch.tensor([0, 5, 10], device=DEV)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.ivf_search(q, rows, ids, off, torch.zeros(2, 1025, dtype=torch.int64, device=DEV), 1, 5)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.ivf_search(q, rows, ids, off, torch.zeros(2, 1, dtype=torch.int64, device=DEV), 1025, 5)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.ivf_search(q[:, :48], rows[:, :48], ids, off, torch.zeros(2, 1, dtype=torch.int64, device=DEV), 1, 5)
    with pytest.raises(_lib.MatchmakerB200Error):       # rows narrower than the queries
        interaction.ivf_search(q, rows[:, :32].contiguous(), ids, off, torch.zeros(2, 1, dtype=torch.int64, device=DEV), 1, 5)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.flat_ip_topk(q, rows[:, :32].contiguous(), 1)


def _clustered(n, dim, n_clusters, seed, nq=64):
    g = torch.Generator().manual_seed(seed)
    centers = torch.nn.functional.normalize(torch.randn(n_clusters, dim, generator=g), dim=1)
    lab = torch.randint(0, n_clusters, (n,), generator=g)
    x = centers[lab] + 0.35 * torch.randn(n, dim, generator=g) / dim ** 0.5
    ql = torch.randint(0, n_clusters, (nq,), generator=g)
    q = centers[ql] + 0.35 * torch.randn(nq, dim, generator=g) / dim ** 0.5
    return x, q


@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_coarse_stage_is_exact(dtype):
    x, q = _clustered(4000, 128, 40, seed=1)
    idx = IVFIndexer(_cfg(dtype, nlist=64, nprobe=8, dim=128))
    idx.prepare([x.numpy()])
    p = idx.coarse(q.to(DEV).to(idx.store_dtype if dtype == "float16" else torch.float32))
    c = idx.centroids.cpu()
    c_seen = c.half().float() if dtype == "float16" else c
    qq = q.half().float() if dtype == "float16" else q
    s = torch.gather(qq.double() @ c_seen.double().T, 1, p.cpu())
    O.flat_ip_check_exact(qq, c_seen, torch.arange(64), s.float(), p, 8)


@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_full_probe_equals_flat_index(dtype):
    x, q = _clustered(6000, 64, 20, seed=2)
    ids = np.arange(6000, dtype=np.int64) * 7 - 9000
    ivf = IVFIndexer(_cfg(dtype, nlist=32, nprobe=32))
    ivf.prepare([x.numpy()])
    ivf.index([ids], [x.numpy()])
    flat = FlatIPIndexer(_cfg(dtype))
    flat.index([ids], [x.numpy()])
    s, i = ivf.search(q.numpy(), 100)
    fs, fi = flat.search(q.numpy(), 100)
    if dtype == "float16":
        xs, qs = x.half().float(), q.half().float()
        O.flat_ip_check_exact(qs, xs, torch.from_numpy(ids), torch.from_numpy(s), torch.from_numpy(i), 100)
        O.flat_ip_check_exact(qs, xs, torch.from_numpy(ids), torch.from_numpy(fs), torch.from_numpy(fi), 100)
    else:   # one list holding every row, probed by every query: the fp32-storage checker of the scan tests
        whole, probes = torch.tensor([0, 6000]), torch.zeros(q.shape[0], 1, dtype=torch.int64)
        for got_s, got_i in ((s, i), (fs, fi)):
            V.ivf_check_split(q, x, torch.from_numpy(ids), whole, probes, torch.from_numpy(got_s), torch.from_numpy(got_i), 100)
    assert (i == fi).mean() > 0.99
    assert_close_rel(torch.from_numpy(s), torch.from_numpy(fs), what="scores")


def test_recall_is_monotone_in_nprobe():
    x, q = _clustered(20000, 64, 100, seed=3, nq=128)
    ids = np.arange(20000, dtype=np.int64)
    ivf = IVFIndexer(_cfg(nlist=128, nprobe=1))
    ivf.prepare([x.numpy()])
    ivf.index([ids], [x.numpy()])
    flat = FlatIPIndexer(_cfg())
    flat.index([ids], [x.numpy()])
    _, fi = flat.search(q.numpy(), 100)
    recalls = []
    for nprobe in (1, 2, 4, 8, 16, 32, 128):
        ivf.nprobe = nprobe
        _, i = ivf.search(q.numpy(), 100)
        recalls.append(np.mean([len(set(a) & set(b)) for a, b in zip(i.tolist(), fi.tolist())]))
    assert all(b >= a for a, b in zip(recalls, recalls[1:])), recalls
    assert recalls[-1] == 100


@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_kmeans_iteration_matches_fp64_oracle(dtype):
    x, _ = _clustered(5000, 64, 30, seed=4)
    idx = IVFIndexer(_cfg(dtype, nlist=40))
    xd = x.to(DEV).to(idx.store_dtype)
    c0 = torch.nn.functional.normalize(x[:40].clone(), dim=1)
    new, assign, _ = idx.kmeans_step(xd, c0.to(DEV))
    c_seen = c0.half().float() if dtype == "float16" else c0
    ref_a, ref_c, gap = V.kmeans_step(xd.float().cpu(), c_seen)
    sure = gap > 1e-3
    assert torch.equal(assign.cpu()[sure], ref_a[sure])
    err = (new.cpu().double() - ref_c).norm(dim=1) / ref_c.norm(dim=1).clamp_min(1e-30)
    assert float(err[ref_c.norm(dim=1) > 0].max()) < 1e-3


def test_kmeans_is_deterministic_unit_norm_and_monotone():
    x, _ = _clustered(40 * 50, 64, 50, seed=5)
    a = IVFIndexer(_cfg("float32", nlist=50))
    ca = a.train([x.numpy()])
    cb = IVFIndexer(_cfg("float32", nlist=50)).train([x.numpy()])
    assert torch.equal(ca, cb)
    assert torch.allclose(ca.norm(dim=1), torch.ones(50, device=DEV), atol=1e-5)
    obj, splits = a.train_objective, a.train_splits
    for t in range(1, len(obj)):
        if splits[t - 1] == 0:
            assert obj[t] >= obj[t - 1] - 1e-6 * abs(obj[t - 1]), (obj, splits)
    a.set_centroids(ca)
    a.index([np.arange(len(x))], [x.numpy()])
    assert int((a.list_offsets[1:] - a.list_offsets[:-1]).min()) > 0     # n >= 39 * nlist: no empty list
    f16 = IVFIndexer(_cfg("float16", nlist=50))
    assert torch.equal(f16.train([x.numpy()]), IVFIndexer(_cfg("float16", nlist=50)).train([x.numpy()]))


def test_kmeans_needs_a_point_per_list():
    with pytest.raises(_lib.MatchmakerB200Error):
        IVFIndexer(_cfg(nlist=100)).prepare([np.random.default_rng(0).normal(size=(99, 64)).astype(np.float16)])


def test_two_shards_sharing_centroids_merge_to_the_whole_index():
    x, q = _clustered(8000, 64, 30, seed=6)
    ids = torch.arange(8000) * 3 - 100
    whole = IVFIndexer(_cfg(nlist=32, nprobe=6))
    whole.prepare([x.numpy()])
    whole.index([ids.numpy()], [x.numpy()])
    parts = []
    for lo, hi in ((0, 4000), (4000, 8000)):
        p = IVFIndexer(_cfg(nlist=32, nprobe=6))
        p.set_centroids(whole.centroids)
        p.add_sorted(x[lo:hi].to(DEV).half(), ids[lo:hi].to(DEV))
        parts.append(p.search_device(q.to(DEV).half(), 100))
    s, i = interaction.topk_merge(torch.cat([parts[0][0], parts[1][0]], 1), torch.cat([parts[0][1], parts[1][1]], 1), 100)
    ws, wi = whole.search_device(q.to(DEV).half(), 100)
    assert torch.equal(i, wi) and torch.equal(s, ws)


def test_drop_in_behaviour(tmp_path):
    x, q = _clustered(5000, 64, 20, seed=7)
    ids = np.arange(5000, dtype=np.int64) * 2 - 3000
    idx = IVFIndexer(_cfg(nlist=32, nprobe=4))
    idx.prepare([x[:2500].numpy(), x[2500:].numpy()])
    idx.index([ids[:2500], ids[2500:]], [x[:2500].numpy(), x[2500:].numpy()])
    s, i = idx.search(q.numpy().astype(np.float16), 10)
    assert isinstance(s, np.ndarray) and s.dtype == np.float32 and i.dtype == np.int64 and s.shape == (64, 10)
    s1, i1 = idx.search(q[3].numpy(), 10)               # 1-D query
    assert np.array_equal(i1[0], i[3])
    path = str(tmp_path / "faiss.index")
    idx.save(path)
    back = IVFIndexer(_cfg(nlist=32, nprobe=4))
    back.load(path)
    s2, i2 = back.search(q.numpy(), 10)
    assert np.array_equal(s2, s) and np.array_equal(i2, i)
    wide = IVFIndexer(_cfg(nlist=32, nprobe=4))
    wide.load(path, {"faiss_ivf_search_probe_count": 32})
    assert wide.nprobe == 32
    s3, _ = wide.search(q.numpy(), 10)
    assert np.all(s3 >= s - 1e-3 * np.abs(s))           # rank j over a superset of lists is never worse
    with pytest.raises(_lib.MatchmakerB200Error):
        IVFIndexer(_cfg("float32", nlist=32)).load(path)
    blob = torch.load(path)
    blob["world"] = 2
    torch.save(blob, path)
    with pytest.raises(_lib.MatchmakerB200Error):
        IVFIndexer(_cfg(nlist=32)).load(path)


def test_search_unique_matches_the_maxp_loop():
    x, q = _clustered(4000, 64, 20, seed=8, nq=8)
    ids = (np.arange(4000) // 4).astype(np.int64)        # four vectors per passage
    idx = IVFIndexer(_cfg(nlist=16, nprobe=4))
    idx.prepare([x.numpy()])
    idx.index([ids], [x.numpy()])
    s, i = idx.search_unique(q.numpy(), 10, 200)
    hs, hi = idx.search(q.numpy(), 200)
    loop = E.maxp_loop(hs, hi, 10)
    for a in range(8):
        assert [int(v) for v in i[a, :len(loop[a])]] == [int(p) for p, _ in loop[a]]


def test_search_device_replays_in_a_cuda_graph():
    x, q = _clustered(6000, 64, 20, seed=9)
    idx = IVFIndexer(_cfg(nlist=32, nprobe=8))
    idx.prepare([x.numpy()])
    idx.index([np.arange(6000)], [x.numpy()])
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


def test_scan_kernel_sass_uses_wgmma_and_tma():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump not available")
    txt = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s+Function : ", txt)
    ivf = [f for f in funcs if f.startswith("_Z") and "flat_ip_tc_kernel" in f.split("\n", 1)[0]
           and "Lb1E" in f.split("\n", 1)[0]]
    assert len(ivf) == 4, [f.split("\n", 1)[0] for f in funcs if "flat_ip_tc_kernel" in f.split("\n", 1)[0]]
    for f in ivf:
        body = [l for l in f.splitlines() if "HGMMA" in l and "gdesc[URZ]" not in l]
        assert body, "no wgmma in the IVF scan"
        assert "UTMALDG" in f, "no TMA load in the IVF scan"
