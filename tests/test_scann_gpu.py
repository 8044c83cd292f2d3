"""AH (faiss_index_type "scann") index on the GPU: the code scan and the reorder against the CPU oracle bit for bit, the
training, and the drop-in behaviour of retrieval.ScaNNIndexer."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import ah_oracle as A
import colbert_e2e_oracle as E
from conftest import ROOT
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.retrieval import FlatIPIndexer, ScaNNIndexer
from matchmaker_b200.retrieval import scann_index as S

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cfg(dtype="float16", dim=64, top_n=100, hit=None):
    qs = {"top_n": top_n}
    if hit is not None:
        qs["index_hit_top_n"] = hit
    return {"token_dim": dim, "faiss_use_gpu": False, "token_dtype": dtype, "query_sets": {"test": qs}}


def _layout(n, nlist, seed):
    """Leaf offsets with an empty leaf 0, a one-row leaf 1 and leaf 2 holding half the rows; the rest random."""
    rng = np.random.default_rng(seed)
    sizes = np.zeros(nlist, dtype=np.int64)
    sizes[1] = 1
    sizes[2] = n // 2
    sizes[3:] = rng.multinomial(n - int(sizes.sum()), np.ones(nlist - 3) / (nlist - 3))
    off = np.zeros(nlist + 1, dtype=np.int64)
    off[1:] = np.cumsum(sizes)
    return torch.from_numpy(off)


def _clustered(n, dim, k, seed, nq=64):
    g = torch.Generator().manual_seed(seed)
    c = torch.nn.functional.normalize(torch.randn(k, dim, generator=g), dim=1)
    x = c[torch.randint(0, k, (n,), generator=g)] + 0.4 * torch.randn(n, dim, generator=g) / dim ** 0.5
    q = c[torch.randint(0, k, (nq,), generator=g)] + 0.4 * torch.randn(nq, dim, generator=g) / dim ** 0.5
    return x.half(), q.half()


def _probe_table(nq, nprobe, nlist, g):
    """Distinct leaf ids per row: even rows probe leaves 0, 1, 2 (empty, one row, half the rows) first and then others,
    odd rows a random set; every third row ends in a -1 filler."""
    rows = []
    for r in range(nq):
        if r % 2 == 0:
            head = torch.arange(min(3, nprobe))
            rows.append(torch.cat([head, 3 + torch.randperm(nlist - 3, generator=g)[:nprobe - len(head)]]))
        else:
            rows.append(torch.randperm(nlist, generator=g)[:nprobe])
    p = torch.stack(rows)
    if nprobe > 1:
        p[::3, -1] = -1
    return p


def _scan_inputs(dim, nq, nprobe, nlist, n, seed):
    g = torch.Generator().manual_seed(seed)
    tables = torch.randint(-6, 7, (nq, dim // 2, 16), generator=g).float() / 4
    codes = torch.randint(0, 256, (n, dim // 4), generator=g, dtype=torch.int64).to(torch.uint8)
    off = _layout(n, nlist, seed=seed)
    probes = _probe_table(nq, nprobe, nlist, g)
    bias = torch.randint(-8, 9, (nq, nprobe), generator=g).float() / 2
    return tables, codes, off, probes, bias


@pytest.mark.parametrize("case", [(64, 1, 5000, 3, 200, 4000), (64, 100, 1, 8, 50, 6000), (128, 100, 64, 16, 40, 12000),
                                  (128, 1024, 8, 5, 30, 3000), (768, 100, 32, 8, 20, 6000), (768, 1024, 16, 4, 10, 8000),
                                  (768, 1, 24, 6, 12, 2000), (128, 1024, 20, 2, 400, 3000)])
def test_scan_matches_oracle_bit_for_bit(case):
    """Dyadic tables and biases: every sum is exact in fp32 whatever its order, and integer-valued scores tie a lot, so
    the shortlist (scores and positions under (score desc, position asc)) must equal the oracle's exactly.  Leaf 0 is
    empty, leaf 1 holds one row and leaf 2 half the rows (longer than kr); probes are distinct within a row and some
    are -1.  In the last case most queries probe fewer than kr rows, so the (-3.4028235e38, -1) tail is compared too."""
    dim, kr, nq, nprobe, nlist, n = case
    tables, codes, off, probes, bias = _scan_inputs(dim, nq, nprobe, nlist, n, seed=dim + kr + nq)
    for row in probes:
        live = row[row >= 0]
        assert live.unique().numel() == live.numel()
    max_len = int((off[1:] - off[:-1]).max())
    s, p = interaction.ah_search(tables.to(DEV), codes.to(DEV), off.to(DEV), probes.to(DEV), bias.to(DEV), kr, max_len)
    rs, rp = A.scan(tables, codes, off, probes, bias, kr)
    if case[-3:] == (2, 400, 3000):
        assert bool((rp == -1).any())
    assert torch.equal(p.cpu(), rp)
    assert torch.equal(s.cpu().double(), rs)


def test_scan_with_an_understated_max_list_len_keeps_each_slot_full():
    """max_list_len 40 gives slots of 64 entries, while the leaves hold about 190 rows (one 1 500): every (query, probe)
    keeps its 64 best rows, and the query's shortlist is the best kr of those."""
    dim, kr, nq, nprobe, nlist, n = 64, 100, 12, 4, 10, 3000
    tables, codes, off, probes, bias = _scan_inputs(dim, nq, nprobe, nlist, n, seed=8)
    s, p = interaction.ah_search(tables.to(DEV), codes.to(DEV), off.to(DEV), probes.to(DEV), bias.to(DEV), kr, 40)
    rs, rp = A.scan_slots(tables, codes, off, probes, bias, kr, 64)
    assert torch.equal(p.cpu(), rp)
    assert torch.equal(s.cpu().double(), rs)


def test_scan_query_batching_is_exact(monkeypatch):
    dim, kr, nq, nprobe, nlist, n = 64, 50, 300, 6, 40, 5000
    g = torch.Generator().manual_seed(5)
    tables = (torch.randint(-6, 7, (nq, dim // 2, 16), generator=g).float() / 4).to(DEV)
    codes = torch.randint(0, 256, (n, dim // 4), generator=g, dtype=torch.int64).to(torch.uint8).to(DEV)
    off = _layout(n, nlist, 1).to(DEV)
    probes = torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(nq)]).to(DEV)
    bias = torch.zeros(nq, nprobe, device=DEV)
    whole = interaction.ah_search(tables, codes, off, probes, bias, kr, n)
    monkeypatch.setattr(interaction, "AH_WORKSPACE_CAP", 1 << 20)
    parts = interaction.ah_search(tables, codes, off, probes, bias, kr, n)
    assert torch.equal(whole[0], parts[0]) and torch.equal(whole[1], parts[1])


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("dim,kr,top_n", [(64, 100, 10), (128, 1024, 1000), (768, 300, 100)])
def test_reorder_matches_oracle_bit_for_bit(dtype, dim, kr, top_n):
    """Integer-valued rows and queries: every product and sum is exact, so scores and the (score desc, id asc) order
    must equal the oracle's; shortlists hold void entries, and ids do not follow positions."""
    n, nq = 3000, 20
    g = torch.Generator().manual_seed(dim + kr)
    rows = torch.randint(-3, 4, (n, dim), generator=g).to(dtype)
    q = torch.randint(-3, 4, (nq, dim), generator=g).to(dtype)
    ids = torch.randperm(n, generator=g) * 5 - 7000
    sl = torch.stack([torch.randperm(n, generator=g)[:kr] for _ in range(nq)])
    sl[1, kr // 2:] = -1
    sl[2, :] = -1
    sl[3, 1:] = -1
    s, i = interaction.ah_reorder(q.to(DEV), rows.to(DEV), ids.to(DEV), sl.to(DEV), top_n)
    rs, ri = A.reorder(q, rows, ids, sl, top_n)
    assert torch.equal(i.cpu(), ri)
    assert torch.equal(s.cpu().double(), rs)


def test_search_rejects_sizes_outside_the_envelope():
    codes = torch.zeros(10, 24, dtype=torch.uint8, device=DEV)          # dim 96
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.ah_search(torch.zeros(1, 48, 16, device=DEV), codes, torch.tensor([0, 10], device=DEV),
                              torch.zeros(1, 1, dtype=torch.int64, device=DEV), torch.zeros(1, 1, device=DEV), 10, 10)
    codes = torch.zeros(10, 16, dtype=torch.uint8, device=DEV)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.ah_search(torch.zeros(1, 32, 16, device=DEV), codes, torch.tensor([0, 10], device=DEV),
                              torch.zeros(1, 1, dtype=torch.int64, device=DEV), torch.zeros(1, 1, device=DEV), 1025, 10)
    with pytest.raises(_lib.MatchmakerB200Error, match="top_n"):
        ScaNNIndexer(_cfg(top_n=2000))


def _train(x, dim, dtype="float16"):
    idx = ScaNNIndexer(_cfg(dtype, dim=dim))
    idx.index([np.arange(x.shape[0])], [x.numpy()])
    return idx


def test_training_is_monotone_deterministic_and_anisotropic():
    x, _ = _clustered(20000, 128, 40, seed=1)
    a, b = _train(x, 128), _train(x, 128)
    assert len(a.train_loss) == S.AH_ROUNDS + 1
    assert all(l1 <= l0 * (1 + 1e-12) for l0, l1 in zip(a.train_loss, a.train_loss[1:])), a.train_loss
    assert torch.equal(a.ivf.centroids, b.ivf.centroids) and torch.equal(a.codebook, b.codebook)
    assert torch.equal(a.codes, b.codes) and torch.equal(a.ids, b.ids)
    # the error along the data point, (e . x/|x|)^2, is smaller with the anisotropic codebook and codes than with the
    # isotropic start
    xs = a.rows.float()
    leaf = torch.repeat_interleave(torch.arange(a.nlist, device=DEV), a.list_offsets[1:] - a.list_offsets[:-1])
    r = xs - a.ivf.centroids[leaf]
    xh = S.unit_rows(xs)
    iso = a.codebook_iso
    e_iso = r.double() - S.decode(iso, S.nearest_codes(r, iso))
    e_ah = r.double() - S.decode(a.codebook.double(), S.unpack_codes(a.codes))
    par_iso, par_ah = ((e_iso * xh).sum(1) ** 2).mean(), ((e_ah * xh).sum(1) ** 2).mean()
    assert par_ah < par_iso, (float(par_ah), float(par_iso))


@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_full_probe_with_a_shortlist_of_every_row_equals_the_flat_index(dtype):
    """n = 1000 rows: 31 leaves, all probed; kr = 1000 shortlists every row, so the reorder ranks the whole set.
    Integer-valued data keeps both indexes' scores exact."""
    g = torch.Generator().manual_seed(2)
    x = torch.randint(-3, 4, (1000, 64), generator=g).float()
    q = torch.randint(-3, 4, (40, 64), generator=g).float()
    ids = np.arange(1000, dtype=np.int64) * 3 - 500
    idx = ScaNNIndexer(_cfg(dtype, hit=1000))
    idx.index([ids], [x.numpy()])
    assert idx.nlist == 31 and idx.nprobe == 31
    flat = FlatIPIndexer({"token_dim": 64, "faiss_use_gpu": True, "token_dtype": dtype})
    flat.index([ids], [x.numpy()])
    s, i = idx.search(q.numpy(), 100)
    fs, fi = flat.search(q.numpy(), 100)
    assert np.array_equal(i, fi) and np.array_equal(s, fs)


def _recall(got, exact):
    return float(np.mean([len(set(a) & set(b)) / len(b) for a, b in zip(got.tolist(), exact.tolist())]))


def test_recall_does_not_fall_as_nprobe_or_the_shortlist_grow():
    """Unclustered rows, so a query's neighbours spread over many leaves."""
    g = torch.Generator().manual_seed(3)
    x, q = torch.randn(40000, 128, generator=g).half(), torch.randn(200, 128, generator=g).half()
    ids = np.arange(40000, dtype=np.int64)
    idx = ScaNNIndexer(_cfg(dim=128, top_n=10, hit=100))
    idx.index([ids], [x.numpy()])
    flat = FlatIPIndexer({"token_dim": 128, "faiss_use_gpu": True, "token_dtype": "float16"})
    flat.index([ids], [x.numpy()])
    _, exact = flat.search(q.numpy(), 10)
    by_probe = []
    for nprobe in (1, 4, 16, 64, idx.nlist):
        idx.nprobe = nprobe
        by_probe.append(_recall(idx.search(q.numpy(), 10)[1], exact))
    assert all(b >= a for a, b in zip(by_probe, by_probe[1:])) and by_probe[-1] > by_probe[0], by_probe
    idx.nprobe = 16
    by_kr = []
    for kr in (10, 40, 160, 640):
        idx.top_n = kr
        by_kr.append(_recall(idx.search(q.numpy(), 10)[1], exact))
    assert all(b >= a for a, b in zip(by_kr, by_kr[1:])) and by_kr[-1] > by_kr[0], by_kr


@pytest.mark.parametrize("n,hit", [(8000, 100), (1000, 1000)])
def test_two_shards_sharing_the_training_merge_to_the_whole_index(n, hit):
    """Every row gets the same code in a shard as in the whole index.  Each shard shortlists its own kr best rows, a
    superset of its share of the whole index's shortlist, so the merged result is never worse rank by rank; with a
    shortlist of every row (n = kr = 1000) it is the same result."""
    x, q = _clustered(n, 64, 30, seed=4)
    ids = torch.arange(n) * 3 - 100
    whole = ScaNNIndexer(_cfg(hit=hit))
    whole.index([ids.numpy()], [x.numpy()])
    code_of = dict(zip(whole.ids.tolist(), whole.codes.cpu()))
    parts = []
    for lo, hi in ((0, n // 2), (n // 2, n)):
        p = ScaNNIndexer(_cfg(hit=hit))
        p._leaves(whole.nlist, whole.nprobe)
        p.ivf.set_centroids(whole.ivf.centroids)
        p.codebook = whole.codebook
        p.add(x[lo:hi].to(DEV), ids[lo:hi].to(DEV))
        assert all(torch.equal(code_of[i], c) for i, c in zip(p.ids.tolist(), p.codes.cpu()))
        parts.append(p.search_device(q.to(DEV), 100))
    s, i = interaction.topk_merge(torch.cat([parts[0][0], parts[1][0]], 1), torch.cat([parts[0][1], parts[1][1]], 1), 100)
    ws, wi = whole.search_device(q.to(DEV), 100)
    assert torch.all(s >= ws)
    if hit >= n:
        assert torch.equal(i, wi) and torch.equal(s, ws)


def test_drop_in_sequence_of_dense_retrieval(tmp_path):
    """prepare (a no-op), index, save into a directory created beforehand, load(path), search -- with the reference's
    config shape (faiss_use_gpu False, query sets with index_hit_top_n)."""
    x, q = _clustered(5000, 64, 20, seed=5)
    ids = np.arange(5000, dtype=np.int64) * 2 - 3000
    cfg = _cfg(top_n=10, hit=50)
    cfg["query_sets"]["other"] = {"top_n": 7}
    idx = ScaNNIndexer(cfg)
    assert idx.top_n == 50
    idx.prepare([x[:2500].numpy(), x[2500:].numpy()])
    idx.index([ids[:2500], ids[2500:]], [x[:2500].numpy(), x[2500:].numpy()])
    s, i = idx.search(q.numpy(), 10)
    assert isinstance(s, np.ndarray) and s.dtype == np.float32 and i.dtype == np.int64 and s.shape == (64, 10)
    s1, i1 = idx.search(q[3].numpy(), 10)
    assert np.array_equal(i1[0], i[3])
    path = tmp_path / "scann-index"
    os.makedirs(path)
    idx.save(str(path))
    assert sum(os.path.getsize(f) for f in path.iterdir()) > 0
    back = ScaNNIndexer(cfg)
    back.load(str(path))
    s2, i2 = back.search(q.numpy(), 10)
    assert np.array_equal(s2, s) and np.array_equal(i2, i)
    with pytest.raises(_lib.MatchmakerB200Error):
        ScaNNIndexer(_cfg("float32", top_n=10)).load(str(path))
    os.rename(path / "rank0of1.pt", path / "rank0of2.pt")
    with pytest.raises(_lib.MatchmakerB200Error):
        ScaNNIndexer(cfg).load(str(path))


def test_search_unique_matches_the_maxp_loop():
    x, q = _clustered(4000, 64, 20, seed=6, nq=8)
    ids = (np.arange(4000) // 4).astype(np.int64)
    idx = ScaNNIndexer(_cfg(top_n=10, hit=200))
    idx.index([ids], [x.numpy()])
    s, i = idx.search_unique(q.numpy(), 10, 200)
    hs, hi = idx.search(q.numpy(), 200)
    loop = E.maxp_loop(hs, hi, 10)
    for a in range(8):
        assert [int(v) for v in i[a, :len(loop[a])]] == [int(p) for p, _ in loop[a]]


def test_search_device_replays_in_a_cuda_graph():
    x, q = _clustered(6000, 64, 20, seed=7)
    idx = ScaNNIndexer(_cfg())
    idx.index([np.arange(6000)], [x.numpy()])
    qd = q.to(DEV)
    ref_s, ref_i = idx.search_device(qd, 100)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gs, gi = idx.search_device(qd, 100)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(gs, ref_s) and torch.equal(gi, ref_i)


def test_ptxas_reports_no_spills_in_the_scan_kernel(tmp_path):
    from matchmaker_b200 import build
    src = os.path.join(ROOT, "matchmaker_b200", "csrc", "ah.cu")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "ah.o")],
                       capture_output=True, text=True, check=True)
    m = re.search(r"Function properties for \S*ah_scan_kernel\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", r.stderr)
    assert m, r.stderr[-2000:]
    assert m.groups() == ("0", "0", "0")


def test_add_memory_is_bounded_by_the_chunk_not_by_n(monkeypatch):
    """Coding 400 000 rows of dim 256 takes the stored index (the sorted rows, codes, ids), the leaf ids and their sort
    (at most 128 B per row here) and scratch bounded by _CHUNK rows -- not fp32 / fp64 copies of the whole shard, which
    would be more than 4 GB."""
    dim, n, chunk = 256, 400_000, 4096
    x, _ = _clustered(20000, dim, 20, seed=9)
    idx = ScaNNIndexer(_cfg(dim=dim))
    idx.index([np.arange(20000)], [x.numpy()])
    monkeypatch.setattr(S, "_CHUNK", chunk)
    big = torch.randn(n, dim, generator=torch.Generator(device=DEV).manual_seed(0), device=DEV).half()
    ids = torch.arange(n, device=DEV)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx.add(big, ids)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    stored = n * dim * 2 + n * dim // 4 + n * 8
    scratch = chunk * dim * 8 * 40 + (256 << 20)     # fp64 coding temporaries of one chunk, the coarse search's lists
    assert peak <= stored + 128 * n + scratch, (peak, stored, scratch)
    assert idx.codes.shape == (n, dim // 4) and int(idx.list_offsets[-1]) == n
