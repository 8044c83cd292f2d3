"""Residual token codes without a GPU: the numpy format's packing and bucket properties, the four C entry points, the
indexer's construction envelope, and the compiled residual kernels (wgmma, mbarrier waits, TMA query loads, spills)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import colbert_residual_oracle as R
from matchmaker_b200 import _lib, build


@pytest.mark.parametrize("bits", [1, 2])
def test_pack_puts_dimension_d_at_its_bit_position(bits):
    dim = 64
    for d in (0, 1, 5, 7, 8, 33, 63):
        c = np.zeros((1, dim), dtype=np.uint8)
        c[0, d] = (1 << bits) - 1
        p = R.pack(c, bits)
        assert p.shape == (1, dim * bits // 8)
        byte, shift = d * bits // 8, bits * (d % (8 // bits))
        expect = np.zeros_like(p)
        expect[0, byte] = ((1 << bits) - 1) << shift
        assert np.array_equal(p, expect)
        assert np.array_equal(R.unpack(p, bits, dim), c)


@pytest.mark.parametrize("bits,dim", [(1, 64), (2, 128), (2, 768), (1, 768)])
def test_codes_are_in_range_and_decode_into_their_bucket(bits, dim):
    rows, lids, base, cutoff, weight = R.synth(600, dim, 7, bits, seed=dim + bits)
    c = R.codes(rows, lids, base, cutoff)
    assert c.max() < (1 << bits)
    assert np.array_equal(R.unpack(R.encode(rows, lids, base, cutoff, bits), bits, dim), c)
    r = R.residuals(rows, lids, base)
    lo = np.concatenate([np.full((dim, 1), -np.inf, np.float32), cutoff], axis=1)
    hi = np.concatenate([cutoff, np.full((dim, 1), np.inf, np.float32)], axis=1)
    d = np.arange(dim)[None, :]
    assert (lo[d, c] <= r).all() and (r < hi[d, c]).all()
    # a residual exactly on a cutoff counts that cutoff
    z = np.nonzero(lids == 0)[0][0]
    assert (c[z] >= 1).all()
    # quantile weights lie in their own bucket, so the decoded value does too (up to the fp16 roundings)
    w = weight.astype(np.float32)
    assert (w >= lo - 1e-2 * np.abs(lo).clip(1)).all() and (w <= hi + 1e-2 * np.abs(hi).clip(1)).all()
    dec = R.decode(R.encode(rows, lids, base, cutoff, bits), lids, base, weight, bits)
    assert dec.dtype == np.float16 and dec.shape == rows.shape


def test_library_exports_the_residual_entry_points():
    for name in ("mmb200_residual_encode", "mmb200_residual_decode", "mmb200_ivf_search_residual",
                 "mmb200_maxsim_store_residual_fwd"):
        assert name in _lib.SIGNATURES
        assert hasattr(_lib.load(), name)


def test_indexer_rejects_configurations_outside_the_envelope():
    torch = pytest.importorskip("torch")
    from matchmaker_b200.retrieval import ColBERTResidualIndexer
    base = {"token_dim": 128, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": 8,
            "faiss_ivf_search_probe_count": 2, "colbert_residual_bits": 2}
    for bad in ({"colbert_residual_bits": 3}, {"colbert_residual_bits": 0}, {"token_dtype": "float32"},
                {"token_dim": 96}, {"token_dim": 1088}):
        with pytest.raises(_lib.MatchmakerB200Error):
            ColBERTResidualIndexer({**base, **bad}, device=torch.device("cpu"))


def _ptxas(src):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", os.devnull],
                       capture_output=True, text=True, check=True)
    return dict(re.findall(r"Compiling entry function '(\S+)'.*?\n\s*(\d+ bytes stack frame.*?)\n", r.stderr, re.S))


def _spill_stores(line):
    return int(re.search(r"(\d+) bytes spill stores", line).group(1))


def test_residual_kernels_do_not_add_spills():
    """The max-sim over codes does not spill.  The scan's consumers are the gather scan's: the residual scan spills no
    more than the gather kernel of the same list capacity, up to one spilled loop counter (16 bytes)."""
    ms = {k: v for k, v in _ptxas("maxsim.cu").items() if "maxsim_tc_residual_kernel" in k}
    assert len(ms) == 16, list(ms)
    for name, line in ms.items():
        assert "0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
    fi = _ptxas("flat_ip.cu")
    for epl in (32, 64):
        gather = [v for k, v in fi.items() if f"flat_ip_tc_gather_kernelI6__halfLi{epl}E" in k]
        resid = [v for k, v in fi.items() if f"flat_ip_tc_residual_kernelILi{epl}E" in k]
        assert len(gather) == 1 and len(resid) == 2, (epl, list(fi))
        for line in resid:
            assert _spill_stores(line) <= _spill_stores(gather[0]) + 16, (epl, line, gather[0])


@pytest.fixture(scope="module")
def sass():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        out = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump unavailable: {e}")
    funcs, name = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


@pytest.mark.parametrize("needle,count", [("flat_ip_tc_residual_kernel", 4), ("maxsim_tc_residual_kernel", 16)])
def test_residual_kernels_are_wgmma_kernels_with_tma_queries(sass, needle, count):
    ks = {k: v for k, v in sass.items() if needle in k}
    assert len(ks) == count, list(ks)
    for name, text in ks.items():
        assert any("HGMMA" in l and "gdesc[URZ]" not in l for l in text.splitlines()), f"{name}: no wgmma"
        assert "SYNCS.PHASECHK" in text, f"{name}: no mbarrier wait"
        assert "UTMALDG" in text, f"{name}: the query tiles are not loaded by TMA"
        assert "LDGSTS" not in text, f"{name}: the passage tile is decoded, not copied"


@pytest.mark.parametrize("chunk", [5, 64, 1 << 16])
def test_list_means_are_sequential_fp64_sums_of_whole_lists(chunk, monkeypatch):
    """The bases: per list, the fp64 sum of its rows in ascending row order over the count, cast to fp16, whatever the
    host chunking (chunks smaller than a list included); an empty list gives zeros."""
    torch = pytest.importorskip("torch")
    from matchmaker_b200.retrieval import colbert_residual
    monkeypatch.setattr(colbert_residual, "MEAN_CHUNK_ROWS", chunk)
    rng = np.random.default_rng(chunk)
    nlist, n, dim = 9, 700, 64
    a = rng.integers(0, nlist - 1, n)          # list nlist - 1 stays empty
    a[:300] = 3                                # one list larger than the small chunks
    x = (rng.standard_normal((n, dim)) * 50).astype(np.float16)
    got = colbert_residual.list_means_f16(torch.from_numpy(x), torch.from_numpy(a), nlist)
    ref = np.zeros((nlist, dim), dtype=np.float16)
    for l in range(nlist):
        s = np.zeros(dim, dtype=np.float64)
        rows = np.nonzero(a == l)[0]
        for r in rows:
            s += x[r].astype(np.float64)
        ref[l] = (s / max(1, len(rows))).astype(np.float16)
    assert np.array_equal(got.view(np.int16), ref.view(np.int16))
    assert not got[nlist - 1].any()


def _residual_file(dim=64, bits=2, nlist=4, world=1, rank=0):
    """A residual index file as the format was first written: three passages of 2, 0 and 3 rows from passage 7 on."""
    torch = pytest.importorskip("torch")
    g = torch.Generator().manual_seed(bits)
    n = 5
    return {"centroids": torch.nn.functional.normalize(torch.randn(nlist, dim, generator=g), dim=1),
            "base": torch.randn(nlist, dim, generator=g).half(), "weight": torch.randn(dim, 1 << bits, generator=g).half(),
            "cutoff": torch.randn(dim, (1 << bits) - 1, generator=g), "bits": bits, "dim": dim,
            "codes": torch.randint(0, 256, (n, dim * bits // 8), generator=g, dtype=torch.uint8),
            "list_ids": torch.tensor([0, 2, 2, 3, 0], dtype=torch.int32), "row_index": torch.tensor([0, 4, 1, 2, 3]),
            "list_offsets": torch.tensor([0, 2, 2, 4, 5]), "offsets": torch.tensor([0, 2, 2, 5]), "d_lo": 7,
            "n_docs": 12, "nlist": nlist, "nprobe": 2, "rank": rank, "world": world}


def test_residual_file_loads_and_saves_in_its_format(tmp_path):
    torch = pytest.importorskip("torch")
    from matchmaker_b200.retrieval import ColBERTResidualIndexer
    cfg = {"token_dim": 64, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": 4,
           "faiss_ivf_search_probe_count": 1, "colbert_residual_bits": 2}
    blob = _residual_file()
    path = str(tmp_path / "res.pt")
    torch.save(blob, path)
    idx = ColBERTResidualIndexer(cfg, device=torch.device("cpu"))
    idx.load(path)
    for name, got in (("codes", idx.store), ("list_ids", idx.list_ids), ("base", idx.base), ("weight", idx.weight),
                      ("cutoff", idx.cutoff), ("row_index", idx.row_index), ("list_offsets", idx.list_offsets),
                      ("offsets", idx.offsets)):
        assert torch.equal(got, blob[name]), name
    assert torch.equal(idx.row_ids, torch.tensor([7, 7, 9, 9, 9]))
    assert (idx.d_lo, idx.d_hi, idx.n_docs, idx.max_doc_len, idx.max_list_len, idx.nprobe) == (7, 10, 12, 3, 2, 2)
    idx.save(str(tmp_path / "again.pt"))
    again = torch.load(str(tmp_path / "again.pt"))
    assert again.keys() == blob.keys()
    for k in blob:
        assert torch.equal(again[k], blob[k]) if isinstance(blob[k], torch.Tensor) else again[k] == blob[k], k
    for bad in (_residual_file(bits=1), _residual_file(dim=128)):
        torch.save(bad, path)
        with pytest.raises(_lib.MatchmakerB200Error, match="codes"):
            ColBERTResidualIndexer(cfg, device=torch.device("cpu")).load(path)
    torch.save(_residual_file(world=2), path)
    with pytest.raises(_lib.MatchmakerB200Error, match="world size"):
        ColBERTResidualIndexer(cfg, device=torch.device("cpu")).load(path)
