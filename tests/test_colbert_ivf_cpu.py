"""Host-side pieces of the IVF token index for ColBERT retrieval (retrieval.ColBERTIVFIndexer): the list layout, the
fingerprint checks of load(), the stage-1 oracle against a plain loop, and the binding of the gather scan."""
import numpy as np
import pytest
import torch

import colbert_ivf_oracle as CV
from matchmaker_b200 import _lib
from matchmaker_b200.retrieval import ColBERTIVFIndexer

CPU = torch.device("cpu")


def _cfg(dim=64, nlist=8, nprobe=2, dtype="float16"):
    return {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": dtype, "faiss_ivf_list_count": nlist,
            "faiss_ivf_search_probe_count": nprobe}


def test_layout_from_an_assignment_keeps_store_order_within_lists():
    g = torch.Generator().manual_seed(1)
    nlist = 9
    assign = torch.randint(0, nlist, (500,), generator=g)
    assign[assign == 4] = 5                       # list 4 empty
    idx = ColBERTIVFIndexer(_cfg(nlist=nlist), device=CPU)
    row_index, off = idx.ivf._layout(assign)
    ref_rows, ref_off = CV.layout(assign, nlist)
    assert torch.equal(off, ref_off) and torch.equal(row_index, ref_rows)
    assert int(off[4]) == int(off[5])
    for l in range(nlist):
        seg = row_index[off[l]:off[l + 1]]
        assert bool((assign[seg] == l).all()) and bool((seg[1:] > seg[:-1]).all())
    assert torch.equal(torch.sort(row_index).values, torch.arange(500))


def _saved(tmp_path, world=1, rank=0, dtype="torch.float16", n_rows=40, d_lo=0, d_hi=5, nlist=8, dim=64):
    path = str(tmp_path / "tok.ivf")
    torch.save({"centroids": torch.nn.functional.normalize(torch.randn(nlist, dim), dim=1),
                "row_index": torch.arange(n_rows), "list_offsets": torch.tensor([0] + [n_rows] * nlist),
                "nlist": nlist, "nprobe": 3, "token_dtype": dtype, "rank": rank,
                "fingerprint": {"n_rows": n_rows, "d_lo": d_lo, "d_hi": d_hi, "world": world}},
               path if world == 1 else f"{path}.rank{rank}of{world}")
    return path


def test_load_restores_the_quantizer_and_nprobe(tmp_path):
    path = _saved(tmp_path)
    idx = ColBERTIVFIndexer(_cfg(nprobe=2), device=CPU)
    idx.load(path)
    assert idx.nprobe == 3 and idx.nlist == 8 and idx.ivf.centroids.shape == (8, 64)
    idx.load(path, {"faiss_ivf_search_probe_count": 7})
    assert idx.nprobe == 7


def test_load_rejects_another_world_size_or_dtype(tmp_path):
    (tmp_path / "one").mkdir()
    path = _saved(tmp_path / "one", world=1)
    idx = ColBERTIVFIndexer(_cfg(), device=CPU)
    idx._world = lambda: (1, 2)
    with pytest.raises(_lib.MatchmakerB200Error, match="world size"):
        idx.load(path)                         # saved by one rank, loaded by rank 1 of 2
    bad = _saved(tmp_path, world=2, rank=0)
    torch.save(torch.load(f"{bad}.rank0of2"), bad)   # a two-rank shard under the one-rank name
    with pytest.raises(_lib.MatchmakerB200Error, match="world size"):
        ColBERTIVFIndexer(_cfg(), device=CPU).load(bad)
    idx = ColBERTIVFIndexer(_cfg(), device=CPU)
    idx._world = lambda: (0, 2)
    idx.load(bad)                              # the same world size loads
    with pytest.raises(_lib.MatchmakerB200Error, match="token_dtype"):
        ColBERTIVFIndexer(_cfg(), device=CPU).load(_saved(tmp_path, dtype="torch.float32"))


@pytest.mark.parametrize("store_rows,d_lo,d_hi,ok", [(40, 0, 5, True), (41, 0, 5, False), (40, 1, 6, False)])
def test_a_loaded_layout_is_used_only_for_the_store_it_was_built_for(tmp_path, store_rows, d_lo, d_hi, ok):
    idx = ColBERTIVFIndexer(_cfg(), device=CPU)
    idx.load(_saved(tmp_path))
    idx.store = torch.zeros(store_rows, 64, dtype=torch.float16)
    idx.d_lo, idx.d_hi = d_lo, d_hi
    saved = idx._saved_layout
    if ok:
        idx._set_layout(saved[1], saved[2])
        assert idx.max_list_len == 40 and idx.row_index.numel() == 40
    else:
        with pytest.raises(_lib.MatchmakerB200Error, match="re-index"):
            idx._set_layout(saved[1], saved[2])


def _stage1_case(seed, nq=3, lq=6, n_rows=120, nlist=7, nprobe=3):
    g = torch.Generator().manual_seed(seed)
    scores = torch.randint(-6, 7, (nq, lq, n_rows), generator=g).float()      # many exact ties
    live = torch.ones(nq, lq, dtype=torch.bool)
    live[1, 4:] = False
    row_pid = torch.sort(torch.randint(0, 30, (n_rows,), generator=g)).values
    assign = torch.randint(0, nlist, (n_rows,), generator=g)
    probes = torch.stack([torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(lq)]) for _ in range(nq)])
    probes[0, 0, 1:] = -1                                                      # a token probing one list
    return scores, live, row_pid, assign, probes


@pytest.mark.parametrize("seed,kp,cap", [(0, 4, 4096), (1, 1, 4096), (2, 50, 4096), (3, 8, 5)])
def test_stage1_oracle_matches_a_plain_loop(seed, kp, cap):
    scores, live, row_pid, assign, probes = _stage1_case(seed)
    assert CV.candidates(scores, live, row_pid, assign, probes, kp, cap) == \
        CV.candidates_loop(scores, live, row_pid, assign, probes, kp, cap)


def test_stage1_oracle_uses_only_probed_lists_and_padding_probes_nothing():
    scores, live, row_pid, assign, probes = _stage1_case(5)
    got = CV.candidates(scores, live, row_pid, assign, probes, 1000, 4096)
    for a in range(scores.shape[0]):
        allowed = set()
        for t in range(scores.shape[1]):
            if live[a, t]:
                allowed |= set(row_pid[CV.probed_rows(assign, probes[a, t])].tolist())
        assert set(got[a]) == allowed        # k' above every list size: the whole probed union
    # a query whose tokens are all padding has no candidates, whatever its probes
    live[2] = False
    assert CV.candidates(scores, live, row_pid, assign, probes, 4, 4096)[2] == {}
    assert not bool(CV.probed_rows(assign, torch.tensor([-1, -1])).any())


def test_gather_scan_symbol_is_bound():
    assert "mmb200_ivf_search_gather" in _lib.SIGNATURES
    lib = _lib.load()
    assert lib.mmb200_ivf_search_gather.argtypes == _lib.SIGNATURES["mmb200_ivf_search_gather"][1]
    # a null row_index is refused before any device work
    rc = lib.mmb200_ivf_search_gather(*([None] * 9), 1, 1, 1, 1, 1, 1, 64, 1, _lib.F16, None)
    assert rc == _lib.ERR_INVALID


def test_index_before_prepare_raises():
    idx = ColBERTIVFIndexer(_cfg(), device=CPU)
    with pytest.raises(_lib.MatchmakerB200Error, match="centroids"):
        idx.index([np.zeros(3, dtype=np.int64)], [np.zeros((3, 64), dtype=np.float16)])


def _blobs_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]) if isinstance(a[k], torch.Tensor) else a[k] == b[k], k


def test_e4m3_layout_file_loads_and_saves_in_its_format(tmp_path):
    """An IVF token layout of an E4M3 store as the format was first written: it loads into an E4M3 indexer only, a
    re-index must reproduce its store scale, and a save of the same layout writes the same keys and values."""
    dim, nlist, n_rows = 128, 8, 40
    blob = {"centroids": torch.nn.functional.normalize(torch.randn(nlist, dim), dim=1),
            "row_index": torch.arange(n_rows), "list_offsets": torch.tensor([0] + [n_rows] * nlist), "nlist": nlist,
            "nprobe": 3, "token_dtype": "torch.float16", "store_dtype": "float8_e4m3", "store_scale": 5,
            "fingerprint": {"n_rows": n_rows, "d_lo": 0, "d_hi": 5, "world": 1}, "rank": 0}
    path = str(tmp_path / "fp8.ivf")
    torch.save(blob, path)
    fp8 = dict(_cfg(dim=dim), colbert_store_dtype="float8_e4m3")
    with pytest.raises(_lib.MatchmakerB200Error, match="colbert_store_dtype"):
        ColBERTIVFIndexer(_cfg(dim=dim), device=CPU).load(path)
    with pytest.raises(_lib.MatchmakerB200Error, match="colbert_store_dtype"):
        ColBERTIVFIndexer(fp8, device=CPU).load(_saved(tmp_path, dim=dim))     # an fp16 layout
    idx = ColBERTIVFIndexer(fp8, device=CPU)
    idx.load(path)
    assert idx.nprobe == 3 and idx.tokens.loaded_scale == 5
    # what index() leaves behind on the same store: its rows, passages and scale, and the loaded layout
    idx.store = torch.zeros(n_rows, dim, dtype=torch.float8_e4m3fn)
    idx.store_scale, idx.d_lo, idx.d_hi = 5, 0, 5
    idx._set_layout(*idx._saved_layout[1:])
    idx.save(str(tmp_path / "again.ivf"))
    _blobs_equal(torch.load(str(tmp_path / "again.ivf")), blob)
