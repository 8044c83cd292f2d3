"""TKL store without a GPU: the encode folder round trip, refused folders, the chunk-slot count, passage shards and the
rank merge under gloo with void pairs, and the store-mode kernels in the library's SASS."""
import os
import re
import shutil
import socket
import subprocess

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from matchmaker_b200 import _lib, sharding
from matchmaker_b200.rankers.tkl import chunk_documents, chunk_slots
from matchmaker_b200.retrieval.colbert_e2e import doc_offsets_from_id_mapping
from matchmaker_b200.retrieval.tk_store import local_pairs, merge
from matchmaker_b200.retrieval.tkl_store import CHUNK_FILE, TKLStoreWriter, load_chunk_meta, void_pairs
from matchmaker_b200.retrieval.token_storage import TokenStorageWriter, load_token_storage

DIM = 8


def _passages(rng):
    """Passages with 0, 1, 2, 3, 4, 7 and 50 packed chunks on increasing slots with gaps (dropped middle chunks), a
    partly masked last chunk, and an empty last passage."""
    out = []
    for n in [3, 0, 1, 50, 2, 4, 7, 0]:
        slots = np.sort(rng.choice(50, size=n, replace=False)) if n < 50 else np.arange(50)
        mask = np.ones((n, 40), dtype=np.uint8)
        if n:
            mask[-1, 17:] = 0
        chunks = rng.standard_normal((n, 40, DIM)).astype(np.float32)
        out.append((chunks, mask, slots))
    return out


def test_writer_loader_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    ps = _passages(rng)
    w = TKLStoreWriter(str(tmp_path), DIM, 2000)
    for i, (c, m, s) in enumerate(ps):
        w.add(str(i), c, m, s)
    w.close()
    assert sorted(f for f in os.listdir(tmp_path) if f.startswith("tkl_chunks_")) == \
        [CHUNK_FILE.format(i) for i in range(len(w.storage))]
    storage, idm, seq_ids, infos = load_token_storage(str(tmp_path), DIM, 2000, "float32")
    assert len(storage) > 1 and seq_ids == [str(i) for i in range(len(ps))]
    meta = load_chunk_meta(str(tmp_path), 2000, storage)
    rows = np.concatenate(storage)
    rec = np.concatenate(meta)
    off = doc_offsets_from_id_mapping(idm)
    assert len(off) - 1 == len(ps) - 1          # the empty last passage has no row, so no offset
    for i, (c, m, s) in enumerate(ps):
        b, lo, hi = infos[str(i)]
        assert hi - lo == 40 * len(c)
        if i < len(off) - 1:
            assert off[i + 1] - off[i] == 40 * len(c)
        r = storage[b][lo:hi]
        np.testing.assert_array_equal(r, (c * m[..., None]).reshape(-1, DIM))   # masked rows stored as zeros
        mb = meta[b][lo // 40:hi // 40]
        np.testing.assert_array_equal(mb["mask"], m)
        np.testing.assert_array_equal(mb["slot"], s)
    assert len(rows) == 40 * len(rec)


def test_bad_folders_are_refused(tmp_path):
    with pytest.raises(_lib.MatchmakerB200Error, match="% 40"):
        TKLStoreWriter(str(tmp_path / "a"), DIM, 1000 + 20)
    plain = tmp_path / "b"
    w = TokenStorageWriter(str(plain), DIM, 400, "float32")
    w.add("0", np.ones((40, DIM), dtype=np.float32))
    w.close()
    storage = load_token_storage(str(plain), DIM, 400, "float32")[0]
    with pytest.raises(_lib.MatchmakerB200Error, match="not a TKL store"):
        load_chunk_meta(str(plain), 400, storage)
    with pytest.raises(_lib.MatchmakerB200Error, match="% 40"):
        load_chunk_meta(str(plain), 410, storage)
    w = TKLStoreWriter(str(tmp_path / "c"), DIM, 400)
    with pytest.raises(_lib.MatchmakerB200Error, match="increasing"):
        w.add("0", np.ones((2, 40, DIM)), np.ones((2, 40)), np.array([3, 3]))
    with pytest.raises(_lib.MatchmakerB200Error, match="do not fit"):
        w.add("0", np.ones((11, 40, DIM)), np.ones((11, 40)), np.arange(11))


def test_chunk_slots_is_the_packing_piece_count():
    for L in [1, 5, 6, 44, 45, 46, 400, 1100, 1999, 2000]:
        assert chunk_slots(L) == chunk_documents(torch.zeros(1, L, 4), torch.ones(1, L))[3]
    assert chunk_slots(2000) == 50


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
        has_chunks = torch.from_numpy(np.diff(off[d_lo:d_hi + 1]) > 0)
        live = (pair_d >= 0) & has_chunks[pair_d.clamp(min=0)] if d_hi > d_lo else torch.zeros_like(pair_d, dtype=bool)
        s, i = void_pairs(full_scores, ids, live.view(cand.shape))
        out[rank] = merge(s, i, k) + ((d_lo, d_hi),)
    finally:
        dist.destroy_process_group()


def test_passage_shards_void_pairs_and_merge_under_gloo():
    # row offsets in whole 40-row chunks; passages 1 and 4 have no chunk, passage 7 (past the offsets) is the empty last
    off = 40 * np.array([0, 3, 3, 10, 12, 12, 21, 30], dtype=np.int64)
    world = 2
    cand = torch.tensor([[6, 0, -1, 3, 1, 5, 7], [2, 4, -1, -1, 5, 0, 6]], dtype=torch.int64)
    g = torch.Generator().manual_seed(0)
    full = torch.randn(cand.shape, generator=g)
    full[1, 4] = full[1, 5] = 0.25                     # a tie broken by id
    k = 6
    with mp.Manager() as mgr:
        out = mgr.dict()
        mp.spawn(_rank_main, args=(world, _free_port(), off, cand, full, k, out), nprocs=world, join=True)
        res = dict(out)
    assert res[0][2][1] == res[1][2][0] and res[1][2][1] == len(off) - 1
    live_docs = {d for d in range(len(off) - 1) if off[d + 1] > off[d]}
    for r in range(cand.shape[0]):
        items = [(float(full[r, j]), int(cand[r, j])) for j in range(cand.shape[1]) if int(cand[r, j]) in live_docs]
        items += [(float("-inf"), -1)] * (world * cand.shape[1])
        items.sort(key=lambda x: (-x[0], x[1]))
        for rank in range(world):
            s, i, _ = res[rank]
            assert [(float(a), int(b)) for a, b in zip(s[r], i[r])] == items[:k], (rank, r)


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def sass():
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump unavailable: {e}")
    if out.returncode != 0:
        pytest.skip("cuobjdump failed: " + out.stderr[-200:])
    funcs, name = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


def _local(text):
    return [l for l in text.splitlines() if re.search(r"\b(LDL|STL)(\.\S+)?\b", l)]


def test_store_mode_instantiations_in_the_library(sass):
    ts = {k: v for k, v in sass.items() if "tkl_ts_kernel" in k}
    store_ts = {k: v for k, v in ts.items() if re.search(r"tkl_ts_kernelILi\dELb1E", k)}
    assert {re.search(r"ILi(\d)E", k).group(1) for k in store_ts} == {"0", "1"}
    ffma = {k: v for k, v in sass.items() if re.search(r"tkl_window_kernelILi(12|16)ELb0ELb1E", k)}
    assert {re.search(r"ILi(\d+)E", k).group(1) for k in ffma} == {"12", "16"}
    plan = {k: v for k, v in sass.items() if "tkl_plan_store_kernel" in k}
    assert len(plan) == 1
    # the FFMA and plan store kernels touch no local memory
    for name, text in list(ffma.items()) + list(plan.items()):
        assert not _local(text), f"{name}: local-memory traffic in the SASS: {_local(text)[:3]}"
    # the tensor-core store kernels are TMA-fed wgmma kernels and spill no more than their padded instantiation (the
    # embedding-saturation kernel at 80 registers already keeps a few values in local memory)
    for name, text in store_ts.items():
        assert "UTMALDG" in text and "HGMMA" in text, name
        sat = re.search(r"ILi(\d)E", name).group(1)
        padded = [v for k, v in ts.items() if re.search(rf"tkl_ts_kernelILi{sat}ELb0E", k)]
        assert len(padded) == 1 and len(_local(text)) <= len(_local(padded[0])), name
