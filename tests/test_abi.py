"""The C-ABI library builds, loads on a CPU-only box, exports every symbol the public header declares,
and fails loudly (no CPU fallback) when asked to compute without a GPU."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT
from matchmaker_b200 import _lib


def _header_symbols():
    syms = []
    inc = os.path.join(ROOT, "include")
    for f in sorted(os.listdir(inc)):
        if f.endswith(".h"):
            txt = open(os.path.join(inc, f)).read()
            syms += re.findall(r"MMB200_API\s+[\w\s\*]+?\b(mmb200_\w+)\s*\(", txt)
    return sorted(set(syms))


def test_library_is_built():
    assert os.path.isfile(_lib.LIB_PATH), "run `python -m matchmaker_b200.build` (or __graft_entry__.build())"


def test_exports_every_declared_symbol():
    syms = _header_symbols()
    assert len(syms) >= 6
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/ but not exported"
    assert sorted(_lib.SIGNATURES) == syms, "ctypes SIGNATURES out of sync with include/matchmaker_b200.h"


def test_version_and_error_string():
    lib = _lib.load()
    assert lib.mmb200_version() == 100
    assert isinstance(_lib.last_error(), str)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_fails_loudly_without_gpu():
    from matchmaker_b200 import interaction
    q = torch.zeros(1, 4, 64, dtype=torch.float16)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.maxsim(q, q)  # CPU tensors are rejected: there is no CPU fallback
    lib = _lib.load()
    rc = lib.mmb200_device_info(-1, None, None, None)
    assert rc == _lib.ERR_CUDA and "CUDA" in _lib.last_error()


@pytest.mark.parametrize("sm_count", [148, 132, 8, 1])
def test_flat_ip_plan_invariants(sm_count):
    """Host-side work decomposition of the exact top-k search (pure arithmetic, runs without a GPU): every passage tile
    belongs to exactly one range, the grid is a whole number of clusters that fits the device, query blocks are never
    dropped when clusters are formed, and the workspace covers thresholds, candidate lists and per-range candidates."""
    lib = _lib.load()
    out = (ctypes.c_int32 * 8)()
    for nq in (1, 127, 128, 129, 1300, 6400, 100000):
        for n_pass in (1, 255, 256, 257, 70000, 1100000, 8800000):
            for k in (1, 100, 256, 257, 1000, 1024):
                assert lib.mmb200_flat_ip_plan(nq, n_pass, k, sm_count, out) == _lib.OK, _lib.last_error()
                n_qb, n_tiles, n_ranges, tpr, grid, cl, ws_lo, ws_hi = [int(v) for v in out]
                ws = (ws_lo & 0xffffffff) | ((ws_hi & 0xffffffff) << 32)
                assert n_qb == (nq + 127) // 128 and n_tiles == (n_pass + 127) // 128   # 128 x 128 score tiles
                assert 1 <= n_ranges <= 32 and n_ranges * tpr >= n_tiles and (n_ranges - 1) * tpr < n_tiles
                assert cl in (1, 2, 4) and grid >= cl and grid % cl == 0 and grid <= max(cl, sm_count)
                n_groups = (n_qb + cl - 1) // cl
                assert grid <= cl * n_groups * n_ranges          # no CTA without a work item
                cap = 1024 if k <= 256 else 2048
                assert ws >= nq * 4 + grid * 128 * cap * 8       # thresholds + one candidate list per row per CTA
                kpad = (k + 31) // 32 * 32
                assert ws >= nq * n_ranges * kpad * 12           # (score, id) candidates per query and range
    assert lib.mmb200_flat_ip_plan(0, 10, 1, sm_count, out) == _lib.ERR_INVALID
    assert lib.mmb200_flat_ip_plan(10, 10, 1025, sm_count, out) == _lib.ERR_INVALID


def test_training_pair_envelope_and_saved_size():
    """Host-side contract of the tensor-core training pair (pure arithmetic, no GPU): the envelope the Python layer routes
    on, and the size of the opaque state the forward leaves for the backward."""
    lib = _lib.load()
    ok = lib.mmb200_kernel_pool_train_tc_supported
    assert ok(30, 200, 300, 21) == 1 and ok(30, 180, 300, 11) == 1 and ok(32, 2000, 320, 32) == 1 and ok(1, 1, 4, 1) == 1
    assert ok(33, 200, 300, 21) == 0      # more than 32 query terms: FFMA backward (the forward runs per 32-row block)
    assert ok(30, 200, 324, 21) == 0      # the query-gradient accumulator holds 320 columns
    assert ok(30, 200, 302, 21) == 0      # 16-byte rows
    assert ok(30, 200, 300, 33) == 0
    assert lib.mmb200_kernel_pool_saved_floats(7, 200) == 7 * (33 * 200 + 32)
    assert lib.mmb200_kernel_pool_saved_floats(0, 200) == 0
