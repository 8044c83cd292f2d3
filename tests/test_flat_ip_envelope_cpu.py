"""The shared cases of the flat-IP envelope tests (tests/flat_ip_cases.py), checked without a GPU: the fp64 oracle equals
the fp32 CPU oracles on the matrix inputs, the inputs hold the preconditions the GPU tests rely on, the routing
restatement agrees with the library's own plan, the rows between them claim every instantiation of the kernel body
compiled into the library and every edge the matrix is there for.  Also the empty query batch at the C ABI."""
import ctypes
import re
import shutil
import subprocess

import pytest
import torch

import flat_ip_cases as C
import ivf_oracle
from matchmaker_b200 import _lib
from oracle import interaction_oracle as O

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
ENV = ("MMB200_FLATIP_CLUSTER", "MMB200_FLATIP_RANGES")


@pytest.mark.parametrize("row", C.MATRIX, ids=str)
def test_oracle_equals_the_fp32_cpu_oracles(row):
    """On the matrix inputs the fp32 CPU sums of oracle.flat_ip_search / ivf_oracle.ivf_search are exact too."""
    c = C.make_case(row)
    exp_s, exp_i = C.expected(row)
    ids = C.row_ids(row, c)
    if row.mode == "flat":
        s, i = O.flat_ip_search(c.q.float(), c.p.float(), ids, row.k)
    else:
        s, i = ivf_oracle.ivf_search(c.q.float(), c.p.float(), ids, c.offsets, c.probes, row.k)
    assert torch.equal(i, exp_i)
    assert torch.equal(s, exp_s)


def _scores(c):
    return c.q.double() @ c.p.double().T


@pytest.mark.parametrize("row", C.MATRIX, ids=str)
def test_cases_hold_their_preconditions(row):
    c = C.make_case(row)
    exp_s, exp_i = C.expected(row)
    s = _scores(c)
    cand = torch.ones_like(s, dtype=torch.bool) if row.mode == "flat" else C.candidates(c)
    ids = C.row_ids(row, c)
    assert torch.unique(ids).numel() == ids.numel(), "ids must be distinct"
    if row.regime == "neg":
        assert (s[cand] < 0).all(), "a candidate scores >= 0"
        if row.mode == "flat":
            assert row.n % C.BN, "n must leave a ragged last tile"
    if row.regime == "tie":
        top = s.masked_fill(~cand, float("-inf"))
        for r in range(s.shape[0]):
            sr = top[r][cand[r]]
            kth = float(exp_s[r, row.k - 1])
            above, at = int((sr > kth).sum()), int((sr == kth).sum())
            assert above < row.k < above + at, f"query {r}: no tie run straddles rank {row.k}"
            assert at >= row.run, f"query {r}: the run is not at rank {row.k}"
        if row.ids == "extreme":
            assert (exp_i == C.I64_MIN).any(1).all() and (exp_i == -1).any(1).all(), "the smallest run ids must win"
            assert not (exp_i == C.I64_MAX).any(), "INT64_MAX must lose its tie"
    if row.mode == "flat":
        return
    # ivf / residual: the store holds the list rows at row_index; padding rows outrank every candidate ("neg"), or
    # reach the top score ("tie")
    assert torch.equal(c.store[c.row_index], c.p)
    assert torch.equal(c.store_ids[c.row_index], c.ids)
    pad = torch.ones(c.store.shape[0], dtype=torch.bool)
    pad[c.row_index] = False
    assert pad.any()
    ps = c.q.double() @ c.store[pad].double().T
    best = s.masked_fill(~cand, float("-inf")).max(1).values
    if row.regime == "neg":
        assert (ps.min(1).values > best).all(), "padding rows must outrank the candidates"
    if row.regime == "tie":
        assert (ps.min(1).values >= best).all(), "padding rows must reach the top score"
    if row.mode == "residual":
        assert all((c.store_lists[c.row_index[c.offsets[l]:c.offsets[l + 1]]] == l).all() for l in range(len(row.lists)))
    if row.regime == "neg":   # the rows just past each probed list (the next list) outrank everything probed
        nlist = len(row.lists)
        for r in range(s.shape[0]):
            for l in c.probes[r].tolist():
                if 0 <= l < nlist - 1 and row.lists[l + 1]:
                    nxt = s[r, int(c.offsets[l + 1]): int(c.offsets[l + 2])]
                    assert nxt.min() > best[r], f"query {r}: list {l + 1} does not outrank list {l}"
    probed = torch.bincount(c.probes[(c.probes >= 0) & (c.probes < len(row.lists))], minlength=len(row.lists))
    if "a list probed by more than 128 queries" in C.features(row):
        assert int(probed[torch.tensor(row.lists).argmax()]) == row.nq > C.BM
    if row.nprobe > 1 and row.regime != "neg":
        assert (c.probes == -1).any() and (c.probes >= len(row.lists)).any()
    for r in range(s.shape[0]):
        p = c.probes[r][c.probes[r] >= 0]
        assert torch.unique(p).numel() == p.numel(), "duplicate probes"


def test_rows_claim_what_the_routing_gives_them():
    every = set().union(*(C.dispatched(r) for r in C.MATRIX))
    expect = ({C.inst(C.FLAT, t, cl, e, False) for t in ("__half", "__nv_bfloat16") for cl in (1, 2, 4) for e in (32, 64)}
              | {C.inst(C.FLAT, t, 1, e, True) for t in ("__half", "__nv_bfloat16") for e in (32, 64)}
              | {C.inst(C.IVF_GATHER, t, e) for t in ("__half", "__nv_bfloat16") for e in (32, 64)}
              | {C.inst(C.RESIDUAL, e, b) for e in (32, 64) for b in (1, 2)}
              | {C.inst(C.FLAT_FP8, cl, e) for cl in (1, 2, 4) for e in (32, 64)}
              | {C.inst(C.GATHER_FP8, e) for e in (32, 64)})
    assert len(expect) == 32
    assert every == expect


def test_every_row_is_needed():
    """Between them the rows hold every instantiation and every required edge, and each row holds one that no other row
    does: deleting a row fails this test."""
    feats = [C.features(r) for r in C.MATRIX]
    assert C.REQUIRED_FEATURES <= set().union(*feats), sorted(C.REQUIRED_FEATURES - set().union(*feats))
    for k, row in enumerate(C.MATRIX):
        others = [j for j in range(len(C.MATRIX)) if j != k]
        own = (C.dispatched(row) - set().union(*(C.dispatched(C.MATRIX[j]) for j in others))) \
            | ((feats[k] & C.REQUIRED_FEATURES) - set().union(*(feats[j] for j in others)))
        assert own, f"{row} holds nothing another row does not"


PLAN_SHAPES = [(r.nq, r.n, r.k) for r in C.MATRIX if r.mode == "flat"] + [
    (6400, 1_100_000, 100), (1, 10 ** 6, 1), (1280, 128, 1024), (1152, 7000, 32), (200, 40000, 257)]


@pytest.mark.parametrize("sm_count", [132, 114])
@pytest.mark.parametrize("overrides", [(None, None), ("1", None), ("2", "1"), ("4", "32"), (None, "7"), ("3", "0")])
def test_plan_restatement_matches_the_library(monkeypatch, sm_count, overrides):
    """mmb200_flat_ip_plan (no device needed) against flat_ip_cases.plan, with the overrides (3 and 0 are ignored)."""
    lib = _lib.load()
    for name, v in zip(ENV, overrides):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, v)
    cl = int(overrides[0]) if overrides[0] else None
    ranges = int(overrides[1]) if overrides[1] else None
    for nq, n, k in PLAN_SHAPES:
        out = (ctypes.c_int32 * 8)()
        assert lib.mmb200_flat_ip_plan(nq, n, k, sm_count, out) == _lib.OK, _lib.last_error()
        pl = C.plan(nq, n, k, sm_count, cl, ranges)
        got = dict(zip(("n_qblocks", "n_tiles", "n_ranges", "tiles_per_range", "grid", "cl"), out[:6]))
        got["workspace"] = (out[6] & 0xffffffff) | ((out[7] & 0xffffffff) << 32)
        assert got == {key: pl[key] for key in got}, (nq, n, k)


def _normalise(kernel: str, args: str) -> str:
    vals = [re.sub(r"^\((int|bool)\)", "", a.strip()) for a in args.split(",")]
    if kernel == C.FLAT:
        vals[3] = {"0": "false", "1": "true"}.get(vals[3], vals[3])
    return kernel + "<" + ",".join(vals) + ">"


@pytest.fixture(scope="module")
def instantiations():
    """The instantiations of the kernel body compiled into the library, from the demangled SASS function names."""
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
        if out.returncode != 0:
            pytest.skip("cuobjdump failed: " + out.stderr[-200:])
        names = re.findall(r"Function : (\S+)", out.stdout)
        dem = subprocess.run([DEMANGLE], input="\n".join(names), capture_output=True, text=True, timeout=60)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump / c++filt unavailable: {e}")
    if dem.returncode != 0:
        pytest.skip("c++filt failed: " + dem.stderr[-200:])
    pattern = re.compile(r"\b(" + "|".join(C.KERNELS) + r")<([^>]*)>")
    found = []
    for line in dem.stdout.splitlines():
        m = pattern.search(line)
        if m:
            found.append(_normalise(m.group(1), m.group(2)))
    return found


def test_every_compiled_instantiation_is_claimed_by_a_row(instantiations):
    assert len(instantiations) == len(set(instantiations)) == 32, sorted(instantiations)
    claimed = set().union(*(C.dispatched(r) for r in C.MATRIX))
    assert set(instantiations) == claimed, (sorted(set(instantiations) - claimed), sorted(claimed - set(instantiations)))


def test_empty_query_batch_is_accepted_at_the_abi():
    """nq = 0 with the null pointers torch hands out for empty tensors returns OK without touching the device; the sizes
    are still checked, and one query needs its tensors."""
    lib = _lib.load()
    n = None
    assert lib.mmb200_flat_ip_topk(n, n, n, n, n, n, 0, 0, 1000, 64, 10, _lib.F16, 0, n) == _lib.OK, _lib.last_error()
    assert lib.mmb200_flat_ip_topk(n, n, n, n, n, n, 0, 0, 1000, 64, 2000, _lib.F16, 0, n) == _lib.ERR_INVALID
    assert lib.mmb200_flat_ip_topk(n, n, n, n, n, n, 0, 0, 1000, 60, 10, _lib.F16, 0, n) == _lib.ERR_INVALID
    assert lib.mmb200_flat_ip_topk(n, n, n, n, n, n, 0, -1, 1000, 64, 10, _lib.F16, 0, n) == _lib.ERR_INVALID
    rc = lib.mmb200_flat_ip_topk(n, n, n, n, n, n, 0, 1, 1000, 64, 10, _lib.F16, 0, n)
    assert rc == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
