"""The shared cases of the kernel-pooling store-mode envelope tests (tests/kernel_pool_store_cases.py), checked without a
GPU: the store-mode instantiations compiled into the library are exactly the 11 the matrix claims, every row claims what
the routing gives its shape and holds an instantiation or a required edge no other row does, the fp64 reference is the
pinned TK / TK-Sparse store oracle, and the built inputs hold the preconditions the GPU tests rely on."""
import re
import shutil
import subprocess

import pytest
import torch

import kernel_pool_cases as KP
import kernel_pool_store_cases as C
import tk_store_cases as TKC
from matchmaker_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
INSTANTIATION = re.compile(r"\b(" + "|".join(C.KERNELS) + r")<([^>]*)>")


@pytest.fixture(scope="module")
def instantiations():
    """The store-mode instantiations compiled into the library, from the demangled SASS function names."""
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
    found = []
    for line in dem.stdout.splitlines():
        m = INSTANTIATION.search(line)
        if m:
            found.append(C.inst(m.group(1), *re.findall(r"\d+", m.group(2))))
    return found


def test_compiled_store_instantiations_are_exactly_the_claimed_eleven(instantiations):
    assert len(instantiations) == len(set(instantiations)) == 11, sorted(instantiations)
    assert set(instantiations) == C.EVERY
    assert set().union(*(row.claims for row in C.MATRIX)) == C.EVERY


def test_rows_claim_what_the_routing_gives_them():
    for row in C.MATRIX:
        assert set(row.claims) == C.dispatched(row.Lq, row.D, row.K, row.L), str(row)
        assert row.impls == (("tcgen05", "simt") if row.Lq <= C.TS_MAX_LQ else ("simt",)), str(row)


def test_routing_restatement():
    assert [C.ts_store_kb(k) for k in (1, 5, 11, 12, 13, 21, 22, 24, 25, 32)] == [12, 12, 11, 12, 24, 21, 24, 24, 32, 32]
    assert C.simt_store_inst(11, 48) == (12, 1) and C.simt_store_inst(11, 49) == (12, 2)
    assert C.simt_store_inst(21, 300) == (24, 2) and C.simt_store_inst(32, 1) == (32, 1)
    assert C.ts_accepts(128, 4) and not C.ts_accepts(129, 4) and not C.ts_accepts(8, 30)
    assert C.auto_impl(128, 64) == "tcgen05" and C.auto_impl(129, 64) == "simt"
    # the FFMA kernel's D edge on an H100: D = 484 is the last of the <32, 2> plan (padded stride 484; 488 pads to 492)
    assert C.D_EDGE == 484 and C.simt_accepts(484, 32, 300) and not C.simt_accepts(488, 32, 300)
    assert C.simt_d_edge(5, 8) == 828 and not C.simt_accepts(832, 5, 8)
    assert C.impls(129, 488, 32, 300) == ()


def test_every_row_is_needed():
    """Between them the rows hold every instantiation and every required edge, and each row holds one that no other row
    does: deleting a row fails this test."""
    feats = [C.features(r) for r in C.MATRIX]
    assert C.REQUIRED_FEATURES <= set().union(*feats), sorted(C.REQUIRED_FEATURES - set().union(*feats))
    for k, row in enumerate(C.MATRIX):
        others = [j for j in range(len(C.MATRIX)) if j != k]
        own = (set(row.claims) - set().union(*(C.MATRIX[j].claims for j in others))) \
            | ((feats[k] & C.REQUIRED_FEATURES) - set().union(*(feats[j] for j in others)))
        assert own, f"{row} holds nothing another row does not"


@pytest.mark.parametrize("gate", [False, True], ids=["tk", "tk_sparse"])
@pytest.mark.parametrize("L", [1, 9, 40])
def test_reference_is_the_tk_store_oracle(L, gate):
    c = C.make_case(11, 5, 16, L, 2, seed=L + 3 * gate, gate=gate, min_pairs=50)
    ref = C.reference(c)
    t = C.truncated(c)   # store_oracle reads whole passages
    o = TKC.store_oracle(c.q, c.qm.double(), t.clean_buf[:t.n_rows], t.off, c.pair_q, c.pair_d, c.mu, c.sigma, c.alpha,
                         c.weight, t.clean_gate)
    assert torch.equal(torch.isneginf(o), c.void()) and torch.equal(torch.isneginf(ref["score"]), c.void())
    torch.testing.assert_close(ref["score"], o, rtol=1e-12, atol=1e-12)


def _passages(c: C.Case):
    return [(int(c.off[d]), int(c.off[d + 1]), bool(c.referenced[d])) for d in range(len(c.off) - 1)]


@pytest.mark.parametrize("gate", [False, True], ids=["plain", "gate"])
@pytest.mark.parametrize("row", C.MATRIX, ids=str)
def test_cases_hold_their_preconditions(row, gate):
    c = C.row_case(row, gate)
    P = len(c.pair_q)
    store, tail = c.buf[:c.n_rows], c.buf[c.n_rows:]
    # poison only in unreferenced passages, each right after a referenced passage of length % 8 != 0
    ps = _passages(c)
    finite = torch.isfinite(store).all(1)
    for i, (a, b, ref) in enumerate(ps):
        if ref:
            assert finite[a:b].all(), f"{row}: a referenced passage holds a non-finite row"
        else:
            assert (~finite[a:b]).all() and b - a == C.POISON_ROWS
            assert i > 0 and ps[i - 1][2] and (ps[i - 1][1] - ps[i - 1][0]) % 8 != 0
            assert torch.isnan(store[a:b]).any() and torch.isposinf(store[a:b]).any() and torch.isneginf(store[a:b]).any()
    assert any(not r for _, _, r in ps) and torch.isfinite(c.clean_buf).all()
    # the store is a view; the rows past it are NaN; the last passage is referenced, of length 1..7 (mod 8)
    a, b, ref = ps[-1]
    assert ref and b == c.n_rows and (b - a) % 8 != 0 and torch.isnan(tail).all() and len(tail) > 0
    assert (c.pair_d == len(ps) - 1).any()
    # gates: >= 0 with about a quarter exactly 0 on the referenced rows, NaN on the poisoned ones
    if gate:
        live = torch.cat([torch.arange(a, b) for a, b, r in ps if r])
        gl = c.gate[live]
        assert (gl >= 0).all() and 0.15 < float((gl == 0).double().mean()) < 0.35
        assert torch.isnan(c.gate[~torch.isin(torch.arange(c.n_rows), live)]).all()
    # pairs: enough for several per CTA on both grids; the pairs of one query adjacent; no unreferenced passage
    assert P >= C.MIN_PAIRS
    assert P // min(C.SM_H100, P) >= 9 and P // min(P, 4 * C.SM_H100) >= 2
    assert (c.pair_q[1:] >= c.pair_q[:-1]).all()
    assert c.referenced[c.pair_d[c.pair_d >= 0].long()].all()
    # tile counts interleaved, void pairs (pair_d -1 and the empty passage) between non-void ones, every pair repeated
    tiles = c.tiles()
    possible = {min(3, (min(n, row.L) + 127) // 128) for n in C.passage_lengths(row.L)} | {0}
    assert set(tiles.tolist()) == possible
    for qi in range(int(c.pair_q.max()) + 1):
        windows = tiles[c.pair_q == qi].unfold(0, len(C.TILE_PATTERN), 1)
        assert all(set(w.tolist()) == possible for w in windows), f"{row}: tile counts not interleaved"
    void = c.void()
    same_q = c.pair_q[1:] == c.pair_q[:-1]
    assert not (void[1:] & void[:-1] & same_q).any()
    assert (c.pair_d == -1).any() and (void & (c.pair_d >= 0)).any()
    u, inv = c.unique_pairs()
    assert (torch.bincount(inv[inv >= 0]) >= 2).all()
    # passages longer than max_doc_len are truncated
    lens = (c.off[1:] - c.off[:-1])[c.pair_d[c.pair_d >= 0].long()]
    assert (lens > row.L).any()
    assert len(u) * row.Lq * row.L * row.K <= 5e7, f"{row}: the fp64 reference would be too large"
