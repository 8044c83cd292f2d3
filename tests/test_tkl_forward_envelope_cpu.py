"""The shared cases of the TKL forward envelope tests (tests/tkl_forward_cases.py), checked without a GPU: the library holds
exactly the TKL forward instantiations the matrix claims and no profiling one, every row claims what the routing gives
its shape and holds something no other row does, the corpus builder keeps its invariants, the float32 hill selection is
the oracle's, and interaction.tkl_kernel_set_covers answers what the plan kernel's float32 cover test answers."""
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import tkl_forward_cases as F
from matchmaker_b200 import _lib, interaction
from oracle import interaction_oracle as O

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
TEMPLATED = re.compile(r"\b(tkl_window_kernel|tkl_ts_kernel)<([^>]*)>")
PLAIN = re.compile(r"\b(tkl_plan_kernel|tkl_plan_store_kernel|tkl_hills_kernel|tkl_slot_map_kernel)\(")


@pytest.fixture(scope="module")
def instantiations():
    """The TKL forward kernels compiled into the library, from the demangled SASS function names."""
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
        m = TEMPLATED.search(line)
        if m:
            found.append(F.inst(m.group(1), *[a.strip() for a in m.group(2).split(",")]))
            continue
        m = PLAIN.search(line)
        if m:
            found.append(m.group(1))
    return found


def test_library_holds_exactly_the_claimed_forward_kernels(instantiations):
    assert len(instantiations) == len(set(instantiations)) == len(F.EVERY) == 12, sorted(instantiations)
    assert set(instantiations) == F.EVERY
    assert not any(re.match(r"tkl_window_kernel<\d+, true", i) for i in instantiations), "profiling build shipped"
    assert set().union(*(row.claims for row in F.MATRIX)) == F.EVERY | F.PLAN_CLAIMS | F.FFMA_CLAIMS


def test_rows_claim_what_the_routing_gives_them():
    for row in F.MATRIX:
        assert row.claims == F.routed_claims(row.entry, row.impl, row.sat, row.K, row.Lq, row.D, row.C, row.n), str(row)
        assert (F.tc_fits(row.Lq, row.K) if row.impl == "tcgen05" else F.ffma_fits(row.D, row.K)), str(row)
    # on the SM count of the GPU at hand too: the FFMA split claims hold there
    for row in F.MATRIX:
        assert row.claims == F.routed_claims(row.entry, row.impl, row.sat, row.K, row.Lq, row.D, row.C, row.n,
                                             F.sm_count()), str(row)


def test_routing_restatement():
    assert [F.kb(k) for k in (1, 11, 12, 13, 16)] == [12, 12, 12, 16, 16]
    assert F.plan_path(1024, 64, 40) == ("smem", "ballot") and F.plan_path(1025, 65, 40) == ("global", "general")
    # fewer documents than SMs: segments of chunk slots, at most C of them
    assert F.ffma_split(5, 4, 132) == (4, 20) and F.ffma_split(1, 130, 132) == (130, 130)
    assert F.ffma_split(7, 65, 132) == (33, 231) and F.ffma_split(132, 65, 132) == (1, 132)
    assert F.ffma_split(600, 65, 132) == (1, 264)
    # the FFMA plan: D = 300 with K <= 12 fits, with K = 13 it does not; D = 356 fits neither
    assert F.ffma_fits(300, 12) and not F.ffma_fits(300, 13) and not F.ffma_fits(356, 1) and F.ffma_fits(44, 16)
    assert F.tc_fits(32, 16) and not F.tc_fits(40, 13) and F.tc_fits(40, 12)
    assert F.n_windows(1) == 6 and F.n_windows(130) == 2586


def test_every_row_is_needed():
    """Between them the rows hold every claim and required edge, and each row holds one that no other row does:
    deleting a row fails this test."""
    feats = [F.features(r) for r in F.MATRIX]
    assert F.REQUIRED_FEATURES <= set().union(*feats), sorted(F.REQUIRED_FEATURES - set().union(*feats))
    for k, row in enumerate(F.MATRIX):
        others = [j for j in range(len(F.MATRIX)) if j != k]
        own = (set(row.claims) - set().union(*(F.MATRIX[j].claims for j in others))) \
            | ((feats[k] & F.REQUIRED_FEATURES) - set().union(*(feats[j] for j in others)))
        assert own, f"{row} holds nothing another row does not"


@pytest.mark.parametrize("row", F.MATRIX, ids=str)
def test_builder_invariants(row):
    c = F.build(row.Lq, row.D, row.C, row.K, row.n, seed=F.seed(row))
    n_chunks = c.chunk_mask.shape[0]
    assert len(c.pair_q) == len(c.pair_d) == row.n
    slots = c.doc_slots
    ref = slots[slots >= 0]
    # every chunk referenced once except the poison, which is non-finite and referenced by no slot
    assert sorted(ref.tolist() + c.poison) == list(range(n_chunks))
    assert len(c.poison) == F.N_DOCS // 2
    for p in c.poison:
        assert not torch.isfinite(c.chunks[p]).any() and torch.isnan(c.chunks[p]).any() and torch.isinf(c.chunks[p]).any()
    assert torch.isfinite(c.chunks[ref.long()]).all() and torch.isnan(c.store_base[n_chunks:]).all()
    # passages: empty ones, a full one, dropped middle slots, partly masked last chunks, the last packed slot at every
    # residue mod 3 (and at C - 1)
    n_per = (slots >= 0).sum(1)
    assert (n_per == 0).any() and (n_per == row.C).any()
    last = [int((s >= 0).nonzero().max()) for s in slots if (s >= 0).any()]
    assert (row.C - 1) in last
    if row.C >= 3:
        assert {l % F.TILE_SLOTS for l in last} == {0, 1, 2}
        assert any((s[:l] < 0).any() for s, l in zip(slots[(n_per > 0)], last)), "no dropped middle slot"
    partial = (c.chunk_mask.sum(1) < F.CHUNK)
    assert partial[ref.long()].any()
    # pairs: void ones when there are four or more, every live combination at least twice when pairs outnumber them
    uniq, inv = c.unique()
    assert len(uniq) <= 64 and (inv >= 0).any()
    if row.n >= 4:
        assert (c.pair_d < 0).any()
    if row.n >= 8:
        assert (torch.bincount(inv[inv >= 0]) >= 2).all()
    # the padded layout holds the same chunks in slot order
    q, qm, ch, cm, packed = F.gathered(c)
    assert packed.numel() == row.n * row.C and ch.shape[0] == int(packed.sum()) and torch.isfinite(ch).all()


def test_continuous_case_reaches_the_layernorm_region():
    c = F.continuous_case(40, 32, 8, 11, seed=5)
    w = c.params["sat_emb_reduce1_weight"]
    red = (c.q.double() @ w.double())
    # exact in float32: the float32 product of the row with the weight is the double one
    assert torch.equal((c.q @ w).double(), red)
    ref = F.reference(c, "embedding")
    assert F.continuous_share(c, ref) >= 0.1
    lens = set(ref["lengths"][ref["lengths"] > 0].unique().tolist())
    assert set(range(1, 31)) <= lens, sorted(set(range(1, 31)) - lens)


@pytest.mark.parametrize("W", [3, 6, 16, 26, 44, 45, 257])
def test_hills_restatement_is_the_oracle(W):
    x = F.hill_rows(64, W, seed=W)
    cs = (np.random.default_rng(W).random(15) + 0.5).astype(np.float32)
    score, orig, top, top15 = F.top_hills_f32(x, cs)
    ws = torch.from_numpy(x).double()
    o = ws.clone()
    o[o == 0] = -9900
    ti, t15 = O.tkl_top_hills(o)
    assert torch.equal(torch.from_numpy(top), ti)
    assert torch.equal(torch.from_numpy(top15).double(), t15)
    o[o <= -9900] = 0
    assert torch.equal(torch.from_numpy(orig).double(), o)
    np.testing.assert_allclose(score, (t15 * torch.from_numpy(cs).double()).sum(1).numpy(), rtol=1e-6, atol=1e-6)


def test_host_cover_is_the_plan_kernels_float32_test():
    mu, sg = F.ULP_GAP_SET
    mu32, sg32 = np.float32(mu), np.float32(sg)
    assert F.cover_sweep_f64(mu32, sg32) and not F.plan_cover_f32(mu32, sg32)
    assert not interaction.tkl_kernel_set_covers(torch.tensor(mu32), torch.tensor(sg32))
    ms, ss = F.near_touching_sets(100_000, 6, seed=1)
    got = np.array([interaction.tkl_kernel_set_covers(torch.from_numpy(m), torch.from_numpy(s)) for m, s in zip(ms, ss)])
    want = np.array([F.plan_cover_f32(m, s) for m, s in zip(ms, ss)])
    assert (got == want).all(), int((got != want).sum())
    assert 0.05 < want.mean() < 0.95
    # the double sweep disagrees on some of them in both directions
    f64 = np.array([F.cover_sweep_f64(m, s) for m, s in zip(ms[:20_000], ss[:20_000])])
    assert (f64 & ~want[:20_000]).any() and (~f64 & want[:20_000]).any()


def test_host_cover_cache_follows_the_tensor_version():
    mu, sg = torch.linspace(-0.9, 1.0, 11), torch.full((11,), 0.1)
    assert interaction.tkl_kernel_set_covers(mu, sg)
    sg.fill_(0.001)
    assert not interaction.tkl_kernel_set_covers(mu, sg)
    assert interaction.tkl_kernel_set_covers(torch.zeros(1), torch.full((1,), 0.1))


def test_host_cover_cache_survives_address_reuse():
    """A freed kernel set's address goes to the next tensor at version 0: the cached answer must not follow it."""
    for i in range(50):
        covering = i % 2 == 0
        sg = torch.full((11,), 0.1 if covering else 0.001)
        mu = torch.linspace(-0.9, 1.0, 11)
        assert interaction.tkl_kernel_set_covers(mu.view(-1), sg.view(-1)) == covering, i
        assert interaction.tkl_kernel_set_covers(mu, sg) == covering, i
        del mu, sg
