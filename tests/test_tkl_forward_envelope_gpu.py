"""The TKL forward at every compiled instantiation against fp64 (tests/tkl_forward_cases.py): the padded and the store
entry on both kernels and saturations, the plan kernel's shared-memory and global prefix and its ballot and general
pass, the FFMA segment split and several documents per CTA; the embedding saturation inside the continuous region of its
LayerNorm; the hill selection bit for bit against a float32 restatement; every mask element type; and the host's cover
answer against what the device does with it."""
import dataclasses
import functools

import numpy as np
import pytest
import torch

import tkl_forward_cases as F
from matchmaker_b200 import interaction

pytestmark = pytest.mark.gpu
DEV = "cuda"
IMPLS = ("simt", "tcgen05")
BAR = 1e-3   # of the pair's largest window: the terms of a window are bounded by it


def _auto_impl(case: F.Case, Lq: int, K: int) -> str:
    p = case.params
    return "tcgen05" if F.tc_fits(Lq, K) and interaction.tkl_kernel_set_covers(p["mu"], p["sigma"]) else "simt"


def _check(got: torch.Tensor, case: F.Case, ref: dict, what: str) -> float:
    """Window scores of every pair against the fp64 windows of its distinct pair; returns the worst error / scale."""
    uniq, inv = case.unique()
    g = got.cpu()
    assert g.shape == (len(inv), F.n_windows(case.C)), what
    assert torch.isfinite(g).all(), f"{what}: poison reached a window"
    assert (g[inv < 0] == 0).all(), f"{what}: a void pair scored"
    first = torch.full((len(uniq),), -1, dtype=torch.long)
    for i, u in enumerate(inv.tolist()):
        if u >= 0 and first[u] < 0:
            first[u] = i
    live = (inv >= 0).nonzero().flatten()
    assert torch.equal(g[live], g[first[inv[live]]]), f"{what}: repeats of a pair differ"
    gu, r = g[first].double(), ref["orig_score"]
    assert ((gu == 0) == (r == 0)).all(), f"{what}: exact-zero windows must stay exactly zero"
    assert (gu != 0).sum() > gu.shape[0], f"{what}: hardly any window scored"
    scale = r.abs().amax(dim=1, keepdim=True).clamp(min=1e-30)
    err = ((gu - r).abs() / scale).max().item()
    assert err <= BAR, f"{what}: worst error / scale {err:.3e}"
    _, _, top_idx, _ = interaction.tkl_top_hills(g[first].to(DEV), case.params["chunk_scoring"].to(DEV))
    ti, ri = top_idx.cpu(), ref["top_non_overlapping_idx"]
    for b, c in (ti != ri).nonzero().tolist():   # top-3 windows exact, except between windows tied within the bar
        assert abs(r[b, ti[b, c]] - r[b, ri[b, c]]) <= BAR * scale[b, 0], (what, b, c, ti[b].tolist(), ri[b].tolist())
    return err


@pytest.mark.parametrize("row", F.MATRIX, ids=str)
def test_matrix_against_fp64(row, record_property):
    assert row.claims == F.routed_claims(row.entry, row.impl, row.sat, row.K, row.Lq, row.D, row.C, row.n,
                                         F.sm_count()), "the row's claims do not hold on this GPU"
    case = F.build(row.Lq, row.D, row.C, row.K, row.n, seed=F.seed(row))
    assert interaction.tkl_kernel_set_covers(case.params["mu"], case.params["sigma"])
    got = F.windows(case, row.entry, row.sat, row.impl)
    err = _check(got, case, F.reference(case, row.sat), str(row))
    record_property("worst_err_over_scale", f"{err:.2e}")
    print(f"{row}: worst error / scale {err:.2e}")
    # a second run gives the same bits; auto gives what the kernel it routes to gives
    assert torch.equal(F.windows(case, row.entry, row.sat, row.impl), got)
    routed = _auto_impl(case, row.Lq, row.K)
    want = got if routed == row.impl else F.windows(case, row.entry, row.sat, routed)
    assert torch.equal(F.windows(case, row.entry, row.sat, "auto"), want)


@functools.lru_cache(maxsize=None)
def _continuous():
    case = F.continuous_case(40, 32, 8, 11, seed=5)
    ref = F.reference(case, "embedding")
    return case, ref


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("entry", ["padded", "store"])
def test_embedding_saturation_continuous_region(entry, impl, record_property):
    """sat_emb_reduce1 · q_i = len + {0, +-2^-10, +-2^-6, +-0.5} exactly, for the window lengths 1-30 that passage tails
    and dropped slots produce: LayerNorm((red, len)) moves continuously there, so its eps and the scale of red count."""
    case, ref = _continuous()
    share = F.continuous_share(case, ref)
    assert share >= 0.1, f"only {share:.3f} of the live cells inside the LayerNorm's continuous region"
    err = _check(F.windows(case, entry, "embedding", impl), case, ref, f"continuous {entry} {impl}")
    record_property("worst_err_over_scale", f"{err:.2e}")
    print(f"continuous {entry} {impl}: worst error / scale {err:.2e}, share {share:.3f}")


@pytest.mark.parametrize("W", [6, 16, 26, 44, 45, 255, 256, 257, 512, 986, 1286, 2586])
def test_top_hills_bit_for_bit(W):
    cs = (np.random.default_rng(W).random(15) + 0.5).astype(np.float32)
    for B in (1, F.sm_count() * 8 + 1, 3000):   # one document, one past the grid (grid-stride loop), many
        x = F.hill_rows(B, W, seed=W * 7 + B)
        ws = torch.from_numpy(x).to(DEV)
        keep = ws.clone()
        got = interaction.tkl_top_hills(ws, torch.from_numpy(cs).to(DEV))
        torch.cuda.synchronize()
        assert torch.equal(ws, keep), "the window scores were modified"
        for name, a, b in zip(("score", "orig_score", "top_idx", "top15"), got, F.top_hills_f32(x, cs)):
            assert torch.equal(a.cpu(), torch.from_numpy(b)), f"W={W} B={B}: {name} differs"


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("entry", ["padded", "store"])
def test_mask_element_types(entry, impl):
    case = F.build(12, 32, 4, 11, 40, seed=77)
    sat = "embedding"
    base = F.windows(case, entry, sat, impl, mask_dtype=torch.float32)
    assert (base != 0).any()
    for dt in (torch.bool, torch.uint8, torch.int32, torch.int64):
        assert torch.equal(F.windows(case, entry, sat, impl, mask_dtype=dt), base), dt
    if entry == "store":
        ones_q, ones_c = torch.ones_like(case.q_mask), torch.ones_like(case.chunk_mask)
        assert torch.equal(F.windows(case, entry, sat, impl, q_mask=None), F.windows(case, entry, sat, impl, q_mask=ones_q))
        assert torch.equal(F.windows(case, entry, sat, impl, chunk_mask=None),
                           F.windows(case, entry, sat, impl, chunk_mask=ones_c))
        assert torch.equal(F.windows(case, entry, sat, impl, q_mask=None, chunk_mask=None),
                           F.windows(case, entry, sat, impl, q_mask=ones_q, chunk_mask=ones_c))


def _cover_sets():
    """The one-ulp-gap set, then near-touching sets on which the float32 and the double cover tests agree and disagree,
    six of each of the four kinds."""
    sets = [tuple(np.float32(v) for v in F.ULP_GAP_SET)]
    ms, ss = F.near_touching_sets(20_000, 6, seed=3)
    kinds = {}
    for m, s in zip(ms, ss):
        k = (F.plan_cover_f32(m, s), F.cover_sweep_f64(m, s))
        if len(kinds.setdefault(k, [])) < 6:
            kinds[k].append((m, s))
    assert len(kinds) == 4 and all(len(v) == 6 for v in kinds.values()), {k: len(v) for k, v in kinds.items()}
    return sets + [x for v in kinds.values() for x in v]


@pytest.mark.parametrize("entry", ["padded", "store"])
def test_cover_routing(entry):
    """impl="auto" never leaves the windows at zero and stays within the fp64 bar of the FFMA kernel, which tests the
    activations themselves; a forced tensor-core call scores exactly when the host says the set covers."""
    case = F.build(12, 32, 3, 6, 16, seed=91)
    for n, (mu, sg) in enumerate(_cover_sets() if entry == "padded" else _cover_sets()[:1]):
        c = dataclasses.replace(case, params=dict(case.params, mu=torch.from_numpy(mu), sigma=torch.from_numpy(sg)))
        covers = interaction.tkl_kernel_set_covers(c.params["mu"], c.params["sigma"])
        assert covers == F.plan_cover_f32(mu, sg), n
        simt = F.windows(c, entry, "log", "simt").double().cpu()
        auto = F.windows(c, entry, "log", "auto").double().cpu()
        tc = F.windows(c, entry, "log", "tcgen05").double().cpu()
        assert (simt != 0).any(), n
        assert (auto != 0).any(), f"set {n}: impl='auto' left every window at zero (host cover {covers})"
        scale = simt.abs().amax(dim=1, keepdim=True).clamp(min=1e-30)
        assert ((auto - simt).abs() <= BAR * scale).all(), n
        assert bool((tc != 0).any()) == covers, f"set {n}: host cover {covers}, forced tensor-core call disagrees"
