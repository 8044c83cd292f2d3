"""TKL backward (tkl_bwd_kernel, csrc/tkl_bwd.cu) across its envelope against fp64 autograd of the oracle restatement, with
the top-3 window choice conditioned on the kernel's (tests/tkl_oracle.py); the forward kernels at the same shapes."""
import pytest
import torch

import tkl_oracle as T
from conftest import assert_close_rel
from matchmaker_b200 import _lib, autograd, interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
SATS = ["embedding", "log"]
GRAD_REL = 2e-3        # worst error / largest reference entry, per gradient tensor
H100_SMEM_OPTIN = 227 * 1024

# (B, Lq, Ld, D, K) and what each shape exercises
SHAPES = {
    "b5_lq14_d32_k11": (5, 14, 420, 32, 11),      # the original single-shape check
    "config5": (20, 40, 2000, 300, 11),           # Lq = 40, two passes of the 256-column loop, trailing chunks dropped
    "k12_d44_lq33": (6, 33, 300, 44, 12),         # last K of the KB = 12 kernels; D not a multiple of 32; Lq > 32
    "k13_d64_lq30": (6, 30, 250, 64, 13),         # first K of the KB = 16 kernels
    "k16_lq32": (4, 32, 200, 128, 16),            # Lq * K = 512, the tensor-core forward's limit
    "lq1_d4_one_chunk": (3, 1, 20, 4, 11),        # W = 6: clamped and duplicate gathered slots, overlapping hills
    "600_docs": (600, 8, 90, 32, 11),             # more documents than 2 x SMs: each CTA walks several documents
    "d356_k16": (3, 20, 400, 356, 16),            # the largest D the backward's shared-memory plan holds at K > 12
}


def _ffma_forward_fits(D, K):
    """The FFMA forward's shared-memory plan (mmb200_tkl_window_scores, tkl.cu) fits in an H100's 227 KB opt-in."""
    KB = 12 if K <= 12 else 16
    dp = (D + 3) & ~3
    dp += 4 if ((dp >> 2) & 1) == 0 else 0
    floats = 2 * 40 * dp + 40 * 41 + 40 * (40 * KB + 1) + 40 * 41 + 3 * 40 + 4 * KB + 16 + 20 * KB + 20 * 40 * KB
    return floats * 4 <= H100_SMEM_OPTIN


def _forward_impls(Lq, D, K):
    return (["simt"] if _ffma_forward_fits(D, K) else []) + (["tcgen05"] if Lq * K <= 512 else [])


def _chunk(d, dm):
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    return (cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous(),
            cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous(), packed, pieces)


def _case(B, Lq, Ld, D, K, seed, zero_padding=True):
    """Random lengths (document 0 full, document 1 a one-row query, document 2 shorter than a chunk), an exact match of
    query row 0 in every document so that the mu = 1 kernel fires, covering kernel set."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    q_len = torch.randint(1, Lq + 1, (B,), generator=g)
    d_len = torch.randint(1, Ld + 1, (B,), generator=g)
    q_len[0], d_len[0] = Lq, Ld
    if B > 2:
        q_len[1], d_len[2] = 1, min(Ld, 17)
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    if zero_padding:
        q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    for b in range(B):
        d[b, int(d_len[b]) // 2] = q[b, 0]
    params = T.covering_params(K, D, g)
    assert interaction.tkl_kernel_set_covers(params["mu"], params["sigma"])
    return {"q": q, "qm": qm, "d": d, "dm": dm, "params": params, "gout": torch.randn(B, generator=g)}


def _cuda_forward_backward(c, sat, chunked):
    """autograd.tkl_interaction forward + backward.  Returns (score, orig, top_idx, grads as in tkl_oracle)."""
    chunks, cmask, packed, pieces = chunked
    qm, cm = c["qm"], cmask
    p = c["params"]
    sp, red = T.sat_args(p, sat)
    leaves = {"q": c["q"], "chunks": chunks, "dense_weight": p["dense_weight"], "sat": sp, "sat_red": red,
              "chunk_scoring": p["chunk_scoring"]}
    leaves = {k: None if v is None else v.to(DEV).requires_grad_(True) for k, v in leaves.items()}
    score, orig, top_idx, _ = autograd.tkl_interaction(
        leaves["q"], qm.to(DEV), leaves["chunks"], cm.to(DEV), packed.to(DEV), pieces, p["mu"].to(DEV),
        p["sigma"].to(DEV), leaves["dense_weight"], sat, leaves["sat"], leaves["sat_red"], leaves["chunk_scoring"])
    score.backward(c["gout"].to(DEV))
    grads = {k: None if v is None else v.grad.detach().cpu() for k, v in leaves.items()}
    return score.detach().cpu(), orig.cpu(), top_idx.cpu(), grads


def _bwd(c, sat, chunked, top_idx, orig, gout=None, masks=None):
    """interaction.tkl_bwd on given windows: (grad_q, grad_chunks, grad_dense, grad_chunk_scoring, grad_sat, grad_red)."""
    chunks, cmask, packed, pieces = chunked
    qm, cm = masks if masks is not None else (c["qm"], cmask)
    p = c["params"]
    sp, red = T.sat_args(p, sat)
    out = interaction.tkl_bwd(c["q"].to(DEV), qm.to(DEV), chunks.to(DEV), cm.to(DEV), packed.to(DEV), pieces,
                              p["mu"].to(DEV), p["sigma"].to(DEV), p["dense_weight"].to(DEV), sat, sp.to(DEV),
                              None if red is None else red.to(DEV), p["chunk_scoring"].to(DEV), top_idx.to(DEV),
                              orig.to(DEV), (c["gout"] if gout is None else gout).to(DEV))
    return tuple(None if t is None else t.cpu() for t in out)


def _check_window_choice(top_idx, sec, what):
    """The kernel's top-3 windows are the oracle's on every document whose competing windows are separated by more than
    1e-3 relative, and on at least 90 % of the documents."""
    ours, ref = top_idx.cpu(), sec["top_non_overlapping_idx"]
    same = (ours == ref).all(dim=1)
    for b in (~same).nonzero().flatten().tolist():
        a, r = sec["orig_score"][b][ours[b]], sec["orig_score"][b][ref[b]]
        assert torch.allclose(a, r, rtol=1e-3), f"{what}: doc {b} picked windows {ours[b].tolist()} over {ref[b].tolist()}"
    assert same.double().mean() >= 0.9, f"{what}: windows agree on {same.double().mean():.2%} of the documents"


def _check_grads(grads, ref, sat, what):
    """Every gradient within GRAD_REL of its tensor's largest reference entry; prints the worst ratio of each."""
    names = ["q", "chunks", "dense_weight", "chunk_scoring", "sat"] + (["sat_red"] if sat == "embedding" else [])
    for name in names:
        a, b = grads[name].double().view(-1), ref[name].double().view(-1)
        assert a.shape == b.shape, f"{what} grad {name}: shape"
        scale = b.abs().max().item()
        err = (a - b).abs().max().item()
        print(f"TKL-BWD {what} grad {name}: max err {err:.3e} / scale {scale:.3e} = {err / max(scale, 1e-300):.2e}")
        assert scale > 0, f"{what} grad {name}: the reference gradient is all zero"
        assert err <= GRAD_REL * scale, f"{what} grad {name}: max err {err:.3e} vs scale {scale:.3e}"


def _check_exact_zeros(grads, ref, qm, cmask, covered, what):
    """Masked query rows, masked chunk rows and chunk rows outside every gathered window carry exactly zero gradient,
    in the kernel and in the reference."""
    for side, g in (("kernel", grads), ("reference", ref)):
        assert (g["q"][qm == 0] == 0).all(), f"{what}: {side} gradient on masked query rows"
        assert (g["chunks"][cmask == 0] == 0).all(), f"{what}: {side} gradient on masked chunk rows"
        assert (g["chunks"][~covered] == 0).all(), f"{what}: {side} gradient on rows no gathered window covers"


def _check_forward(c, sat, chunked, sec, impl, what):
    chunks, cmask, packed, pieces = chunked
    p = c["params"]
    sp, red = T.sat_args(p, sat)
    ws = interaction.tkl_window_scores(c["q"].to(DEV), c["qm"].to(DEV), chunks.to(DEV), cmask.to(DEV), packed.to(DEV),
                                       pieces, p["mu"].to(DEV), p["sigma"].to(DEV), p["dense_weight"].to(DEV), sat,
                                       sp.to(DEV), None if red is None else red.to(DEV), impl=impl)
    score, orig, top_idx, _ = interaction.tkl_top_hills(ws, p["chunk_scoring"].to(DEV))
    assert_close_rel(orig, sec["orig_score"], what=f"{what} orig_score")
    assert ((orig.cpu() == 0) == (sec["orig_score"] == 0)).all(), f"{what}: exact-zero windows"
    _check_window_choice(top_idx, sec, what)
    ref_score = T.conditional_score(sec["orig_score"], p["chunk_scoring"].double(), top_idx)
    assert_close_rel(score, ref_score, what=f"{what} score")


@pytest.mark.parametrize("sat", SATS)
@pytest.mark.parametrize("name", list(SHAPES))
def test_backward_vs_conditional_fp64_autograd(name, sat):
    B, Lq, Ld, D, K = SHAPES[name]
    c = _case(B, Lq, Ld, D, K, seed=B * 1000 + Lq * 10 + K)
    chunked = _chunk(c["d"], c["dm"])
    chunks, cmask, packed, pieces = chunked
    if name == "config5":
        assert pieces == 50 and int(packed.sum()) < B * pieces, "the packing must have dropped trailing chunks"
    if name == "lq1_d4_one_chunk":
        assert pieces == 1
    score, orig, top_idx, grads = _cuda_forward_backward(c, sat, chunked)
    ref_score, sec, ref = T.reference_grads(c["q"], c["qm"], chunks, cmask, packed, pieces, c["params"], sat, c["gout"],
                                            top_idx=top_idx)
    what = f"{name}/{sat}"
    _check_window_choice(top_idx, sec, what)
    assert_close_rel(score, ref_score, what=f"{what} score")
    _check_grads(grads, ref, sat, what)
    _check_exact_zeros(grads, ref, c["qm"], cmask, T.covered_rows(top_idx, packed, pieces), what)
    for impl in _forward_impls(Lq, D, K):
        _check_forward(c, sat, chunked, sec, impl, f"{what} forward {impl}")


@pytest.mark.parametrize("sat", SATS)
def test_window_edges_empty_documents_and_dropped_chunks(sat):
    """Best windows placed by exact matches at 0, 1, W-2 and W-1 (clamped neighbours, duplicate slots); an empty document
    and an empty query (every window a sentinel: no gradient at all, no share of any parameter gradient); a best window
    next to a chunk that the packing dropped."""
    B, Lq, Ld, D, K = 7, 6, 200, 64, 11
    c = _case(B, Lq, Ld, D, K, seed=77, zero_padding=False)
    q, d, qm, dm = c["q"], c["d"], c["qm"], c["dm"]
    qm[:] = 1
    dm[:] = 1
    d.copy_(torch.randn(B, Ld, D, generator=torch.Generator().manual_seed(78)) * 0.4)   # no other exact matches
    W = (5 * 40 - 30) // 2 + 1
    # window w spans positions 2w .. 2w+29: only the target window holds both matches
    targets = {0: (0, 1), 1: (2, 30), 2: (168, 197), 3: (198, 199)}
    best = {0: 0, 1: 1, 2: W - 2, 3: W - 1}
    for b, (p0, p1) in targets.items():
        d[b, p0], d[b, p1] = q[b, 0], q[b, 1]
    dm[4] = 0                                # empty document
    qm[5] = 0                                # empty query
    dm[6, 80:120] = 0                        # chunk slot 2 dropped by the packing ...
    d[6, 78], d[6, 79] = q[6, 0], q[6, 1]    # ... right after the best window's matches
    q.mul_(qm.unsqueeze(-1))
    d.mul_(dm.unsqueeze(-1))
    chunked = _chunk(d, dm)
    chunks, cmask, packed, pieces = chunked
    assert pieces == 5 and not packed[4 * 5:5 * 5].any() and not bool(packed[6 * 5 + 2])
    score, orig, top_idx, grads = _cuda_forward_backward(c, sat, chunked)
    ref_score, sec, ref = T.reference_grads(q, qm, chunks, cmask, packed, pieces, c["params"], sat, c["gout"],
                                            top_idx=top_idx)
    for b, w in best.items():
        assert int(top_idx[b, 0]) == w and int(sec["top_non_overlapping_idx"][b, 0]) == w, f"doc {b}: best window"
    assert (orig[4] == 0).all() and (orig[5] == 0).all() and (sec["orig_score"][4:6] == 0).all()
    nb6 = T.gathered_windows(top_idx[6:7], W)[0].tolist()
    assert any(2 * w + 29 >= 80 and orig[6, w] != 0 for w in nb6), "a gathered window must reach into the dropped chunk"
    what = f"edges/{sat}"
    _check_window_choice(top_idx, sec, what)
    assert_close_rel(score, ref_score, what=f"{what} score")
    _check_grads(grads, ref, sat, what)
    _check_exact_zeros(grads, ref, qm, cmask, T.covered_rows(top_idx, packed, pieces), what)
    assert score[4] == 0 and score[5] == 0
    assert (grads["q"][4:6] == 0).all()
    # the two empty documents contribute exactly nothing: the batch without them gives bit-identical gradients
    keep = [0, 1, 2, 3, 6]
    full = _bwd(c, sat, chunked, top_idx, orig)
    sub = {"q": q[keep], "qm": qm[keep], "params": c["params"], "gout": c["gout"][keep]}
    sub_chunked = _chunk(d[keep], dm[keep])
    part = _bwd(sub, sat, sub_chunked, top_idx[keep], orig[keep])
    assert torch.equal(full[0][keep], part[0])
    doc5_rows = int(packed[:5 * 5].sum()), int(packed[:6 * 5].sum())
    assert (full[1][doc5_rows[0]:doc5_rows[1]] == 0).all()
    assert torch.equal(torch.cat([full[1][:doc5_rows[0]], full[1][doc5_rows[1]:]]), part[1])
    for i in range(2, 6):
        if full[i] is not None:
            assert torch.equal(full[i], part[i]), f"parameter gradient {i} changed by the empty documents"


@pytest.mark.parametrize("sat", SATS)
def test_documents_sharing_a_cta_match_single_document_runs(sat):
    """B = 600 > 2 x SMs, so every CTA walks several documents and reuses its shared accumulators.  A document's arithmetic
    is confined to one CTA: its gradient rows must be bit-identical to the same document run alone, and the parameter
    gradients equal the sum of the single-document runs."""
    B, Lq, Ld, D, K = SHAPES["600_docs"]
    c = _case(B, Lq, Ld, D, K, seed=600)
    chunked = _chunk(c["d"], c["dm"])
    chunks, cmask, packed, C = chunked
    _, orig, top_idx, _ = _cuda_forward_backward(c, sat, chunked)
    full = _bwd(c, sat, chunked, top_idx, orig)
    starts = torch.cat([torch.zeros(1, dtype=torch.long), packed.view(B, C).sum(1).cumsum(0)])
    summed = [torch.zeros_like(t) if t is not None else None for t in full[2:]]
    for b in range(B):
        r0, r1 = int(starts[b]), int(starts[b + 1])
        one = {"q": c["q"][b:b + 1], "qm": c["qm"][b:b + 1], "params": c["params"], "gout": c["gout"][b:b + 1]}
        single = _bwd(one, sat, (chunks[r0:r1], cmask[r0:r1], packed[b * C:(b + 1) * C], C), top_idx[b:b + 1],
                      orig[b:b + 1])
        if b in (0, 1, 2, 131, 263, 264, 389, 527, 598, 599):
            assert torch.equal(single[0], full[0][b:b + 1]), f"doc {b}: grad_q differs from the single-document run"
            assert torch.equal(single[1], full[1][r0:r1]), f"doc {b}: grad_chunks differs from the single-document run"
        for acc, t in zip(summed, single[2:]):
            if acc is not None:
                acc += t
    for i, (acc, t) in enumerate(zip(summed, full[2:])):
        if t is not None:
            torch.testing.assert_close(t, acc, rtol=1e-5, atol=1e-6 * acc.abs().max().item(),
                                       msg=lambda m: f"parameter gradient {i}: {m}")


@pytest.mark.parametrize("name", ["config5", "600_docs"])
def test_backward_is_deterministic(name):
    B, Lq, Ld, D, K = SHAPES[name]
    c = _case(B, Lq, Ld, D, K, seed=4242)
    chunked = _chunk(c["d"], c["dm"])
    for sat in SATS:
        _, orig, top_idx, _ = _cuda_forward_backward(c, sat, chunked)
        a = _bwd(c, sat, chunked, top_idx, orig)
        b = _bwd(c, sat, chunked, top_idx, orig)
        for i, (x, y) in enumerate(zip(a, b)):
            assert (x is None and y is None) or torch.equal(x, y), f"{sat}: output {i} differs between two runs"


@pytest.mark.parametrize("sat", SATS)
def test_mask_dtypes_give_identical_gradients(sat):
    """bool, int64 and float32 masks give bit-identical gradients.  The padding rows hold non-zero data here, so the masks
    alone must keep them out: exactly zero gradient on masked rows, the rest against the fp64 reference."""
    B, Lq, Ld, D, K = SHAPES["k12_d44_lq33"]
    c = _case(B, Lq, Ld, D, K, seed=31, zero_padding=False)
    chunked = _chunk(c["d"], c["dm"])
    chunks, cmask, packed, pieces = chunked
    _, orig, top_idx, _ = _cuda_forward_backward(c, sat, chunked)
    outs = [_bwd(c, sat, chunked, top_idx, orig, masks=(c["qm"].to(dt), cmask.to(dt)))
            for dt in (torch.bool, torch.int64, torch.float32)]
    for other in outs[1:]:
        for i, (x, y) in enumerate(zip(outs[0], other)):
            assert (x is None and y is None) or torch.equal(x, y), f"output {i} depends on the mask dtype"
    _, sec, ref = T.reference_grads(c["q"], c["qm"], chunks, cmask, packed, pieces, c["params"], sat, c["gout"],
                                    top_idx=top_idx)
    grads = dict(zip(["q", "chunks", "dense_weight", "chunk_scoring", "sat", "sat_red"], outs[0]))
    what = f"garbage-padding/{sat}"
    _check_window_choice(top_idx, sec, what)
    _check_grads(grads, ref, sat, what)
    _check_exact_zeros(grads, ref, c["qm"], cmask, T.covered_rows(top_idx, packed, pieces), what)


def _synthetic_bwd(B, Lq, D, K, C=1, sat="log"):
    """interaction.tkl_bwd on random inputs and made-up windows (the envelope checks run on the host before any launch)."""
    g = torch.Generator().manual_seed(D + Lq + K)
    W = (C * 40 - 30) // 2 + 1
    q, chunks = torch.randn(B, Lq, D, generator=g), torch.randn(B * C, 40, D, generator=g)
    params = T.covering_params(K, D, g)
    sp, red = T.sat_args(params, sat)
    top_idx = torch.tensor([[0, W - 1, W // 2]] * B)
    orig = torch.rand(B, W, generator=g) + 0.5
    return interaction.tkl_bwd(q.to(DEV), torch.ones(B, Lq, device=DEV), chunks.to(DEV),
                               torch.ones(B * C, 40, device=DEV), torch.ones(B * C, dtype=torch.bool, device=DEV), C,
                               params["mu"].to(DEV), params["sigma"].to(DEV), params["dense_weight"].to(DEV), sat,
                               sp.to(DEV), None if red is None else red.to(DEV), params["chunk_scoring"].to(DEV),
                               top_idx.to(DEV), orig.to(DEV), torch.randn(B, generator=g).to(DEV))


def test_backward_envelope():
    """D = 356 runs (K = 16 in the shape matrix, K = 12 here); D = 360, Lq > 40 and K > 16 are refused on the host, the
    shared-memory limit with the largest D that fits in the message."""
    gq, gc, *_ = _synthetic_bwd(2, 3, 356, 12)
    assert torch.isfinite(gq).all() and torch.isfinite(gc).all() and gc.abs().max() > 0
    with pytest.raises(_lib.MatchmakerB200Error, match=r"D=360 with K=16 .* \(D <= 356 fits with K <= 16\)"):
        _synthetic_bwd(2, 3, 360, 16)
    with pytest.raises(_lib.MatchmakerB200Error, match=r"D=360 with K=12 .* \(D <= 356 fits with K <= 12\)"):
        _synthetic_bwd(2, 3, 360, 12)
    with pytest.raises(_lib.MatchmakerB200Error, match="Lq <= 40"):
        _synthetic_bwd(2, 41, 32, 11)
    with pytest.raises(_lib.MatchmakerB200Error, match="K <= 16"):
        _synthetic_bwd(2, 3, 32, 17)
