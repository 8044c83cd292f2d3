"""TKL at BERT widths: the wide backward (mmb200_tkl_bwd_wide, tkl_bwd_wide_*_kernel in csrc/tkl_bwd.cu) against fp64
autograd of the oracle restatement with the top-3 window choice conditioned on the kernel's (tests/tkl_oracle.py), its
agreement with the one-CTA-per-document backward where both run, determinism, graph capture and routing; the window-score
forward at D > 356, padded and store; a TKL_sigir20 training step at D = 768; the refusals."""
import copy

import pytest
import torch

import tkl_oracle as T
from conftest import assert_close_rel
from matchmaker_b200 import _lib, autograd, interaction
from matchmaker_b200.rankers.tkl import TKL_sigir20
from oracle import interaction_oracle as O
from test_tkl_bwd_gpu import GRAD_REL, _check_exact_zeros, _check_grads, _check_window_choice, _chunk

pytestmark = pytest.mark.gpu
DEV = "cuda"
SATS = ["embedding", "log"]
NAMES = ["q", "chunks", "dense_weight", "chunk_scoring", "sat", "sat_red"]

# (B, Lq, Ld, D, K) and what each shape exercises.  Lq * K > 512 has no forward past the FFMA kernel's plan: there the
# backward runs on the oracle's own windows and orig_score.
SHAPES = {
    "d360_k12_lq30": (16, 30, 400, 360, 12),        # first D past the one-CTA plan, last K of the KB = 12 kernels
    "d384_k11_minilm": (16, 30, 600, 384, 11),      # MiniLM width, the reference's kernel count
    "d516_k13_lq33": (6, 33, 300, 516, 13),         # a partial feature block (516 = 8 x 64 + 4), first K of KB = 16
    "d384_k16_lq33": (6, 33, 250, 384, 16),         # Lq * K = 528 > 512: no forward, given windows
    "d768_k16_lq40": (4, 40, 300, 768, 16),         # bert-base, Lq = 40, Lq * K = 640: given windows
    "d768_k11_c50": (3, 30, 2000, 768, 11),         # C = 50, trailing chunk slots dropped
    "d768_b300": (300, 8, 90, 768, 11),             # more than 2 x 132 documents
    "d1020_k1_lq1_c1": (5, 1, 20, 1020, 1),         # W = 6: clamped and duplicate windows, overlapping hills; K = 1
    "d1024_k12_lq40": (16, 40, 500, 1024, 12),      # the edge, bert-large
    "d1024_k13_lq40_b1": (1, 40, 1000, 1024, 13),   # one document, Lq * K = 520: given windows
}


def _params(K, D, g):
    p = T.covering_params(K, D, g)
    if K == 1:   # one kernel wide enough to cover [-1, 1] alone
        p["mu"], p["sigma"] = torch.tensor([0.0]), torch.tensor([0.5])
    return p


def _case(B, Lq, Ld, D, K, seed):
    """Random lengths (document 0 full, document 1 a one-row query, document 2 shorter than a chunk: fewer than three
    non-sentinel windows), padding zeroed, an exact match of query row 0 in every document, a covering kernel set."""
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
    q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    for b in range(B):
        d[b, int(d_len[b]) // 2] = q[b, 0]
    params = _params(K, D, g)
    assert interaction.tkl_kernel_set_covers(params["mu"], params["sigma"])
    return {"q": q, "qm": qm, "d": d, "dm": dm, "params": params, "gout": torch.randn(B, generator=g)}


def _args(c, sat, chunked, top_idx, orig, gout=None):
    chunks, cmask, packed, pieces = chunked
    p = c["params"]
    sp, red = T.sat_args(p, sat)
    return (c["q"].to(DEV), c["qm"].to(DEV), chunks.to(DEV), cmask.to(DEV), packed.to(DEV), pieces, p["mu"].to(DEV),
            p["sigma"].to(DEV), p["dense_weight"].to(DEV), sat, sp.to(DEV), None if red is None else red.to(DEV),
            p["chunk_scoring"].to(DEV), top_idx.to(DEV), orig.to(DEV), (c["gout"] if gout is None else gout).to(DEV))


def _run(fn, *args):
    return dict(zip(NAMES, (None if t is None else t.cpu() for t in fn(*args))))


def _forward(c, sat, chunked):
    chunks, cmask, packed, pieces = chunked
    p = c["params"]
    sp, red = T.sat_args(p, sat)
    ws = interaction.tkl_window_scores(c["q"].to(DEV), c["qm"].to(DEV), chunks.to(DEV), cmask.to(DEV), packed.to(DEV),
                                       pieces, p["mu"].to(DEV), p["sigma"].to(DEV), p["dense_weight"].to(DEV), sat,
                                       sp.to(DEV), None if red is None else red.to(DEV))
    return ws, interaction.tkl_top_hills(ws, p["chunk_scoring"].to(DEV))


def _windows(c, sat, chunked, Lq, K):
    """(top_idx, orig_score): the kernels' where the forward takes the shape, else the fp64 oracle's."""
    if Lq * K <= 512:
        _, (_, orig, top_idx, _) = _forward(c, sat, chunked)
        return top_idx.cpu(), orig.cpu()
    chunks, cmask, packed, pieces = chunked
    _, sec, _ = T.reference_grads(c["q"], c["qm"], chunks, cmask, packed, pieces, c["params"], sat, c["gout"])
    return sec["top_non_overlapping_idx"], sec["orig_score"].float()


@pytest.mark.parametrize("sat", SATS)
@pytest.mark.parametrize("name", list(SHAPES))
def test_wide_backward_vs_conditional_fp64_autograd(name, sat):
    B, Lq, Ld, D, K = SHAPES[name]
    c = _case(B, Lq, Ld, D, K, seed=B * 1000 + Lq * 10 + K + D)
    chunked = _chunk(c["d"], c["dm"])
    chunks, cmask, packed, pieces = chunked
    if name == "d768_k11_c50":
        assert pieces == 50 and int(packed.sum()) < B * pieces, "the packing must have dropped chunk slots"
    if name == "d1020_k1_lq1_c1":
        assert pieces == 1
    top_idx, orig = _windows(c, sat, chunked, Lq, K)
    grads = _run(interaction.tkl_bwd_wide, *_args(c, sat, chunked, top_idx, orig))
    _, sec, ref = T.reference_grads(c["q"], c["qm"], chunks, cmask, packed, pieces, c["params"], sat, c["gout"],
                                    top_idx=top_idx)
    what = f"{name}/{sat}"
    _check_window_choice(top_idx, sec, what)
    _check_grads(grads, ref, sat, what)
    _check_exact_zeros(grads, ref, c["qm"], cmask, T.covered_rows(top_idx, packed, pieces), what)


@pytest.mark.parametrize("sat", SATS)
@pytest.mark.parametrize("D", [32, 300, 356])
def test_wide_backward_agrees_with_the_one_cta_backward(D, sat):
    """Where both run, the two backward kernels agree within the bar, and each is held to fp64."""
    B, Lq, Ld, K = 12, 30, 700, 11
    c = _case(B, Lq, Ld, D, K, seed=D + 7)
    chunked = _chunk(c["d"], c["dm"])
    chunks, cmask, packed, pieces = chunked
    assert interaction.tkl_bwd_route(Lq, D, K) == "tkl_bwd"
    top_idx, orig = _windows(c, sat, chunked, Lq, K)
    args = _args(c, sat, chunked, top_idx, orig)
    wide, one = _run(interaction.tkl_bwd_wide, *args), _run(interaction.tkl_bwd, *args)
    _, sec, ref = T.reference_grads(c["q"], c["qm"], chunks, cmask, packed, pieces, c["params"], sat, c["gout"],
                                    top_idx=top_idx)
    _check_grads(wide, ref, sat, f"D{D}/{sat} wide")
    _check_grads(one, ref, sat, f"D{D}/{sat} one-CTA")
    _check_grads(wide, one, sat, f"D{D}/{sat} wide vs one-CTA")


@pytest.mark.parametrize("D", [384, 1024])
def test_wide_backward_is_deterministic(D):
    B, Lq, Ld, K = 16, 30, 1100, 11
    c = _case(B, Lq, Ld, D, K, seed=4243)
    chunked = _chunk(c["d"], c["dm"])
    for sat in SATS:
        top_idx, orig = _windows(c, sat, chunked, Lq, K)
        args = _args(c, sat, chunked, top_idx, orig)
        a, b = _run(interaction.tkl_bwd_wide, *args), _run(interaction.tkl_bwd_wide, *args)
        for k in NAMES:
            assert (a[k] is None and b[k] is None) or torch.equal(a[k], b[k]), f"{sat}: {k} differs between two runs"


def _leaves(c, sat, chunked):
    chunks, _, _, _ = chunked
    p = c["params"]
    sp, red = T.sat_args(p, sat)
    leaves = {"q": c["q"], "chunks": chunks, "dense_weight": p["dense_weight"], "sat": sp, "sat_red": red,
              "chunk_scoring": p["chunk_scoring"]}
    return {k: None if v is None else v.to(DEV).clone().requires_grad_(True) for k, v in leaves.items()}


def _autograd_step(c, sat, chunked, leaves, gout):
    _, cmask, packed, pieces = chunked
    p = c["params"]
    score, orig, top_idx, _ = autograd.tkl_interaction(
        leaves["q"], c["qm_dev"], leaves["chunks"], c["cm_dev"], c["packed_dev"], pieces, c["mu_dev"], c["sigma_dev"],
        leaves["dense_weight"], sat, leaves["sat"], leaves["sat_red"], leaves["chunk_scoring"])
    live = [v for v in leaves.values() if v is not None]
    return (score, orig, top_idx) + torch.autograd.grad((score * gout).sum(), live)


def _device_case(c, chunked):
    _, cmask, packed, _ = chunked
    c.update(qm_dev=c["qm"].to(DEV), cm_dev=cmask.to(DEV), packed_dev=packed.to(DEV),
             mu_dev=c["params"]["mu"].to(DEV), sigma_dev=c["params"]["sigma"].to(DEV))


@pytest.mark.parametrize("sat", SATS)
def test_graph_replay_of_the_autograd_step_gives_the_eager_bits(sat):
    B, Lq, Ld, D, K = 16, 30, 1100, 768, 11
    c = _case(B, Lq, Ld, D, K, seed=99)
    chunked = _chunk(c["d"], c["dm"])
    _device_case(c, chunked)
    gout = c["gout"].to(DEV)
    eager = _autograd_step(c, sat, chunked, _leaves(c, sat, chunked), gout)
    # each run gets leaves of its own: a leaf whose gradient accumulator was made on another stream would make the
    # captured backward wait on that stream
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # warm-up on a side stream, as graph capture requires
        _autograd_step(c, sat, chunked, _leaves(c, sat, chunked), gout)
    torch.cuda.current_stream().wait_stream(side)
    leaves = _leaves(c, sat, chunked)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _autograd_step(c, sat, chunked, leaves, gout)
    graph.replay()
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(eager, captured)):
        assert torch.equal(x, y), f"output {i} of the replayed step differs from the eager step"


@pytest.mark.parametrize("sat", SATS)
@pytest.mark.parametrize("D", [300, 768])
def test_autograd_routes_by_width(D, sat):
    """autograd.tkl_interaction gives exactly the bits of the backward its route names: the one-CTA kernel at D <= 356,
    the wide kernel at D = 768."""
    B, Lq, Ld, K = 8, 30, 600, 11
    c = _case(B, Lq, Ld, D, K, seed=D)
    chunked = _chunk(c["d"], c["dm"])
    _device_case(c, chunked)
    route = interaction.tkl_bwd_route(Lq, D, K)
    assert route == ("tkl_bwd" if D <= 356 else "tkl_bwd_wide")
    leaves = _leaves(c, sat, chunked)
    _, orig, top_idx, *grads = _autograd_step(c, sat, chunked, leaves, c["gout"].to(DEV))
    direct = getattr(interaction, route)(*_args(c, sat, chunked, top_idx, orig))
    direct = dict(zip(NAMES, direct))
    live = [k for k in leaves if leaves[k] is not None]
    for k, gk in zip(live, grads):
        assert torch.equal(gk, direct[k].view_as(gk)), f"{k}: autograd is not the {route} backward"


def _store_slots(packed, pieces):
    """The slot table [B, C] of the padded batch: the packed index of every slot, -1 where the packing dropped it."""
    pk = packed.view(-1).bool()
    idx = torch.cumsum(pk.int(), 0) - 1
    return torch.where(pk, idx, torch.full_like(idx, -1)).view(-1, pieces).int()


@pytest.mark.parametrize("sat", SATS)
@pytest.mark.parametrize("D", [360, 768, 1024])
def test_forward_at_bert_widths(D, sat):
    """Padded and store window scores past the one-CTA backward's width: fp64 within 1e-3 of each pair's largest window,
    exact zeros exact, the top-3 windows, and the store bit-identical to the padded path on the same chunks."""
    B, Lq, Ld, K = 16, 30, 1100, 11
    c = _case(B, Lq, Ld, D, K, seed=D * 3 + len(sat))
    chunked = _chunk(c["d"], c["dm"])
    chunks, cmask, packed, pieces = chunked
    ws, (score, orig, top_idx, _) = _forward(c, sat, chunked)
    p = c["params"]
    p64 = {k: v.double() for k, v in p.items()}
    _, sec = O.tkl_interaction(c["q"].double(), c["qm"].double(), chunks.double(), cmask.double(), packed, pieces, p64,
                               sat)
    ref = sec["orig_score"]
    err = (orig.cpu().double() - ref).abs()
    scale = ref.abs().amax(dim=1, keepdim=True)
    assert (err <= 1e-3 * scale).all(), f"D{D}/{sat}: worst window error / pair scale {(err / scale).max():.3e}"
    assert ((orig.cpu() == 0) == (ref == 0)).all(), f"D{D}/{sat}: exact-zero windows"
    _check_window_choice(top_idx, sec, f"D{D}/{sat} forward")
    assert_close_rel(score, T.conditional_score(ref, p64["chunk_scoring"], top_idx), what=f"D{D}/{sat} score")
    sp, red = T.sat_args(p, sat)
    store = interaction.tkl_store_window_scores(
        c["q"].to(DEV), c["qm"].to(DEV), chunks.to(DEV), cmask.to(DEV), _store_slots(packed, pieces).to(DEV),
        torch.arange(B, device=DEV), torch.arange(B, device=DEV), p["mu"].to(DEV), p["sigma"].to(DEV),
        p["dense_weight"].to(DEV), sat, sp.to(DEV), None if red is None else red.to(DEV))
    assert torch.equal(store, ws), f"D{D}/{sat}: the store windows differ from the padded path"


def _ref_model_score(m, q, d, qm, dm, top_idx):
    """TKL_sigir20.forward of ``m`` with the interaction stage replaced by the oracle, conditioned on ``top_idx``."""
    query_ctx, _ = m.forward_representation(q, qm, m.positional_features_q[:, :q.shape[1], :])
    chunks2, cmask2, packed, pieces = m.chunk_documents(d, dm)
    docs_packed, pad_packed = chunks2[packed], cmask2[packed]
    docs_ctx, _ = m.forward_representation(docs_packed, pad_packed,
                                           m.positional_features_d[:, :docs_packed.shape[1], :])
    chunks = docs_ctx[:, m.overlap:-m.overlap, :]
    cmask = pad_packed[:, m.overlap:-m.overlap]
    params = {"mu": m.mu, "sigma": m.sigma, "dense_weight": m.dense.weight.view(-1),
              "chunk_scoring": m.chunk_scoring.view(-1), "sat_emb_reduce1_weight": m.sat_emb_reduce1.weight.view(-1),
              "sat_normer_weight": m.sat_normer.weight, "sat_normer_bias": m.sat_normer.bias,
              "saturation_linear_weight": m.saturation_linear.weight.view(-1),
              "saturation_linear_bias": m.saturation_linear.bias,
              "saturation_linear2_weight": m.saturation_linear2.weight.view(-1),
              "saturation_linear2_bias": m.saturation_linear2.bias,
              "saturation_linear3_weight": m.saturation_linear3.weight.view(-1),
              "saturation_linear3_bias": m.saturation_linear3.bias, "kernel_mult0": m.kernel_mult[0].reshape(-1)}
    _, sec = O.tkl_interaction(query_ctx, qm, chunks, cmask, packed, pieces, params, m.saturation_type)
    return T.conditional_score(sec["orig_score"], params["chunk_scoring"], top_idx), sec


@pytest.mark.parametrize("sat", SATS)
def test_tkl_ranker_training_step_at_bert_base_width(sat):
    """A TKL_sigir20 training step at D = 768 (12 heads, 1 layer): every parameter gradient and both input-embedding
    gradients against an fp64 copy of the model whose interaction stage is the oracle, on the kernel's windows."""
    torch.manual_seed(768)
    B, Lq, Ld, D = 4, 30, 300, 768
    mu = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
    m = TKL_sigir20(D, mu, [0.001] + [0.1] * 10, 12, 1, 100, 2000, True, True, sat)
    with torch.no_grad():   # parameters away from their constant initial values, so that every gradient is exercised
        for n, prm in m.named_parameters():
            if prm.requires_grad and n not in ("positional_features_q", "positional_features_d"):
                prm.add_(torch.randn_like(prm) * 0.05)
    g = torch.Generator().manual_seed(769)
    q, d = torch.randn(B, Lq, D, generator=g), torch.randn(B, Ld, D, generator=g)
    q_len, d_len = torch.tensor([Lq, 7, 19, 1]), torch.tensor([Ld, 120, 17, 263])
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    gout = torch.randn(B, generator=g)
    m64 = copy.deepcopy(m).double().train()
    m = m.to(DEV).train()
    qd, dd = q.to(DEV).requires_grad_(True), d.to(DEV).requires_grad_(True)
    assert interaction.tkl_bwd_route(Lq, D, len(mu)) == "tkl_bwd_wide"
    score, sec_k = m(qd, dd, qm.to(DEV), dm.to(DEV), output_secondary_output=True)
    (score * gout.to(DEV)).sum().backward()
    top_idx = sec_k["top_non_overlapping_idx"].cpu()
    q64, d64 = q.double().requires_grad_(True), d.double().requires_grad_(True)
    ref_score, sec = _ref_model_score(m64, q64, d64, qm.double(), dm.double(), top_idx)
    _check_window_choice(top_idx, sec, f"ranker/{sat}")
    assert_close_rel(score, ref_score, what=f"ranker/{sat} score")
    (ref_score * gout.double()).sum().backward()
    pairs = [(n, p.grad, p64.grad) for (n, p), (_, p64) in zip(m.named_parameters(), m64.named_parameters())]
    pairs += [("input q", qd.grad, q64.grad), ("input d", dd.grad, d64.grad)]
    checked = 0
    for n, a, b in pairs:
        if b is None or not b.any():
            assert a is None or not a.any(), f"{n}: the fp64 model gives it no gradient, the kernel step does"
            continue
        err = (a.cpu().double() - b).abs().max().item()
        scale = b.abs().max().item()
        assert err <= GRAD_REL * scale, f"ranker/{sat} grad {n}: max err {err:.3e} vs scale {scale:.3e}"
        checked += 1
    assert checked >= 10


def _synthetic_wide(B, Lq, D, K, C=1, sat="log"):
    g = torch.Generator().manual_seed(D + Lq + K)
    W = (C * 40 - 30) // 2 + 1
    q, chunks = torch.randn(B, Lq, D, generator=g), torch.randn(B * C, 40, D, generator=g)
    params = T.covering_params(K, D, g)
    sp, red = T.sat_args(params, sat)
    return interaction.tkl_bwd_wide(q.to(DEV), torch.ones(B, Lq, device=DEV), chunks.to(DEV),
                                    torch.ones(B * C, 40, device=DEV), torch.ones(B * C, dtype=torch.bool, device=DEV),
                                    C, params["mu"].to(DEV), params["sigma"].to(DEV), params["dense_weight"].to(DEV),
                                    sat, sp.to(DEV), None if red is None else red.to(DEV),
                                    params["chunk_scoring"].to(DEV), torch.tensor([[0, W - 1, W // 2]] * B).to(DEV),
                                    (torch.rand(B, W, generator=g) + 0.5).to(DEV), torch.randn(B, generator=g).to(DEV))


def test_wide_backward_envelope():
    """D = 1024 runs; D = 1028, D = 770, Lq = 41 and K = 17 are refused on the host with the envelope in the message."""
    for sat in SATS:
        gq, gc, *_ = _synthetic_wide(2, 3, 1024, 16, sat=sat)
        assert torch.isfinite(gq).all() and torch.isfinite(gc).all() and gc.abs().max() > 0
    for B, Lq, D, K in ((2, 3, 1028, 12), (2, 3, 770, 12), (2, 41, 768, 11), (2, 3, 768, 17)):
        with pytest.raises(_lib.MatchmakerB200Error, match=r"TKL wide backward: .*outside its envelope"):
            _synthetic_wide(B, Lq, D, K)
        assert interaction.tkl_bwd_route(Lq, D, K) is None
