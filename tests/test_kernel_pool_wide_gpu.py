"""Kernel-pooling training at BERT widths (512 < D <= 1024, D % 64 == 0): the saving tensor-core forward and the wide
tensor-core backward (csrc/kernel_pool_wide.cu) at every compiled instantiation (tests/kernel_pool_wide_cases.py),
against fp64 autograd of the restatement in tests/kernel_pool_cases.py, with the error measure of
test_kernel_pool_envelope_gpu.py; determinism, CUDA-graph replay, and the rankers built over BERT embeddings.

Before this backward existed, every backward call here raised "kernel_pool backward supports embedding dim <= 512";
test_rankers_train_at_bert_width checks that the FFMA route still does."""
import pytest
import torch

import kernel_pool_cases as C
import kernel_pool_wide_cases as W
from matchmaker_b200 import _lib, autograd, interaction
from oracle import interaction_oracle as O
from test_kernel_pool_envelope_gpu import GRADS, _backward, _check_exact_zeros, _check_forward, _check_grads, _dev, _forward, _inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _train_step(c, args, clamp_min=C.DEFAULT_FLOOR, bias=0.0):
    train = _forward(c, args, clamp_min=clamp_min, bias=bias, save=True)
    return train, _backward(c, args, train["per_kernel_query"], clamp_min=clamp_min, saved=train["saved"])


@pytest.mark.parametrize("gate", [False, True], ids=["plain", "gate"])
@pytest.mark.parametrize("row", W.MATRIX, ids=str)
def test_matrix_forward_and_backward_vs_fp64(row, gate, record_property):
    c = W.row_case(row, gate)
    ref = C.reference(c)
    assert C.floor_margin(ref["aS"], c.qm, C.DEFAULT_FLOOR) > 1e-2
    assert interaction.kernel_pool_train_supported(row.Lq, row.Ld, row.D, row.K)
    args = _inputs(c)
    plain = _forward(c, args, impl="tcgen05")
    _check_forward(plain, ref, c, "tensor-core forward")
    train, got = _train_step(c, args)
    for key in ("score", "per_kernel", "per_kernel_query"):
        assert torch.equal(train[key], plain[key]), f"training forward {key} differs from the inference forward"
    where = f"{W.g_inst(row.K, gate)} D={row.D}"
    _check_grads(got, ref, where, record_property, few=C.few_term_pairs(c.qm))
    _check_exact_zeros(got, c, where)
    if row.empty_doc:
        assert (got["grad_q"][-1] == 0).all() and (got["grad_d"][-1] == 0).all()
    again = _backward(c, args, train["per_kernel_query"], saved=train["saved"])
    for name in GRADS:
        assert (got[name] is None and again[name] is None) or torch.equal(got[name], again[name]), f"{where} {name}: run to run"


@pytest.mark.parametrize("K", W.CLAMP_KS)
def test_clamp_floor_and_bias(K, record_property):
    """IDCM's 1e-4 floor and bias at D = 768: at least 10 % of the live entries below the floor, none within 1 % of it."""
    c = W.clamp_case(K)
    ref = C.reference(c, clamp_min=C.IDCM_FLOOR, bias=0.37)
    assert C.below_floor_fraction(ref["aS"], c.qm, C.IDCM_FLOOR) >= 0.1
    assert C.floor_margin(ref["aS"], c.qm, C.IDCM_FLOOR) > 1e-2
    args = _inputs(c)
    train, got = _train_step(c, args, clamp_min=C.IDCM_FLOOR, bias=0.37)
    _check_forward(train, ref, c, "training forward")
    _check_grads(got, ref, f"clamp {W.g_inst(K, False)}", record_property, few=C.few_term_pairs(c.qm))


def test_cuda_graph_replay_equals_eager():
    """The training step (saving forward + wide backward) captured in a CUDA graph gives the eager step's bits."""
    c = W.row_case(W.MATRIX[1], True)
    args = _inputs(c)
    alpha, gate, gout = _dev(c.alpha), _dev(c.gate), _dev(c.gout)

    def step():
        out = interaction.kernel_pool(*args, alpha=alpha, log_scale=c.log_scale, doc_gate=gate, want_per_kernel=True,
                                      save_for_backward=True)
        res = interaction.kernel_pool_bwd(*args, alpha, out["per_kernel_query"], gout, c.log_scale, doc_gate=gate,
                                          saved=out["saved"])
        return (out["score"], out["per_kernel"]) + tuple(res)

    eager = step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, captured):
        assert torch.equal(a, b)


def test_empty_batch():
    """B = 0 at D = 768: empty per-pair gradients, zero weight and alpha gradients."""
    c = C.make_case(1, 5, 20, 768, 11, seed=6, gate=True)
    c.q, c.d, c.qm, c.dm, c.gate, c.gout = c.q[:0], c.d[:0], c.qm[:0], c.dm[:0], c.gate[:0], c.gout[:0]
    args = _inputs(c)
    train, got = _train_step(c, args)
    assert train["score"].shape == (0,) and train["saved"].numel() == 0
    assert got["grad_q"].shape == (0, 5, 768) and got["grad_d"].shape == (0, 20, 768) and got["grad_gate"].shape == (0, 20)
    assert torch.equal(got["grad_weight"].cpu(), torch.zeros(11)) and torch.equal(got["grad_alpha"].cpu(), torch.zeros(11))
    cq, cw, ca = _dev(c.q).requires_grad_(True), _dev(c.weight).requires_grad_(True), _dev(c.alpha).requires_grad_(True)
    score, _ = autograd.kernel_pool(cq, *args[1:6], cw, ca, c.log_scale)
    assert score.grad_fn.tc
    score.sum().backward()
    assert torch.equal(cw.grad.cpu(), torch.zeros(11)) and torch.equal(ca.grad.cpu(), torch.zeros(11))


# --- the rankers over BERT-width embeddings ---------------------------------------------------------------------------

TK_MU = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
TK_SIGMA = [0.1] * 11


def _model(name, D):
    from matchmaker_b200.rankers import get_model_class
    if name == "KNRM":
        return get_model_class("knrm").from_config({"knrm_kernels": 11}, D)
    cfg = {"tk_kernels_mu": TK_MU, "tk_kernels_sigma": TK_SIGMA, "tk_att_heads": 8, "tk_att_layer": 1, "tk_att_ff_dim": 256,
           "max_doc_length": 200, "tk_use_diff_posencoding": True, "tk_mix_hybrid_context": True, "tk_att_proj_dim": 32}
    return get_model_class("TK" if name == "ECAI20_TK" else "TK_Sparse").from_config(cfg, D)


class _Tap:
    """Wraps autograd.kernel_pool: keeps its inputs (retaining the gradients of the non-leaf ones) and its route."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def __call__(self, q, d, q_mask, d_mask, mu, sigma, weight, alpha=None, log_scale=1.0, doc_gate=None, **kw):
        for t in (q, d, doc_gate):
            if t is not None and t.requires_grad and not t.is_leaf:
                t.retain_grad()
        out = self.inner(q, d, q_mask, d_mask, mu, sigma, weight, alpha, log_scale, doc_gate, **kw)
        self.calls.append(dict(q=q, d=d, qm=q_mask, dm=d_mask, mu=mu, sigma=sigma, weight=weight, alpha=alpha,
                               log_scale=log_scale, gate=doc_gate, tc=out[0].grad_fn.tc))
        return out


@pytest.mark.parametrize("name", ["ECAI20_TK", "KNRM", "CIKM20_TK_Sparse"])
def test_rankers_train_at_bert_width(name, monkeypatch, record_property):
    """The ranker at D = 768 runs forward and loss.backward() on the tensor-core training pair, and the gradients that
    reach the interaction's inputs and parameters are fp64 autograd's of the oracle function (kernel_pool_knrm /
    _tk / _tk_sparse) on the same inputs.  The FFMA route (autograd.KP_TRAIN_IMPL = "simt") still refuses D = 768."""
    torch.manual_seed(31)
    D, B, Lq, Ld = 768, 4, 12, 90
    m = _model(name, D).to(DEV)
    c = C.make_case(B, Lq, Ld, D, 11, seed=41)
    c.d = W.no_exact_matches(c.d, 41)   # KNRM scores the raw embeddings with its sigma = 1e-4 kernel
    q, d, qm, dm = _dev(c.q).requires_grad_(True), _dev(c.d).requires_grad_(True), _dev(c.qm), _dev(c.dm)
    gout = _dev(c.gout)
    tap = _Tap(autograd.kernel_pool)
    monkeypatch.setattr(autograd, "kernel_pool", tap)
    out = m(q, d, qm, dm)
    score = out[0] if isinstance(out, tuple) else out
    (score * gout).sum().backward()
    (call,) = tap.calls
    assert call["tc"], "the ranker did not take the tensor-core training pair"
    # fp64 autograd of the oracle function on the interaction's inputs
    x = {k: None if call[k] is None else call[k].detach().double().cpu().requires_grad_(True)
         for k in ("q", "d", "gate")}
    w64 = call["weight"].detach().double().cpu().view(-1).requires_grad_(True)
    a64 = None if call["alpha"] is None else call["alpha"].detach().double().cpu().view(-1).requires_grad_(True)
    qm64, dm64 = qm.double().cpu(), dm.double().cpu()
    mu64, sg64 = call["mu"].double().cpu().view(-1), call["sigma"].double().cpu().view(-1)
    if name == "KNRM":
        s64, _ = O.kernel_pool_knrm(x["q"], x["d"], qm64, dm64, mu64, sg64, w64)
    elif name == "ECAI20_TK":
        s64, _ = O.kernel_pool_tk(x["q"], x["d"], qm64, dm64, mu64, sg64, a64, w64)
    else:
        s64, _ = O.kernel_pool_tk_sparse(x["q"], x["d"], qm64, dm64, x["gate"], mu64, sg64, a64, w64)
    s64.backward(c.gout.double())
    assert (score.detach().double().cpu() - s64.detach()).abs().max() <= 1e-3 * s64.abs().max() + 1e-6
    got = {"grad_q": call["q"].grad, "grad_d": call["d"].grad, "grad_weight": call["weight"].grad.view(-1),
           "grad_alpha": None if a64 is None else call["alpha"].grad.view(-1),
           "grad_gate": None if x["gate"] is None else call["gate"].grad}
    ref = {"grad_q": x["q"].grad, "grad_d": x["d"].grad, "grad_weight": w64.grad, "grad_alpha": None if a64 is None else a64.grad,
           "grad_gate": None if x["gate"] is None else x["gate"].grad}
    # the magnitudes the tf32 contractions summed (kernel_pool_cases.TF32_SUMMED), from the same restatement
    case = C.Case(x["q"].detach(), x["d"].detach(), qm64.float(), dm64.float(), mu64.float(), sg64.float(),
                  None if a64 is None else a64.detach().float(), w64.detach().float(),
                  None if x["gate"] is None else x["gate"].detach().float(), c.gout, call["log_scale"])
    summed = C.reference(case)
    ref["summed_q"], ref["summed_d"] = summed["summed_q"], summed["summed_d"]
    _check_grads(got, ref, f"{name} D={D}", record_property, few=C.few_term_pairs(c.qm))
    params = [p for p in m.parameters() if p.requires_grad]
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in params)
    # the FFMA backward stops at D = 512
    monkeypatch.setattr(autograd, "KP_TRAIN_IMPL", "simt")
    m.zero_grad()
    out = m(q, d, qm, dm)
    score = out[0] if isinstance(out, tuple) else out
    with pytest.raises(_lib.MatchmakerB200Error, match="512"):
        score.sum().backward()
