"""Kernel-pooling variants of SURVEY 8(f) row 3 against golden vectors recorded from the reference's own classes
(CIKM20_TK_Sparse, Conv_KNRM) and against the oracle restatement (IDCM's ESM scorer): the document-term gate, the
n x n n-gram cross match, the 1e-4 clamp floor + bias.  Forward on both kernels (tensor-core / FFMA), gradients against fp64
autograd of the oracle."""
import pytest
import torch

from conftest import assert_close_rel, load_golden
from matchmaker_b200 import autograd, interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
IMPLS = ["simt", "tcgen05"]


def _c(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


@pytest.mark.parametrize("impl", IMPLS)
def test_golden_tk_sparse_interaction(impl):
    g = load_golden("tk_sparse")
    out = interaction.kernel_pool(*_c(g["q_ctx"], g["d_ctx"], g["q_mask"], g["d_mask"], g["mu"], g["sigma"], g["weight"]),
                                  alpha=g["alpha"].to(DEV), log_scale=1.0, want_per_kernel=True, impl=impl,
                                  doc_gate=g["doc_gate"].to(DEV))
    assert_close_rel(out["per_kernel"], g["per_kernel"], what="per_kernel")
    assert_close_rel(out["score"], g["score"], what="score")


def test_tk_sparse_class_matches_reference_golden():
    from matchmaker_b200.rankers.tk_sparse import CIKM20_TK_Sparse
    g = load_golden("tk_sparse")
    emb, heads, layers, proj, ff, max_len = [int(x) for x in g["cfg"]]
    m = CIKM20_TK_Sparse(emb, g["mu"].tolist(), g["sigma"].tolist(), heads, layers, proj, ff, max_len, True)
    missing, unexpected = m.load_state_dict({k[4:]: v for k, v in g.items() if k.startswith("sd__")}, strict=True)
    assert not missing and not unexpected
    m = m.to(DEV).eval()
    with torch.no_grad():
        score, stop = m(*_c(g["q"], g["d"], g["q_mask"], g["d_mask"]))
    assert_close_rel(stop, g["document_stop_words"], what="document_stop_words")
    assert_close_rel(score, g["score"], rel=2e-3, what="TK-Sparse class score")


@pytest.mark.parametrize("impl", IMPLS)
def test_gate_seeded_vs_oracle_cfg2_shape(impl):
    """BASELINE config-2 token shape (Lq 30, Ld 200, D 300, 21 kernels) with a gate that is 0 for a third of the terms,
    fractional elsewhere; also clamp_min = 1e-4 and a bias (IDCM's ESM constants) on the same inputs."""
    mu, sg = O.tk_21_kernels()
    mu, sg = torch.tensor(mu), torch.tensor(sg)
    g = torch.Generator().manual_seed(9)
    w = (torch.rand(21, generator=g) - 0.5) * 0.03
    alpha = torch.rand(21, generator=g) + 0.5
    q, d, qm, dm = O.synth_kernel_pool_inputs(9, 30, 200, 300, seed=77)
    gate = torch.relu(torch.randn(9, 200, generator=g) + 0.4) * dm
    ref, sec = O.kernel_pool_tk_sparse(q, d, qm, dm, gate, mu, sg, alpha, w)
    out = interaction.kernel_pool(*_c(q, d, qm, dm, mu, sg, w), alpha=alpha.to(DEV), want_per_kernel=True, impl=impl,
                                  doc_gate=gate.to(DEV))
    assert_close_rel(out["per_kernel"], sec["per_kernel"], what="per_kernel (gate)")
    qn, dn = torch.nn.functional.normalize(q, dim=-1), torch.nn.functional.normalize(d, dim=-1)
    bias = torch.tensor([0.37])
    ref_esm = O.idcm_esm_patch_scores(qn, dn, qm, dm, mu, sg, alpha, w, bias)
    out_esm = interaction.kernel_pool(*_c(qn, dn, qm, dm, mu, sg, w), alpha=alpha.to(DEV), want_per_kernel=True, impl=impl,
                                      clamp_min=1e-4, bias=0.37)
    assert_close_rel(out_esm["score"], ref_esm, what="ESM score (clamp 1e-4 + bias)")


@pytest.mark.parametrize("impl", IMPLS)
def test_golden_conv_knrm_cross_match(impl):
    g = load_golden("conv_knrm")
    n = int(g["cfg"][1])
    K = int(g["cfg"][2])
    w = g["dense_weight"].view(n * n, K)
    total = torch.zeros(g["score"].shape[0], device=DEV)
    blk = 0
    for i in range(n):
        for t in range(n):
            out = interaction.kernel_pool(*_c(g[f"qg{i}"], g[f"dg{t}"], g["q_mask"], g["d_mask"], g["mu"], g["sigma"], w[blk]),
                                          alpha=None, log_scale=0.01, want_per_kernel=True, impl=impl)
            assert_close_rel(out["per_kernel"], g["all_grams"][:, blk * K:(blk + 1) * K], what=f"per_kernel block {blk}")
            total += out["score"]
            blk += 1
    assert_close_rel(total, g["score"], rel=2e-3, what="conv-knrm score")


def test_conv_knrm_class_matches_reference_golden():
    from matchmaker_b200.rankers.conv_knrm import Conv_KNRM
    g = load_golden("conv_knrm")
    emb, n, K, conv_out = [int(x) for x in g["cfg"]]
    m = Conv_KNRM(emb, n, K, conv_out)
    missing, unexpected = m.load_state_dict({k[4:]: v for k, v in g.items() if k.startswith("sd__")}, strict=True)
    assert not missing and not unexpected
    m = m.to(DEV).eval()
    with torch.no_grad():
        score = m(*_c(g["q"], g["d"], g["q_mask"], g["d_mask"]))
    assert_close_rel(score, g["score"], rel=2e-3, what="Conv-KNRM class score")
    m.train()
    s = m(*_c(g["q"], g["d"], g["q_mask"], g["d_mask"]))
    s.sum().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())


@pytest.mark.parametrize("train_impl", ["auto", "simt"])   # tensor-core training pair / FFMA backward
@pytest.mark.parametrize("shape", [(4, 9, 37, 32), (5, 30, 200, 300), (150, 12, 130, 64)])
def test_gate_backward_vs_fp64_autograd_of_oracle(shape, train_impl, monkeypatch):
    monkeypatch.setattr(autograd, "KP_TRAIN_IMPL", train_impl)
    B, Lq, Ld, D = shape
    K = 11
    g = torch.Generator().manual_seed(3)
    mu = torch.tensor([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9])
    sg = torch.full((K,), 0.1)
    w = torch.randn(K, generator=g) * 0.1
    alpha = torch.rand(K, generator=g) + 0.5
    q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=5)
    gate = (torch.rand(B, Ld, generator=g) * 1.5) * dm
    gate[0, 3] = 0.0
    gout = torch.randn(B, generator=g)
    q64, d64 = q.double().requires_grad_(True), d.double().requires_grad_(True)
    g64, w64, a64 = gate.double().requires_grad_(True), w.double().requires_grad_(True), alpha.double().requires_grad_(True)
    s64, _ = O.kernel_pool_tk_sparse(q64, d64, qm.double(), dm.double(), g64, mu.double(), sg.double(), a64, w64)
    s64.backward(gout.double())
    cq, cd = q.to(DEV).requires_grad_(True), d.to(DEV).requires_grad_(True)
    cg, cw, ca = gate.to(DEV).requires_grad_(True), w.to(DEV).requires_grad_(True), alpha.to(DEV).requires_grad_(True)
    score, _ = autograd.kernel_pool(cq, cd, qm.to(DEV), dm.to(DEV), mu.to(DEV), sg.to(DEV), cw, ca, 1.0, doc_gate=cg)
    assert score.grad_fn.tc == (train_impl == "auto")
    assert_close_rel(score, s64.float(), what="score")
    score.backward(gout.to(DEV))

    def close(a, b, what):
        a, b = a.double().cpu(), b.double()
        scale = b.abs().max().item()
        err = (a - b).abs().max().item()
        assert err <= 2e-3 * scale + 1e-9, f"{what}: max err {err:.3e} vs scale {scale:.3e}"

    close(cg.grad, g64.grad, "grad gate")
    close(cq.grad, q64.grad, "grad q")
    close(cd.grad, d64.grad, "grad d")
    close(cw.grad, w64.grad, "grad weight")
    close(ca.grad, a64.grad, "grad alpha")
