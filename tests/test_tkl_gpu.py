"""TKL interaction kernels vs the golden vectors of the reference's TKL_sigir20 and the oracle."""
import pytest
import torch

from conftest import assert_close_rel, load_golden
from matchmaker_b200 import interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _sat_args(params, sat):
    if sat == "embedding":
        p = torch.cat([params["sat_normer_weight"], params["sat_normer_bias"], params["saturation_linear_weight"],
                       params["saturation_linear_bias"], params["saturation_linear2_weight"],
                       params["saturation_linear2_bias"], params["saturation_linear3_weight"],
                       params["saturation_linear3_bias"]])
        return p, params["sat_emb_reduce1_weight"]
    return params["kernel_mult0"], None


IMPLS = ["simt", "tcgen05"]   # the FFMA kernel (tkl.cu) and the TMA + wgmma kernel (tkl_ts.cu); the impl name is historical


def _run(g, params, sat, impl="auto"):
    sp, red = _sat_args(params, sat)
    ws = interaction.tkl_window_scores(g["q_ctx"].to(DEV), g["q_mask"].to(DEV), g["doc_chunks_ctx"].to(DEV),
                                       g["doc_chunk_mask"].to(DEV), g["packed_indices"].to(DEV), int(g["chunk_pieces"]),
                                       params["mu"].to(DEV), params["sigma"].to(DEV), params["dense_weight"].to(DEV), sat,
                                       sp.to(DEV), None if red is None else red.to(DEV), impl=impl)
    return ws, interaction.tkl_top_hills(ws, params["chunk_scoring"].to(DEV))


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("sat", ["embedding", "log"])
def test_golden_tkl(sat, impl):
    g = load_golden(f"tkl_{sat}")
    params = {k[3:]: v for k, v in g.items() if k.startswith("p__")}
    ws, (score, orig, top_idx, top15) = _run(g, params, sat, impl)
    assert_close_rel(orig, g["orig_score"], what="orig_score")
    assert torch.equal(top_idx.cpu(), g["top_non_overlapping_idx"]), "top-3 window indices must be bit-exact"
    assert_close_rel(top15, g["top_k_non_overlapping"], what="top15")
    assert_close_rel(score, g["score"], what="score")
    # exact-zero windows (fully padded regions) must come out as exact zeros
    assert ((orig.cpu() == 0) == (g["orig_score"] == 0)).all()


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("sat", ["embedding", "log"])
@pytest.mark.parametrize("shape", [(3, 40, 2000, 64), (2, 7, 95, 32), (150, 12, 400, 32), (1, 5, 20, 16), (4, 32, 121, 300)])
def test_seeded_vs_oracle(shape, sat, impl):
    B, Lq, Ld, D = shape
    g = torch.Generator().manual_seed(Ld + Lq)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    q_len = torch.randint(1, Lq + 1, (B,), generator=g)
    d_len = torch.randint(1, Ld + 1, (B,), generator=g)
    d_len[0] = Ld
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    chunks = cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    cmask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    K = 11
    params = {"mu": torch.tensor([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]), "sigma": torch.full((K,), 0.1),
              "dense_weight": torch.randn(K, generator=g) * 0.1, "chunk_scoring": torch.rand(15, generator=g) + 0.5,
              "sat_emb_reduce1_weight": torch.randn(D, generator=g) * 0.3,
              "sat_normer_weight": torch.rand(2, generator=g) + 0.5, "sat_normer_bias": torch.randn(2, generator=g) * 0.1,
              "saturation_linear_weight": torch.randn(2, generator=g) * 0.014, "saturation_linear_bias": torch.tensor([100.0]),
              "saturation_linear2_weight": torch.randn(2, generator=g) * 0.014, "saturation_linear2_bias": torch.tensor([100.0]),
              "saturation_linear3_weight": torch.randn(2, generator=g) * 0.014, "saturation_linear3_bias": torch.tensor([100.0]),
              "kernel_mult0": torch.rand(K, generator=g) + 0.5}
    ref_score, sec = O.tkl_interaction(q, qm, chunks, cmask, packed, pieces, params, sat)
    gd = {"q_ctx": q, "q_mask": qm, "doc_chunks_ctx": chunks, "doc_chunk_mask": cmask, "packed_indices": packed,
          "chunk_pieces": torch.tensor(pieces)}
    ws, (score, orig, top_idx, top15) = _run(gd, params, sat, impl)
    assert_close_rel(orig, sec["orig_score"], what="orig_score")
    assert ((orig.cpu() == 0) == (sec["orig_score"] == 0)).all(), "exact-zero windows"
    same = (top_idx.cpu() == sec["top_non_overlapping_idx"]).all(dim=1)
    # index ties: a different-but-equal-valued window may be picked only if the scores tie within tolerance
    for b in (~same).nonzero().flatten().tolist():
        a = sec["orig_score"][b][top_idx.cpu()[b]]
        r = sec["orig_score"][b][sec["top_non_overlapping_idx"][b]]
        assert torch.allclose(a, r, rtol=1e-3), f"doc {b}: picked windows differ beyond tolerance"
    assert same.float().mean() > 0.9
    assert_close_rel(score.cpu()[same], ref_score[same], what="score")


def _tkl_params(D, g, K=11):
    return {"mu": torch.tensor([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]), "sigma": torch.full((K,), 0.1),
            "dense_weight": torch.randn(K, generator=g) * 0.1, "chunk_scoring": torch.rand(15, generator=g) + 0.5,
            "sat_emb_reduce1_weight": torch.randn(D, generator=g) * 0.05,
            "sat_normer_weight": torch.rand(2, generator=g) + 0.5, "sat_normer_bias": torch.randn(2, generator=g) * 0.1,
            "saturation_linear_weight": torch.randn(2, generator=g) * 0.014, "saturation_linear_bias": torch.tensor([100.0]),
            "saturation_linear2_weight": torch.randn(2, generator=g) * 0.014, "saturation_linear2_bias": torch.tensor([100.0]),
            "saturation_linear3_weight": torch.randn(2, generator=g) * 0.014, "saturation_linear3_bias": torch.tensor([100.0]),
            "kernel_mult0": torch.rand(K, generator=g) + 0.5}


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("sat", ["embedding", "log"])
def test_baseline_cfg5_shape_vs_oracle(sat, impl):
    """BASELINE config 5 token shape (Lq=40, Ld=2000, D=300, 11 kernels), B=20 documents (more than one GPU's share of
    128/8): MSMARCO-document-shaped lengths so that trailing chunks are dropped by the packing (sigir20_tkl.py:159-162),
    one full-length document, one shorter than a window, one empty query row pattern.  Window scores within 1e-3, the
    exact-zero windows exactly zero, the top-3 window ids bit-exact, final score within 1e-3."""
    B, Lq, Ld, D = 20, 40, 2000, 300
    g = torch.Generator().manual_seed(555)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    q_len = torch.randint(3, Lq + 1, (B,), generator=g)
    d_len = (torch.randn(B, generator=g) * 500 + 1100).round().clamp(100, Ld).long()
    d_len[0], d_len[1], d_len[2], d_len[3] = Ld, 17, 40, 1999
    q_len[0], q_len[4] = Lq, 1
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    for b in range(B):   # exact matches so that the mu = 1.0 kernel fires
        d[b, int(d_len[b]) // 2] = q[b, 0]
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    assert pieces == 50 and int(packed.sum()) < B * pieces, "the packing must have dropped trailing chunks"
    chunks = cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    cmask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    params = _tkl_params(D, g)
    ref_score, sec = O.tkl_interaction(q, qm, chunks, cmask, packed, pieces, params, sat)
    gd = {"q_ctx": q, "q_mask": qm, "doc_chunks_ctx": chunks, "doc_chunk_mask": cmask, "packed_indices": packed,
          "chunk_pieces": torch.tensor(pieces)}
    ws, (score, orig, top_idx, top15) = _run(gd, params, sat, impl)
    assert orig.shape == (B, 986)
    assert_close_rel(orig, sec["orig_score"], what="orig_score")
    assert ((orig.cpu() == 0) == (sec["orig_score"] == 0)).all(), "exact-zero windows"
    assert torch.equal(top_idx.cpu(), sec["top_non_overlapping_idx"]), "top-3 window ids must be bit-exact"
    assert_close_rel(top15, sec["top_k_non_overlapping"], what="top15")
    assert_close_rel(score, ref_score, what="score")
    # batch-order independence, bit-exact: a document's windows do not depend on its neighbours or on how the
    # documents are split over CTAs
    perm = torch.randperm(B, generator=g)
    cd2p, cp2p, packedp, _ = O.tkl_chunk_documents(d[perm], dm[perm])
    gp = {"q_ctx": q[perm], "q_mask": qm[perm], "doc_chunks_ctx": cd2p[packedp][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous(),
          "doc_chunk_mask": cp2p[packedp][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous(), "packed_indices": packedp,
          "chunk_pieces": torch.tensor(pieces)}
    wsp, (scorep, _, top_idxp, _) = _run(gp, params, sat, impl)
    assert torch.equal(wsp.cpu(), ws.cpu()[perm]) and torch.equal(top_idxp.cpu(), top_idx.cpu()[perm])
    assert torch.equal(scorep.cpu(), score.cpu()[perm])


@pytest.mark.parametrize("impl", IMPLS)
def test_chunk_holes_and_many_documents(impl):
    """Non-prefix document masks: an all-padding chunk in the middle of a document is dropped by the packing and must
    behave as zeros (not as stale data); more documents than SMs; D not a multiple of 32."""
    B, Lq, Ld, D = 170, 9, 330, 44
    g = torch.Generator().manual_seed(808)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    qm = (torch.arange(Lq).unsqueeze(0) < torch.randint(1, Lq + 1, (B, 1), generator=g)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < torch.randint(1, Ld + 1, (B, 1), generator=g)).float()
    dm[0] = 1.0
    dm[0, 75:130] = 0        # chunk slot 2 (positions 80..119) is entirely padding
    dm[1] = 1.0
    dm[1, 0:45] = 0          # leading empty chunk
    dm[2] = (torch.rand(Ld, generator=g) < 0.5).float()   # holes everywhere
    dm[3] = 0                # empty document
    q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    chunks = cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    cmask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    params = _tkl_params(D, g)
    for sat in ("embedding", "log"):
        ref_score, sec = O.tkl_interaction(q, qm, chunks, cmask, packed, pieces, params, sat)
        gd = {"q_ctx": q, "q_mask": qm, "doc_chunks_ctx": chunks, "doc_chunk_mask": cmask, "packed_indices": packed,
              "chunk_pieces": torch.tensor(pieces)}
        ws, (score, orig, top_idx, top15) = _run(gd, params, sat, impl)
        assert_close_rel(orig, sec["orig_score"], what=f"orig_score ({sat})")
        assert ((orig.cpu() == 0) == (sec["orig_score"] == 0)).all()
        same = (top_idx.cpu() == sec["top_non_overlapping_idx"]).all(dim=1)
        assert same.float().mean() > 0.97
        assert_close_rel(score.cpu()[same], ref_score[same], what=f"score ({sat})")


def test_kernel_set_without_cover_takes_the_ffma_kernel():
    """Narrow kernels that leave parts of [-1, 1] without any activation: the window token count is then NOT the mask
    count (sigir20_tkl.py:210 tests the activations), the plan kernel detects it on the device and the FFMA kernel,
    which tests the activations themselves, produces the result; forcing the tensor-core kernel alone leaves the output of
    the memset (all zero), which is how the test knows which kernel ran."""
    B, Lq, Ld, D, K = 3, 6, 200, 32, 3
    g = torch.Generator().manual_seed(4)
    # one-hot embeddings: every cosine is exactly 0 or 1, so a position either fires the mu = 1 kernel fully or
    # activates nothing at all (no value lands in the band where fp32 denormals and flush-to-zero would disagree)
    q = torch.nn.functional.one_hot(torch.randint(0, D, (B, Lq), generator=g), D).float()
    d = torch.nn.functional.one_hot(torch.randint(0, D, (B, Ld), generator=g), D).float()
    qm, dm = torch.ones(B, Lq), torch.ones(B, Ld)
    dm[1, 150:] = 0
    d = d * dm.unsqueeze(-1)
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    chunks = cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    cmask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    params = _tkl_params(D, g)
    params.update(mu=torch.tensor([1.0, 0.5, -0.5]), sigma=torch.tensor([0.001, 0.01, 0.01]),
                  dense_weight=torch.tensor([0.3, -0.2, 0.1]), kernel_mult0=torch.ones(3))
    ref_score, sec = O.tkl_interaction(q, qm, chunks, cmask, packed, pieces, params, "log")
    gd = {"q_ctx": q, "q_mask": qm, "doc_chunks_ctx": chunks, "doc_chunk_mask": cmask, "packed_indices": packed,
          "chunk_pieces": torch.tensor(pieces)}
    ws, (score, orig, top_idx, top15) = _run(gd, params, "log", "auto")
    assert_close_rel(orig, sec["orig_score"], what="orig_score")
    assert ((orig.cpu() == 0) == (sec["orig_score"] == 0)).all()
    ws_tc, _ = _run(gd, params, "log", "tcgen05")
    assert (ws_tc == 0).all(), "the tensor-core kernel must decline a kernel set without cover"


def test_dropin_class_matches_reference_golden():
    from matchmaker_b200.rankers.tkl import TKL_sigir20
    for sat in ("embedding", "log"):
        g = load_golden(f"tkl_{sat}")
        emb, heads, layers, ff = [int(x) for x in g["cfg"]]
        params = {k[3:]: v for k, v in g.items() if k.startswith("p__")}
        m = TKL_sigir20(emb, params["mu"].tolist(), params["sigma"].tolist(), heads, layers, ff, 2000, True, True, sat)
        sd = {k[4:]: v for k, v in g.items() if k.startswith("sd__")}
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not unexpected and all(k.startswith("positional_features") for k in missing), (missing, unexpected)
        m = m.to(DEV).eval()
        with torch.no_grad():
            score, sec = m(g["q"].to(DEV), g["d"].to(DEV), g["q_mask"].to(DEV), g["d_mask"].to(DEV),
                           output_secondary_output=True)
        assert_close_rel(score, g["score"], rel=2e-3, what=f"TKL class score ({sat})")
        assert torch.equal(sec["top_non_overlapping_idx"].cpu(), g["top_non_overlapping_idx"])


@pytest.mark.parametrize("sat", ["embedding", "log"])
def test_backward_vs_fp64_autograd_of_oracle(sat):
    """Gradients of the TKL interaction stage against torch autograd (fp64) through the oracle restatement."""
    from matchmaker_b200 import autograd
    B, Lq, Ld, D, K = 5, 14, 420, 32, 11
    g = torch.Generator().manual_seed(123)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    q_len = torch.tensor([14, 9, 3, 14, 1])
    d_len = torch.tensor([420, 300, 61, 33, 200])
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    q, d = q * qm.unsqueeze(-1), d * dm.unsqueeze(-1)
    for b in range(B):
        d[b, 7] = q[b, 0]
    cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
    chunks = cd2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    cmask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
    params = {"mu": torch.tensor([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]), "sigma": torch.full((K,), 0.1),
              "dense_weight": torch.randn(K, generator=g) * 0.1, "chunk_scoring": torch.rand(15, generator=g) + 0.5,
              "sat_emb_reduce1_weight": torch.randn(D, generator=g) * 0.3,
              "sat_normer_weight": torch.rand(2, generator=g) + 0.5, "sat_normer_bias": torch.randn(2, generator=g) * 0.1,
              "saturation_linear_weight": torch.randn(2, generator=g) * 0.5, "saturation_linear_bias": torch.tensor([3.0]),
              "saturation_linear2_weight": torch.randn(2, generator=g) * 0.2, "saturation_linear2_bias": torch.tensor([2.0]),
              "saturation_linear3_weight": torch.randn(2, generator=g) * 0.5, "saturation_linear3_bias": torch.tensor([1.0]),
              "kernel_mult0": torch.rand(K, generator=g) + 0.5}
    gout = torch.randn(B, generator=g)
    # fp64 reference gradients through the oracle
    leaf = {k: v.double().clone().requires_grad_(True) for k, v in params.items() if k not in ("mu", "sigma")}
    p64 = dict(leaf, mu=params["mu"].double(), sigma=params["sigma"].double())
    q64 = q.double().clone().requires_grad_(True)
    c64 = chunks.double().clone().requires_grad_(True)
    s64, sec64 = O.tkl_interaction(q64, qm.double(), c64, cmask.double(), packed, pieces, p64, sat)
    s64.backward(gout.double())
    # CUDA path
    sp, red = _sat_args(params, sat)
    cq = q.to(DEV).requires_grad_(True)
    cc = chunks.to(DEV).requires_grad_(True)
    cdw = params["dense_weight"].to(DEV).requires_grad_(True)
    csp = sp.to(DEV).requires_grad_(True)
    cred = None if red is None else red.to(DEV).requires_grad_(True)
    ccs = params["chunk_scoring"].to(DEV).requires_grad_(True)
    score, orig, top_idx, top15 = autograd.tkl_interaction(cq, qm.to(DEV), cc, cmask.to(DEV), packed.to(DEV), pieces,
                                                           params["mu"].to(DEV), params["sigma"].to(DEV), cdw, sat, csp, cred, ccs)
    assert torch.equal(top_idx.cpu(), sec64["top_non_overlapping_idx"]), "window selection must agree for the gradient check"
    assert_close_rel(score, s64.float(), what="score")
    score.backward(gout.to(DEV))

    def close(a, b, what):
        a, b = a.double().cpu(), b.double()
        scale = b.abs().max().item()
        err = (a - b).abs().max().item()
        assert err <= 2e-3 * scale + 1e-9, f"{what}: max err {err:.3e} vs scale {scale:.3e}"

    close(cq.grad, q64.grad, "grad q_ctx")
    close(cc.grad, c64.grad, "grad chunks")
    close(cdw.grad, leaf["dense_weight"].grad, "grad dense")
    close(ccs.grad, leaf["chunk_scoring"].grad, "grad chunk_scoring")
    if sat == "embedding":
        ref_sp = torch.cat([leaf["sat_normer_weight"].grad, leaf["sat_normer_bias"].grad,
                            leaf["saturation_linear_weight"].grad, leaf["saturation_linear_bias"].grad,
                            leaf["saturation_linear2_weight"].grad, leaf["saturation_linear2_bias"].grad,
                            leaf["saturation_linear3_weight"].grad, leaf["saturation_linear3_bias"].grad])
        close(csp.grad, ref_sp, "grad saturation params")
        close(cred.grad, leaf["sat_emb_reduce1_weight"].grad, "grad sat_emb_reduce1")
    else:
        close(csp.grad, leaf["kernel_mult0"].grad, "grad kernel_mult")


def test_tkl_class_trains():
    from matchmaker_b200.rankers.tkl import TKL_sigir20
    g = load_golden("tkl_embedding")
    emb, heads, layers, ff = [int(x) for x in g["cfg"]]
    params = {k[3:]: v for k, v in g.items() if k.startswith("p__")}
    m = TKL_sigir20(emb, params["mu"].tolist(), params["sigma"].tolist(), heads, layers, ff, 2000, True, True, "embedding")
    m.load_state_dict({k[4:]: v for k, v in g.items() if k.startswith("sd__")}, strict=False)
    m = m.to(DEV).train()
    s = m(g["q"].to(DEV), g["d"].to(DEV), g["q_mask"].to(DEV), g["d_mask"].to(DEV))
    s.sum().backward()
    for name in ("dense.weight", "chunk_scoring", "saturation_linear.weight", "sat_emb_reduce1.weight", "mixer"):
        p = dict(m.named_parameters())[name]
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0, name
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.contextualizer.parameters())
