"""The differentiable all-pairs max-sim (in-batch negatives, colbert.py:154-162) on the GPU: autograd.maxsim_allpairs
and the backward kernels of mmb200_maxsim_allpairs_bwd.

On small-integer inputs every fp32 sum is exact, so scores, argmax and gradients are held bit for bit to the fp64
oracle, with NaN / +-inf wherever no pair reads.  With one query the gradients are those of the pairs backward, two runs
give the same bits, and at the reference configuration on real values the gradients meet the bar of the pairs autograd
test against fp64 autograd of the reference expression (worst error / scale recorded as test properties)."""
import copy

import pytest
import torch

import maxsim_cases as C
import maxsim_inbatch_cases as I
from conftest import assert_close_rel
from matchmaker_b200 import _lib, autograd, interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _exact(got, ref, what):
    got = got.detach().cpu().to(ref.dtype)
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    bad = got != ref
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.numel()} differ, first at {bad.nonzero()[0].tolist()}: "
                           f"{got[bad][0].item()} vs {ref[bad][0].item()}")


def _leaf_followed_by_nan(t: torch.Tensor, dtype) -> torch.Tensor:
    """t on the device as a leaf that requires grad, with one more slab of NaN after it in memory."""
    big = torch.full((t.shape[0] + 1,) + tuple(t.shape[1:]), float("nan"), dtype=dtype, device=DEV)
    big[: t.shape[0]] = t.to(dtype).to(DEV)
    return big[: t.shape[0]].detach().requires_grad_(True)


@pytest.mark.parametrize("s", I.MATRIX, ids=str)
def test_autograd_bit_exact_on_integer_inputs(s):
    c = I.make_case(s)
    score, arg = C.oracle(c)
    ref_q, ref_d = I.oracle_grads(c, arg, s.n_d)
    qp, dp = I.poisoned(c, s)
    cq, cd = _leaf_followed_by_nan(qp, s.dtype), _leaf_followed_by_nan(dp, s.dtype)
    qm, dm = c.qm.to(DEV), c.dm.to(DEV)
    gout = c.gout.view(s.n_q, s.n_d).to(DEV)
    ref_idx = not s.own
    out = autograd.maxsim_allpairs(cq, qm, cd, dm, reference_mask_indexing=ref_idx)
    _exact(out, score.view(s.n_q, s.n_d), f"{s} score")
    out.backward(gout)
    # autograd hands back the inputs' dtype: the exact fp32 gradient rounded once
    _exact(cq.grad, ref_q.to(s.dtype), f"{s} grad_q (autograd)")
    _exact(cd.grad, ref_d.to(s.dtype), f"{s} grad_d (autograd)")
    with torch.no_grad():
        s2, am = interaction.maxsim_allpairs(cq, qm, cd, dm, reference_mask_indexing=ref_idx, return_argmax=True)
    _exact(s2, score.view(s.n_q, s.n_d), f"{s} score (argmax forward)")
    _exact(am, arg, f"{s} argmax")
    gq, gd = interaction.maxsim_allpairs_bwd(cq.detach(), cd.detach(), gout, am)
    _exact(gq, ref_q, f"{s} grad_q")
    _exact(gd, ref_d, f"{s} grad_d")
    assert (gq.cpu()[~c.qm.bool()] == 0).all()
    gq2, gd2 = interaction.maxsim_allpairs_bwd(cq.detach(), cd.detach(), gout, am)
    assert torch.equal(gq, gq2) and torch.equal(gd, gd2)


@pytest.mark.parametrize("dtype", [C.H, C.BF, C.F32], ids=lambda t: C.SHORT[t])
@pytest.mark.parametrize("dim,Lq", [(128, 32), (768, 30), (100, 20)])
def test_one_query_is_the_pairs_backward(dtype, dim, Lq):
    """n_q = 1 on real values: bit-identical to interaction.maxsim_bwd(..., docs_per_query=n_d)."""
    n_d, Ld = 9, 150
    g = torch.Generator().manual_seed(dim + Lq)
    q = (torch.randn(1, Lq, dim, generator=g) * 0.3).to(dtype).to(DEV)
    d = (torch.randn(n_d, Ld, dim, generator=g) * 0.3).to(dtype).to(DEV)
    qm = (torch.rand(1, Lq, generator=g) > 0.2).long().to(DEV)
    dm = (torch.rand(n_d, Ld, generator=g) > 0.2).long().to(DEV)
    gout = torch.randn(1, n_d, generator=g).to(DEV)
    s_all, am_all = interaction.maxsim_allpairs(q, qm, d, dm, return_argmax=True)
    s_pair, am_pair = interaction.maxsim(q, d, qm, dm, docs_per_query=n_d, return_argmax=True)
    assert torch.equal(am_all, am_pair) and torch.equal(s_all.view(-1), s_pair)
    gq, gd = interaction.maxsim_allpairs_bwd(q, d, gout, am_all)
    pq, pd = interaction.maxsim_bwd(q, d, gout.view(-1), am_pair, docs_per_query=n_d)
    assert torch.equal(gq, pq) and torch.equal(gd, pd)


def _real_batch(n, Lq, Ld, dim, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(n, Lq, dim, generator=g) * 0.3).to(dtype)
    d = (torch.randn(n, Ld, dim, generator=g) * 0.3).to(dtype)
    qm = (torch.arange(Lq).unsqueeze(0) < torch.randint(5, Lq + 1, (n, 1), generator=g)).long()
    dm = (torch.arange(Ld).unsqueeze(0) < torch.randint(20, Ld + 1, (n, 1), generator=g)).long()
    dm[0] = 1
    return q, qm, d, dm, torch.randn(n, n, generator=g)


@pytest.mark.parametrize("dtype", [C.H, C.BF, C.F32], ids=lambda t: C.SHORT[t])
def test_autograd_at_the_reference_configuration(dtype, record_property):
    """32 x 32 in-batch pairs at dim 768, Lq 30, Ld 200 on real values (reference mask indexing), against fp64 autograd
    of oracle.maxsim_allpairs: scores to 1e-3; gradients to 1e-3 (bf16: 2^-8, the unit roundoff of the bf16 gradient
    autograd returns) except where the top-2 margin of a token's scores does not decide its argmax in fp32.  Two runs
    give the same bits."""
    n, Lq, Ld, dim = 32, 30, 200, 768
    q, qm, d, dm, gout = _real_batch(n, Lq, Ld, dim, dtype, 3232)
    ref, rq, rd = I.reference_autograd(q, qm, d, dm, gout, own=False)
    grads = []
    for _ in range(2):
        cq, cd = q.to(DEV).requires_grad_(True), d.to(DEV).requires_grad_(True)
        out = autograd.maxsim_allpairs(cq, qm.to(DEV), cd, dm.to(DEV), reference_mask_indexing=True)
        out.backward(gout.to(DEV))
        grads.append((out.detach(), cq.grad, cd.grad))
    assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1])), "two runs differ"
    out, gq, gd = grads[0]
    assert_close_rel(out, ref, what="score")
    S = torch.einsum("aid,bjd->abij", q.double(), d.double())
    S = S.masked_fill(~dm.bool()[:, None, None, :], C.FILL)      # pair (a, b) masked with row a (colbert.py:158)
    top = S.topk(2, dim=-1)
    live = qm.bool()[:, None, :].expand(n, n, Lq)
    amb = live & ((top.values[..., 0] - top.values[..., 1]) <= 1e-4 * top.values[..., 0].abs().clamp(min=1.0))
    keep_q = torch.ones(n, Lq, dtype=torch.bool)
    keep_d = torch.ones(n, Ld, dtype=torch.bool)
    for a, b, i in amb.nonzero().tolist():
        keep_q[a, i] = False
        keep_d[b, top.indices[a, b, i]] = False
    record_property("ambiguous tokens", int(amb.sum()))
    bar = 2.0 ** -8 if dtype == C.BF else 1e-3
    for name, got, want, keep in (("grad_q", gq, rq, keep_q), ("grad_d", gd, rd, keep_d)):
        got, want = got.double().cpu()[keep], want[keep]
        scale = want.abs().max().item()
        record_property(f"{C.SHORT[dtype]} {name} worst error / scale", f"{(got - want).abs().max().item() / scale:.2e}")
        assert_close_rel(got, want, rel=bar, what=name)


class _TinyEncoder(torch.nn.Module):
    """Stand-in for the HF encoder: embedding + linear, returns (hidden,)."""

    class _Cfg:
        hidden_size = 48

    def __init__(self, vocab=100):
        super().__init__()
        self.config = self._Cfg()
        self.emb = torch.nn.Embedding(vocab, 48)
        self.lin = torch.nn.Linear(48, 48)

    def forward(self, input_ids=None, attention_mask=None, **kw):
        return (torch.tanh(self.lin(self.emb(input_ids))),)


def _tokens(B, L, g):
    lens = torch.randint(2, L + 1, (B,), generator=g)
    ids = torch.randint(1, 100, (B, L), generator=g)
    mask = (torch.arange(L).unsqueeze(0) < lens.unsqueeze(1)).long()
    return {"input_ids": (ids * mask).to(DEV), "attention_mask": mask.to(DEV)}


@pytest.mark.parametrize("dim", [64, 128])
def test_inbatch_loss_trains_the_model(dim):
    """An in-batch cross-entropy over ColBERT.forward_inbatch_aggregation reaches compressor.weight, with the gradient
    of the same model scored by the reference expression in torch; no_grad scores are those of
    interaction.maxsim_allpairs, and with grad at dim 64 / 128, Lq <= 32 (fp16) the scores are the no_grad bits."""
    from matchmaker_b200.rankers.colbert import ColBERT, ColBERTConfig
    torch.manual_seed(dim)
    g = torch.Generator().manual_seed(dim)
    m = ColBERT(ColBERTConfig(bert_model=_TinyEncoder(), compression_dim=dim)).to(DEV)
    ref_m = copy.deepcopy(m)
    q, d = _tokens(8, 16, g), _tokens(8, 60, g)
    target = torch.arange(8, device=DEV)

    def loss_of(model, scorer):
        qv, dv = model.forward_representation(q), model.forward_representation(d)
        return torch.nn.functional.cross_entropy(scorer(model, qv, dv), target)

    loss = loss_of(m, lambda mm, qv, dv: mm.forward_inbatch_aggregation(qv, q["attention_mask"], dv, d["attention_mask"]))
    loss.backward()
    ref = loss_of(ref_m, lambda mm, qv, dv: O.maxsim_allpairs(qv, q["attention_mask"], dv, d["attention_mask"]))
    ref.backward()
    assert_close_rel(loss.detach(), ref.detach(), what="loss")
    assert m.compressor.weight.grad.abs().sum() > 0
    assert_close_rel(m.compressor.weight.grad, ref_m.compressor.weight.grad, rel=1e-3, what="compressor.weight.grad")
    assert_close_rel(m.bert_model.lin.weight.grad, ref_m.bert_model.lin.weight.grad, rel=1e-3, what="encoder grad")

    with torch.autocast("cuda", dtype=torch.float16):
        qv, dv = m.forward_representation(q), m.forward_representation(d)
    assert qv.dtype == torch.float16
    assert qv.requires_grad and dv.requires_grad
    with torch.no_grad():   # vectors that require grad, scored without grad: the inference call
        s0 = m.forward_inbatch_aggregation(qv, q["attention_mask"], dv, d["attention_mask"])
        s_int = interaction.maxsim_allpairs(qv, q["attention_mask"], dv, d["attention_mask"],
                                            reference_mask_indexing=True)
    assert s0.grad_fn is None and torch.equal(s0, s_int)
    # with grad: the argmax forward of the queries-on-M kernel, whose scores are the inference bits
    s1 = m.forward_inbatch_aggregation(qv, q["attention_mask"], dv, d["attention_mask"])
    assert s1.grad_fn is not None and torch.equal(s1.detach(), s0)
    s2 = m.forward_inbatch_aggregation(qv, q["attention_mask"], dv, d["attention_mask"], reference_mask_indexing=False)
    with torch.no_grad():
        s3 = interaction.maxsim_allpairs(qv, q["attention_mask"], dv, d["attention_mask"])
    assert torch.equal(s2.detach(), s3)


def test_empty_batch():
    """No pairs: empty scores; a side that has rows gets a zero gradient."""
    for n_q, n_d in ((0, 0), (3, 0), (0, 2)):
        q = torch.full((n_q, 30, 768), float("nan"), dtype=C.H, device=DEV, requires_grad=True)
        d = torch.full((n_d, 200, 768), float("nan"), dtype=C.H, device=DEV, requires_grad=True)
        qm = torch.ones(n_q, 30, dtype=torch.long, device=DEV)
        dm = torch.ones(n_d, 200, dtype=torch.long, device=DEV)
        out = autograd.maxsim_allpairs(q, qm, d, dm)
        assert out.shape == (n_q, n_d)
        out.sum().backward()
        assert q.grad.shape == q.shape and d.grad.shape == d.shape
        assert (q.grad == 0).all() and (d.grad == 0).all()


@pytest.mark.parametrize("Lq", [30, 75])
@pytest.mark.parametrize("reference_mask_indexing", [True, False], ids=["reference-indexing", "own-masks"])
def test_no_grad_scoring_of_vectors_that_require_grad_is_the_inference_call(Lq, reference_mask_indexing):
    """Vectors produced with grad, scored under torch.no_grad() (logging, metrics, a teacher): the same bits as
    interaction.maxsim_allpairs, which at dim 768 runs the tensor-core kernel (not the SIMT argmax forward), no graph,
    and Lq 75, beyond the argmax forward's envelope, still scores."""
    q, qm, d, dm, _ = _real_batch(6, Lq, 120, 768, C.H, 768 + Lq)
    q, qm, d, dm = q.to(DEV).requires_grad_(True), qm.to(DEV), d.to(DEV).requires_grad_(True), dm.to(DEV)
    with torch.no_grad():
        got = autograd.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=reference_mask_indexing)
        want = interaction.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=reference_mask_indexing)
    assert got.grad_fn is None and torch.equal(got, want)


def test_training_beyond_the_argmax_envelope_is_refused():
    """Dim 768 at Lq 75: the SIMT argmax kernel's query tile no longer fits in shared memory, so the training forward is
    refused by the host (MatchmakerB200Error, no kernel runs); without grad the tensor cores still score it."""
    q, qm, d, dm, _ = _real_batch(4, 75, 64, 768, C.H, 75)
    q, qm, d, dm = q.to(DEV), qm.to(DEV), d.to(DEV), dm.to(DEV)
    s = autograd.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True)
    assert_close_rel(s, O.maxsim_allpairs(q.double().cpu(), qm.cpu(), d.double().cpu(), dm.cpu()), what="no-grad score")
    with pytest.raises(_lib.MatchmakerB200Error):
        autograd.maxsim_allpairs(q.requires_grad_(True), qm, d, dm, reference_mask_indexing=True)
