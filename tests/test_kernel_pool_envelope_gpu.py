"""Kernel pooling across its whole instantiation matrix (tests/kernel_pool_cases.py): every compiled instantiation of the
tensor-core and FFMA forward and backward, with padded kernel slots, distinct per-kernel sigmas, the document gate, the
KNRM form and IDCM's 1e-4 floor, against fp64 autograd of one restatement of the oracle.

Bars: per_kernel and S 1e-3 (assert_close_rel); the score 1e-3 of the magnitude summed (assert_score_close); gradients 1e-3
of the largest entry of each tensor, 3e-3 on the tensor-core backward for pairs with at most 4 live query terms
(test_train_pair_few_query_terms_bound), plus there the tf32 operand rounding of the magnitude each element summed
(kernel_pool_cases.TF32_SUMMED).  The worst error / scale of every gradient is recorded per instantiation as a
test property (``--junitxml``)."""
import pytest
import torch

import kernel_pool_cases as C
from conftest import assert_close_rel
from matchmaker_b200 import _lib, autograd, interaction
from test_kernel_pool_gpu import assert_score_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRADS = ("grad_q", "grad_d", "grad_alpha", "grad_weight", "grad_gate")


def _dev(t):
    return None if t is None else t.to(DEV)


def _inputs(c: C.Case, mask_dtype=None):
    qm, dm = (c.qm, c.dm) if mask_dtype is None else (c.qm.to(mask_dtype), c.dm.to(mask_dtype))
    return [_dev(t) for t in (c.q, c.d, qm, dm, c.mu, c.sigma, c.weight)]


def _forward(c, args, impl="auto", clamp_min=C.DEFAULT_FLOOR, bias=0.0, save=False):
    return interaction.kernel_pool(*args, alpha=_dev(c.alpha), log_scale=c.log_scale, doc_gate=_dev(c.gate),
                                   want_per_kernel=True, want_per_kernel_query=True, impl="auto" if save else impl,
                                   clamp_min=clamp_min, bias=bias, save_for_backward=save)


def _backward(c, args, S, clamp_min=C.DEFAULT_FLOOR, saved=None):
    res = interaction.kernel_pool_bwd(*args, _dev(c.alpha), S, _dev(c.gout), c.log_scale, doc_gate=_dev(c.gate),
                                      clamp_min=clamp_min, saved=saved)
    torch.cuda.synchronize()
    return dict(zip(GRADS, list(res) + [None] * (5 - len(res))))


def _check_grads(got, ref, where, record, few=None):
    """1e-3 of the largest reference entry of each gradient tensor.  ``few`` marks the tensor-core backward: a [B] mask
    of pairs with at most 4 live query terms, whose per-pair gradients are held to 3e-3; and every grad_q / grad_d element
    is also allowed kernel_pool_cases.TF32_SUMMED times the magnitude its tf32 contraction summed.  Records the worst
    error / scale."""
    for name in GRADS:
        a, b = got[name], ref[name]
        assert (a is None) == (b is None), f"{where} {name}: present {a is not None}, expected {b is not None}"
        if b is None:
            continue
        a, b = a.double().cpu(), b.double()
        assert a.shape == b.shape, f"{where} {name}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
        scale = b.abs().max().item()
        assert scale > 0, f"{where} {name}: the reference gradient is all zero"
        err = (a - b).abs()
        record(f"{where} {name}", f"{err.max().item() / scale:.2e}")
        if few is not None and name in ("grad_q", "grad_d"):
            err = (err - C.TF32_SUMMED * ref["summed_" + name[-1]]).clamp(min=0)
        if few is not None and name != "grad_alpha" and name != "grad_weight":
            many_err = err[~few].max().item() if (~few).any() else 0.0
            few_err = err[few].max().item() if few.any() else 0.0
            assert many_err <= 1e-3 * scale, f"{where} {name}: max err {many_err:.3e} vs scale {scale:.3e}"
            assert few_err <= 3e-3 * scale, f"{where} {name} (<= 4 query terms): max err {few_err:.3e} vs scale {scale:.3e}"
        else:
            assert err.max().item() <= 1e-3 * scale, f"{where} {name}: max err {err.max().item():.3e} vs scale {scale:.3e}"


def _check_exact_zeros(got, c: C.Case, where):
    """Masked query / document rows, and document rows whose gate is 0, get exactly no gradient; nor does the gate of a
    masked document row."""
    assert (got["grad_q"].cpu()[c.qm == 0] == 0).all(), f"{where}: gradient on a masked query row"
    assert (got["grad_d"].cpu()[c.dm == 0] == 0).all(), f"{where}: gradient on a masked document row"
    if c.gate is not None:
        assert (got["grad_d"].cpu()[c.gate == 0] == 0).all(), f"{where}: gradient on a document row whose gate is 0"
        assert (got["grad_gate"].cpu()[c.dm == 0] == 0).all(), f"{where}: gate gradient on a masked document row"


def _check_forward(out, ref, c: C.Case, what):
    assert_score_close(out["score"], ref["score"], ref["per_kernel"], c.weight, what=f"{what} score")
    assert_close_rel(out["per_kernel"], ref["per_kernel"], what=f"{what} per_kernel")
    valid = c.qm.bool()
    assert_close_rel(out["per_kernel_query"].cpu()[valid], ref["S"][valid], what=f"{what} S (valid query rows)")


@pytest.mark.parametrize("gate", [False, True], ids=["plain", "gate"])
@pytest.mark.parametrize("row", C.MATRIX, ids=str)
def test_matrix_forward_and_backward_vs_fp64(row, gate, record_property):
    c = C.row_case(row, gate)
    ref = C.reference(c)
    assert C.floor_margin(ref["aS"], c.qm, C.DEFAULT_FLOOR) > 1e-2
    args = _inputs(c)
    # forward on both kernels
    simt = _forward(c, args, impl="simt")
    plain = _forward(c, args, impl="tcgen05")
    _check_forward(simt, ref, c, "FFMA forward")
    _check_forward(plain, ref, c, "tensor-core forward")
    # FFMA backward, from the FFMA forward's S
    where = C.inst(C.SIMT_BWD, C.simt_kb(row.K), 2 if row.D > 256 else 1)
    got = _backward(c, args, simt["per_kernel_query"])
    _check_grads(got, ref, where, record_property)
    _check_exact_zeros(got, c, where)
    if not row.train:
        return
    # training forward: the inference forward plus stores, bit for bit
    train = _forward(c, args, save=True)
    for key in ("score", "per_kernel", "per_kernel_query"):
        assert torch.equal(train[key], plain[key]), f"training forward {key} differs from the inference forward"
    # tensor-core backward: fp64, exact zeros, run to run
    where = C.inst(C.TC_BWD, C.tc_kb(row.K), gate)
    got = _backward(c, args, train["per_kernel_query"], saved=train["saved"])
    _check_grads(got, ref, where, record_property, few=C.few_term_pairs(c.qm))
    _check_exact_zeros(got, c, where)
    again = _backward(c, args, train["per_kernel_query"], saved=train["saved"])
    for name in GRADS:
        assert (got[name] is None and again[name] is None) or torch.equal(got[name], again[name]), f"{where} {name}: run to run"


@pytest.mark.parametrize("K", C.CLAMP_KS)
def test_clamp_floor_and_bias(K, record_property, monkeypatch):
    """IDCM's ESM scorer: the 1e-4 floor on alpha S, and the Linear bias.  At least 10 % of the live (pair, query row,
    kernel) entries lie below the floor, none within 1 % of it: fp32 and fp64 agree on the side of every entry, so the
    gradients must be those of fp64 autograd through torch.clamp -- 0 below the floor."""
    c = C.clamp_case(K)
    ref = C.reference(c, clamp_min=C.IDCM_FLOOR, bias=0.37)
    assert C.below_floor_fraction(ref["aS"], c.qm, C.IDCM_FLOOR) >= 0.1
    assert C.floor_margin(ref["aS"], c.qm, C.IDCM_FLOOR) > 1e-2
    args = _inputs(c)
    # forward on both kernels; the bias shifts the score exactly
    for impl in ("simt", "tcgen05"):
        out = _forward(c, args, impl=impl, clamp_min=C.IDCM_FLOOR, bias=0.37)
        _check_forward(out, ref, c, f"{impl} forward")
        unbiased = _forward(c, args, impl=impl, clamp_min=C.IDCM_FLOOR)
        assert torch.equal(out["score"], unbiased["score"] + 0.37), f"{impl}: the bias does not shift the score exactly"
        assert torch.equal(out["per_kernel"], unbiased["per_kernel"])
    # both backward kernels
    simt = _forward(c, args, impl="simt", clamp_min=C.IDCM_FLOOR)
    got = _backward(c, args, simt["per_kernel_query"], clamp_min=C.IDCM_FLOOR)
    _check_grads(got, ref, f"clamp {C.inst(C.SIMT_BWD, C.simt_kb(K), 1)}", record_property)
    train = _forward(c, args, clamp_min=C.IDCM_FLOOR, bias=0.37, save=True)
    got = _backward(c, args, train["per_kernel_query"], clamp_min=C.IDCM_FLOOR, saved=train["saved"])
    _check_grads(got, ref, f"clamp {C.inst(C.TC_BWD, C.tc_kb(K), False)}", record_property, few=C.few_term_pairs(c.qm))
    # through autograd on both training routes.  The bias is a plain float of the API: it has no gradient.
    for impl in ("auto", "simt"):
        monkeypatch.setattr(autograd, "KP_TRAIN_IMPL", impl)
        cq, cd = _dev(c.q).requires_grad_(True), _dev(c.d).requires_grad_(True)
        cw, ca = _dev(c.weight).requires_grad_(True), _dev(c.alpha).requires_grad_(True)
        score, _ = autograd.kernel_pool(cq, cd, args[2], args[3], args[4], args[5], cw, ca, c.log_scale,
                                        clamp_min=C.IDCM_FLOOR, bias=0.37)
        assert score.grad_fn.tc == (impl == "auto")
        score.backward(_dev(c.gout))
        got = {"grad_q": cq.grad, "grad_d": cd.grad, "grad_alpha": ca.grad, "grad_weight": cw.grad, "grad_gate": None}
        _check_grads(got, ref, f"clamp autograd {impl} K={K}", record_property,
                     few=C.few_term_pairs(c.qm) if impl == "auto" else None)


def _autograd_run(c: C.Case):
    cq, cd = _dev(c.q).requires_grad_(True), _dev(c.d).requires_grad_(True)
    cw, ca = _dev(c.weight).requires_grad_(True), _dev(c.alpha).requires_grad_(True)
    args = _inputs(c)
    score, _ = autograd.kernel_pool(cq, cd, args[2], args[3], args[4], args[5], cw, ca, c.log_scale)
    tc = score.grad_fn.tc
    score.backward(_dev(c.gout))
    return tc, {"grad_q": cq.grad, "grad_d": cd.grad, "grad_alpha": ca.grad, "grad_weight": cw.grad, "grad_gate": None}


@pytest.mark.parametrize("Lq,D,tc", [(8, 320, True), (8, 324, False), (32, 64, True), (33, 64, False), (8, 512, False)])
def test_autograd_route_at_envelope_edges(Lq, D, tc, record_property):
    """autograd.kernel_pool takes the tensor-core training pair exactly inside its envelope (D <= 320, Lq <= 32) and the
    FFMA backward outside it, up to its own limit D = 512; either way the gradients are fp64 autograd's."""
    c = C.make_case(3, Lq, 40, D, 12, seed=70 + Lq + D)
    assert interaction.kernel_pool_train_supported(Lq, 40, D, 12) == tc
    got_tc, got = _autograd_run(c)
    assert got_tc == tc
    _check_grads(got, C.reference(c), f"route Lq={Lq} D={D}", record_property, few=C.few_term_pairs(c.qm) if tc else None)


def test_out_of_envelope_raises_on_the_host():
    """D = 516 (past the FFMA backward's 512) and K = 33 (past the 32 kernel slots) are refused by the host's argument
    checks, before any launch, with MatchmakerB200Error; the stream stays usable."""
    c = C.make_case(2, 8, 40, 516, 12, seed=3)
    args = _inputs(c)
    out = _forward(c, args)   # the forward serves D = 516
    with pytest.raises(_lib.MatchmakerB200Error, match="invalid argument.*512"):
        _backward(c, args, out["per_kernel_query"])
    cq = _dev(c.q).requires_grad_(True)
    score, _ = autograd.kernel_pool(cq, *args[1:6], _dev(c.weight).requires_grad_(True), _dev(c.alpha), c.log_scale)
    assert not score.grad_fn.tc
    with pytest.raises(_lib.MatchmakerB200Error, match="invalid argument.*512"):
        score.sum().backward()
    c = C.make_case(2, 8, 40, 64, 33, seed=4)
    args = _inputs(c)
    for impl in ("auto", "simt", "tcgen05"):
        with pytest.raises(_lib.MatchmakerB200Error, match="invalid argument.*K <= 32"):
            _forward(c, args, impl=impl)
    S = torch.zeros(2, 8, 33, device=DEV)
    with pytest.raises(_lib.MatchmakerB200Error, match="invalid argument.*K <= 32"):
        _backward(c, args, S)
    with pytest.raises(_lib.MatchmakerB200Error, match="invalid argument.*K <= 32"):
        autograd.kernel_pool(_dev(c.q).requires_grad_(True), *args[1:6], args[6], _dev(c.alpha), c.log_scale)
    torch.cuda.synchronize()
    ok = C.make_case(2, 8, 40, 64, 12, seed=5)
    _check_forward(_forward(ok, _inputs(ok)), C.reference(ok, grads=False), ok, "after the refusals")


@pytest.mark.parametrize("kernel", ["tensor-core", "FFMA"])
def test_mask_dtypes_give_identical_gradients(kernel):
    """bool, int64 and float32 masks select the same rows: bit-identical forward outputs and gradients.  The padding rows
    hold data, so only the masks keep them out."""
    c = C.make_case(7, 20, 70, 64, 12, seed=91, gate=True)
    assert (c.q[c.qm == 0] != 0).any() and (c.d[c.dm == 0] != 0).any()
    runs = []
    for mdt in (torch.float32, torch.bool, torch.int64):
        args = _inputs(c, mdt)
        if kernel == "tensor-core":
            out = _forward(c, args, save=True)
            got = _backward(c, args, out["per_kernel_query"], saved=out["saved"])
        else:
            out = _forward(c, args, impl="simt")
            got = _backward(c, args, out["per_kernel_query"])
        runs.append((out, got))
    ref = C.reference(c)
    _check_grads(runs[0][1], ref, f"mask dtypes {kernel}", lambda *a: None,
                 few=C.few_term_pairs(c.qm) if kernel == "tensor-core" else None)
    for out, got in runs[1:]:
        for key in ("score", "per_kernel", "per_kernel_query"):
            assert torch.equal(out[key], runs[0][0][key]), key
        for name in GRADS:
            assert torch.equal(got[name], runs[0][1][name]), name


@pytest.mark.parametrize("train_impl", ["auto", "simt"])
def test_empty_batch(train_impl, monkeypatch):
    """B = 0: empty outputs on every forward, empty per-pair gradients and zero parameter gradients on both backward
    kernels and through autograd."""
    monkeypatch.setattr(autograd, "KP_TRAIN_IMPL", train_impl)
    c = C.make_case(1, 5, 20, 32, 11, seed=6, gate=True)
    c.q, c.d, c.qm, c.dm, c.gate, c.gout = c.q[:0], c.d[:0], c.qm[:0], c.dm[:0], c.gate[:0], c.gout[:0]
    args = _inputs(c)
    for impl in ("auto", "simt", "tcgen05"):
        out = _forward(c, args, impl=impl)
        assert out["score"].shape == (0,) and out["per_kernel"].shape == (0, 11) and out["per_kernel_query"].shape == (0, 5, 11)
    train = _forward(c, args, save=True)
    assert train["score"].shape == (0,) and train["saved"].numel() == 0
    for saved in (None, train["saved"]):
        got = _backward(c, args, train["per_kernel_query"], saved=saved)
        assert got["grad_q"].shape == (0, 5, 32) and got["grad_d"].shape == (0, 20, 32) and got["grad_gate"].shape == (0, 20)
        assert torch.equal(got["grad_weight"].cpu(), torch.zeros(11)) and torch.equal(got["grad_alpha"].cpu(), torch.zeros(11))
    cq, cd = _dev(c.q).requires_grad_(True), _dev(c.d).requires_grad_(True)
    cw, ca, cg = _dev(c.weight).requires_grad_(True), _dev(c.alpha).requires_grad_(True), _dev(c.gate).requires_grad_(True)
    score, pk = autograd.kernel_pool(cq, cd, args[2], args[3], args[4], args[5], cw, ca, c.log_scale, doc_gate=cg)
    assert score.shape == (0,) and pk.shape == (0, 11)
    score.sum().backward()
    assert cq.grad.shape == cq.shape and cd.grad.shape == cd.shape and cg.grad.shape == cg.shape
    assert torch.equal(cw.grad.cpu(), torch.zeros(11)) and torch.equal(ca.grad.cpu(), torch.zeros(11))
