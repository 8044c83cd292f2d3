"""The store mode of kernel pooling (``interaction.kernel_pool_store``) across its whole instantiation matrix
(tests/kernel_pool_store_cases.py), on every kernel that takes each shape, without and with the gate:

- against fp64 (``kernel_pool_cases.reference`` over the gathered passages): the score within 1e-3 of the magnitude
  summed (assert_score_close); void pairs and passages without rows exactly -inf;
- the store's contract: bit-identical to ``interaction.kernel_pool`` on the padded gather with the same ``impl``;
- bit for bit invariant under repeated (query, passage) pairs, a permuted pair order, a second run, ``auto`` against the
  kernel the routing names, and the poisoned rows (NaN / +-inf in unreferenced passages and past the end of the store
  view) against the same store with finite rows there.

Every launch has at least 1 200 pairs, so every CTA of both grids walks several pairs of mixed tile counts.  The worst
error / scale per instantiation is recorded as a test property (``--junitxml``).  Then the targeted edges: Lq > 128,
truncation at max_doc_len, the query mask forms, the KNRM form, IDCM's floor and bias, the FFMA kernel's D edge, an empty
pair list, and ``TKDocumentStore.rerank`` ties and tails."""
import dataclasses

import numpy as np
import pytest
import torch

import kernel_pool_cases as KP
import kernel_pool_store_cases as C
import tk_store_cases as TKC
from matchmaker_b200 import _lib, interaction
from matchmaker_b200.rankers.tk import ECAI20_TK
from matchmaker_b200.rankers.tk_sparse import CIKM20_TK_Sparse
from matchmaker_b200.retrieval import TKDocumentStore
from test_kernel_pool_gpu import assert_score_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAD_CHUNK_FLOATS = 1 << 25    # fp32 elements of one padded gather (128 MB)


def _smem_optin() -> int:
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def _on_dev(c: C.Case, clean: bool = False) -> dict:
    """The case's tensors on the GPU; the store stays a view of its buffer (rows past it: NaN, or finite when clean)."""
    buf = (c.clean_buf if clean else c.buf).to(DEV)
    gate = c.clean_gate if clean else c.gate
    t = {k: getattr(c, k) for k in ("q", "qm", "off", "pair_q", "pair_d", "mu", "sigma", "alpha", "weight")}
    t = {k: None if v is None else v.to(DEV) for k, v in t.items()}
    t.update(store=buf[:c.n_rows], gate=None if gate is None else gate.to(DEV))
    assert t["store"].data_ptr() == buf.data_ptr() and t["store"].is_contiguous()
    return t


def _score(c: C.Case, t: dict, impl: str, pair_q=None, pair_d=None, q_mask="case", **kw):
    """``interaction.kernel_pool_store`` on the case (its pairs, its query mask) unless told otherwise."""
    return interaction.kernel_pool_store(t["q"], t["qm"] if isinstance(q_mask, str) else q_mask, t["store"], t["off"],
                                         t["pair_q"] if pair_q is None else pair_q,
                                         t["pair_d"] if pair_d is None else pair_d, t["mu"], t["sigma"], t["weight"],
                                         t["alpha"], log_scale=c.log_scale, max_doc_len=c.L, impl=impl, gate=t["gate"],
                                         **kw)


def _padded(c: C.Case, t: dict, pair_q, pair_d, impl: str, q_mask="case", **kw) -> torch.Tensor:
    """``interaction.kernel_pool`` on the pairs gathered into [pairs, max_doc_len, D] (tk_store_cases.gather_padded), in
    chunks."""
    out = []
    step = max(1, PAD_CHUNK_FLOATS // (c.L * c.q.shape[2]))
    for i in range(0, len(pair_q), step):
        pq, pd = pair_q[i:i + step], pair_d[i:i + step]
        d, dm, dg = TKC.gather_padded(t["store"], c.off, pd, c.L, t["gate"])
        qi = pq.long().to(DEV)
        qm = t["qm"][qi] if isinstance(q_mask, str) else (None if q_mask is None else q_mask[qi])
        out.append(interaction.kernel_pool(t["q"][qi], d, qm, dm, t["mu"], t["sigma"], t["weight"], t["alpha"],
                                           log_scale=c.log_scale, impl=impl, doc_gate=dg, **kw)["score"])
    return torch.cat(out)


def _check_fp64(s, ref, c: C.Case, what: str) -> float:
    """Void pairs exactly -inf, the rest finite and within assert_score_close's bar; returns the worst error / scale."""
    s = s.double().cpu()
    void = c.void()
    assert torch.isneginf(s[void]).all(), f"{what}: a void pair or a passage without rows does not score -inf"
    assert torch.isfinite(s[~void]).all(), f"{what}: a pair with rows does not score a finite value"
    assert_score_close(s[~void], ref["score"][~void], ref["per_kernel"][~void], c.weight, what=what)
    b = ref["score"][~void]
    scale = (ref["per_kernel"][~void].abs() * c.weight.double().abs().view(1, -1)).sum(1)
    return float(((s[~void] - b).abs() / torch.maximum(b.abs(), 1e-2 * scale)).max())


def _check_contract(s, c: C.Case, t: dict, impl: str, what: str, **kw):
    """Bit-identical to the padded path on every unique (query, passage), and every repeat of a pair gives its bits."""
    u, inv = c.unique_pairs()
    live = inv >= 0
    first = torch.full((len(u),), -1, dtype=torch.int64)
    first.scatter_reduce_(0, inv[live], torch.nonzero(live).view(-1), reduce="amin", include_self=False)
    s = s.cpu()
    assert torch.equal(s[live], s[first[inv[live]]]), f"{what}: repeats of one (query, passage) differ"
    assert (torch.bincount(inv[live]) >= 2).all(), "every (query, passage) appears more than once"
    pad = _padded(c, t, u[:, 0].to(torch.int32), u[:, 1].to(torch.int32), impl, **kw).cpu()
    bad = torch.nonzero(s[first] != pad).view(-1)
    assert len(bad) == 0, f"{what}: {len(bad)}/{len(u)} unique pairs differ from the padded path, first {u[bad[0]].tolist()}"


@pytest.mark.parametrize("gate", [False, True], ids=["plain", "gate"])
@pytest.mark.parametrize("row", C.MATRIX, ids=str)
def test_matrix_vs_fp64_padded_path_and_invariances(row, gate, record_property):
    c = C.row_case(row, gate)
    ref = C.reference(c)
    t = _on_dev(c)
    clean = _on_dev(c, clean=True)
    perm = torch.randperm(len(c.pair_q), generator=torch.Generator().manual_seed(row.seed))
    impls = C.impls(row.Lq, row.D, row.K, row.L, _smem_optin())
    assert set(impls) == set(row.impls)
    got = {}
    for impl in impls:
        where = f"{C.instantiation(impl, row.K, row.L)} {'gate' if gate else 'plain'}"
        s = got[impl] = _score(c, t, impl)
        record_property(where, f"{_check_fp64(s, ref, c, where):.2e}")
        _check_contract(s, c, t, impl, where)
        assert torch.equal(_score(c, t, impl), s), f"{where}: run to run"
        sp = _score(c, t, impl, pair_q=t["pair_q"][perm.to(DEV)], pair_d=t["pair_d"][perm.to(DEV)])
        assert torch.equal(sp, s[perm.to(DEV)]), f"{where}: a permuted pair order changes the bits"
        assert torch.equal(_score(c, clean, impl), s), f"{where}: the poisoned rows change the scores"
    assert torch.equal(_score(c, t, "auto"), got[C.auto_impl(row.Lq, row.D)]), "auto is not the routed kernel"


def test_long_query_is_refused_by_the_tensor_cores_and_auto_takes_ffma():
    c = C.make_case(11, 130, 64, 60, 3, seed=31, min_pairs=300)
    t = _on_dev(c)
    with pytest.raises(_lib.MatchmakerB200Error, match="not supported by the tensor-core kernel"):
        _score(c, t, "tcgen05")
    simt = _score(c, t, "simt")
    assert torch.equal(_score(c, t, "auto"), simt)
    _check_fp64(simt, C.reference(c), c, "Lq 130 FFMA")


@pytest.mark.parametrize("L", [40, 100])
@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
def test_max_doc_len_truncates_to_the_first_rows(impl, L):
    """max_doc_len below the longest passage: each passage is scored over its first max_doc_len rows -- fp64 over those
    rows, and the bits of the store in which the passages physically end there."""
    c = C.make_case(21, 30, 64, 300, 3, seed=40 + L, gate=True, min_pairs=300)
    assert int((c.off[1:] - c.off[:-1]).max()) > L
    cut = dataclasses.replace(c, L=L)
    s = _score(cut, _on_dev(cut), impl)
    _check_fp64(s, C.reference(cut), cut, f"{impl} max_doc_len {L}")
    short = C.truncated(cut)
    assert torch.equal(_score(short, _on_dev(short), impl), s)


@pytest.mark.parametrize("Lq", [40, 64])
@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
def test_query_mask_forms(impl, Lq):
    """Every mask dtype gives the bits of the bool mask.  q_mask=None gives the padded path's bits with q_mask=None and
    fp64's score with every query row live; it gives the bits of an all-true mask on the FFMA kernel, and on the
    tensor-core kernel where every 32-row query block is full (a partial last block with a mask packs its rows into
    sub-streams of 8 / 16 lanes, which adds the document rows in another order)."""
    c = C.make_case(11, Lq, 64, 100, 3, seed=50 + Lq, min_pairs=300)
    assert not c.qm.all()
    t = _on_dev(c)
    base = _score(c, t, impl)
    for dt in (torch.uint8, torch.int32, torch.int64, torch.float32, torch.float16, torch.float64):
        assert torch.equal(_score(c, t, impl, q_mask=t["qm"].to(dt)), base), f"mask dtype {dt}"
    none = _score(c, t, impl, q_mask=None)
    every = dataclasses.replace(c, qm=torch.ones_like(c.qm))
    _check_fp64(none, C.reference(every), every, f"{impl} q_mask None")
    _check_contract(none, c, t, impl, f"{impl} q_mask None", q_mask=None)
    if impl == "simt" or Lq % 32 == 0:
        assert torch.equal(_score(c, t, impl, q_mask=torch.ones_like(t["qm"])), none)


@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
def test_knrm_form_at_k11(impl):
    """KNRM: no alpha, log_scale 0.01, its 11 kernels (the exact <11> tensor-core instantiation)."""
    c = C.make_case(11, 30, 300, 200, 3, seed=61, knrm=True, min_pairs=300)
    assert c.alpha is None and c.log_scale == 0.01
    t = _on_dev(c)
    s = _score(c, t, impl)
    _check_fp64(s, C.reference(c), c, f"{impl} KNRM")
    _check_contract(s, c, t, impl, f"{impl} KNRM")


IDCM_SEEDS = {8: 13, 40: 100}   # seeds whose live entries all lie more than 1 % from the floor


def idcm_case(Lq: int) -> C.Case:
    """IDCM's form over a store: normalised rows, alpha, and the kernel at mu = -0.9 given sigma 0.05, so that its
    activations fall far below the 1e-4 floor (kernel_pool_cases.clamp_case)."""
    c = C.make_case(11, Lq, 64, 100, 3, seed=IDCM_SEEDS[Lq], normalise=True, min_pairs=300)
    lo, s = int(torch.argmin(c.mu)), int(torch.argmin(c.sigma))
    c.sigma[lo], c.sigma[s] = c.sigma[s].item(), c.sigma[lo].item()
    return c


@pytest.mark.parametrize("Lq", [8, 40])
@pytest.mark.parametrize("impl", ["tcgen05", "simt"])
def test_idcm_floor_and_bias(impl, Lq):
    """IDCM's 1e-4 floor with at least 10 % of the live entries below it and none within 1 % of it; the bias shifts
    every score exactly (score(bias) == score(0) + bias in fp32), also over several query blocks (Lq 40)."""
    c = idcm_case(Lq)
    ref = C.reference(c, clamp_min=KP.IDCM_FLOOR, bias=0.37)
    assert KP.below_floor_fraction(ref["aS"], ref["qm"], KP.IDCM_FLOOR) >= 0.1
    assert KP.floor_margin(ref["aS"], ref["qm"], KP.IDCM_FLOOR) > 1e-2
    t = _on_dev(c)
    s = _score(c, t, impl, clamp_min=KP.IDCM_FLOOR, bias=0.37)
    _check_fp64(s, ref, c, f"{impl} IDCM floor")
    _check_contract(s, c, t, impl, f"{impl} IDCM floor", clamp_min=KP.IDCM_FLOOR, bias=0.37)
    unbiased = _score(c, t, impl, clamp_min=KP.IDCM_FLOOR)
    assert torch.equal(s, unbiased + 0.37), "the bias does not shift the score exactly"


def _kernel_names(fn) -> list:
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "kernel_pool" in e.name]


@pytest.mark.parametrize("K,L", [(25, 300), (5, 8)])
def test_ffma_d_edge(K, L):
    """At the last D of the FFMA kernel's shared-memory plan it scores; 4 columns more are refused with an error, and no
    kernel-pooling kernel is launched.  ``auto`` refuses them too where the tensor-core kernel does not take the shape
    (Lq > 128)."""
    edge = C.simt_d_edge(K, L, _smem_optin())
    c = C.make_case(K, 130, edge, L, 2, seed=70 + K, min_pairs=40)
    t = _on_dev(c)
    names = _kernel_names(lambda: _check_fp64(_score(c, t, "auto"), C.reference(c), c, f"FFMA at D {edge}"))
    assert any("kernel_pool_fwd_simt_store" in n for n in names), names
    past = C.make_case(K, 130, edge + 4, L, 2, seed=71 + K, min_pairs=40)
    tp = _on_dev(past)
    for impl in ("simt", "auto"):
        def refused():
            with pytest.raises(_lib.MatchmakerB200Error, match="embedding dim too large"):
                _score(past, tp, impl)
        assert _kernel_names(refused) == []
    _check_fp64(_score(c, t, "simt"), C.reference(c), c, "after the refusals")


def test_empty_pair_list():
    c = C.make_case(11, 30, 64, 60, 2, seed=80, min_pairs=10)
    t = _on_dev(c)
    none = torch.zeros(0, dtype=torch.int32, device=DEV)
    for impl in ("auto", "tcgen05", "simt"):
        s = _score(c, t, impl, pair_q=none, pair_d=none)
        assert s.shape == (0,) and s.dtype == torch.float32 and s.device.type == "cuda"


# ---------------------------------------------------------------------------------------------------------------------
# TKDocumentStore.rerank
# ---------------------------------------------------------------------------------------------------------------------
def _model(sparse: bool, D: int):
    torch.manual_seed(9)
    mu, sigma = TKC.kernels(11)
    if sparse:
        m = CIKM20_TK_Sparse(D, mu.tolist(), sigma.tolist(), att_heads=4, att_layer=1, att_proj_dim=32, att_ff_dim=64,
                             max_length=64, use_diff_posencoding=True)
    else:
        m = ECAI20_TK(D, mu.tolist(), sigma.tolist(), att_heads=4, att_layer=1, att_ff_dim=64, max_length=64,
                      use_diff_posencoding=True, mix_hybrid_context=True)
    with torch.no_grad():
        m.kernel_bin_weights.weight.uniform_(-0.05, 0.05)
    return m.cuda().eval()


@pytest.mark.parametrize("sparse", [False, True], ids=["tk", "tk_sparse"])
def test_rerank_ties_tails_and_void_queries(sparse):
    """640 candidates per query over a store of 700 passages: two passages with identical rows (and gates) tie exactly
    and come out in ascending id order; a query with 40 void candidates asked for all 640 ends in 40 (-inf, -1); a query
    whose candidates are all -1 gets only (-inf, -1).  Scores are the store kernel's bits, ranked (score desc, id asc)."""
    D, n_docs, nq, Lq, C_ = 64, 700, 3, 12, 640
    g = torch.Generator().manual_seed(3)
    lens = torch.randint(1, 61, (n_docs,), generator=g)
    off = np.concatenate([[0], np.cumsum(lens.numpy())])
    rows = torch.randn(int(off[-1]), D, generator=g)
    gates = torch.rand(int(off[-1]), generator=g) + 0.1
    a, b = 17, 401                                     # passage b is a copy of passage a
    lens_b = int(lens[a])
    rows_l, gates_l, lens_l = [], [], lens.clone()
    lens_l[b] = lens_b
    for d in range(n_docs):
        src = a if d == b else d
        rows_l.append(rows[off[src]:off[src + 1]])
        gates_l.append(gates[off[src]:off[src + 1]])
    rows, gates = torch.cat(rows_l), torch.cat(gates_l)
    idm = np.repeat(np.arange(n_docs), lens_l.numpy())
    model = _model(sparse, D)
    cfg = {"token_dim": D, "faiss_use_gpu": True, "token_dtype": "float32"}
    st = TKDocumentStore(cfg, model)
    st.index([idm], [rows.numpy().astype(np.float32)], [gates.numpy().astype(np.float32)] if sparse else None)
    q = torch.randn(nq, Lq, D, generator=g).cuda()
    qm = torch.ones(nq, Lq, device="cuda")
    qm[1, 7:] = 0
    others = torch.tensor([d for d in range(n_docs) if d not in (a, b)])
    cand = torch.full((nq, C_), -1, dtype=torch.int64)
    for r in range(2):   # distinct candidates, both copies among them
        row = torch.cat([torch.tensor([b, a]), others[torch.randperm(len(others), generator=g)[:C_ - 2]]])
        cand[r] = row[torch.randperm(C_, generator=g)]
    void = torch.randperm(C_, generator=g)
    void = void[(cand[1, void] != a) & (cand[1, void] != b)][:40]
    cand[1, void] = -1
    cand[2] = -1
    cand = cand.cuda()
    s, ids = st.rerank(q, qm, cand, top_n=C_ + 10)
    assert s.shape == (nq, C_) and ids.shape == (nq, C_)
    pq = torch.arange(nq, device="cuda", dtype=torch.int32).repeat_interleave(C_)
    extra = {"gate": st.gate} if sparse else {}
    with torch.no_grad():
        flat = model.score_store(q, qm, st.rows, st.offsets, pq, cand.view(-1).to(torch.int32),
                                 max_doc_len=st.max_doc_len, **extra).view(nq, C_).cpu()
    cand, s, ids = cand.cpu(), s.cpu(), ids.cpu()
    for r in range(nq):
        live = [(float(flat[r, j]), int(cand[r, j])) for j in range(C_) if cand[r, j] >= 0]
        assert all(np.isfinite(v) for v, _ in live)
        exp = sorted(live, key=lambda x: (-x[0], x[1])) + [(float("-inf"), -1)] * (C_ - len(live))
        assert [(float(v), int(i)) for v, i in zip(s[r], ids[r])] == exp, f"query {r}"
        if r < 2:
            pos = {int(i): j for j, i in enumerate(ids[r].tolist())}
            assert s[r, pos[a]] == s[r, pos[b]] and pos[b] == pos[a] + 1, "identical passages do not tie in id order"
    assert (ids[1, -40:] == -1).all() and torch.isneginf(s[1, -40:]).all()
    assert (ids[2] == -1).all() and torch.isneginf(s[2]).all()
