"""ColBERT max-sim across its whole instantiation matrix (tests/maxsim_cases.py): every compiled instantiation of the
queries-on-M, documents-on-M and SIMT forward kernels and of the two backward kernels, at the reference configuration
(dim 768, Lq 30, Ld 200), at the tile, query-chunk and shared-memory edges, in store mode and for in-batch scoring.

The inputs are small integers, so every kernel's fp32 arithmetic is exact: scores, argmax and gradients are held
bit-exactly to the fp64 oracle (colbert.py:68-75 with an explicit argmax).  NaN / +-inf in masked query tokens, masked
document rows, rows past a passage's max_doc_len and the memory after the document tensor must change nothing.  The
end-to-end autograd test runs real values at the reference configuration against fp64 autograd of the reference
expression; its worst error / scale per gradient is recorded as a test property (``--junitxml``).  The e4m3 and
residual store rows are held bit-exactly to the fp64 store oracle, to the 16-bit kernel on the same values, and under a
permutation of their pairs; the premise of the exact e4m3 rows (the FP8 MMA sums below 2^11 grains exactly, subnormals
kept) has its own test."""
import ctypes
import functools

import pytest
import torch

import maxsim_cases as C
from conftest import assert_close_rel
from matchmaker_b200 import _lib, autograd, interaction

pytestmark = pytest.mark.gpu
DEV = "cuda"


@functools.lru_cache(maxsize=None)
def _smem() -> int:
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


@functools.lru_cache(maxsize=2)
def _prepared(row: C.Row):
    """Inputs on the device (clean, and poisoned with NaN / inf where nothing may read), the oracle's results."""
    c = C.make_case(row)
    score, arg = C.oracle(c, fill=row.mode != "store")
    P = {"c": c, "score": score, "arg": arg, "qm": c.qm.to(DEV), "dm": c.dm.to(DEV),
         "q": c.q.to(row.dtype).to(DEV), "d": c.d.to(row.dtype).to(DEV)}
    if row.mode == "store":
        P["store"], P["offsets"] = c.store.to(row.dtype).to(DEV), c.offsets.to(DEV)
        P["pair_q"], P["pair_d"] = c.pair_q.to(DEV), c.pair_d.to(DEV)
        return P
    qp, dp = C.poisoned(c, row)
    P["qp"] = qp.to(row.dtype).to(DEV)
    # one more document of NaN after the last: rows >= Ld of the last document are never read
    big = torch.full((row.n_d + 1,) + tuple(dp.shape[1:]), float("nan"), dtype=row.dtype, device=DEV)
    big[: row.n_d] = dp.to(row.dtype).to(DEV)
    P["dp"] = big[: row.n_d]
    P["pair_q"], P["pair_d"], P["pair_dm"] = (t.to(torch.int32).to(DEV) for t in (c.pair_q, c.pair_d, c.pair_dm))
    return P


def _call(row: C.Row, P, impl: str, argmax: bool = False, poisoned: bool = True):
    if row.mode == "store":
        return interaction.maxsim_store(P["q"], P["store"], P["offsets"], P["pair_q"], P["pair_d"], row.Ld, impl=impl)
    q, d = (P["qp"], P["dp"]) if poisoned else (P["q"], P["d"])
    if row.mode == "pairs":
        return interaction.maxsim(q, d, P["qm"], P["dm"], docs_per_query=row.dpq, impl=impl, return_argmax=argmax)
    if not argmax:
        return interaction.maxsim_allpairs(q, P["qm"], d, P["dm"], impl=impl, reference_mask_indexing=True).view(-1)
    return interaction.maxsim(q, d, P["qm"], P["dm"], pair_q=P["pair_q"], pair_d=P["pair_d"], pair_dmask=P["pair_dm"],
                              impl=impl, return_argmax=True)


def _exact(got, ref, what):
    got = got.detach().cpu().to(ref.dtype)
    assert got.shape == ref.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}"
    bad = got != ref
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.numel()} differ, first at {bad.nonzero()[0].tolist()}: "
                           f"{got[bad][0].item()} vs {ref[bad][0].item()}")


@functools.lru_cache(maxsize=2)
def _coded(row: C.Row, bits: int):
    """An e4m3 or residual store row on the device, with its oracle scores."""
    c = C.make_store_case(row, bits)
    P = {"c": c, "score": C.store_oracle(c, row.Ld), "offsets": c.offsets.to(DEV),
         "pair_q": c.pair_q.to(torch.int32).to(DEV), "pair_d": c.pair_d.to(torch.int32).to(DEV)}
    if row.dtype == C.E4:
        store8 = c.store.float().to(C.E4)
        nan = torch.isnan(c.store)
        assert bool(((store8.view(torch.uint8)[nan] & 0x7F) == 0x7F).all())   # the e4m3 NaN, in rows no pair reads
        P["q"], P["store"] = c.q.float().to(C.E4).to(DEV), store8.to(DEV)
    else:
        P["q"] = c.q.half().to(DEV)
        P["codes"], P["list_ids"] = c.codes.to(DEV), c.list_ids.to(DEV)
        P["base"], P["weight"] = c.base.to(DEV), c.weight.to(DEV)
        P["store"] = c.store.half().to(DEV)   # the decoded rows (NaN where the poison list stands)
    return P


def _call_coded(row: C.Row, P, key, pair_q=None, pair_d=None):
    pq = P["pair_q"] if pair_q is None else pair_q
    pd = P["pair_d"] if pair_d is None else pair_d
    if key[0] == "score":
        return interaction.maxsim_store(P["q"], P["store"], P["offsets"], pq, pd, row.Ld, impl=key[1])
    return interaction.maxsim_store_residual(P["q"], P["codes"], P["list_ids"], P["base"], P["weight"], key[1],
                                             P["offsets"], pq, pd, row.Ld)


def _coded_rows_bit_exact(row: C.Row):
    """Every path of an e4m3 / residual store row against the fp64 store oracle; two runs; a permutation of the pairs;
    the 16-bit documents-on-M kernel on the same values (e4m3) or on the decoded rows (residual) where it takes the
    shape."""
    runs = C.runs(row, _smem())
    fp16_docm = C.route(C.H, row.Lq, row.Ld, row.dim, "tcgen05_docm", store=True, smem=_smem())
    for key, name in runs.items():
        P = _coded(row, 0 if key[0] == "score" else key[1])
        if name is None:
            with pytest.raises(_lib.MatchmakerB200Error):
                _call_coded(row, P, key)
            continue
        got = _call_coded(row, P, key)
        _exact(got, P["score"], f"{row} {key} ({name})")
        assert torch.equal(_call_coded(row, P, key), got), f"{row} {key}: two runs differ"
        perm = torch.randperm(row.n_pairs, generator=torch.Generator().manual_seed(row.seed)).to(DEV)
        permuted = _call_coded(row, P, key, P["pair_q"][perm], P["pair_d"][perm])
        assert torch.equal(permuted, got[perm]), f"{row} {key}: permuted pairs"
        if fp16_docm is not None and key != ("score", "tcgen05_docm"):
            q16 = P["q"].half() if row.dtype == C.E4 else P["q"]
            h = interaction.maxsim_store(q16, P["store"].half(), P["offsets"], P["pair_q"], P["pair_d"], row.Ld,
                                         impl="tcgen05_docm")
            assert torch.equal(h, got), f"{row} {key}: the fp16 kernel {fp16_docm} on the same values differs"


@pytest.mark.parametrize("row", C.MATRIX, ids=str)
def test_scores_bit_exact_on_every_path(row):
    if row.coded:
        return _coded_rows_bit_exact(row)
    runs = C.runs(row, _smem())
    for impl in C.IMPLS:
        if runs[("score", impl)] is None:
            with pytest.raises(_lib.MatchmakerB200Error):
                _call(row, _prepared(row), impl)
            continue
        for poisoned in ((True,) if row.mode == "store" else (False, True)):
            got = _call(row, _prepared(row), impl, poisoned=poisoned)
            _exact(got, _prepared(row)["score"], f"{row} {impl} ({runs[('score', impl)]}) poisoned={poisoned}")


@pytest.mark.parametrize("row", [r for r in C.MATRIX if r.mode in ("pairs", "inbatch")], ids=str)
def test_argmax_bit_exact_on_both_producers(row):
    runs = C.runs(row, _smem())
    P = _prepared(row)
    by_kernel = {}
    for impl in C.ARGMAX_IMPLS:
        name = runs[("argmax", impl)]
        if name is None:
            with pytest.raises(_lib.MatchmakerB200Error):
                _call(row, P, impl, argmax=True)
            continue
        for poisoned in (False, True):
            s, am = _call(row, P, impl, argmax=True, poisoned=poisoned)
            _exact(s, P["score"], f"{row} {impl} ({name}) score")
            _exact(am, P["arg"], f"{row} {impl} ({name}) argmax poisoned={poisoned}")
            by_kernel[name.split("<")[0]] = am
    if C.QM in by_kernel and C.SIMT in by_kernel:
        assert torch.equal(by_kernel[C.QM], by_kernel[C.SIMT])


@pytest.mark.parametrize("row", [r for r in C.MATRIX if r.mode == "pairs"], ids=str)
def test_backward_bit_exact(row):
    """interaction.maxsim_bwd from the oracle's argmax: fp32 grad_q and grad_d equal the gradient written out from it,
    with exact zeros in masked, unselected and padding positions, and the same bits run to run."""
    P = _prepared(row)
    c = P["c"]
    arg = P["arg"].to(torch.int32).to(DEV)
    gout = c.gout.to(DEV)
    gq, gd = interaction.maxsim_bwd(P["qp"], P["dp"], gout, arg, row.dpq)
    ref_q, ref_d = C.oracle_grads(c, P["arg"], row.dpq)
    _exact(gq, ref_q, f"{row} grad_q")
    _exact(gd, ref_d, f"{row} grad_d")
    assert (gq.cpu()[~c.qm.bool()] == 0).all() and (gd.cpu()[~c.dm.bool()] == 0).all()
    gq2, gd2 = interaction.maxsim_bwd(P["qp"], P["dp"], gout, arg, row.dpq)
    assert torch.equal(gq, gq2) and torch.equal(gd, gd2)


@pytest.mark.parametrize("dtype", [C.H, C.BF, C.F32], ids=lambda t: C.SHORT[t])
def test_autograd_at_the_reference_configuration(dtype, record_property):
    """autograd.maxsim end to end on real values at dim 768, Lq 30, Ld 200 (f16 under autocast, as the reference
    trains), against fp64 autograd of colbert.py:68-75 on the same values.  Scores to 1e-3; gradients to 1e-3 (bf16:
    2^-8, the unit roundoff of the bf16 gradient autograd returns) except where the top-2 margin of a token's scores
    does not decide its argmax in fp32."""
    n_q, dpq, n_d, Lq, Ld, dim = 4, 3, 11, 30, 200, 768
    g = torch.Generator().manual_seed(768)
    q = (torch.randn(n_q, Lq, dim, generator=g) * 0.3).to(dtype)
    d = (torch.randn(n_d, Ld, dim, generator=g) * 0.3).to(dtype)
    qm = (torch.arange(Lq).unsqueeze(0) < torch.randint(5, Lq + 1, (n_q, 1), generator=g)).long()
    dm = (torch.arange(Ld).unsqueeze(0) < torch.randint(20, Ld + 1, (n_d, 1), generator=g)).long()
    dm &= (torch.rand(n_d, Ld, generator=g) > 0.05).long()
    dm[0] = 1
    gout = torch.randn(n_d, generator=g)
    ref, rq, rd = C.reference_autograd(q, d, qm, dm, dpq, gout)
    cq, cd = q.to(DEV).requires_grad_(True), d.to(DEV).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16, enabled=dtype == C.H):
        out = autograd.maxsim(cq, cd, qm.to(DEV), dm.to(DEV), docs_per_query=dpq)
    out.backward(gout.to(DEV))
    assert_close_rel(out, ref, what="score")
    # tokens whose two best scores lie within fp32 reach of each other: their gradient may go to either row
    S = torch.bmm(q.double().repeat_interleave(dpq, 0)[:n_d], d.double().transpose(1, 2))
    S = S.masked_fill(~dm.bool().unsqueeze(1), C.FILL)
    top = S.topk(2, dim=-1)
    live = qm.bool().repeat_interleave(dpq, 0)[:n_d]
    amb = live & ((top.values[..., 0] - top.values[..., 1]) <= 1e-4 * top.values[..., 0].abs().clamp(min=1.0))
    keep_q = torch.ones(n_q, Lq, dtype=torch.bool)
    keep_d = torch.ones(n_d, Ld, dtype=torch.bool)
    for p, i in amb.nonzero().tolist():
        keep_q[p // dpq, i] = False
        keep_d[p, top.indices[p, i]] = False
    record_property("ambiguous tokens", int(amb.sum()))
    bar = 2.0 ** -8 if dtype == C.BF else 1e-3
    for name, got, want, keep in (("grad_q", cq.grad, rq, keep_q), ("grad_d", cd.grad, rd, keep_d)):
        got, want = got.double().cpu()[keep], want[keep]
        scale = want.abs().max().item()
        record_property(f"{C.SHORT[dtype]} {name} worst error / scale", f"{(got - want).abs().max().item() / scale:.2e}")
        assert_close_rel(got, want, rel=bar, what=name)


def test_empty_batch():
    """No pairs: empty scores and argmax, empty gradients; queries without documents get a zero gradient."""
    q = torch.empty(0, 30, 768, dtype=C.H, device=DEV)
    d = torch.empty(0, 200, 768, dtype=C.H, device=DEV)
    qm = torch.empty(0, 30, dtype=torch.long, device=DEV)
    dm = torch.empty(0, 200, dtype=torch.long, device=DEV)
    s, am = interaction.maxsim(q, d, qm, dm, return_argmax=True)
    assert s.shape == (0,) and am.shape == (0, 30)
    gq, gd = interaction.maxsim_bwd(q, d, s, am)
    assert gq.shape == q.shape and gd.shape == d.shape
    cq, cd = q.clone().requires_grad_(True), d.clone().requires_grad_(True)
    autograd.maxsim(cq, cd, qm, dm).sum().backward()
    assert cq.grad.shape == q.shape and cd.grad.shape == d.shape
    q2 = torch.ones(2, 30, 768, dtype=C.H, device=DEV, requires_grad=True)
    out = autograd.maxsim(q2, d, None, dm)
    assert out.shape == (0,)
    out.sum().backward()
    assert q2.grad is not None and (q2.grad == 0).all()


EDGE_DIMS = list(range(64, 1025, 64)) + [100, 1088]


@pytest.mark.parametrize("train", [False, True], ids=["auto", "training"])
@pytest.mark.parametrize("dim", EDGE_DIMS)
def test_envelope_edge_per_dim(dim, train):
    """The last Lq that runs at this dim (``auto``; with the argmax: the training forward) matches the oracle; the next
    one is refused by the host with MatchmakerB200Error and launches nothing."""
    last = C.last_lq(C.H, dim, train, _smem())
    assert last >= 1
    Ld = 9
    g = torch.Generator().manual_seed(dim + 7 * train)
    for Lq in (last, last + 1):
        q = torch.randint(-3, 4, (1, Lq, dim), generator=g).float()
        d = torch.randint(-3, 4, (1, Ld, dim), generator=g).float()
        qm = torch.ones(1, Lq, dtype=torch.long)
        dm = torch.ones(1, Ld, dtype=torch.long)
        dm[0, -2] = 0
        cq, cd = q.half().to(DEV), d.half().to(DEV)
        if Lq == last:
            got = interaction.maxsim(cq, cd, qm.to(DEV), dm.to(DEV), return_argmax=train)
            p = torch.zeros(1, dtype=torch.long)
            score, arg = C.oracle(C.Case(q, d, qm, dm, p, p, p, torch.ones(1)))
            _exact(got[0] if train else got, score, f"dim {dim} Lq {Lq}")
            if train:
                _exact(got[1], arg, f"dim {dim} Lq {Lq} argmax")
            continue
        out = torch.full((1,), 12345.0, device=DEV)
        am = torch.full((1, Lq), -7, dtype=torch.int32, device=DEV) if train else None
        cqm, cdm = qm.to(DEV), dm.to(DEV)
        lib = _lib.load()
        rc = lib.mmb200_maxsim_fwd(cq.data_ptr(), cd.data_ptr(), cqm.data_ptr(), cdm.data_ptr(), None, None, None,
                                   out.data_ptr(), None if am is None else am.data_ptr(), 1, 1, 1, 1, Lq, Ld, dim,
                                   _lib.F16, _lib.MASK_I64, _lib.IMPL_AUTO, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc in (_lib.ERR_INVALID, _lib.ERR_UNSUPPORTED), f"dim {dim} Lq {Lq}: rc {rc}"
        torch.cuda.synchronize()
        assert out.item() == 12345.0 and (am is None or (am == -7).all()), "a kernel ran"
        with pytest.raises(_lib.MatchmakerB200Error):
            interaction.maxsim(cq, cd, cqm, cdm, return_argmax=train)


def _one_row_passages(q: torch.Tensor, rows: torch.Tensor):
    """maxsim_store over e4m3 passages of one row each with a one-token query: the dot product of every row."""
    n = rows.shape[0]
    off = torch.arange(n + 1, dtype=torch.int64, device=DEV)
    pd = torch.arange(n, dtype=torch.int32, device=DEV)
    return interaction.maxsim_store(q.view(1, 1, -1).to(C.E4).to(DEV), rows.to(C.E4).to(DEV), off,
                                    torch.zeros(n, dtype=torch.int32, device=DEV), pd, 1)


def test_fp8_mma_accumulates_exactly():
    """The premise of the exact e4m3 rows, at dim 1024 (32 k32 steps): sums of products below 2^11 grains come out
    exact in both e4m3 kernels (max-sim and the flat top-k), whatever the order: partial sums at the bound before the
    last k32 step with a +-1 product in it, a large early sum cancelled back to a small total, and the grain at 2^-9
    (e4m3 subnormals).  Fails if the FP8 MMA drops low bits of its accumulator or flushes subnormal inputs."""
    dim = 1024
    q = torch.zeros(dim, dtype=torch.float64)
    rows = []
    # 2046 in the first 992 dimensions (511 products of 4, one of 2), then +-1 in the last k32 step
    qa = q.clone()
    qa[:512] = 2.0
    qa[1000] = 1.0
    for last in (1.0, -1.0):
        r = torch.zeros(dim, dtype=torch.float64)
        r[:511], r[511] = 2.0, 1.0
        r[1000] = last
        rows.append(r)
    # +1024 in the first 16 steps, -1020 in the next 8, +1 in the last: 5 out of a mass of 2045
    qb = q.clone()
    qb[:512], qb[512:767], qb[1000] = 2.0, 4.0, 1.0
    r = torch.zeros(dim, dtype=torch.float64)
    r[:512], r[512:767], r[1000] = 1.0, -1.0, 1.0
    rows.append(r)
    # the grain at 2^-9: one subnormal product, and 2047 of them
    sub1 = torch.zeros(dim, dtype=torch.float64)
    sub1[1023] = 2.0 ** -9
    sub2 = torch.zeros(dim, dtype=torch.float64)
    sub2[:1023] = 2.0 ** -9
    sub2[1023] = 2.0 ** -8
    cases = [(qa, rows[0]), (qa, rows[1]), (qb, rows[2]), (torch.ones(dim, dtype=torch.float64), sub1),
             (torch.ones(dim, dtype=torch.float64), sub2)]
    for i, (qq, r) in enumerate(cases):
        assert torch.equal(qq.to(C.E4).double(), qq) and torch.equal(r.to(C.E4).double(), r)
        grain = 2.0 ** -9 if (r != r.round()).any() else 1.0
        mass = float((qq * r).abs().sum()) / grain
        assert mass < C.E4M3_EXACT_GRAINS, (i, mass)
        want = float((qq * r).sum())
        got = _one_row_passages(qq, r.view(1, -1)).item()
        assert got == want, f"case {i}: max-sim {got} vs {want} (mass {mass} grains)"
        s, _ = interaction.flat_ip_topk(qq.view(1, -1).to(C.E4).to(DEV), r.view(1, -1).to(C.E4).to(DEV), 1)
        assert s.item() == want, f"case {i}: flat top-k {s.item()} vs {want}"


@pytest.mark.parametrize("dim", list(range(64, 1025, 64)))
def test_e4m3_and_residual_envelope_edge_per_dim(dim):
    """The last Lq each coded store kernel runs at this dim matches the oracle, and the next one is refused."""
    g = torch.Generator().manual_seed(dim)
    off = torch.tensor([0, 5, 9], dtype=torch.int64)
    pq, pd = torch.tensor([0, 0, 0], dtype=torch.int32), torch.tensor([1, -1, 0], dtype=torch.int32)
    kinds = [("residual", b, C.last_lq_residual(dim, b, _smem())) for b in C.RESIDUAL_BITS]
    if dim % 128 == 0:
        kinds.append(("e4m3", 0, C.last_lq_e4m3(dim, _smem())))
    for kind, bits, last in kinds:
        for Lq in (last, last + 1):
            q = torch.randint(-1, 2, (1, Lq, dim), generator=g).double()
            if kind == "e4m3":
                store = torch.randint(-2, 3, (9, dim), generator=g).double()
                c = C.StoreCase(q, store, off, pq.long(), pd.long())
                call = functools.partial(interaction.maxsim_store, q.float().to(C.E4).to(DEV),
                                         store.float().to(C.E4).to(DEV))
            else:
                base = torch.randint(-1, 2, (2, dim), generator=g).half()
                weight = torch.randint(-2, 3, (dim, 1 << bits), generator=g).half()
                raw = torch.randint(0, 1 << bits, (9, dim), generator=g)
                lid = torch.tensor([0, 1, 0, 1, 0, 1, 1, 0, 0], dtype=torch.int32)
                import colbert_residual_oracle as RO
                packed = torch.from_numpy(RO.pack(raw.numpy().astype("uint8"), bits))
                dec = RO.decode(packed.numpy(), lid.numpy(), base.numpy(), weight.numpy(), bits)
                c = C.StoreCase(q, torch.from_numpy(dec.astype("float64")), off, pq.long(), pd.long())
                call = functools.partial(interaction.maxsim_store_residual, q.half().to(DEV), packed.to(DEV),
                                         lid.to(DEV), base.to(DEV), weight.to(DEV), bits)
            args = (off.to(DEV), pq.to(DEV), pd.to(DEV), 7)
            if Lq == last:
                _exact(call(*args), C.store_oracle(c, 7), f"{kind} b{bits} dim {dim} Lq {Lq}")
            else:
                with pytest.raises(_lib.MatchmakerB200Error):
                    call(*args)
