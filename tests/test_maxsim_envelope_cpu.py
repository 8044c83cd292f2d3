"""The shared cases of the max-sim envelope tests (tests/maxsim_cases.py), checked without a GPU: the fp64 oracle is
torch autograd of colbert.py:68-75 except where its tie rule is documented to differ, every row claims what the routing
rules give it, the rows between them claim every max-sim instantiation compiled into the library and every launch
configuration the matrix is there for, and the inputs hold the preconditions the GPU tests rely on.  Also the empty batch
at the C ABI."""
import ctypes
import re
import shutil
import subprocess

import pytest
import torch

import maxsim_cases as C
from matchmaker_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
INSTANTIATION = re.compile(r"\b(" + "|".join(C.KERNELS) + r")<([^>]*)>")
PAIRS_ROWS = [r for r in C.MATRIX if r.mode == "pairs" and r.n_pairs * r.Lq * r.Ld * r.dim <= 3e7]


def _close(a, b, what):
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-9, msg=lambda m: f"{what}: {m}")


@pytest.mark.parametrize("shape", [(2, 3, 5, 7, 9, 16), (3, 2, 5, 30, 40, 64), (1, 1, 1, 1, 1, 8), (2, 4, 8, 33, 20, 12)])
def test_oracle_is_torch_autograd_on_real_values(shape):
    """Tie-free real values, masks with holes, a fully masked document, a masked query token, the last query partial."""
    n_q, dpq, n_d, Lq, Ld, dim = shape
    g = torch.Generator().manual_seed(sum(shape))
    q, d = torch.randn(n_q, Lq, dim, generator=g), torch.randn(n_d, Ld, dim, generator=g)
    qm = (torch.rand(n_q, Lq, generator=g) > 0.2).long()
    dm = (torch.rand(n_d, Ld, generator=g) > 0.3).long()
    qm[0, 0] = dm[0, 0] = 1
    if n_d > 2:
        dm[2] = 0
        d[1] *= -300.0            # real scores far below -1000: the fill wins where document 1 has a masked row
    p = torch.arange(n_d)
    c = C.Case(q, d, qm, dm, p // dpq, p, p, torch.randn(n_d, generator=g))
    score, arg = C.oracle(c)
    gq, gd = C.oracle_grads(c, arg, dpq)
    ref, rq, rd = C.reference_autograd(q, d, qm, dm, dpq, c.gout)
    _close(score, ref, "score")
    _close(gq, rq, "grad_q")
    _close(gd, rd, "grad_d")


@pytest.mark.parametrize("row", PAIRS_ROWS, ids=str)
def test_oracle_is_torch_autograd_on_the_matrix_inputs_but_for_the_fill_tie(row):
    """On the matrix's integer inputs (exact ties between real rows, fill wins, fully masked documents and queries) the
    oracle and torch autograd agree exactly, but for one documented difference: where a real row scores exactly -1000
    after a masked row, torch's first-index max picks the masked row (whose gradient the fill assignment drops), while
    the kernels and the oracle let the real row win."""
    c = C.make_case(row)
    score, arg = C.oracle(c)
    gq, gd = C.oracle_grads(c, arg, row.dpq)
    ref, rq, rd = C.reference_autograd(c.q, c.d, c.qm, c.dm, row.dpq, c.gout)
    assert torch.equal(score, ref)
    tie = row.Ld >= 8 and row.n_d > C.TIE1000_DOC
    if tie:
        qi = int(c.pair_q[C.TIE1000_DOC])
        assert int(arg[C.TIE1000_DOC, 0]) == C.TIE1000_REAL
        g = float(c.gout[C.TIE1000_DOC])
        rq[qi, 0] += g * c.d[C.TIE1000_DOC, C.TIE1000_REAL].double()
        rd[C.TIE1000_DOC, C.TIE1000_REAL] += g * c.q[qi, 0].double()
    assert torch.equal(gq, rq)
    assert torch.equal(gd, rd)


def test_rows_claim_what_the_routing_gives_them():
    every = set()
    for row in C.MATRIX:
        assert set(row.claims) == C.dispatched(row), str(row)
        every |= set(row.claims)
    T = [C.TNAME[t] for t in (C.H, C.BF)]
    expect = ({C.inst(C.TC, t, k, n) for t in T for k in (1, 2) for n in (1, 2, 3, 4)}
              | {C.inst(C.QM, t, a, s) for t in T for a, s in ((False, False), (True, False), (False, True))}
              | {C.inst(k, C.TNAME[t]) for k in (C.SIMT, C.BWD_D, C.BWD_Q) for t in (C.H, C.BF, C.F32)}
              | {C.inst(C.TC_FP8, k, n) for k in (1, 2) for n in (1, 2, 3, 4)}
              | {C.inst(C.TC_RES, k, n, b) for k in (1, 2) for n in (1, 2, 3, 4) for b in (1, 2)})
    assert len(expect) == 55
    assert every == expect


def test_every_row_is_needed():
    """Between them the rows hold every instantiation and every required configuration, and each row holds one that no
    other row does: deleting a row fails this test."""
    feats = [C.features(r) for r in C.MATRIX]
    assert C.REQUIRED_FEATURES <= set().union(*feats), sorted(C.REQUIRED_FEATURES - set().union(*feats))
    for k, row in enumerate(C.MATRIX):
        others = [j for j in range(len(C.MATRIX)) if j != k]
        own = (set(row.claims) - set().union(*(C.MATRIX[j].claims for j in others))) \
            | ((feats[k] & C.REQUIRED_FEATURES) - set().union(*(feats[j] for j in others)))
        assert own, f"{row} holds nothing another row does not"


def test_launch_configurations_and_envelope_edges():
    """The reference configuration's launch, and the Lq limits per dim on an H100 (232 448 B of shared memory)."""
    assert C.route(C.H, 30, 200, 768, "auto") == "maxsim_tc_kernel<__half,2,1>"
    assert C.tc_launch(30, 768, C.SMEM_OPTIN_H100) == {"kbs": 2, "nc": 1, "qslots": 2, "stages": 3}
    assert C.route(C.H, 30, 200, 768, "auto", argmax=True) == "maxsim_simt_kernel<__half>"
    auto = {dim: C.last_lq(C.H, dim, False) for dim in range(64, 1025, 64)}
    train = {dim: C.last_lq(C.H, dim, True) for dim in range(64, 1025, 64)}
    assert {d for d, lq in auto.items() if lq == 96} == {640, 768, 832, 960}
    assert {d for d, lq in auto.items() if lq == 64} == {896, 1024}
    assert all(lq == 128 for d, lq in auto.items() if d not in (640, 768, 832, 896, 960, 1024))
    assert train[768] == 74 and train[1024] == 56 and train[384] == 128 and train[448] == 127
    assert C.last_lq(C.BF, 768, False) == 96 and C.last_lq(C.BF, 768, True) == 74
    assert C.last_lq(C.F32, 768, False) == 74   # f32 runs on the SIMT kernel only


def test_e4m3_and_residual_envelopes():
    """plan_tc over e4m3 (1-byte elements) and over residual codes (16-bit tiles beside the weight table) on an H100."""
    e4 = {dim: C.last_lq_e4m3(dim) for dim in range(128, 1025, 128)}
    assert set(e4.values()) == {128}
    one_slot = {dim: min([lq for lq in range(1, 129) if C.plan_tc(lq, dim, C.SMEM_OPTIN_H100, 1)["qslots"] == 1]
                         or [0]) for dim in e4}
    assert one_slot == {128: 0, 256: 0, 384: 0, 512: 0, 640: 0, 768: 97, 896: 97, 1024: 65}
    assert C.plan_tc(128, 1024, C.SMEM_OPTIN_H100, 1) == {"kbs": 2, "nc": 4, "qslots": 1, "stages": 2}
    for bits in (1, 2):
        res = {dim: C.last_lq_residual(dim, bits) for dim in range(64, 1025, 64)}
        assert {d for d, lq in res.items() if lq == 96} == ({640, 768, 832, 960} if bits == 1 else {640, 768, 832})
        assert {d for d, lq in res.items() if lq == 64} == ({896, 1024} if bits == 1 else {896, 960, 1024})
        assert res[704] == 128 and all(lq == 128 for d, lq in res.items() if d < 640)
        for lq in range(1, 65):
            assert C.plan_tc(lq, 1024, C.SMEM_OPTIN_H100, 2, C.residual_extra(1024, bits))["stages"] == 2
    assert C.route_e4m3(30, 768, "simt") is None and C.route_e4m3(30, 768, "tcgen05") is None
    assert C.route_e4m3(30, 768, "auto") == C.route_e4m3(30, 768, "tcgen05_docm") == "maxsim_tc_fp8_kernel<2,1>"
    assert C.route_e4m3(30, 704, "auto") is None and C.route_e4m3(129, 128, "auto") is None


CODED_ROWS = [(r, b) for r in C.MATRIX if r.coded for b in ((0,) if r.dtype == C.E4 else C.RESIDUAL_BITS)]


@pytest.mark.parametrize("row,bits", CODED_ROWS, ids=lambda v: str(v) if isinstance(v, C.Row) else f"b{v}")
def test_store_cases_hold_their_preconditions(row, bits):
    """e4m3 and residual store rows: exact inputs, the layout the row claims, and inputs that would change the result if
    a kernel read past a window (neg rows), flushed subnormals (the subnormal passage) or read a poisoned row."""
    c = C.make_store_case(row, bits)
    score = C.store_oracle(c, row.Ld)
    assert not torch.isnan(score).any(), "a window holds a poisoned row"
    lens = c.offsets[1:] - c.offsets[:-1]
    void = (c.pair_d < 0) | (lens[c.pair_d.clamp(min=0)] == 0)
    assert torch.equal(torch.isinf(score), void) and bool((score[void] < 0).all())
    assert int(c.offsets[-1]) == c.store.shape[0]
    if row.dtype == C.E4:
        C.assert_exact_e4m3(c, row.Ld)
    else:
        assert torch.equal(c.q, c.q.round()) and float(c.q.abs().max()) <= 3
        live = ~torch.isnan(c.store)
        assert torch.equal(c.store[live], c.store[live].round()) and float(c.store[live].abs().max()) <= 5
        assert torch.isnan(c.base[-1]).all() and not torch.isnan(c.base[:-1]).any()
    if row.pairs > 1:
        assert tuple(lens[: len(C.LAYOUT)].tolist()) == C.LAYOUT and (lens > row.Ld).any()
        assert (c.pair_d == -1).any()
        last = c.store.shape[0] - 1
        assert any(c.window(d, row.Ld)[1] - 1 == last for d in c.pair_d.tolist()), "no window ends at the last row"
        assert (c.pair_q[1:] != c.pair_q[:-1]).all(), "the query must change every pair"
        returns = [p for p in range(2, c.pair_q.numel()) if int(c.pair_q[p]) in c.pair_q[max(0, p - 3):p - 1].tolist()]
        assert returns, "no pair comes back to an earlier query"
        hot = c.pair_q[c.pair_d == C.LAYOUT.index(257)]
        assert hot.numel() > row.n_q and torch.unique(hot).numel() >= min(row.n_q, 2)
        referenced = set(c.pair_d.tolist())
        assert all(d in referenced for d in range(row.n_d) if d != c.poison_doc)
    if row.regime == "neg":
        live = ~void
        assert (C.store_oracle(c, row.Ld, extra=1)[live] != score[live]).all(), "reading one more row changes nothing"
        for p in live.nonzero().flatten().tolist():
            a, b = c.window(int(c.pair_d[p]), row.Ld)
            assert (c.q[c.pair_q[p]] @ c.store[a:b].T < 0).all()
    else:
        assert torch.isnan(c.store).any(), "no poison"
        if row.pairs > 1:
            a, b = int(c.offsets[c.poison_doc]), int(c.offsets[c.poison_doc + 1])
            assert b > a and torch.isnan(c.store[a:b]).all() and c.poison_doc not in c.pair_d.tolist()
    if c.subnormal_doc >= 0:
        a, b = int(c.offsets[c.subnormal_doc]), int(c.offsets[c.subnormal_doc + 1])
        sub = c.store[a:b]
        assert ((sub.abs() < C.E4M3_MIN_NORMAL) & (sub != 0)).any(1).all() and (sub.abs() < C.E4M3_MIN_NORMAL).all()
        sel = c.pair_d == c.subnormal_doc
        assert sel.any() and (C.store_oracle(c, row.Ld, flush=True)[sel] != score[sel]).all(), "flushing changes nothing"


def test_cases_hold_their_preconditions():
    for row in C.MATRIX:
        if row.coded:
            continue
        c = C.make_case(row)
        for t in (c.q, c.d, c.gout):
            assert torch.equal(t, t.round()) and t.abs().max() <= 8
            assert torch.equal(t.to(C.BF).float(), t) and torch.equal(t.to(C.H).float(), t)
        # every product sum the kernels form stays an exact fp32 integer
        assert (c.q.abs().sum(-1).max() * 8 * row.Lq) < 2 ** 24
        score, arg = C.oracle(c, fill=row.mode != "store")
        live = c.qm.bool()[c.pair_q]
        if row.mode == "pairs" and row.Ld >= 8 and row.n_d > C.REALTIE_DOC:
            assert (arg[C.FILL_DOC, 0] == -1).item(), f"{row}: the fill does not win"
            assert (arg[C.TIE1000_DOC, 0] == C.TIE1000_REAL).item() and not c.dm[C.TIE1000_DOC, C.TIE1000_MASKED]
            assert (arg[C.REALTIE_DOC, 1] == C.REALTIE_ROWS[0]).item(), f"{row}: no tie between real rows"
        if row.mode == "store":
            assert (c.lens > row.Ld).any() and torch.isnan(c.store[-1]).all()
        else:
            assert (~c.dm.bool()).any() and (~live).any()
            if row.mode == "pairs" and row.Ld > 1:
                assert (arg[live] == -1).any(), f"{row}: no live token where the fill wins"


@pytest.fixture(scope="module")
def instantiations():
    """The max-sim instantiations compiled into the library, from the demangled SASS function names."""
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
        if out.returncode != 0:
            pytest.skip("cuobjdump failed: " + out.stderr[-200:])
        names = re.findall(r"Function : (\S+)", out.stdout)
        dem = subprocess.run([DEMANGLE], input="\n".join(names), capture_output=True, text=True, timeout=60)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump / c++filt unavailable: {e}")
    if dem.returncode != 0:
        pytest.skip("c++filt failed: " + dem.stderr[-200:])
    found = set()
    for line in dem.stdout.splitlines():
        m = INSTANTIATION.search(line)
        if m:
            found.add(C.inst(m.group(1), *[a.strip() for a in m.group(2).split(",")]))
    return found


def test_every_compiled_instantiation_is_claimed_by_a_row(instantiations):
    for kernel in C.KERNELS:
        assert any(n.startswith(kernel + "<") for n in instantiations), f"no {kernel} in the library"
    claimed = set().union(*(row.claims for row in C.MATRIX))
    missing = sorted(instantiations - claimed)
    assert not missing, f"compiled but claimed by no row of maxsim_cases.MATRIX: {missing}"
    assert len(instantiations) == 55


def test_every_maxsim_and_flat_ip_kernel_belongs_to_a_matrix():
    """Every kernel named maxsim_*_kernel or flat_ip_tc*_kernel in the library's SASS is named by the KERNELS of an
    instantiation matrix (maxsim_cases, flat_ip_cases, and the in-batch backward's own list): a new kernel family fails
    here until it has rows."""
    import flat_ip_cases
    import test_maxsim_inbatch_bwd_cpu
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
        if out.returncode != 0:
            pytest.skip("cuobjdump failed: " + out.stderr[-200:])
        names = re.findall(r"Function : (\S+)", out.stdout)
        dem = subprocess.run([DEMANGLE], input="\n".join(names), capture_output=True, text=True, timeout=60)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump / c++filt unavailable: {e}")
    found = set(re.findall(r"\b(maxsim_\w*_kernel|flat_ip_tc\w*_kernel)<", dem.stdout))
    owned = set(C.KERNELS) | set(flat_ip_cases.KERNELS) | set(test_maxsim_inbatch_bwd_cpu.KERNELS)
    assert found, "no max-sim or flat-IP kernel in the library"
    assert not found - owned, f"kernels no instantiation matrix names: {sorted(found - owned)}"


def test_empty_batch_is_accepted_at_the_abi():
    """n_q = n_d = n_pairs = 0 with the null pointers torch hands out for empty tensors: both entry points return OK
    without touching the device; a non-empty batch still needs its tensors."""
    lib = _lib.load()
    n = None
    Lq, Ld, dim = 30, 200, 768
    rc = lib.mmb200_maxsim_fwd(n, n, n, n, n, n, n, n, n, 0, 0, 0, 1, Lq, Ld, dim, _lib.F16, _lib.MASK_NONE,
                               _lib.IMPL_AUTO, n)
    assert rc == _lib.OK, _lib.last_error()
    rc = lib.mmb200_maxsim_bwd(n, n, n, n, n, n, 0, 0, 0, 1, Lq, Ld, dim, _lib.F16, n)
    assert rc == _lib.OK, _lib.last_error()
    rc = lib.mmb200_maxsim_fwd(n, n, n, n, n, n, n, n, n, 1, 1, 1, 1, Lq, Ld, dim, _lib.F16, _lib.MASK_NONE,
                               _lib.IMPL_AUTO, n)
    assert rc == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
    rc = lib.mmb200_maxsim_bwd(n, n, n, n, n, n, 1, 1, 1, 1, Lq, Ld, dim, _lib.F16, n)
    assert rc == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
    buf = (ctypes.c_float * 4)()
    rc = lib.mmb200_maxsim_fwd(n, n, n, n, n, n, n, ctypes.addressof(buf), n, 0, 0, 1, 1, Lq, Ld, dim, _lib.F16,
                               _lib.MASK_NONE, _lib.IMPL_AUTO, n)
    assert rc == _lib.ERR_INVALID, "pairs without queries or documents"
