"""The shared cases of the kernel-pooling envelope tests (tests/kernel_pool_cases.py), checked without a GPU: the fp64
reference is the oracle functions it stands for, every row claims what the dispatch rules give it, the rows between them
claim every instantiation compiled into the library, and the cases hold the preconditions the GPU tests rely on.  Also the
empty batch at the C ABI."""
import ctypes
import re
import shutil
import subprocess

import pytest
import torch

import kernel_pool_cases as C
from matchmaker_b200 import _lib
from oracle import interaction_oracle as O

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
INSTANTIATION = re.compile(r"\b(" + "|".join(C.KERNELS) + r")<(\d+),\s*(\w+)>")


def _leaves(c: C.Case):
    return {k: (None if v is None else v.double().clone().requires_grad_(True))
            for k, v in (("q", c.q), ("d", c.d), ("alpha", c.alpha), ("weight", c.weight), ("gate", c.gate))}


def _close(a, b, what):
    torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-14, msg=lambda m: f"{what}: {m}")


def _check(ref, score, per_kernel, S, leaves, valid, grads=("q", "d", "alpha", "weight", "gate")):
    _close(ref["score"], score.detach(), "score")
    if per_kernel is not None:
        _close(ref["per_kernel"], per_kernel.detach(), "per_kernel")
    if S is not None:
        _close(ref["S"][valid], S.detach()[valid], "S (valid query rows)")
    for name in grads:
        if leaves[name] is not None:
            _close(ref["grad_" + name], leaves[name].grad, "grad_" + name)


SMALL = [(3, 5, 9, 8, 11), (2, 1, 1, 4, 1), (4, 7, 30, 12, 24)]


@pytest.mark.parametrize("shape", SMALL)
def test_reference_is_the_tk_oracle(shape):
    c = C.make_case(*shape, seed=sum(shape))
    ref = C.reference(c)
    x = _leaves(c)
    score, sec = O.kernel_pool_tk(x["q"], x["d"], c.qm.double(), c.dm.double(), c.mu.double(), c.sigma.double(),
                                  x["alpha"], x["weight"])
    score.backward(c.gout.double())
    _check(ref, score, sec["per_kernel"], sec["per_kernel_query"], x, c.qm.bool())


@pytest.mark.parametrize("shape", SMALL)
def test_reference_is_the_tk_sparse_oracle(shape):
    c = C.make_case(*shape, seed=sum(shape) + 1, gate=True)
    ref = C.reference(c)
    x = _leaves(c)
    score, sec = O.kernel_pool_tk_sparse(x["q"], x["d"], c.qm.double(), c.dm.double(), x["gate"], c.mu.double(),
                                         c.sigma.double(), x["alpha"], x["weight"])
    score.backward(c.gout.double())
    assert ref["grad_gate"].abs().max() > 0
    _check(ref, score, sec["per_kernel"], sec["per_kernel_query"], x, c.qm.bool())


@pytest.mark.parametrize("shape", SMALL)
def test_reference_is_the_knrm_oracle(shape):
    c = C.make_case(*shape, seed=sum(shape) + 2, knrm=True)
    assert c.alpha is None and c.log_scale == 0.01
    ref = C.reference(c)
    x = _leaves(c)
    score, sec = O.kernel_pool_knrm(x["q"], x["d"], c.qm.double(), c.dm.double(), c.mu.double(), c.sigma.double(),
                                    x["weight"])
    score.backward(c.gout.double())
    _check(ref, score, sec["per_kernel"], sec["per_kernel_query"], x, c.qm.bool())


@pytest.mark.parametrize("K", C.CLAMP_KS)
def test_reference_is_the_idcm_esm_oracle(K):
    """The ESM scorer takes embeddings its caller has normalised (sigir21_idcm.py:164-178); the kernels, like the cosine
    module, normalise themselves.  The oracle is fed the same fp64 normalisation, so its gradients reach q and d."""
    c = C.clamp_case(K)
    ref = C.reference(c, clamp_min=C.IDCM_FLOOR, bias=0.37)
    x = _leaves(c)
    tiny = O.tiny_value_of_dtype(torch.float64)
    qn = x["q"] / (x["q"].norm(p=2, dim=-1, keepdim=True) + tiny)
    dn = x["d"] / (x["d"].norm(p=2, dim=-1, keepdim=True) + tiny)
    score = O.idcm_esm_patch_scores(qn, dn, c.qm.double(), c.dm.double(), c.mu.double(), c.sigma.double(),
                                    x["alpha"], x["weight"], torch.tensor([0.37], dtype=torch.float64))
    score.backward(c.gout.double())
    assert ref["grad_q"].abs().max() > 0
    _check(ref, score, None, None, x, None)


def test_rows_claim_what_the_dispatch_rules_give_them():
    for row in C.MATRIX:
        assert set(row.claims) == C.dispatched(row.Lq, row.Ld, row.D, row.K), str(row)
        assert C.activation_elements(row) <= 1e7, f"{row}: the fp64 reference would be too large"
    every = ({C.inst(k, kb, s) for k in (C.TS_FWD, C.TC_BWD) for kb in (11, 12, 21, 24, 32) for s in (False, True)}
             | {C.inst(k, kb, v) for k in (C.SIMT_FWD, C.SIMT_BWD) for kb in (12, 24, 32) for v in (1, 2)})
    assert len(every) == 32
    assert set().union(*(row.claims for row in C.MATRIX)) == every
    assert any(row.B > 132 for row in C.MATRIX), "no row walks several pairs per CTA"


def test_cases_hold_their_preconditions():
    """Distinct kernel sets; exact matches; no live alpha S within 1 % of the floor; the clamp cases put at least 10 % of
    their entries below IDCM's floor."""
    for row in C.MATRIX:
        for gate in (False, True):
            c = C.row_case(row, gate)
            K = row.K
            assert c.mu.unique().numel() == K and c.sigma.unique().numel() == K and c.weight.unique().numel() == K
            assert float(c.sigma.min()) >= 0.05 - 1e-6 and float(c.sigma.max()) <= 0.3 + 1e-6
            if K > 2:
                assert not torch.equal(c.sigma, c.sigma.sort(descending=True).values), f"{row}: sigma in order"
            ref = C.reference(c, grads=False)
            assert C.floor_margin(ref["aS"], c.qm, C.DEFAULT_FLOOR) > 1e-2, f"{row} gate={gate}"
            # every pair has a live cosine of 1 (the exact match)
            cos = O.cosine_matrix(c.q.double(), c.d.double()) * c.qm.double().unsqueeze(-1) * c.dm.double().unsqueeze(1)
            if row.Lq * row.Ld > 1:
                assert (cos.flatten(1).max(1).values > 1 - 1e-12).all(), str(row)
            if gate:
                assert (c.gate == 0).any() and (c.gate > 0).any() and (c.gate >= 0).all()
    for K in C.CLAMP_KS:
        c = C.clamp_case(K)
        ref = C.reference(c, clamp_min=C.IDCM_FLOOR, grads=False)
        assert C.below_floor_fraction(ref["aS"], c.qm, C.IDCM_FLOOR) >= 0.1, K
        assert C.floor_margin(ref["aS"], c.qm, C.IDCM_FLOOR) > 1e-2, K


@pytest.fixture(scope="module")
def instantiations():
    """The kernel-pooling instantiations compiled into the library, from the demangled SASS function names."""
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
            found.add(C.inst(m.group(1), m.group(2), m.group(3)))
    return found


def test_every_compiled_instantiation_is_claimed_by_a_row(instantiations):
    for kernel in C.KERNELS:
        assert any(n.startswith(kernel + "<") for n in instantiations), f"no {kernel} in the library"
    claimed = set().union(*(row.claims for row in C.MATRIX))
    missing = sorted(instantiations - claimed)
    assert not missing, f"compiled but claimed by no row of kernel_pool_cases.MATRIX: {missing}"
    assert len(instantiations) == 32


def test_empty_batch_is_accepted_at_the_abi():
    """B = 0 with the null pointers torch hands out for empty tensors: every entry point returns OK without touching the
    device (mu / sigma / weight are host arrays here; nothing reads them)."""
    lib = _lib.load()
    K, Lq, Ld, D = 11, 5, 20, 32
    par = (ctypes.c_float * K)()
    p = ctypes.addressof(par)
    n = None
    rc = lib.mmb200_kernel_pool_fwd_ex(n, n, n, n, n, p, p, n, p, n, n, n, n, 0, Lq, Ld, D, K, 1.0, 1e-10, 0.0,
                                       _lib.MASK_NONE, _lib.IMPL_AUTO, n)
    assert rc == _lib.OK, _lib.last_error()
    rc = lib.mmb200_kernel_pool_fwd_train(n, n, n, n, n, p, p, n, p, n, n, n, n, 0, Lq, Ld, D, K, 1.0, 1e-10, 0.0,
                                          _lib.MASK_NONE, n)
    assert rc == _lib.OK, _lib.last_error()
    rc = lib.mmb200_kernel_pool_bwd_ex(n, n, n, n, n, p, p, n, p, n, n, n, n, n, n, n, n, 0, Lq, Ld, D, K, 1.0, 1e-10,
                                       _lib.MASK_NONE, n)
    assert rc == _lib.OK, _lib.last_error()
    rc = lib.mmb200_kernel_pool_bwd_saved(n, n, n, n, n, p, p, n, p, n, n, n, n, n, n, n, n, n, 0, Lq, Ld, D, K, 1.0,
                                          1e-10, _lib.MASK_NONE, n)
    assert rc == _lib.OK, _lib.last_error()
    # a non-empty batch still needs its tensors
    rc = lib.mmb200_kernel_pool_fwd_ex(n, n, n, n, n, p, p, n, p, n, n, n, n, 1, Lq, Ld, D, K, 1.0, 1e-10, 0.0,
                                       _lib.MASK_NONE, _lib.IMPL_AUTO, n)
    assert rc == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
