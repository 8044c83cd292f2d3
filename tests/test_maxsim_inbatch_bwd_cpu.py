"""The all-pairs (in-batch) max-sim backward without a GPU: the gradient written out from an explicit argmax is fp64
torch autograd of the reference expression (colbert.py:154-162) and of its own-masks form, the integer cases hold what
the GPU tests rely on, the C ABI validates before it needs a device, and both backward kernels are compiled for every
dtype without spills."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

import maxsim_cases as C
import maxsim_inbatch_cases as I
from matchmaker_b200 import _lib, build, interaction

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
KERNELS = ("maxsim_allpairs_bwd_d_kernel", "maxsim_allpairs_bwd_q_kernel")


def _close(a, b, what):
    torch.testing.assert_close(a.double(), b.double(), rtol=1e-12, atol=1e-9, msg=lambda m: f"{what}: {m}")


SHAPES = [(3, 3, 5, 7, 16), (4, 4, 30, 40, 64), (1, 1, 1, 1, 8), (2, 5, 9, 12, 12), (5, 2, 6, 20, 24)]


# the reference mask indexing needs n_q == n_d
@pytest.mark.parametrize("shape,own", [(s, own) for s in SHAPES for own in (False, True) if own or s[0] == s[1]],
                         ids=lambda v: "own-masks" if v is True else "reference-indexing" if v is False else str(v))
def test_written_out_gradient_is_torch_autograd_on_real_values(shape, own):
    n_q, n_d, Lq, Ld, dim = shape
    g = torch.Generator().manual_seed(sum(shape) + own)
    q, d = torch.randn(n_q, Lq, dim, generator=g), torch.randn(n_d, Ld, dim, generator=g)
    qm = (torch.rand(n_q, Lq, generator=g) > 0.2).long()
    dm = (torch.rand(n_d, Ld, generator=g) > 0.3).long()
    qm[0, 0] = dm[0, 0] = 1
    if n_d > 2:
        dm[2] = 0                 # a fully masked document (own masks) / mask row (reference indexing)
        d[1] *= -300.0            # real scores far below -1000: the fill wins wherever document 1's mask has a hole
    p = torch.arange(n_q * n_d)
    pq, pd = p // n_d, p % n_d
    c = C.Case(q, d, qm, dm, pq, pd, pd if own else pq, torch.randn(n_q * n_d, generator=g))
    score, arg = C.oracle(c)
    gq, gd = I.oracle_grads(c, arg, n_d)
    ref, rq, rd = I.reference_autograd(q, qm, d, dm, c.gout, own)
    if not own:   # the reference expression keeps fp64; the own-masks loop writes into an fp32 tensor
        _close(score.view(n_q, n_d), ref, "score")
    else:
        torch.testing.assert_close(score.view(n_q, n_d).float().double(), ref)
    _close(gq, rq, "grad_q")
    _close(gd, rd, "grad_d")


@pytest.mark.parametrize("s", [s for s in I.MATRIX if s.n_q * s.n_d * s.Lq * s.Ld * s.dim <= 2e8], ids=str)
def test_written_out_gradient_is_torch_autograd_on_the_integer_cases_but_for_the_fill_tie(s):
    """Exactly equal, but for one documented difference: where a real row scores exactly -1000 after a masked row,
    torch's first-index max picks the masked row (whose gradient the fill assignment drops), while the kernels and the
    oracle let the real row win."""
    c = I.make_case(s)
    score, arg = C.oracle(c)
    gq, gd = I.oracle_grads(c, arg, s.n_d)
    ref, rq, rd = I.reference_autograd(c.q, c.qm, c.d, c.dm, c.gout, s.own)
    assert torch.equal(score.view(s.n_q, s.n_d), ref)
    if s.special:
        p = I.TIE_DOC    # pair (0, TIE_DOC)
        assert int(arg[p, 0]) == C.TIE1000_REAL
        g = float(c.gout[p])
        rq[0, 0] += g * c.d[I.TIE_DOC, C.TIE1000_REAL].double()
        rd[I.TIE_DOC, C.TIE1000_REAL] += g * c.q[0, 0].double()
    assert torch.equal(gq, rq)
    assert torch.equal(gd, rd)


def test_cases_hold_their_preconditions():
    seen = set()
    for s in I.MATRIX:
        c = I.make_case(s)
        for t in (c.q, c.d, c.gout):
            assert torch.equal(t, t.round()) and t.abs().max() <= 8
            assert torch.equal(t.to(C.BF).float(), t) and torch.equal(t.to(C.H).float(), t)
        assert (c.q.abs().sum(-1).max() * 8 * s.Lq) < 2 ** 24
        score, arg = C.oracle(c)
        live = c.qm.bool()[c.pair_q]
        assert (arg[live] >= 0).any(), f"{s}: no gradient at all"
        if s.special:
            assert int(arg[I.FILL_DOC, 0]) == -1, f"{s}: the fill does not win"
            assert int(arg[I.TIE_DOC, 0]) == C.TIE1000_REAL
            seen.add("fill")
        if s.realtie:
            a = 1 if s.n_q > 1 else 0
            assert int(arg[a * s.n_d + I.REALTIE_DOC, 1]) == C.REALTIE_ROWS[0], f"{s}: no tie between real rows"
            seen.add("real tie")
        if s.n_q >= 3:
            assert not c.qm[s.n_q - 1].any()
            seen.add("masked query")
        if s.n_d > I.MASKED_DOC:
            assert not c.dm[I.MASKED_DOC].any()
            seen.add("masked document")
        seen |= {C.SHORT[s.dtype] + f" dim {s.dim}", f"Ld {s.Ld}", "own" if s.own else "ref"}
        seen |= {"n_q 1"} if s.n_q == 1 else set()
        seen |= {"n_d 1"} if s.n_d == 1 else set()
        seen |= {"n_q != n_d"} if s.n_q != s.n_d else set()
        seen |= {"dim 768 Lq 74"} if (s.dim, s.Lq) == (768, 74) else set()
        seen |= {"dim 768 Lq 30"} if (s.dim, s.Lq) == (768, 30) else set()
        seen |= {"grad_d over several (a, i) chunks"} if s.n_q * s.Lq > I.BWD_CHUNK else set()
        seen |= {"grad_q over several document chunks"} if s.n_d > I.BWD_CHUNK else set()
    need = ({"fill", "real tie", "masked query", "masked document", "own", "ref", "n_q 1", "n_d 1", "n_q != n_d",
             "dim 768 Lq 74", "dim 768 Lq 30", "grad_d over several (a, i) chunks", "grad_q over several document chunks"} | {f"Ld {n}" for n in (1, 127, 129, 200)}
            | {f"{t} dim {n}" for t in ("f16", "bf16", "f32") for n in (64, 100, 768)}
            | {f"{t} dim 128" for t in ("f16", "bf16")})
    assert need <= seen, sorted(need - seen)


def test_abi_validates_before_it_needs_a_device():
    lib = _lib.load()
    n = None
    Lq, Ld, dim = 30, 200, 768
    rc = lib.mmb200_maxsim_allpairs_bwd(n, n, n, n, n, n, 0, 0, Lq, Ld, dim, _lib.F16, n)
    assert rc == _lib.OK, _lib.last_error()
    for n_q, n_d in ((1, 1), (32, 32), (0, 3), (3, 0)):
        rc = lib.mmb200_maxsim_allpairs_bwd(n, n, n, n, n, n, n_q, n_d, Lq, Ld, dim, _lib.F16, n)
        assert rc == _lib.ERR_INVALID and "null pointer" in _lib.last_error(), (n_q, n_d)
    # n_q * n_d = 2^31 - 1 passes the count check (and stops at the null pointers); 2^31 and beyond are refused
    rc = lib.mmb200_maxsim_allpairs_bwd(n, n, n, n, n, n, 2 ** 31 - 1, 1, Lq, Ld, dim, _lib.F16, n)
    assert rc == _lib.ERR_INVALID and "null pointer" in _lib.last_error()
    buf = (ctypes.c_float * 4)()
    p = ctypes.addressof(buf)
    for n_q, n_d in ((2 ** 16, 2 ** 15), (2 ** 31, 1), (3, 2 ** 40)):
        rc = lib.mmb200_maxsim_allpairs_bwd(p, p, p, p, p, p, n_q, n_d, Lq, Ld, dim, _lib.F16, n)
        assert rc == _lib.ERR_INVALID and "2^31" in _lib.last_error(), (n_q, n_d)
    for bad in ((-1, 2, Lq, Ld, dim), (2, -1, Lq, Ld, dim), (2, 2, 0, Ld, dim), (2, 2, Lq, 0, dim), (2, 2, Lq, Ld, 0)):
        rc = lib.mmb200_maxsim_allpairs_bwd(p, p, p, p, p, p, *bad, _lib.F16, n)
        assert rc == _lib.ERR_INVALID and "bad shape" in _lib.last_error(), bad
    rc = lib.mmb200_maxsim_allpairs_bwd(p, p, p, p, p, p, 2, 2, Lq, Ld, dim, 99, n)
    assert rc == _lib.ERR_INVALID and "dtype" in _lib.last_error()


@pytest.mark.parametrize("mode", ["no_grad", "inference_mode", "detached", "grad"])
def test_autograd_takes_the_argmax_path_only_when_a_gradient_is_wanted(monkeypatch, mode):
    """Under torch.no_grad() / inference_mode, or with inputs that require no grad, autograd.maxsim_allpairs is exactly
    interaction.maxsim_allpairs (no argmax, nothing saved), also for vectors that require grad; only with grad mode on
    and an input requiring grad does it run the argmax forward.  The kernels are replaced by a recorder, so this runs
    without a GPU."""
    from matchmaker_b200 import autograd
    calls = []

    def fake(q, q_mask, d, d_mask, impl="auto", reference_mask_indexing=False, return_argmax=False):
        calls.append({"return_argmax": return_argmax, "reference_mask_indexing": reference_mask_indexing})
        out = torch.zeros(q.shape[0], d.shape[0])
        return (out, torch.zeros(q.shape[0] * d.shape[0], q.shape[1], dtype=torch.int32)) if return_argmax else out

    monkeypatch.setattr(interaction, "maxsim_allpairs", fake)
    q = torch.zeros(3, 4, 8, requires_grad=mode != "detached")
    d = torch.zeros(3, 5, 8, requires_grad=mode != "detached")
    qm, dm = torch.ones(3, 4), torch.ones(3, 5)
    if mode == "no_grad":
        with torch.no_grad():
            out = autograd.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True)
    elif mode == "inference_mode":
        with torch.inference_mode():
            out = autograd.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True)
    else:
        out = autograd.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True)
    assert calls == [{"return_argmax": mode == "grad", "reference_mask_indexing": True}]
    assert (out.grad_fn is not None) == (mode == "grad")


def test_python_entry_point_refuses_cpu_tensors():
    q, d = torch.zeros(2, 3, 8), torch.zeros(4, 5, 8)
    with pytest.raises(_lib.MatchmakerB200Error, match="CUDA"):
        interaction.maxsim_allpairs_bwd(q, d, torch.zeros(2, 4), torch.zeros(8, 3, dtype=torch.int32))


@pytest.fixture(scope="module")
def sass_names():
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
        if out.returncode != 0:
            pytest.skip("cuobjdump failed: " + out.stderr[-200:])
        names = re.findall(r"Function : (\S+)", out.stdout)
        dem = subprocess.run([DEMANGLE], input="\n".join(names), capture_output=True, text=True, timeout=60)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump / c++filt unavailable: {e}")
    return dem.stdout


def test_every_instantiation_is_compiled(sass_names):
    found = set(re.findall(r"\b(maxsim_allpairs_bwd_[dq]_kernel)<([^>]*)>", sass_names))
    assert found == {(k, t) for k in KERNELS for t in ("__half", "__nv_bfloat16", "float")}, sorted(found)


def test_ptxas_reports_no_spills():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "maxsim_host.cu")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True,
                       text=True, check=True)
    reports = re.findall(r"Compiling entry function '(\S+)'.*?\n(.*?spill.*?)\n", r.stderr, re.S)
    ours = [(n, line) for n, line in reports if "maxsim_allpairs_bwd" in n]
    assert len(ours) == 6, [n for n, _ in reports]
    for name, line in ours:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
