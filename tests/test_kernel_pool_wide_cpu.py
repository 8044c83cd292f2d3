"""The BERT-width kernel-pooling training pair without a GPU: its envelope at the C ABI, the exported symbols, what the
compiler made of the wide backward's kernels, and that the GPU test's matrix (tests/kernel_pool_wide_cases.py) claims
every compiled instantiation of them."""
import ctypes
import re
import shutil
import subprocess

import pytest

import kernel_pool_cases as C
import kernel_pool_wide_cases as W
from matchmaker_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
DEMANGLE = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
G_INSTANTIATION = re.compile(r"\b(" + W.G_PASS + r")<(\d+),\s*(\w+)>")


def test_envelope():
    ok = _lib.load().mmb200_kernel_pool_train_tc_supported
    assert ok(30, 200, 768, 11) == 1 and ok(32, 2000, 1024, 32) == 1 and ok(1, 1, 576, 1) == 1
    assert ok(30, 200, 516, 11) == 0      # not whole 64-feature blocks (and past the FFMA backward's 512)
    assert ok(30, 200, 1088, 11) == 0     # past BERT-large
    assert ok(30, 200, 324, 11) == 0      # between the two tensor-core backward envelopes
    assert ok(30, 200, 512, 11) == 0      # 320 < D <= 512 stays on the FFMA backward
    assert ok(33, 200, 768, 11) == 0
    assert ok(30, 200, 768, 33) == 0
    for Lq, Ld, D, K in [(30, 200, 768, 11), (32, 2000, 1024, 32), (30, 200, 516, 11), (30, 200, 1088, 11),
                         (30, 200, 324, 11), (33, 200, 768, 11), (30, 200, 320, 21), (1, 1, 4, 1)]:
        assert bool(ok(Lq, Ld, D, K)) == (C.train_ok(Lq, Ld, D, K) or W.wide_ok(Lq, Ld, D, K)), (Lq, Ld, D, K)


def test_workspace_size():
    """2 B K floats (the per-pair weight and alpha terms) everywhere but the wide envelope, which adds 16-byte-aligned
    room for G1, G2^T and the normalisation terms: B (65 Ldp + 32) floats with Ldp = Ld rounded up to 64."""
    ws = _lib.load().mmb200_kernel_pool_bwd_saved_workspace_floats
    assert ws(7, 30, 200, 300, 21) == 2 * 7 * 21
    assert ws(7, 30, 200, 516, 21) == 2 * 7 * 21
    assert ws(7, 30, 200, 768, 21) == 296 + 7 * (65 * 256 + 32)      # 2 * 7 * 21 = 294, rounded up to 296
    assert ws(3, 32, 2000, 1024, 32) == 2 * 3 * 32 + 3 * (65 * 2048 + 32)
    assert ws(0, 30, 200, 768, 11) == 0


def test_symbols_are_exported():
    lib = _lib.load()
    for name in ("mmb200_kernel_pool_bwd_saved_workspace_floats", "mmb200_kernel_pool_train_tc_supported",
                 "mmb200_kernel_pool_fwd_train", "mmb200_kernel_pool_bwd_saved"):
        assert hasattr(lib, name), name


def test_empty_batch_is_accepted_at_the_abi():
    """B = 0 at D = 768 with the null pointers torch hands out for empty tensors."""
    lib = _lib.load()
    K, Lq, Ld, D = 11, 5, 20, 768
    par = (ctypes.c_float * K)()
    p = ctypes.addressof(par)
    n = None
    rc = lib.mmb200_kernel_pool_fwd_train(n, n, n, n, n, p, p, n, p, n, n, n, n, 0, Lq, Ld, D, K, 1.0, 1e-10, 0.0,
                                          _lib.MASK_NONE, n)
    assert rc == _lib.OK, _lib.last_error()


@pytest.fixture(scope="module")
def sass():
    """{demangled function name: SASS text} of the wide backward's kernels."""
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
        if out.returncode != 0:
            pytest.skip("cuobjdump failed: " + out.stderr[-200:])
        parts = re.split(r"\n\s*Function : (\S+)\n", out.stdout)
        names, bodies = parts[1::2], parts[2::2]
        dem = subprocess.run([DEMANGLE], input="\n".join(names), capture_output=True, text=True, timeout=60)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump / c++filt unavailable: {e}")
    if dem.returncode != 0:
        pytest.skip("c++filt failed: " + dem.stderr[-200:])
    return {d: b for d, b in zip(dem.stdout.splitlines(), bodies) if any(k in d for k in W.KERNELS)}


def _instantiations(sass):
    found = set()
    for name in sass:
        m = G_INSTANTIATION.search(name)
        if m:
            found.add(C.inst(m.group(1), m.group(2), m.group(3)))
        elif W.GRAD + "(" in name:
            found.add(W.GRAD)
    return found


def test_sass_gemms_on_the_tensor_cores_and_no_spills(sass):
    grad = [b for n, b in sass.items() if W.GRAD + "(" in n]
    assert len(grad) == 1
    assert "HGMMA.64x64x8.F32.TF32" in grad[0] and "HGMMA.64x32x8.F32.TF32" in grad[0]
    for name, body in sass.items():
        assert not re.search(r"\b(LDL|STL)\b", body), f"{name}: local-memory spill"


def test_every_compiled_instantiation_is_claimed_by_a_row(sass):
    found = _instantiations(sass)
    claimed = set().union(*(row.claims for row in W.MATRIX))
    every = {W.g_inst(K, g) for K in (11, 12, 21, 24, 32) for g in (False, True)} | {W.GRAD}
    assert len(every) == 11
    assert found == every, f"compiled {sorted(found)} vs expected {sorted(every)}"
    assert claimed == every, f"claimed by the matrix: {sorted(claimed)}"
    assert len(found) == 11


def test_rows_are_in_the_envelope_and_cover_its_edges():
    for row in W.MATRIX:
        assert W.wide_ok(row.Lq, row.Ld, row.D, row.K) and not C.train_ok(row.Lq, row.Ld, row.D, row.K), str(row)
        assert C.activation_elements(row) <= 1e7, f"{row}: the fp64 reference would be too large"
    assert {r.D for r in W.MATRIX} == {576, 768, 1024}
    assert {1, 17, 30, 32} <= {r.Lq for r in W.MATRIX}
    assert {1, 40, 200, 1000, 2000} <= {r.Ld for r in W.MATRIX}
    assert {1, 11, 12, 13, 21, 24, 25, 32} <= {r.K for r in W.MATRIX}
    assert any(r.knrm for r in W.MATRIX) and any(r.empty_doc for r in W.MATRIX)


def test_cases_hold_their_preconditions():
    """No live alpha S within 1 % of the floor; padding rows hold data; the KNRM rows carry the sigma = 1e-4 kernel; the
    clamp cases put at least 10 % of their entries below IDCM's floor."""
    for row in W.MATRIX:
        for gate in (False, True):
            c = W.row_case(row, gate)
            ref = C.reference(c, grads=False)
            assert C.floor_margin(ref["aS"], c.qm, C.DEFAULT_FLOOR) > 1e-2, f"{row} gate={gate}"
            if row.knrm:
                assert c.alpha is None and c.log_scale == 0.01 and float(c.sigma.min()) == pytest.approx(1e-4)
            if row.empty_doc:
                assert (c.dm[-1] == 0).all() and (c.d[-1] != 0).any()
    for K in W.CLAMP_KS:
        c = W.clamp_case(K)
        ref = C.reference(c, clamp_min=C.IDCM_FLOOR, grads=False)
        assert C.below_floor_fraction(ref["aS"], c.qm, C.IDCM_FLOOR) >= 0.1, K
        assert C.floor_margin(ref["aS"], c.qm, C.IDCM_FLOOR) > 1e-2, K
