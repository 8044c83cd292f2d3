"""Static checks on the compiled library (no GPU needed): the hot kernels really are wgmma / TMA kernels for sm_90a,
the operands that are meant to come from registers do, and the MMA / TMA issue loops stay free of the ELECT / R2UR
waterfall loops the compiler emits around such instructions inside `if (lane == 0)` regions."""
import re
import shutil
import subprocess

import pytest

from matchmaker_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

# every tensor-core kernel except the kernel-pooling backward, which loads its tiles with plain coalesced loads
TMA_FED = {"maxsim_qm_kernel", "kernel_pool_ts_kernel", "flat_ip_tc_kernel", "maxsim_tc_kernel", "tkl_ts_kernel"}
# wgmma with the A operand in registers: HGMMA.<shape> Rd, Ra, gdesc[URb], ...
HGMMA_RS = re.compile(r"HGMMA\.\S+\s+R\d+,\s*R\d+,\s*gdesc")


@pytest.fixture(scope="module")
def sass():
    try:
        out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump unavailable: {e}")
    if out.returncode != 0:
        pytest.skip("cuobjdump failed: " + out.stderr[-200:])
    funcs, name = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    assert "sm_90a" in out.stdout, "no sm_90a code in the library"
    return {k: "\n".join(v) for k, v in funcs.items()}


def _kernels(sass, needle):
    ks = {k: v for k, v in sass.items() if needle in k}
    assert ks, f"no kernel matching {needle!r} in the library"
    return ks


def _hgmma_lines(text):
    # the compiler adds a no-op HGMMA on RZ operands around warpgroup fences; only the real ones count
    return [l for l in text.splitlines() if "HGMMA" in l and "gdesc[URZ]" not in l]


@pytest.mark.parametrize("needle", ["maxsim_qm_kernel", "kernel_pool_ts_kernel", "flat_ip_tc_kernel",
                                    "maxsim_tc_kernel", "kernel_pool_bwd_tc_kernel", "tkl_ts_kernel"])
def test_tensor_core_kernels_use_tcgen05_and_tma(sass, needle):
    """The kernels behind impl="tcgen05" (a historical name, kept in the API) are wgmma kernels, TMA-fed where intended."""
    for name, text in _kernels(sass, needle).items():
        assert _hgmma_lines(text), f"{name}: no wgmma (HGMMA) in the SASS"
        if needle in TMA_FED:
            assert "UTMALDG" in text, f"{name}: no TMA tensor load (UTMALDG) in the SASS"
            assert "SYNCS.PHASECHK" in text, f"{name}: no mbarrier wait in the SASS"


def test_kernel_pool_ts_feeds_the_mma_from_registers(sass):
    """The document operand is split into tf32 hi / lo in registers and goes to the tensor core from there: no
    converted copy of the document tile is written to shared memory."""
    for name, text in _kernels(sass, "kernel_pool_ts_kernel").items():
        lines = _hgmma_lines(text)
        assert lines and all(HGMMA_RS.search(l) for l in lines), f"{name}: a wgmma takes its A operand from shared memory"
        assert "USETMAXREG" in text, f"{name}: setmaxnreg is missing"


@pytest.mark.parametrize("needle", ["kernel_pool_ts_kernel", "flat_ip_tc_kernel"])
def test_mma_issue_is_uniform(sass, needle):
    """The waterfall pattern is `<instruction> ... ; @P0 BRA.U.ANY <back>`: no wgmma (HGMMA) and no TMA load of these
    kernels may be followed by one."""
    for name, text in _kernels(sass, needle).items():
        lines = [l for l in text.splitlines() if re.search(r"/\*[0-9a-f]{4}\*/", l)]
        assert any("UTMALDG" in l for l in lines) and _hgmma_lines(text), f"{name}: no TMA load or no wgmma"
        for i, l in enumerate(lines):
            if "UTMALDG" in l or "HGMMA" in l:
                nxt = " ".join(lines[i + 1:i + 3])
                assert "BRA.U.ANY" not in nxt, f"{name}: MMA or TMA issue inside a waterfall loop (issue it under elect.sync)"


def test_flat_ip_uses_multicast_in_the_cluster_instantiations(sass):
    ks = _kernels(sass, "flat_ip_tc_kernel")
    multi = [k for k, v in ks.items() if "UTMALDG" in v and ".MULTICAST" in v.upper()]
    assert multi, "no flat-IP instantiation issues a multicast TMA load"


def test_kernel_pool_backward_is_a_tensor_core_kernel(sass):
    """Both contractions of the backward as wgmma with the embeddings as register A operands: the document-gradient GEMM
    (N = 64 document rows) and the query-gradient GEMM (N = 32 query rows)."""
    for name, text in _kernels(sass, "kernel_pool_bwd_tc_kernel").items():
        lines = _hgmma_lines(text)
        assert all(HGMMA_RS.search(l) for l in lines), f"{name}: a wgmma takes its A operand from shared memory"
        assert any("64x64x8" in l for l in lines) and any("64x32x8" in l for l in lines), f"{name}: expected the two GEMMs"
