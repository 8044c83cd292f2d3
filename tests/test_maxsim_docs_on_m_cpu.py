"""Compiled code of the headline max-sim kernel (no GPU needed): every instantiation of `maxsim_qm_kernel` puts the
document chunk on the MMA's M side and the query tile on N = 32 (`HGMMA.64x32x16`, none of the padded `64x64x16`), and
the descriptors of a chunk's MMAs are stepped in uniform registers: between two consecutive MMAs of a chunk there is no
descriptor rebuilding (`LOP3`) and at most one vector-to-uniform move (`R2UR`, at the second k-block of dim 128)."""
import re
import shutil
import subprocess

import pytest

from matchmaker_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def _hgmma_lines(lines):
    # the compiler adds a no-op HGMMA on RZ operands around warpgroup fences; only the real ones count
    return [l for l in lines if "HGMMA" in l and "gdesc[URZ]" not in l]


@pytest.fixture(scope="module")
def qm_sass():
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
            name = m.group(1) if "maxsim_qm_kernel" in m.group(1) else None
            if name:
                funcs[name] = []
        elif name is not None and re.search(r"/\*[0-9a-f]{4}\*/", line):
            funcs[name].append(line)
    return funcs


def test_documents_on_m(qm_sass):
    # f16 / bf16 x (inference, training) + f16 / bf16 store mode
    assert len(qm_sass) == 6, sorted(qm_sass)
    for name, lines in qm_sass.items():
        mma = _hgmma_lines(lines)
        assert mma and all("HGMMA.64x32x16" in l for l in mma), (name, mma[:4])
        assert not any("64x64x16" in l for l in lines), name


def test_chunk_mmas_step_uniform_descriptors(qm_sass):
    for name, lines in qm_sass.items():
        idx = [i for i, l in enumerate(lines) if "HGMMA.64x32x16" in l]
        # the first MMA of a chunk overwrites (!UPT): the rest follow it without a wait in between
        starts = [i for i in idx if "!UPT" in lines[i]]
        assert starts, name
        for a, b in zip(idx, idx[1:]):
            if "!UPT" in lines[b]:
                continue
            gap = lines[a + 1:b]
            assert not any("LOP3" in l for l in gap), (name, gap)
            assert sum("R2UR" in l for l in gap) <= 1, (name, gap)
            assert not any("DEPBAR" in l for l in gap), (name, gap)
