"""The store-mode entry points of the kernel-pooling forward (kernel_pool_ts_store_kernel, kernel_pool_fwd_simt_store)
are in the library for every kernel count they serve, the tensor-core one TMA-fed wgmma, and none spills to local
memory (no GPU needed)."""
import re
import shutil
import subprocess

import pytest

from matchmaker_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


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
    return {k: "\n".join(v) for k, v in funcs.items()}


@pytest.mark.parametrize("needle,kbs", [("kernel_pool_ts_store_kernel", {11, 12, 21, 24, 32}),
                                        ("kernel_pool_fwd_simt_store", {12, 24, 32})])
def test_store_mode_instantiations_do_not_spill(sass, needle, kbs):
    ks = {k: v for k, v in sass.items() if needle in k}
    assert {int(m) for k in ks for m in re.findall(needle + r"ILi(\d+)E", k)} == kbs
    for name, text in ks.items():
        local = [l for l in text.splitlines() if re.search(r"\b(LDL|STL)\b", l)]
        assert not local, f"{name}: local-memory traffic (spills) in the SASS: {local[:3]}"
        if "ts_store" in needle:
            assert "UTMALDG" in text and "HGMMA" in text, f"{name}: not a TMA-fed wgmma kernel"
