"""The wide TKL backward without a GPU: the exported symbols, the workspace size, the routing query at the edges of both
envelopes, and the new kernels in the library's SASS."""
import os
import re
import shutil
import subprocess

import pytest

from matchmaker_b200 import _lib, interaction

NEW = ("mmb200_tkl_bwd_wide", "mmb200_tkl_bwd_wide_workspace_floats", "mmb200_tkl_bwd_route")
WIDE_KERNELS = ("tkl_bwd_wide_dot_kernel", "tkl_bwd_wide_g_kernel", "tkl_bwd_wide_grad_kernel")
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "matchmaker_b200.h")


def test_new_symbols_are_exported():
    lib = _lib.load()
    text = open(HEADER).read()
    for name in NEW:
        assert name in _lib.SIGNATURES and getattr(lib, name) is not None, name
        assert re.search(rf"MMB200_API\s+\w+\s+{name}\(", text), f"{name} is not declared in the header"
    assert callable(interaction.tkl_bwd_wide) and callable(interaction.tkl_bwd_route)


def _workspace_floats(B, D, K, saturation):
    """Per-document parameter partials (rounded up to 4 floats), then one record per (document, 64-feature block) and
    one per document: [40 x 128] products, 40 + 128 + 40 coefficients."""
    stride = K + 15 + (13 + D if saturation == 0 else K)
    rec = 40 * 128 + 40 + 128 + 40
    return ((B * stride + 3) // 4) * 4 + B * ((D + 63) // 64 + 1) * rec


@pytest.mark.parametrize("B,D,K,sat", [(1, 4, 1, 1), (16, 768, 11, 0), (16, 768, 11, 1), (300, 1024, 16, 0),
                                       (7, 516, 13, 1), (3, 360, 12, 0), (0, 768, 11, 0)])
def test_workspace_size(B, D, K, sat):
    assert _lib.load().mmb200_tkl_bwd_wide_workspace_floats(B, D, K, sat) == _workspace_floats(B, D, K, sat)


def test_routing_at_the_edges():
    route = interaction.tkl_bwd_route
    for K in (12, 16):   # the one-CTA plan stops at D = 356 for both kernel blocks
        assert route(30, 356, K) == "tkl_bwd" and route(30, 360, K) == "tkl_bwd_wide"
    assert route(40, 4, 1) == "tkl_bwd" and route(1, 768, 11) == "tkl_bwd_wide"
    assert route(30, 1024, 16) == "tkl_bwd_wide" and route(30, 1028, 16) is None
    assert route(40, 768, 11) == "tkl_bwd_wide" and route(41, 768, 11) is None and route(41, 300, 11) is None
    assert route(0, 300, 11) is None and route(30, 300, 17) is None and route(30, 300, 0) is None
    assert route(30, 770, 11) is None and route(30, 302, 11) is None and route(30, 0, 11) is None


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


def _sass_needles():
    """The kernel-name needles of tests/test_sass.py's parametrized checks."""
    text = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_sass.py")).read()
    needles = set()
    for lst in re.findall(r"parametrize\(\s*\"needle\"\s*,\s*\[([^\]]*)\]", text):
        needles.update(re.findall(r"\"([^\"]+)\"", lst))
    return needles


def test_wide_kernels_in_the_library_without_local_memory(sass):
    found = {k: v for k, v in sass.items() if any(n in k for n in WIDE_KERNELS)}
    assert {n for n in WIDE_KERNELS if any(n in k for k in found)} == set(WIDE_KERNELS)
    assert len([k for k in found if "tkl_bwd_wide_g_kernel" in k]) == 2   # KB = 12 and 16
    for name, text in found.items():
        local = [l for l in text.splitlines() if re.search(r"\b(LDL|STL)(\.\S+)?\b", l)]
        assert not local, f"{name}: local-memory traffic in the SASS: {local[:3]}"
    needles = _sass_needles()
    assert needles, "no needles found in tests/test_sass.py"
    for name in found:
        assert not any(n in name for n in needles), f"{name} matches a needle of tests/test_sass.py"
