"""Compiler report of the headline max-sim kernel (no GPU needed): no instantiation of `maxsim_qm_kernel` spills, and
the live-row fetch left no pre-pass kernel behind."""
import os
import re
import shutil
import subprocess

import pytest

from matchmaker_b200 import build


def test_maxsim_qm_kernel_does_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "maxsim_qm.cu")
    r = subprocess.run([nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True,
                       text=True, check=True)
    reports = re.findall(r"Compiling entry function '(\S+)'.*?\n(.*?spill.*?)\n", r.stderr, re.S)
    names = [n for n, _ in reports]
    # f16 / bf16 x (inference, training) + f16 / bf16 store mode
    assert len(names) == 6 and all("maxsim_qm_kernel" in n for n in names), names
    for name, line in reports:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in line, (name, line)
    # the consumers' and the helpers' setmaxnreg budgets add up to the launch's registers
    text = open(src).read()
    helper, consumer = (int(x) for x in re.search(r"kRegsHelper = (\d+), kRegsConsumer = (\d+);", text).groups())
    used = {int(x) for x in re.findall(r"Used (\d+) registers", r.stderr)}
    assert used == {(128 * helper + 256 * consumer) // 384}, used
    assert "rows_needed" not in text
