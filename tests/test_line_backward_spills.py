"""CPU: the one-pass line-graph backward (`egc_backward_line_kernel`, csrc/egc_kernels.cu) compiles for sm_90a at every
feature width and norm mode without register spills or a stack frame.

The kernel runs 384 threads, one CTA per SM, so ptxas may give a thread up to 168 registers; a spill would put
local-memory round trips into the per-edge loop.  Needs nvcc (no GPU)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "alignn_b200", "csrc")


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_line_backward_kernel_does_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "egc_kernels.cubin"),
           os.path.join(CSRC, "egc_kernels.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    report = {}
    current = None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current is not None:
            report[current] = tuple(int(v) for v in m.groups())
            current = None
    line = {n: v for n, v in report.items() if "egc_backward_line_kernel" in n}
    shapes = sorted(tuple(int(x) for x in re.search(r"ILi(\d+)ELi(\d+)E", n).groups()) for n in line)
    assert shapes == sorted((d, norm) for d in (32, 64, 128, 256) for norm in (0, 1, 2)), report
    assert all(v == (0, 0, 0) for v in line.values()), line
