"""CPU: the equation-of-state fit kernel (csrc/eos_device.cu) compiles for sm_90a without register spills or a stack frame.
Needs nvcc (no GPU)."""
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
def test_eos_fit_kernel_does_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "eos_device.cubin"),
           os.path.join(CSRC, "eos_device.cu")]
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
    ours = {n: v for n, v in report.items() if "3eos" in n}
    for kernel in ("eos_fit_kernel",):
        assert any(kernel in n for n in ours), sorted(report)
    assert all(v == (0, 0, 0) for v in ours.values()), ours
