"""CPU: the net-torque kernels (csrc/ff_device.cu), the per-crystal ones included, compile for sm_90a without register
spills or a stack frame.  Needs nvcc (no GPU)."""
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
def test_torque_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "ff_device.cubin"),
           os.path.join(CSRC, "ff_device.cu")]
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
    ours = {n: v for n, v in report.items() if "torque_" in n}
    for kernel in ("torque_pc_prep_kernel", "torque_pc_com_kernel", "torque_pc_tau_kernel", "torque_pc_solve_kernel",
                   "torque_pc_apply_kernel", "torque_solve_kernel"):
        assert any(kernel in n for n in ours), sorted(report)
    assert all(v == (0, 0, 0) for v in ours.values()), ours
