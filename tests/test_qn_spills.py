"""CPU: the quasi-Newton step kernels (csrc/qn_device.cu) compile for sm_90a without register spills or a stack frame.
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
def test_qn_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "qn_device.cubin"),
           os.path.join(CSRC, "qn_device.cu")]
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
    ours = {n: v for n, v in report.items() if "2qn" in n}
    for kernel in ("lbfgs_step_kernelILb0", "lbfgs_step_kernelILb1", "bfgs_rows_kernelILb0", "bfgs_rows_kernelILb1",
                   "bfgs_hdr_kernel", "bfgs_rank2_kernel", "bfgs_vtf_kernel", "bfgs_vw_kernel", "bfgs_move_kernelILb0",
                   "bfgs_move_kernelILb1"):
        assert any(kernel in n for n in ours), sorted(report)
    assert all(v == (0, 0, 0) for v in ours.values()), ours
