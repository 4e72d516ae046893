"""CPU: the weight-gradient kernels (csrc/wgrad_tc.cu) compile for sm_90a without register spills, a stack frame or
serialized wgmma.

The kernels run 512 threads per CTA, so ptxas caps a thread at 128 registers; a spill puts local-memory round trips
into the loader or the MMA loop of every chunk of rows.  Needs nvcc (no GPU)."""
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
def test_wgrad_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "wgrad_tc.cubin"),
           os.path.join(CSRC, "wgrad_tc.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    # ptxas -v: "Compiling entry function '<mangled>'" ... "F bytes stack frame, S bytes spill stores, L bytes spill loads"
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
    shapes = lambda kind: sorted(re.search(r"ILi(\d+)ELi(\d+)E", n).groups() for n in report if kind in n)  # noqa: E731
    single = [("256", "256"), ("128", "128"), ("64", "64"), ("32", "32"), ("256", "64"), ("256", "96"), ("64", "96"),
              ("64", "32"), ("32", "64"), ("32", "96")]
    assert shapes("wgrad_bf16x3_kernel") == sorted(single), report
    assert shapes("wgrad_batch_kernel") == sorted([("256", "256"), ("128", "128"), ("64", "64"), ("32", "32")]), report
    kernels = {n: v for n, v in report.items() if "wgrad_bf16x3_kernel" in n or "wgrad_batch_kernel" in n}
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
    # ptxas C7518: a wgmma wait it cannot place makes it serialize every wgmma of the kernel
    serialized = [line for line in res.stderr.splitlines() if "wgmma.mma_async instructions are serialized" in line]
    assert not serialized, serialized
