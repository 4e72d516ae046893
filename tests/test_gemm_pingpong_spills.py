"""CPU: the Linear-layer GEMM kernels (csrc/gemm_tc.cu) compile for sm_90a without register spills, a stack frame or
serialized wgmma.

The kernel runs 384 threads per CTA (ptxas caps a thread at 168 registers) and moves registers from the producer
warpgroup to the two consumer warpgroups with setmaxnreg; a spill puts local-memory round trips into the epilogue or
the MMA loop of every tile, and a serialized wgmma (ptxas C7518) drains the tensor cores after every MMA.  Needs nvcc
(no GPU)."""
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
def test_gemm_kernels_no_spills_stack_or_serialized_wgmma(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "gemm_tc.cubin"),
           os.path.join(CSRC, "gemm_tc.cu")]
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
    gemm = {name: v for name, v in report.items() if "gemm_bf16x3_kernel" in name}
    assert sorted(re.search(r"ILi(\d+)E", n).group(1) for n in gemm) == ["128", "32", "64"], report
    assert all(v == (0, 0, 0) for v in gemm.values()), gemm
    # ptxas C7518: a wgmma wait it cannot place makes it serialize every wgmma of the kernel
    serialized = [line for line in res.stderr.splitlines() if "wgmma.mma_async instructions are serialized" in line]
    assert not serialized, serialized
