"""CPU: every kernel of the batched crystal-graph builder (csrc/crystal_graph_device.cu: the scan in its count, radius
and k-NN modes, shell selection, canonicalisation, ordering and emit) compiles for sm_90a without register spills or a
stack frame.  Needs nvcc (no GPU)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "alignn_b200", "csrc")
KERNELS = ("crystal_scan_kernelILi0E", "crystal_scan_kernelILi1E", "crystal_scan_kernelILi2E", "knn_shell_kernel",
           "knn_canon_kernel", "segment_head_kernel", "order_key_kernel", "unique_flag_kernel", "bond_offsets_kernel",
           "knn_emit_kernel")


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_crystal_graph_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "crystal_graph_device.cubin"),
           os.path.join(CSRC, "crystal_graph_device.cu")]
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
    ours = {n: v for n, v in report.items() if "7crystal" in n}
    for k in KERNELS:
        assert any(k in n for n in ours), (k, sorted(ours))
    assert all(v == (0, 0, 0) for v in ours.values()), ours
