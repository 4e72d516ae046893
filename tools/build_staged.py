"""Build the staged (not yet hardware-validated) kernels into alignn_b200/csrc/staged/libalignn_b200_staged.so.

    python tools/build_staged.py [--force]

Kept apart from libalignn_b200.so on purpose: `__graft_entry__.build()` compiles only alignn_b200/csrc/*.cu, the
shipped library and include/alignn_b200.h contain validated code only.  See alignn_b200/csrc/staged/egc_fused.h."""
import glob
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGED = os.path.join(ROOT, "alignn_b200", "csrc", "staged")
LIB = os.path.join(STAGED, "libalignn_b200_staged.so")


def build(force: bool = False) -> str:
    sources = sorted(glob.glob(os.path.join(STAGED, "*.cu")))
    deps = sources + glob.glob(os.path.join(STAGED, "*.h")) + glob.glob(os.path.join(STAGED, "..", "*.cuh")) + \
        glob.glob(os.path.join(ROOT, "include", "*.h"))
    if force or not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in deps):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
               "-shared", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(STAGED, ".."), "-o", LIB] + sources
        print("[build_staged]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
