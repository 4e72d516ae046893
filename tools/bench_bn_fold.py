#!/usr/bin/env python
"""Per-launch cost of taking train-mode BatchNorm backward statistics in the data-gradient GEMM's epilogue.

    python tools/bench_bn_fold.py [--iters 50] [--json OUT.jsonl]

At each shape where a bench.py step folds (data-gradient GEMMs of the conv layers and of the 64 -> 256 embedding Linear
at the bench's N = 1920, E = 23 040, T = 276 480 rows) it times, with CUDA events over --iters back-to-back launches:
  plain    gemm_gather as without the fold
  fold     gemm_gather(..., bn_bwd=...) + the colsum of its partials
  reduce   bn_backward_reduce + its colsum (what the fold replaces)
and prints ms per launch and the saving plain + reduce - fold.  The device name, power limit and SM clock limit are read
in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_gemm import device_info  # noqa: E402

# (site, M, N = producer width, K = consumer GEMM depth, residual)
SITES = [
    ("egT dgrad, L(g) edge BN", 276480, 256, 256, True),
    ("wT dgrad, angle embedding BN1", 276480, 64, 256, False),
    ("catT dgrad, g edge BN (L(g) node)", 23040, 256, 1024, True),
    ("egT dgrad, g edge BN", 23040, 256, 256, True),
    ("catT dgrad, node BN", 1920, 256, 1024, True),
]


def _time(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bn_fold.py needs a CUDA device")
    from alignn_b200 import ops
    dev = torch.device("cuda")
    info = device_info()
    print(json.dumps(info), flush=True)
    g = torch.Generator(device="cpu").manual_seed(0)
    rows = []
    for site, M, N, K, residual in SITES:
        A = torch.randn(M, K, generator=g).to(dev)
        img = ops.WeightImage((torch.randn(N, K, generator=g) / K ** 0.5).to(dev))
        R = torch.randn(M, N, generator=g).to(dev)
        add0 = torch.randn(M, N, generator=g).to(dev) if residual else None
        vecs = tuple((1.0 + 0.1 * torch.randn(N, generator=g)).to(dev) for _ in range(4))
        C = ops.gemm_gather(A, img, add0=add0)

        def fold():
            _, part = ops.gemm_gather(A, img, add0=add0, bn_bwd=(R,) + vecs)
            ops.colsum(part.view(part.shape[0], 2 * N), 1.0 / M)
        t_plain = _time(lambda: ops.gemm_gather(A, img, add0=add0), args.iters)
        t_fold = _time(fold, args.iters)
        t_reduce = _time(lambda: ops.bn_backward_reduce(R, C, *vecs), args.iters)
        row = {"site": site, "M": M, "N": N, "K": K, "residual": residual, "plain_ms": round(t_plain, 4),
               "fold_ms": round(t_fold, 4), "reduce_ms": round(t_reduce, 4),
               "saving_ms": round(t_plain + t_reduce - t_fold, 4)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del A, img, R, add0, C
    if args.json:
        with open(args.json, "a") as f:
            for row in rows:
                f.write(json.dumps(dict(row, device=info)) + "\n")


if __name__ == "__main__":
    main()
