#!/usr/bin/env python
"""Timing of the batched weight-gradient launch (wgrad_batch, csrc/wgrad_tc.cu) of one bench.py step.

    python tools/bench_wgrad.py [--batch 64] [--atoms 30] [--seconds 0.5] [--json OUT.jsonl]

The problem list is not written by hand: one eager bench.py-configuration step (same model, batch and seed, weight
gradients deferred into the flat gradient buffer) runs with ops.wgrad_batch wrapped, and the problems of its one call
are kept with their real arguments.  That launch is replayed from a CUDA graph for at least --seconds of GPU time
(tools/bench_gemm.py's time_call), timed with CUDA events.  Printed: ms per launch, the operand bytes ops.wgrad_batch
counts (8 K d per problem: A and B read once) as GB/s and as a share of their HBM floor at the H100 SXM data-sheet
3.35 TB/s.  Also timed:
  * the largest problem (the L(g) edge gate, K = T bond pairs) alone, through the batch launch and through the
    single-problem kernel (ops.wgrad, the path of the force-training double backward);
  * an ablation: every problem at d = 128 (one CTA per output block) with twice the rows, against d = 256 (four CTAs per
    output block, each reading half of A's and half of B's channels) with the same bytes.  If d = 128 takes about half
    the time, the duplicate half-width reads of d = 256 cost; if the two take the same time, HBM bounds both.
The device name, power limit and SM clock limit are read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_gemm import HBM_GBS, device_info, time_call  # noqa: E402


def record_problems(args):
    """The (A, B, out) list of the one wgrad_batch call of an eager bench.py step."""
    from alignn_b200 import dp, ops, synthetic
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig
    dev = torch.device("cuda:0")
    torch.manual_seed(123)
    model = ALIGNN(ALIGNNConfig(name="alignn")).to(dev).train()
    g, lg, lat, tgt = synthetic.make_batch(batch_size=args.batch, atoms=args.atoms, k=12, seed=123)
    batch = (g.to(dev), lg.to(dev), lat.to(dev))
    tgt = tgt.to(dev)
    reducer = dp.FlatGradAllReducer(model.parameters())
    reducer.zero_grad()
    (model(batch) - tgt).abs().mean().backward()
    reducer.gather()                                  # builds the flat buffer; later backwards defer into it
    calls = []
    orig = ops.wgrad_batch

    def rec(problems):
        calls.append(list(problems))
        return orig(problems)

    ops.wgrad_batch = rec
    try:
        reducer.zero_grad()
        with reducer.deferring():
            (model(batch) - tgt).abs().mean().backward()
        reducer.gather()
        torch.cuda.synchronize()
    finally:
        ops.wgrad_batch = orig
    if len(calls) != 1:
        raise SystemExit(f"expected one wgrad_batch call per step, saw {len(calls)}")
    return calls[0]


def nbytes(problems):
    return sum(8 * A.shape[0] * A.shape[1] for A, _, _ in problems)


def report(name, ms, b, rows, info):
    floor = b / (HBM_GBS * 1e9) * 1e3
    r = {"case": name, "ms": ms, "bytes": b, "gbs": b / ms / 1e6, "hbm_floor_ms": floor, "frac_of_floor": floor / ms}
    rows.append(dict(r, device=info))
    print(f"{name:52s} {ms:8.4f} {b / 1e9:7.3f} {r['gbs']:7.0f} {floor:8.4f} {r['frac_of_floor']:8.2f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--atoms", type=int, default=30)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None, help="also append one JSON line per case to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad.py needs a CUDA device")
    from alignn_b200 import _lib, ops
    _lib.load()
    info = device_info()
    print(f"# device: {info['torch_device']} | nvidia-smi name, power.limit, clocks.max.sm: {info['nvidia_smi']}")
    problems = record_problems(args)
    d = problems[0][2].shape[0]
    Ks = sorted((A.shape[0] for A, _, _ in problems), reverse=True)
    print(f"# one step: {len(problems)} problems at d = {d}, K = " +
          ", ".join(f"{k} x{Ks.count(k)}" for k in sorted(set(Ks), reverse=True)))
    print(f"{'case':52s} {'ms':>8s} {'GB':>7s} {'GB/s':>7s} {'floor ms':>8s} {'of floor':>8s}")
    rows = []
    ms, _ = time_call(ops.wgrad_batch, (problems,), {}, args.seconds)
    report(f"wgrad_batch<{d}> step launch ({len(problems)} problems)", ms, nbytes(problems), rows, info)

    big = max(problems, key=lambda p: p[0].shape[0])
    K = big[0].shape[0]
    ms, _ = time_call(ops.wgrad_batch, ([big],), {}, args.seconds)
    report(f"wgrad_batch<{d}> K = {K} alone", ms, nbytes([big]), rows, info)
    A, B = big[0].contiguous(), big[1].contiguous()
    ms, _ = time_call(ops.wgrad, (A, B, 1), {}, args.seconds)
    report(f"wgrad<{d},{d}> single-problem kernel, K = {K}", ms, nbytes([big]), rows, info)
    del A, B

    # ablation: the same bytes at d = 256 (TILES = 4) and d = 128 (TILES = 1, twice the rows)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for dd, scale in ((256, 1), (128, 2)):
        prob = []
        for k in Ks:
            A = torch.randn(k * scale, dd, generator=gen, device="cuda")
            prob.append((A, torch.randn(k * scale, dd, generator=gen, device="cuda"), torch.empty(dd, dd, device="cuda")))
        ms, _ = time_call(ops.wgrad_batch, (prob,), {}, args.seconds)
        report(f"ablation: step's K list x{scale} at d = {dd}", ms, nbytes(prob), rows, info)
        del prob
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "a") as fh:
            for r in rows:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
