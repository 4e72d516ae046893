#!/usr/bin/env python
"""Per-shape timing of the Linear-layer GEMM (gemm_nt / gemm_gather) at the shapes one bench.py step launches.

    python tools/bench_gemm.py [--batch 64] [--atoms 30] [--seconds 0.5] [--json OUT.jsonl]

The shapes are not listed by hand: one eager forward + backward of the bench.py model (same config, batch and seed)
runs with ops.gemm_nt / ops.gemm_gather wrapped, and every distinct call (kernel name as in bench.py's kernel table,
M, N, K, addends) is kept with its real arguments.  Each is then replayed from a CUDA graph of back-to-back launches
(no host launch cost in the window) for at least --seconds of GPU time, timed with CUDA events.

Per shape it prints ms per launch; compulsory bytes (A, C and identity addends once each, gathered
tables and their indices once, the weight image) and GB/s; bf16 work (three bf16 products per fp32 product) and
TFLOP/s; and the share of the larger of the two floors at the H100 SXM data-sheet rates (3.35 TB/s HBM3, 989 TFLOP/s
dense BF16), with which floor it is.  The device name, power limit and SM clock limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_GBS = 3350.0
BF16_TFLOPS = 989.0


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001 -- the timings stand without it
        out = f"nvidia-smi unavailable ({e})"
    return {"torch_device": torch.cuda.get_device_name(), "nvidia_smi": out}


def record_calls(args):
    """(key, fn, call args, kwargs, count per step) of every distinct GEMM call of one eager fwd + bwd."""
    from alignn_b200 import ops, synthetic
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig
    dev = torch.device("cuda:0")
    torch.manual_seed(123)
    model = ALIGNN(ALIGNNConfig(name="alignn")).to(dev).train()
    g, lg, lat, tgt = synthetic.make_batch(batch_size=args.batch, atoms=args.atoms, k=12, seed=123)
    batch = (g.to(dev), lg.to(dev), lat.to(dev))
    tgt = tgt.to(dev)
    calls = {}
    orig = {"gemm_nt": ops.gemm_nt, "gemm_gather": ops.gemm_gather}

    def wrap(name):
        fn = orig[name]

        def rec(A, w, bias=None, *a, **kw):
            if name == "gemm_nt":
                res = a[0] if a else kw.get("residual")
                kind = "+residual" if res is not None else ""
            else:
                kind = ("+gather" if kw.get("idx0") is not None else ("+residual" if kw.get("add0") is not None else ""))
                if kw.get("add1") is not None:
                    kind += "+add1" + ("[idx]" if kw.get("idx1") is not None else "")
                kind += "+stats" if kw.get("stats") else ""
            key = (f"{name}<{min(w.N, 256)}>{kind}", A.shape[0], w.N, w.K)
            if key in calls:
                calls[key][4] += 1
            else:
                calls[key] = [key, fn, (A, w, bias) + a, dict(kw), 1]
            return fn(A, w, bias, *a, **kw)
        return rec

    for i in range(2):        # the first pass builds the operand images; the second is the one recorded
        if i == 1:
            calls.clear()
            ops.gemm_nt, ops.gemm_gather = wrap("gemm_nt"), wrap("gemm_gather")
        try:
            model.zero_grad(set_to_none=True)
            (model(batch) - tgt).abs().mean().backward()
            torch.cuda.synchronize()
        finally:
            ops.gemm_nt, ops.gemm_gather = orig["gemm_nt"], orig["gemm_gather"]
    return list(calls.values())


def compulsory_bytes(fn_name, call_args, kw, M, N, K):
    b = 4 * M * K + 4 * M * N + 2 * 2 * N * K              # A in, C out, the two bf16 planes of the weight image
    if call_args[2] is not None:
        b += 4 * N
    if fn_name == "gemm_nt":
        res = call_args[3] if len(call_args) > 3 else kw.get("residual")
        return b + (4 * M * N if res is not None else 0)
    for t, ix in ((kw.get("add0"), kw.get("idx0")), (kw.get("add1"), kw.get("idx1"))):
        if t is None:
            continue
        b += 4 * M * N if ix is None else 4 * t.shape[0] * N + 4 * M   # a gathered table is read once, plus its index
    return b


def time_call(fn, call_args, kw, seconds):
    """ms per launch of fn(*call_args, **kw): a CUDA graph of back-to-back launches, replayed for >= `seconds`."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn(*call_args, **kw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(s):                               # launches per graph: aim at ~50 ms of work per replay
        e0.record()
        fn(*call_args, **kw)
        e1.record()
    torch.cuda.synchronize()
    est = max(e0.elapsed_time(e1), 1e-3)
    per_graph = int(min(2000, max(10, 50.0 / est)))
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=s):
        for _ in range(per_graph):
            fn(*call_args, **kw)
    gr.replay()
    torch.cuda.synchronize()
    e0.record()
    gr.replay()
    e1.record()
    torch.cuda.synchronize()
    replays = max(3, int(seconds * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(replays):
        gr.replay()
    e1.record()
    torch.cuda.synchronize()
    total = e0.elapsed_time(e1)
    return total / (replays * per_graph), total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--atoms", type=int, default=30)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None, help="also append one JSON line per shape to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a CUDA device")
    from alignn_b200 import _lib
    _lib.load()
    info = device_info()
    print(f"# device: {info['torch_device']} | nvidia-smi name, power.limit, clocks.max.sm: {info['nvidia_smi']}")
    print(f"# floors at data-sheet rates: {HBM_GBS:.0f} GB/s HBM, {BF16_TFLOPS:.0f} TFLOP/s dense BF16")
    rows = []
    hdr = (f"{'kernel':44s} {'M':>7s} {'N':>5s} {'K':>5s} {'n/step':>6s} {'ms':>8s} {'MB':>8s} {'GB/s':>7s} "
           f"{'GFLOP':>7s} {'TFLOP/s':>7s} {'floor':>5s} {'of floor':>8s} {'ms/step':>8s}")
    print(hdr)
    total_step = 0.0
    for key, fn, call_args, kw, count in sorted(record_calls(args), key=lambda c: (c[0][0], -c[0][1])):
        name, M, N, K = key
        ms, window = time_call(fn, call_args, kw, args.seconds)
        nbytes = compulsory_bytes(name.split("<")[0], call_args, kw, M, N, K)
        flop = 3 * 2.0 * M * N * K
        t_hbm, t_mma = nbytes / (HBM_GBS * 1e9) * 1e3, flop / (BF16_TFLOPS * 1e12) * 1e3
        floor, which = (t_hbm, "hbm") if t_hbm >= t_mma else (t_mma, "mma")
        total_step += ms * count
        r = {"kernel": name, "M": M, "N": N, "K": K, "launches_per_step": count, "ms": ms, "bytes": nbytes,
             "gbs": nbytes / ms / 1e6, "gflop": flop / 1e9, "tflops": flop / ms / 1e9, "floor": which,
             "frac_of_floor": floor / ms, "ms_per_step": ms * count, "timed_ms": window}
        rows.append(r)
        print(f"{name:44s} {M:7d} {N:5d} {K:5d} {count:6d} {ms:8.4f} {nbytes / 1e6:8.1f} {r['gbs']:7.0f} "
              f"{r['gflop']:7.1f} {r['tflops']:7.1f} {which:>5s} {r['frac_of_floor']:8.2f} {ms * count:8.3f}")
    print(f"# sum over shapes of ms per launch x launches per step: {total_step:.3f} ms")
    if args.json:
        with open(args.json, "a") as fh:
            for r in rows:
                fh.write(json.dumps(dict(r, device=info)) + "\n")


if __name__ == "__main__":
    main()
