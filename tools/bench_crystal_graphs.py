"""Batched crystal-graph construction: the device builder `neighbors.crystal_graphs_device` against the host path
(`crystal_graph(..., "k-nearest")` per structure + `batch` + `.to("cuda")`) on batches of 64 structures drawn with a
seed from tests/golden/sample_structures.npz, at the reference's default k-NN settings (cutoff 8 A, 12 neighbours).

Both paths produce (g, lg) with the bond cosines on the GPU.  Device timings: CUDA events around the build, plus a
synchronise, after warm-up; host timings: wall clock around the host build and the copy, ending in a synchronise.
Prints one JSON line with the GPU name and power limit read in the same run.

    python tools/bench_crystal_graphs.py [--batches 8] [--batch-size 64] [--warmup 2] [--seed 0]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from alignn_b200 import neighbors  # noqa: E402
from alignn_b200.graph import batch  # noqa: E402


def _gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"unavailable ({e})"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_crystal_graphs needs a GPU")
    dev = torch.device("cuda:0")
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    samples = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]]) for i in range(len(z["ids"]))]
    rng = np.random.default_rng(a.seed)
    batches = [[samples[i] for i in rng.choice(len(samples), a.batch_size, replace=False)]
               for _ in range(a.warmup + a.batches)]
    feats = [torch.randn(sum(x.shape[0] for _, x in b), 92, generator=torch.Generator().manual_seed(a.seed)) for b in batches]

    def device_build(i):
        return neighbors.crystal_graphs_device(batches[i], feats[i], device=dev)

    def host_build(i):
        gs, lgs, o = [], [], 0
        for lat, X in batches[i]:
            g, lg = neighbors.crystal_graph(lat, X, feats[i][o:o + X.shape[0]], cutoff=8.0, neighbor_strategy="k-nearest",
                                            max_neighbors=12)
            gs.append(g)
            lgs.append(lg)
            o += X.shape[0]
        return batch(gs).to(dev), batch(lgs).to(dev)

    for i in range(a.warmup):
        device_build(i)
        host_build(i)
    torch.cuda.synchronize()
    dev_ms, host_ms, bonds, pairs = [], [], [], []
    for i in range(a.warmup, a.warmup + a.batches):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        g, lg, _ = device_build(i)
        t1.record()
        torch.cuda.synchronize()
        dev_ms.append(t0.elapsed_time(t1))
        bonds.append(g.num_edges())
        pairs.append(lg.num_edges())
        s = time.perf_counter()
        hg, hlg = host_build(i)
        torch.cuda.synchronize()
        host_ms.append((time.perf_counter() - s) * 1e3)
        assert hg.num_edges() == g.num_edges() and hlg.num_edges() == lg.num_edges()
    name, q = _gpu_info()
    res = {
        "workload": f"{a.batches} batches of {a.batch_size} sample structures, k-nearest, cutoff 8, max_neighbors 12",
        "device_build_ms_median": float(np.median(dev_ms)), "device_build_ms": [round(x, 3) for x in dev_ms],
        "host_build_ms_median": float(np.median(host_ms)), "host_build_ms": [round(x, 3) for x in host_ms],
        "speedup_median": float(np.median(host_ms) / np.median(dev_ms)),
        "bonds_per_batch": bonds, "bond_pairs_per_batch": pairs,
        "gpu": name, "power_limit_and_max_sm_clock": q,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
