#!/usr/bin/env python
"""Batched FIRE relaxation: `relax_structures` against the reference's architecture, one crystal at a time.

Workload: 64 structures drawn with a seed from tests/golden/sample_structures.npz and jittered, the 4 + 4, d = 256,
92-feature ALIGNNAtomWise of tools/bench_force_training.py (seeded weights, eval mode), k-nearest graphs (8 A, 12
neighbours), fmax = 0 so that every crystal takes exactly `--steps` FIRE steps in both arms.

  batched:   relax_structures -- per step one device graph build, one model call and one FIRE launch for the batch;
  per-crystal: for each crystal, every evaluation runs neighbors.crystal_graph on the host, .to("cuda"), the same model
             on a one-crystal batch, and the oracle's FIRE step in numpy (oracle/fire_oracle.py).

Each arm runs three times (alternating); the median wall time (ending in a synchronise) is reported.  One more batched
run with CUDA events around its phases gives the per-step split (build, model, FIRE kernel, read-back; each span runs
from its first enqueue to its last, host work inside it included).  The two arms must end at the same positions.  The
device name, power limit and SM clock limit are read in the same run.

    python tools/bench_relax.py [--structures 64] [--steps 10] [--seed 0]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001 -- the timings stand without it
        out = f"nvidia-smi unavailable ({e})"
    return {"torch_device": torch.cuda.get_device_name(), "nvidia_smi": out}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--structures", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_relax.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from alignn_b200 import neighbors, ops, relax_structures
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    from oracle import fire_oracle as FO

    dev = torch.device("cuda:0")
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    rng = np.random.default_rng(a.seed)
    pick = rng.choice(len(z["ids"]), a.structures, replace=False)
    structs = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]] + rng.normal(scale=0.03, size=(off[i + 1] - off[i], 3)))
               for i in pick]
    sizes = [x.shape[0] for _, x in structs]
    feats = torch.from_numpy(rng.normal(size=(sum(sizes), 92)).astype(np.float32)).to(dev)
    torch.manual_seed(1)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                               atom_input_features=92, gradwise_weight=1.0)
    model = ALIGNNAtomWise(cfg).to(dev).eval()

    def batched():
        r = relax_structures(model, structs, feats, fmax=0.0, steps=a.steps)
        torch.cuda.synchronize()
        return r

    def per_crystal():
        out, o = [], 0
        for lat, X in structs:
            n = X.shape[0]
            f_b = feats[o:o + n].cpu()
            lat_t = torch.tensor(lat, dtype=torch.float32).view(1, 3, 3).to(dev)

            def evaluate(x, lat=lat, f_b=f_b, lat_t=lat_t, n=n):
                g, lg = neighbors.crystal_graph(lat, x, f_b, cutoff=8.0, neighbor_strategy="k-nearest", max_neighbors=12)
                res = model((g.to(dev), lg.to(dev), lat_t))
                return float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy()
            out.append(FO.relax(evaluate, X, fmax=0.0, steps=a.steps))
            o += n
        torch.cuda.synchronize()
        return out

    batched()                                                  # warm-up: module loads, allocator, every kernel shape
    per_crystal()
    ms = {"batched": [], "per_crystal": []}
    res = {}
    for _ in range(3):
        for name, fn in (("batched", batched), ("per_crystal", per_crystal)):
            t = time.perf_counter()
            res[name] = fn()
            ms[name].append((time.perf_counter() - t) * 1e3)
    got, ref = res["batched"], res["per_crystal"]
    P = got.positions.cpu().numpy()
    aoff = got.atom_offsets.cpu().tolist()
    dmax = max(float(np.abs(P[aoff[b]:aoff[b + 1]] - r["positions"]).max()) for b, r in enumerate(ref))
    assert got.nsteps.tolist() == [a.steps] * len(structs) and all(r["nsteps"] == a.steps for r in ref)
    assert dmax <= 1e-5, f"the arms end {dmax} A apart"
    ops.TIMER = ops.KernelTimer()
    try:
        batched()
        summ = ops.TIMER.summary()
    finally:
        ops.TIMER = None
    evals = a.steps + 1
    split = {k[len("relax_"):]: round(summ[k]["total_ms"] / evals, 3) for k in summ if k.startswith("relax_")}
    med_b, med_p = statistics.median(ms["batched"]), statistics.median(ms["per_crystal"])
    out = dict(workload=f"{len(structs)} jittered sample structures ({sum(sizes)} atoms), ALIGNNAtomWise 4+4 d=256, "
                        f"k-nearest 8 A / 12, fmax=0, {a.steps} FIRE steps ({evals} evaluations per crystal)",
               batched_ms=[round(v, 1) for v in ms["batched"]], batched_ms_median=round(med_b, 1),
               per_crystal_ms=[round(v, 1) for v in ms["per_crystal"]], per_crystal_ms_median=round(med_p, 1),
               speedup_median=round(med_p / med_b, 2), batched_ms_per_evaluation_split=split,
               max_position_difference_A=dmax, device=device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
