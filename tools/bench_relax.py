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

--optimize-lattice relaxes the cells too (relax_structures(optimize_lattice=True), ASE's ExpCellFilter): every cell
starts strained and sheared (atoms moved with it), the model computes stress (stresswise_weight=1), and the per-crystal
arm runs the oracle's filtered FIRE (oracle/cell_filter_oracle.py) on the host graph of the current cell.  The largest
difference between the two arms' final positions and cells is reported, with the number of crystals on which they agree
to 1e-5 A and, for every crystal on which they part, whether its 12th-neighbour cut lies inside a distance tie
(`neighbors.knn_cut_is_tied`, at any structure the host arm evaluated), where rounding picks the images the graph
keeps.

    python tools/bench_relax.py [--structures 64] [--steps 10] [--seed 0] [--optimize-lattice]
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
    ap.add_argument("--optimize-lattice", action="store_true", help="relax the cells too (ExpCellFilter)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_relax.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from alignn_b200 import neighbors, ops, relax_structures
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    from oracle import cell_filter_oracle as CF
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
    cell = a.optimize_lattice
    if cell:                                                   # strained, sheared cells, the atoms moved with them
        srng = np.random.default_rng(a.seed + 1)
        Ds = [np.eye(3) + np.diag(srng.uniform(-0.04, 0.04, 3)) + srng.uniform(-0.03, 0.03, (3, 3)) for _ in structs]
        structs = [(lat @ D.T, X @ D.T) for (lat, X), D in zip(structs, Ds)]
    torch.manual_seed(1)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                               atom_input_features=92, gradwise_weight=1.0, stresswise_weight=1.0 if cell else 0.0)
    model = ALIGNNAtomWise(cfg).to(dev).eval()

    def batched():
        r = relax_structures(model, structs, feats, fmax=0.0, steps=a.steps, optimize_lattice=cell)
        torch.cuda.synchronize()
        return r

    visited = []                                               # per crystal: every (cell, x) the host arm evaluated

    def per_crystal():
        out, o = [], 0
        visited.clear()
        for lat, X in structs:
            n = X.shape[0]
            f_b = feats[o:o + n].cpu()
            lat_t = torch.tensor(lat, dtype=torch.float32).view(1, 3, 3).to(dev)

            def evaluate(x, lat=lat, f_b=f_b, lat_t=lat_t, n=n):
                g, lg = neighbors.crystal_graph(lat, x, f_b, cutoff=8.0, neighbor_strategy="k-nearest", max_neighbors=12)
                res = model((g.to(dev), lg.to(dev), lat_t))
                return float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy()

            seen = []
            visited.append(seen)

            def evaluate_cell(c, x, f_b=f_b, n=n, seen=seen):
                seen.append((c, x))
                g, lg = neighbors.crystal_graph(c, x, f_b, cutoff=8.0, neighbor_strategy="k-nearest", max_neighbors=12)
                g.ndata["V"] = torch.full((n,), abs(float(np.dot(np.cross(c[0], c[1]), c[2]))), dtype=torch.float32)
                res = model((g.to(dev), lg.to(dev), torch.tensor(c, dtype=torch.float32).view(1, 3, 3).to(dev)))
                return (float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy(),
                        res["stresses"].detach().reshape(3, 3).cpu().numpy())
            if cell:
                out.append(CF.relax(evaluate_cell, lat, X, fmax=0.0, steps=a.steps))
            else:
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
    extra = {}
    if not cell:
        assert dmax <= 1e-5, f"the arms end {dmax} A apart"
    else:
        # reported, not asserted: the arms' matrix functions (the kernel's Pade, scipy's expm / logm) differ by
        # rounding, and where an atom's 12th and 13th neighbours are equally far (the images x + R and x - R) that
        # rounding picks the image the k-nearest graph keeps, after which the two trajectories part
        Cg = got.cells.cpu().numpy()
        dcell = [float(np.abs(Cg[b] - r["cell"]).max()) for b, r in enumerate(ref)]
        dpos = [float(np.abs(P[aoff[b]:aoff[b + 1]] - r["positions"]).max()) for b, r in enumerate(ref)]
        moved = max(float(np.abs(r["cell"] - lat).max()) for r, (lat, _) in zip(ref, structs))
        agree = sum(p <= 1e-5 and c <= 1e-5 for p, c in zip(dpos, dcell))
        # per crystal: does its 12th-neighbour cut fall inside a distance tie at any structure the host arm evaluated?
        tied = [any(neighbors.knn_cut_is_tied(c, x) for c, x in seen) for seen in visited]
        parted = [b for b in range(len(structs)) if dpos[b] > 1e-5 or dcell[b] > 1e-5]
        extra = {"max_cell_difference_A": max(dcell), "crystals_within_1e-5_A": f"{agree}/{len(structs)}",
                 "crystals_with_a_knn_tie": sum(tied),
                 "parted_crystals": [dict(id=b, positions_A=round(dpos[b], 4), cell_A=round(dcell[b], 4), knn_tie=tied[b])
                                     for b in parted],
                 "every_parted_crystal_has_a_knn_tie": all(tied[b] for b in parted),
                 "max_difference_on_crystals_without_a_tie_A": max([max(dpos[b], dcell[b]) for b in range(len(structs))
                                                                    if not tied[b]], default=0.0),
                 "max_cell_change_A": round(moved, 4)}
    ops.TIMER = ops.KernelTimer()
    try:
        batched()
        summ = ops.TIMER.summary()
    finally:
        ops.TIMER = None
    evals = a.steps + 1
    split = {k[len("relax_"):]: round(summ[k]["total_ms"] / evals, 3) for k in summ if k.startswith("relax_")}
    med_b, med_p = statistics.median(ms["batched"]), statistics.median(ms["per_crystal"])
    what = "ExpCellFilter FIRE on atoms and strained, sheared cells" if cell else "FIRE"
    out = dict(workload=f"{len(structs)} jittered sample structures ({sum(sizes)} atoms), ALIGNNAtomWise 4+4 d=256, "
                        f"k-nearest 8 A / 12, fmax=0, {a.steps} {what} steps ({evals} evaluations per crystal)",
               batched_ms=[round(v, 1) for v in ms["batched"]], batched_ms_median=round(med_b, 1),
               per_crystal_ms=[round(v, 1) for v in ms["per_crystal"]], per_crystal_ms_median=round(med_p, 1),
               speedup_median=round(med_p / med_b, 2), batched_ms_per_evaluation_split=split,
               max_position_difference_A=dmax, **extra, device=device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
