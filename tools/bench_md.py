#!/usr/bin/env python
"""Batched molecular dynamics: `run_md` against the reference's architecture, one crystal at a time.

Workload: 64 structures drawn with a seed from tests/golden/sample_structures.npz and jittered, the 4 + 4, d = 256,
92-feature ALIGNNAtomWise of tools/bench_relax.py (seeded weights, eval mode), k-nearest graphs (8 A, 12 neighbours),
`--ensemble` at 300 K from Maxwell-Boltzmann momenta at 300 K, a 1 fs timestep and `--steps` steps (steps + 1
evaluations per crystal), with the reference's defaults: NVT Berendsen (the default) with taut = 100 timesteps, NVT
Langevin with friction 1e-4 per ASE time unit, NVT Andersen with andersen_prob 0.1.  The stochastic ensembles draw
crystal b's noise from the stream of seed `--seed` + b and draw their structures from the samples with two atoms or
more (Langevin with fixcm rejects one-atom crystals).  Masses are seeded random values in [1, 200] amu.
NPT Berendsen (`--ensemble npt_berendsen`) runs ForceField's taut = 500 fs and taup = 1000 fs at `--pressure-bar`
(default 1.01325 bar, one atmosphere: ASE's own NPTBerendsen example) with `--compressibility` (default 1e-6 / bar, a
solid with a bulk modulus of 100 GPa); the reference passes neither, and its own call cannot run without them.  Its
model is the same with `stresswise_weight=1` (the other ensembles keep the stress off, so their numbers stay
comparable), and each step evaluates the model twice.  NPT Nose-Hoover (`--ensemble npt_nose_hoover`, ASE's NPT) runs
the same structures rotated by `upper_triangular` into the cell form it needs, ForceField's externalstress 0 and
`--ttime` (fs) / `--pfactor` (ASE units); both default to None, the reference's call, with thermostat and barostat off.
Its model also computes stress, and each step evaluates it once.

  batched:     run_md -- per evaluation one device graph build, one model call and one integrator launch for the batch;
  per-crystal: for each crystal, every evaluation runs neighbors.crystal_graph on the host, .to("cuda"), the same model
               on a one-crystal batch, and the oracle's integrator step in numpy (oracle/md_oracle.py, or
               oracle/md_thermostat_oracle.py on the same restated noise stream; for NPT the graph is built on the
               current cell and the integrator is oracle/md_npt_oracle.py or oracle/md_nose_hoover_oracle.py).

Each arm runs three times (alternating); the median wall time (ending in a synchronise) is reported.  One more batched
run with CUDA events around its phases gives the per-evaluation split (build, model, step kernel, read-back; each span
runs from its first enqueue to its last, host work inside it included).  The largest difference between the two arms'
final positions is reported, and per crystal whether its 12th-neighbour cut lies inside a distance tie
(`neighbors.knn_cut_is_tied`) at any structure the host arm evaluated: there rounding picks the images the k-nearest
graph keeps, and the arms may part.  The device name, power limit and SM clock limit are read in the same run.

    python tools/bench_md.py [--ensemble nvt_berendsen|nvt_langevin|nvt_andersen|npt_berendsen|npt_nose_hoover]
                             [--structures 64] [--steps 50] [--seed 0] [--pressure-bar 1.01325] [--compressibility 1e-6]
                             [--ttime FS] [--pfactor AMU_PER_A]
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


def _kept_bonds(lat, X, dev, cutoff=4.0):
    """Bonds eALIGNN keeps in this structure alone: its filter recomputes each bond with the image added as Angstrom
    (DESIGN section 8) and drops those longer than the 4 A inner cutoff, which can drop them all."""
    from alignn_b200 import neighbors
    from alignn_b200.ealignn_atomwise import cartesian_coordinates
    from alignn_b200.graph import lightweight_graph
    g, _, lat_t = neighbors.crystal_graphs_device([(lat, X)], torch.zeros(X.shape[0], 1, device=dev), device=dev,
                                                  neighbor_strategy="radius_graph", cutoff=cutoff, line_graph=False)
    return lightweight_graph(g, cartesian_coordinates(g, lat_t), cutoff)[0].num_edges()


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
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--model", choices=("alignn_atomwise", "ealignn"), default="alignn_atomwise",
                    help="ealignn: a 2+2, d=64 eALIGNNAtomWise on radius_graph 4 A / 12 (the reference's eALIGNN example "
                         "config); the host arm builds each crystal's graph with crystal_graphs_device")
    ap.add_argument("--ensemble", default="nvt_berendsen",
                    choices=("nvt_berendsen", "nvt_langevin", "nvt_andersen", "npt_berendsen", "npt_nose_hoover"))
    ap.add_argument("--pressure-bar", type=float, default=1.01325)
    ap.add_argument("--compressibility", type=float, default=1e-6, help="1/bar")
    ap.add_argument("--ttime", type=float, default=None, help="fs (npt_nose_hoover; default None: no thermostat)")
    ap.add_argument("--pfactor", type=float, default=None, help="amu/A (npt_nose_hoover; default None: no barostat)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from alignn_b200 import maxwell_boltzmann_momenta, neighbors, ops, run_md, upper_triangular
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    from alignn_b200.ealignn_atomwise import eALIGNNAtomWise, eALIGNNAtomWiseConfig
    from oracle import md_nose_hoover_oracle as NH
    from oracle import md_npt_oracle as NO
    from oracle import md_oracle as MO
    from oracle import md_thermostat_oracle as TO

    dev = torch.device("cuda:0")
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    rng = np.random.default_rng(a.seed)
    pool = np.arange(len(z["ids"]))
    npt, nh = a.ensemble == "npt_berendsen", a.ensemble == "npt_nose_hoover"
    if a.ensemble in ("nvt_langevin", "nvt_andersen"):         # Langevin (fixcm) rejects one-atom crystals
        pool = pool[off[1:] - off[:-1] >= 2]
    if a.model == "ealignn":
        # a crystal whose filtered graph keeps no bond cannot run alone (the one-crystal forward has no edges)
        pool = np.array([i for i in pool if _kept_bonds(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]], dev) >= 2 * (off[i + 1] - off[i])])
    pick = rng.choice(pool, min(a.structures, len(pool)), replace=False)
    structs = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]] + rng.normal(scale=0.03, size=(off[i + 1] - off[i], 3)))
               for i in pick]
    if nh:
        structs, _ = upper_triangular(structs)
    sizes = [x.shape[0] for _, x in structs]
    aoff = np.concatenate([[0], np.cumsum(sizes)])
    feats = torch.from_numpy(rng.normal(size=(sum(sizes), 92)).astype(np.float32)).to(dev)
    masses = rng.uniform(1.0, 200.0, sum(sizes))
    p0 = maxwell_boltzmann_momenta(masses, 300.0, rng)
    torch.manual_seed(1)
    ea = a.model == "ealignn"
    if ea:
        model = eALIGNNAtomWise(eALIGNNAtomWiseConfig(name="ealignn_atomwise", atom_input_features=92,
                                                      stresswise_weight=1.0 if npt or nh else 0.0)).to(dev).eval()
        graph = dict(neighbor_strategy="radius_graph", cutoff=4.0, max_neighbors=12)
    else:
        cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                                   atom_input_features=92, gradwise_weight=1.0,
                                   stresswise_weight=1.0 if npt or nh else 0.0)
        model = ALIGNNAtomWise(cfg).to(dev).eval()
        graph = dict(neighbor_strategy="k-nearest", cutoff=8.0, max_neighbors=12)

    def one_crystal(cell, x, f_b):
        """(g, lg, lat) of one crystal as the calculator builds it: on the host for ALIGNNAtomWise; on the device for
        eALIGNN, which needs the graph's frac_coords and images"""
        if ea:
            return neighbors.crystal_graphs_device([(cell, x)], f_b.to(dev), device=dev, **graph)
        g, lg = neighbors.crystal_graph(cell, x, f_b, **graph)
        g.ndata["V"] = torch.full((x.shape[0],), abs(float(np.dot(np.cross(cell[0], cell[1]), cell[2]))),
                                  dtype=torch.float32)
        return g.to(dev), lg.to(dev), torch.tensor(cell, dtype=torch.float32).view(1, 3, 3).to(dev)
    timestep, T0 = 1.0, 300.0

    def batched():
        extra = {} if a.ensemble == "nvt_berendsen" else dict(seed=a.seed)
        if npt:
            extra = dict(pressure=a.pressure_bar, compressibility=a.compressibility)
        if nh:
            extra = dict(ttime=a.ttime, pfactor=a.pfactor)
        r = run_md(model, structs, feats, masses, ensemble=a.ensemble, steps=a.steps, timestep=timestep,
                   temperature_K=T0, momenta=p0, **graph, **extra)
        torch.cuda.synchronize()
        return r

    visited = []                                               # per crystal: every x the host arm evaluated

    def per_crystal():
        out = []
        visited.clear()
        for b, (lat, X) in enumerate(structs):
            sl = slice(aoff[b], aoff[b + 1])
            f_b = feats[sl].cpu()
            seen = []
            visited.append(seen)

            def evaluate(x, lat=lat, f_b=f_b, n=X.shape[0], seen=seen):
                seen.append((lat, x.copy()))
                res = model(one_crystal(lat, x, f_b))
                return float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy()

            def evaluate_cell(cell, x, f_b=f_b, n=X.shape[0], seen=seen):
                seen.append((cell, x.copy()))
                res = model(one_crystal(cell, x, f_b))
                return (float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy(),
                        res["stresses"].detach().reshape(3, 3).cpu().numpy())
            dt = timestep * MO.fs
            if npt:
                out.append(NO.run(evaluate_cell, lat, X, masses[sl], steps=a.steps, dt=dt, temperature_K=T0,
                                  pressure=a.pressure_bar, compressibility=a.compressibility, momenta=p0[sl]))
            elif nh:
                out.append(NH.run(evaluate_cell, lat, X, masses[sl], steps=a.steps, dt=dt, temperature_K=T0,
                                  ttime=None if a.ttime is None else a.ttime * MO.fs, pfactor=a.pfactor,
                                  momenta=p0[sl]))
            elif a.ensemble == "nvt_berendsen":
                out.append(MO.run(evaluate, X, masses[sl], ensemble=MO.NVT_BERENDSEN, steps=a.steps, dt=dt,
                                  temperature_K=T0, taut=100 * dt, momenta=p0[sl]))
            else:
                out.append(TO.run(evaluate, X, masses[sl], ensemble=a.ensemble, steps=a.steps, dt=dt, temperature_K=T0,
                                  noise=TO.PhiloxNoise(a.seed + b), friction=1e-4, andersen_prob=0.1,
                                  momenta=p0[sl]))
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
    T = got.temperature.cpu().numpy()
    dpos = [float(np.abs(P[aoff[b]:aoff[b + 1]] - r["positions"]).max()) for b, r in enumerate(ref)]
    tied = [not ea and any(neighbors.knn_cut_is_tied(c, x) for c, x in seen) for seen in visited]
    parted = [b for b in range(len(structs)) if dpos[b] > 1e-5]
    ops.TIMER = ops.KernelTimer()
    try:
        batched()
        summ = ops.TIMER.summary()
    finally:
        ops.TIMER = None
    evals = (2 if npt else 1) * a.steps + 1
    if npt or nh:
        C = got.cells.cpu().numpy()
        cells_out = dict(cell_moved_max_A=float(np.abs(C[-1] - C[0]).max()),
                         max_cell_difference_A=max(float(np.abs(C[-1, b] - r["cell"]).max()) for b, r in enumerate(ref)),
                         mean_pressure_eV_A3=dict(first=float(got.pressure[0].mean()), last=float(got.pressure[-1].mean())),
                         **({"target_pressure_eV_A3": NO.pressure_au(a.pressure_bar)} if npt else {}))
    else:
        cells_out = {}
    split = {k[len("md_"):]: round(summ[k]["total_ms"] / evals, 3) for k in summ if k.startswith("md_")}
    med_b, med_p = statistics.median(ms["batched"]), statistics.median(ms["per_crystal"])
    what = "eALIGNNAtomWise 2+2 d=64, radius_graph 4 A / 12" if ea else "ALIGNNAtomWise 4+4 d=256, k-nearest 8 A / 12"
    out = dict(workload=f"{len(structs)} jittered sample structures ({sum(sizes)} atoms), {what}, "
                        f"{a.ensemble} 300 K from Maxwell-Boltzmann 300 K, 1 fs, {a.steps} steps "
                        f"({evals} evaluations per crystal)"
                        + (f", {a.pressure_bar} bar, compressibility {a.compressibility} / bar" if npt else "")
                        + (f", upper-triangular cells, ttime {a.ttime} fs, pfactor {a.pfactor}" if nh else ""),
               batched_ms=[round(v, 1) for v in ms["batched"]], batched_ms_median=round(med_b, 1),
               per_crystal_ms=[round(v, 1) for v in ms["per_crystal"]], per_crystal_ms_median=round(med_p, 1),
               speedup_median=round(med_p / med_b, 2), batched_ms_per_evaluation_split=split,
               max_position_difference_A=max(dpos),
               **{"crystals_within_1e-5_A": f"{len(structs) - len(parted)}/{len(structs)}"},
               crystals_with_a_knn_tie=sum(tied),
               parted_crystals=[dict(id=b, positions_A=round(dpos[b], 6), knn_tie=tied[b]) for b in parted],
               max_difference_on_crystals_without_a_tie_A=max([dpos[b] for b in range(len(structs)) if not tied[b]],
                                                               default=0.0),
               mean_temperature_K=dict(first=round(float(T[0].mean()), 1), last=round(float(T[-1].mean()), 1)),
               **cells_out,
               device=device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
