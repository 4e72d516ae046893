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

--optimizer LBFGS or BFGS runs that optimizer in both arms (the per-crystal arm runs oracle/qn_oracle.py's), and
times its kernels alone on the batch: the LBFGS step with a full 100-pair history, and BFGS's update, torch.linalg.eigh
and apply, so that the share taken by eigh is stated.

    python tools/bench_relax.py [--structures 64] [--steps 10] [--seed 0] [--optimize-lattice] [--optimizer FIRE]
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


def qn_kernels_alone(optimizer, sizes, cell, dev, reps=20):
    """CUDA-event times of one quasi-Newton step's kernels on the whole batch, on scripted forces (no model): the LBFGS
    step with a full 100-pair history, or BFGS's update, eigh of every H and apply, each on its own."""
    from alignn_b200 import neighbors, ops
    from alignn_b200.relax import _QuasiNewton
    B, aoff = len(sizes), neighbors.ragged_offsets(sizes)
    N = int(aoff[-1])
    g = torch.randn(N, 3, device=dev) * 0.1
    st = torch.randn(B, 3, 3, device=dev) * 0.01 if cell else None
    aoff_d = torch.from_numpy(aoff).to(dev)
    act = torch.arange(B, dtype=torch.int32, device=dev)
    boff = aoff_d.to(torch.int32)
    pos = torch.randn(N, 3, device=dev, dtype=torch.float64)
    forces = torch.zeros(N, 3, device=dev)
    cops = (None,) * 6
    if cell:
        C0 = torch.eye(3, dtype=torch.float64, device=dev).repeat(B, 1, 1) * 6.0
        cops = (C0, torch.zeros_like(C0), torch.eye(3, dtype=torch.float64, device=dev).repeat(B, 1, 1), C0.clone(),
                torch.zeros_like(C0), torch.zeros(B, 6, device=dev))
    kw = dict(fmax=0.0, steps=10 ** 6, force_multiplier=1.0, stress_wt=1.0)
    q = _QuasiNewton(optimizer, sizes, aoff, 10 ** 6, cell, dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1) / reps, 4)
    if optimizer == "LBFGS":
        # forces that change every step, so that no y.s is zero: precomputed, so that the timed loop is the kernel
        grads = [g + 1e-3 * torch.randn_like(g) for _ in range(101 + reps + 1)]
        it = iter(grads)

        def step():
            ops.lbfgs_step(next(it), st, act, boff, aoff_d, pos, forces, *cops, q.r0, q.f0, q.work, q.s_ring, q.y_ring,
                           q.history, q.istate, **kw)
        for _ in range(100):                                   # fill the 100-pair history
            step()
        out = {"lbfgs_step_full_history": timed(step)}
        out["crystals_still_running"] = int((q.istate[:, 3] == 0).sum())   # every timed step ran on all of them
        return out
    q.step(g, st, act, list(range(B)), boff, aoff_d, pos, forces, cops, kw)
    max_dim = max(q.dims)
    groups = {}
    for b in range(B):
        groups.setdefault(q.dims[b], []).append(b)
    blocks = []
    for d, ids in groups.items():
        base = torch.from_numpy(q.h_off[ids]).to(dev)
        blocks.append((d, ids, base.unsqueeze(1) + torch.arange(d * d, device=dev).unsqueeze(0),
                       torch.tensor(ids, dtype=torch.int32, device=dev)))
    eig = {}

    def update():
        ops.bfgs_update(g, st, act, boff, aoff_d, pos, forces, *cops, q.h_off_d, q.H, q.r0, q.f0, q.r, q.f, q.work,
                        q.istate, max_dim=max_dim, **kw)

    def eigh():
        for d, ids, idx, _ in blocks:
            eig[d] = torch.linalg.eigh(q.H[idx].view(len(ids), d, d))

    def apply():
        for d, ids, _, gid in blocks:
            omega, V = eig[d]
            ops.bfgs_apply(gid, omega.contiguous(), V.contiguous(), aoff_d, pos, *cops[:4], q.r0, q.f0, q.r, q.f, q.work,
                           q.istate, cell=cell)
    eigh()
    out = {"bfgs_update": timed(update), "eigh_all_groups": timed(eigh), "bfgs_apply": timed(apply),
           "size_groups": len(blocks)}
    out["eigh_share"] = round(out["eigh_all_groups"] / (out["bfgs_update"] + out["eigh_all_groups"] + out["bfgs_apply"]), 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--structures", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--optimize-lattice", action="store_true", help="relax the cells too (ExpCellFilter)")
    ap.add_argument("--optimizer", choices=("FIRE", "LBFGS", "BFGS"), default="FIRE")
    ap.add_argument("--model", choices=("alignn_atomwise", "ealignn"), default="alignn_atomwise",
                    help="ealignn: a 2+2, d=64 eALIGNNAtomWise on radius_graph 4 A / 12 (the reference's eALIGNN example "
                         "config); the host arm builds each crystal's graph with crystal_graphs_device")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_relax.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from alignn_b200 import neighbors, ops, relax_structures
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    from alignn_b200.ealignn_atomwise import eALIGNNAtomWise, eALIGNNAtomWiseConfig
    from oracle import cell_filter_oracle as CF
    from oracle import fire_oracle as FO
    from oracle import qn_oracle as QN

    dev = torch.device("cuda:0")
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    rng = np.random.default_rng(a.seed)
    pool = np.arange(len(z["ids"]))
    if a.model == "ealignn":
        # a crystal whose filtered graph keeps no bond cannot run alone (the one-crystal forward has no edges)
        pool = np.array([i for i in pool if _kept_bonds(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]], dev) >= 2 * (off[i + 1] - off[i])])
    pick = rng.choice(pool, min(a.structures, len(pool)), replace=False)
    structs = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]] + rng.normal(scale=0.03, size=(off[i + 1] - off[i], 3)))
               for i in pick]
    sizes = [x.shape[0] for _, x in structs]
    feats = torch.from_numpy(rng.normal(size=(sum(sizes), 92)).astype(np.float32)).to(dev)
    cell = a.optimize_lattice
    # FIRE runs every crystal to the step limit at fmax = 0.  A quasi-Newton step on forces that are exactly zero (a
    # one-atom crystal in a fixed cell) would leave y.s = 0 on the next step, so those stop at fmax = 1e-6 instead.
    fmax = 0.0 if a.optimizer == "FIRE" else 1e-6
    if cell:                                                   # strained, sheared cells, the atoms moved with them
        srng = np.random.default_rng(a.seed + 1)
        Ds = [np.eye(3) + np.diag(srng.uniform(-0.04, 0.04, 3)) + srng.uniform(-0.03, 0.03, (3, 3)) for _ in structs]
        structs = [(lat @ D.T, X @ D.T) for (lat, X), D in zip(structs, Ds)]
    torch.manual_seed(1)
    ea = a.model == "ealignn"
    if ea:
        model = eALIGNNAtomWise(eALIGNNAtomWiseConfig(name="ealignn_atomwise", atom_input_features=92,
                                                      stresswise_weight=1.0 if cell else 0.0)).to(dev).eval()
        graph = dict(neighbor_strategy="radius_graph", cutoff=4.0, max_neighbors=12)
    else:
        cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                                   atom_input_features=92, gradwise_weight=1.0, stresswise_weight=1.0 if cell else 0.0)
        model = ALIGNNAtomWise(cfg).to(dev).eval()
        graph = dict(neighbor_strategy="k-nearest", cutoff=8.0, max_neighbors=12)

    def one_crystal(c, x, f_b):
        """(g, lg, lat) of one crystal as the calculator builds it: on the host for ALIGNNAtomWise; on the device for
        eALIGNN, which needs the graph's frac_coords and images"""
        if ea:
            return neighbors.crystal_graphs_device([(c, x)], f_b.to(dev), device=dev, **graph)
        g, lg = neighbors.crystal_graph(c, x, f_b, **graph)
        g.ndata["V"] = torch.full((x.shape[0],), abs(float(np.dot(np.cross(c[0], c[1]), c[2]))), dtype=torch.float32)
        return g.to(dev), lg.to(dev), torch.tensor(c, dtype=torch.float32).view(1, 3, 3).to(dev)

    def batched():
        r = relax_structures(model, structs, feats, fmax=fmax, steps=a.steps, optimize_lattice=cell, optimizer=a.optimizer,
                             **graph)
        torch.cuda.synchronize()
        return r

    visited = []                                               # per crystal: every (cell, x) the host arm evaluated

    def per_crystal():
        out, o = [], 0
        visited.clear()
        for lat, X in structs:
            n = X.shape[0]
            f_b = feats[o:o + n].cpu()

            def evaluate(x, lat=lat, f_b=f_b, n=n):
                res = model(one_crystal(lat, x, f_b))
                return float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy()

            seen = []
            visited.append(seen)

            def evaluate_cell(c, x, f_b=f_b, n=n, seen=seen):
                seen.append((c, x))
                res = model(one_crystal(c, x, f_b))
                return (float(res["out"].detach() * n), res["grad"].detach().reshape(-1, 3).cpu().numpy(),
                        res["stresses"].detach().reshape(3, 3).cpu().numpy())
            if a.optimizer != "FIRE":
                if cell:
                    out.append(QN.relax_cell(a.optimizer, evaluate_cell, lat, X, fmax=fmax, steps=a.steps))
                else:
                    out.append(QN.relax(a.optimizer, evaluate, X, fmax=fmax, steps=a.steps))
            elif cell:
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
    if a.optimizer == "FIRE":
        assert got.nsteps.tolist() == [a.steps] * len(structs) and all(r["nsteps"] == a.steps for r in ref)
    extra = {}
    if not cell and a.optimizer == "FIRE":
        assert dmax <= 1e-5, f"the arms end {dmax} A apart"
    elif not cell:
        # reported, not asserted: the quasi-Newton updates divide by differences of consecutive forces, which amplify
        # the fp32 differences between the host and the device graph's edge order
        dpos = [float(np.abs(P[aoff[b]:aoff[b + 1]] - r["positions"]).max()) for b, r in enumerate(ref)]
        extra = {"crystals_within_1e-5_A": f"{sum(d <= 1e-5 for d in dpos)}/{len(structs)}",
                 "nsteps_batched": int(got.nsteps.sum()), "nsteps_per_crystal": sum(r["nsteps"] for r in ref)}
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
        tied = [not ea and any(neighbors.knn_cut_is_tied(c, x) for c, x in seen) for seen in visited]
        parted = [b for b in range(len(structs)) if dpos[b] > 1e-5 or dcell[b] > 1e-5]
        extra = {"max_cell_difference_A": max(dcell), "crystals_within_1e-5_A": f"{agree}/{len(structs)}",
                 "crystals_with_a_knn_tie": sum(tied),
                 "parted_crystals": [dict(id=b, positions_A=round(dpos[b], 4), cell_A=round(dcell[b], 4), knn_tie=tied[b])
                                     for b in parted],
                 "every_parted_crystal_has_a_knn_tie": all(tied[b] for b in parted),
                 "max_difference_on_crystals_without_a_tie_A": max([max(dpos[b], dcell[b]) for b in range(len(structs))
                                                                    if not tied[b]], default=0.0),
                 "max_cell_change_A": round(moved, 4),
                 "nsteps_batched": int(got.nsteps.sum()), "nsteps_per_crystal": sum(r["nsteps"] for r in ref)}
    ops.TIMER = ops.KernelTimer()
    try:
        batched()
        summ = ops.TIMER.summary()
    finally:
        ops.TIMER = None
    evals = int(got.nsteps.max()) + 1
    split = {k[len("relax_"):]: round(summ[k]["total_ms"] / evals, 3) for k in summ if k.startswith("relax_")}
    med_b, med_p = statistics.median(ms["batched"]), statistics.median(ms["per_crystal"])
    what = f"ExpCellFilter {a.optimizer} on atoms and strained, sheared cells" if cell else a.optimizer
    if a.optimizer != "FIRE":
        extra["kernels_alone_ms"] = qn_kernels_alone(a.optimizer, sizes, cell, dev)
    model_s = "eALIGNNAtomWise 2+2 d=64, radius_graph 4 A / 12" if ea else "ALIGNNAtomWise 4+4 d=256, k-nearest 8 A / 12"
    out = dict(workload=f"{len(structs)} jittered sample structures ({sum(sizes)} atoms), {model_s}, "
                        f"fmax={fmax}, at most {a.steps} {what} steps",
               batched_ms=[round(v, 1) for v in ms["batched"]], batched_ms_median=round(med_b, 1),
               per_crystal_ms=[round(v, 1) for v in ms["per_crystal"]], per_crystal_ms_median=round(med_p, 1),
               speedup_median=round(med_p / med_b, 2), batched_ms_per_evaluation_split=split,
               max_position_difference_A=dmax, **extra, device=device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
