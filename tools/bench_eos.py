#!/usr/bin/env python
"""Batched E(V) curves and equation-of-state fits: `ev_curve` against the reference's architecture, one strained
structure at a time, and the fit kernel alone against scipy.

Workload: 64 structures drawn with a seed from tests/golden/sample_structures.npz, at the reference's 10 strains
(np.arange(-0.05, 0.05, 0.01)), the 4 + 4, d = 256, 92-feature ALIGNNAtomWise of tools/bench_relax.py (seeded
weights, eval mode), k-nearest graphs (8 A, 12 neighbours), the Murnaghan form.

  batched:     ev_curve -- all 640 strained copies through the device graph builder and the model in chunks of at
               most max_batch_atoms atoms, then one fit launch;
  per-crystal: what the reference's `ev_curve` runs: per strained copy neighbors.crystal_graph on the host, .to("cuda")
               and the same model on a one-crystal batch, then oracle/eos_oracle.py's restatement of ASE's
               EquationOfState.fit with scipy, per crystal.

Each arm runs three times (alternating); the median wall time (ending in a synchronise) is reported, with the largest
parameter differences between the arms over the crystals both fit with status 0.  The fit alone: `fit_eos` on
--fit-rows random Murnaghan rows of 10 points (oracle/eos_oracle.py's random_rows), median of three, against the
oracle's scipy loop on the first --scipy-rows of them, reported as measured on that subset.  The device name, power
limit and SM clock limit are read in the same run.

    python tools/bench_eos.py [--structures 64] [--fit-rows 65536] [--scipy-rows 2048] [--seed 0]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_phonons import device_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--structures", type=int, default=64)
    ap.add_argument("--fit-rows", type=int, default=65536)
    ap.add_argument("--scipy-rows", type=int, default=2048)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eos.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from alignn_b200 import ev_curve, fit_eos, neighbors
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    from alignn_b200.eos import DEFAULT_STRAINS, strained
    from oracle import eos_oracle as EO

    dev = torch.device("cuda:0")
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    rng = np.random.default_rng(a.seed)
    pick = rng.choice(len(off) - 1, min(a.structures, len(off) - 1), replace=False)
    structs = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]]) for i in pick]
    sizes = [x.shape[0] for _, x in structs]
    aoff = np.concatenate([[0], np.cumsum(sizes)])
    feats = torch.from_numpy(rng.normal(size=(sum(sizes), 92)).astype(np.float32)).to(dev)
    torch.manual_seed(1)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                               atom_input_features=92, gradwise_weight=1.0, stresswise_weight=0.0)
    model = ALIGNNAtomWise(cfg).to(dev).eval()
    S = len(DEFAULT_STRAINS)

    def batched():
        r = ev_curve(model, structs, feats)
        torch.cuda.synchronize()
        return r

    def per_crystal():
        params, status, energies = [], [], []
        for b, (lat, X) in enumerate(structs):
            f = feats[aoff[b]:aoff[b + 1]].cpu()
            vol, y = [], []
            for s in DEFAULT_STRAINS:
                lat_s, x_s, v = strained(lat, X, s)
                g, lg = neighbors.crystal_graph(lat_s, x_s, f, cutoff=8.0, neighbor_strategy="k-nearest",
                                                max_neighbors=12)
                res = model((g.to(dev), lg.to(dev), torch.tensor(lat_s, dtype=torch.float32).view(1, 3, 3).to(dev)))
                y.append(float((res["out"].detach().reshape(-1) * float(X.shape[0])).cpu().numpy()[0]))
                res["grad"].detach().cpu()                          # unrelaxed_atoms reads the forces too
                vol.append(v)
            p, st = EO.fit_rows(np.array(vol)[None], np.array(y)[None], "murnaghan")
            params.append(p[0])
            status.append(st[0])
            energies.append(y)
        torch.cuda.synchronize()
        return np.array(params), np.array(status), np.array(energies)

    batched()                                                    # warm-up: module loads, allocator, every shape
    per_crystal()
    ms = {"batched": [], "per_crystal": []}
    res = {}
    for _ in range(3):
        for name, fn in (("batched", batched), ("per_crystal", per_crystal)):
            t = time.perf_counter()
            res[name] = fn()
            ms[name].append((time.perf_counter() - t) * 1e3)
    got = res["batched"]
    P_ref, st_ref, E_ref = res["per_crystal"]
    P = torch.stack([got.e0, got.bulk_modulus, got.bp, got.v0], 1).cpu().numpy()
    st = got.status.cpu().numpy()
    both = (st == 0) & (st_ref == 0)
    dP = (np.abs(P[both] - P_ref[both]) / np.abs(P_ref[both])).max(0) if both.any() else np.full(4, np.nan)
    dE = float((np.abs(got.energies.cpu().numpy() - E_ref) / np.abs(E_ref)).max())

    # ---- the fit alone
    V, E, _ = EO.random_rows("murnaghan", a.fit_rows, S, seed=a.seed)
    v_d, e_d = torch.from_numpy(V).to(dev), torch.from_numpy(E).to(dev)
    fit_eos(v_d, e_d)
    torch.cuda.synchronize()
    fit_ms = []
    for _ in range(3):
        t = time.perf_counter()
        fit = fit_eos(v_d, e_d)
        torch.cuda.synchronize()
        fit_ms.append((time.perf_counter() - t) * 1e3)
    k = min(a.scipy_rows, a.fit_rows)
    t = time.perf_counter()
    P_sc, st_sc = EO.fit_rows(V[:k], E[:k], "murnaghan")
    scipy_ms = (time.perf_counter() - t) * 1e3
    Pf = torch.stack([fit.e0, fit.bulk_modulus, fit.bp, fit.v0], 1)[:k].cpu().numpy()
    ok = (st_sc == 0) & (fit.status[:k].cpu().numpy() == 0)
    dF = (np.abs(Pf[ok] - P_sc[ok]) / np.abs(P_sc[ok])).max(0)

    med_b, med_p = statistics.median(ms["batched"]), statistics.median(ms["per_crystal"])
    out = dict(workload=f"{len(structs)} sample structures ({sum(sizes)} atoms) x {S} strains, ALIGNNAtomWise 4+4 "
                        "d=256, k-nearest 8 A / 12, Murnaghan",
               batched_ms=[round(v, 1) for v in ms["batched"]], batched_ms_median=round(med_b, 1),
               per_crystal_ms=[round(v, 1) for v in ms["per_crystal"]], per_crystal_ms_median=round(med_p, 1),
               speedup_median=round(med_p / med_b, 2),
               statuses_batched=np.bincount(st, minlength=4).tolist(),
               statuses_per_crystal=np.bincount(st_ref, minlength=4).tolist(),
               status_agreement=int((st == st_ref).sum()),
               max_energy_difference_rel=dE,
               max_param_difference_rel_E0_B0_BP_V0=[float(x) for x in dP], crystals_compared=int(both.sum()),
               fit_rows=a.fit_rows, fit_points=S, fit_ms=[round(v, 3) for v in fit_ms],
               fit_ms_median=round(statistics.median(fit_ms), 3),
               fit_statuses=np.bincount(fit.status.cpu().numpy(), minlength=4).tolist(),
               scipy_rows=k, scipy_ms=round(scipy_ms, 1),
               scipy_vs_kernel_max_rel_E0_B0_BP_V0=[float(x) for x in dF],
               device=device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
