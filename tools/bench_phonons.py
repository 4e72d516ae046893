#!/usr/bin/env python
"""Batched phonons: `phonons` against the reference's architecture, one supercell at a time.

Workload: the sample structures of tests/golden/sample_structures.npz with at most `--max-atoms` atoms (38 at 8), the
4 + 4, d = 256, 92-feature ALIGNNAtomWise of tools/bench_relax.py (seeded weights, eval mode), k-nearest graphs (8 A,
12 neighbours), supercell (2, 2, 2), delta 0.01 A, a 100-point q-list per crystal (Gamma-X-M-Gamma-R in fractional
coordinates of its cell), and the reference's DOS: a (20, 20, 20) mesh sampled on 100 points with width 1e-3 eV.
Masses are seeded random values in [1, 200] amu.

  batched:     phonons -- every displaced supercell through the device graph builder and the model in chunks of at most
               max_batch_atoms atoms, one force-constant launch, the dynamical-matrix kernel and torch's eigvalsh in
               blocks, the DOS in torch;
  per-crystal: what `ase_phonon` runs: for each crystal the undisplaced supercell (which ASE evaluates and never reads)
               and its 6n displaced supercells, each through neighbors.crystal_graph on the host, .to("cuda") and the
               same model on a one-crystal batch, then the numpy post-processing of oracle/phonon_oracle.py.

Each arm runs three times (alternating); the median wall time (ending in a synchronise) is reported.  One more batched
run with CUDA events gives the per-span split (each span from its first enqueue to its last, host work inside it
included), and a sweep over max_batch_atoms gives the wall time and peak allocated memory of each chunk size.  The
largest differences between the arms' force constants and band omega^2 are reported, with the kernel names torch's
eigvalsh launches for these shapes and the device name, power limit and SM clock limit, read in the same run.

    python tools/bench_phonons.py [--max-atoms 8] [--seed 0]
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


def qpath(points=100):
    """Gamma-X-M-Gamma-R, `points` fractional q-points."""
    corners = np.array([[0, 0, 0], [0.5, 0, 0], [0.5, 0.5, 0], [0, 0, 0], [0.5, 0.5, 0.5]], dtype=np.float64)
    t = np.linspace(0.0, len(corners) - 1, points)
    i = np.minimum(t.astype(int), len(corners) - 2)
    return corners[i] + (t - i)[:, None] * (corners[i + 1] - corners[i])


def eig_kernels(dev, M, count):
    """Names of the CUDA kernels torch.linalg.eigvalsh launches on [count, M, M] complex128."""
    a = torch.randn(count, M, M, dtype=torch.complex128, device=dev)
    a = a + a.transpose(1, 2).conj()
    torch.linalg.eigvalsh(a, UPLO="U")
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.linalg.eigvalsh(a, UPLO="U")
        torch.cuda.synchronize()
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    return [n[:80] for n in names][:8]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--max-atoms", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_phonons.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    from alignn_b200 import neighbors, ops, phonons
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    from alignn_b200.phonons import DEFAULT_MAX_BATCH_ATOMS, displaced_supercells
    from oracle import phonon_oracle as PO
    from oracle.fire_oracle import scaled_forces

    dev = torch.device("cuda:0")
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    pick = [i for i in range(len(off) - 1) if off[i + 1] - off[i] <= a.max_atoms]
    structs = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]]) for i in pick]
    sizes = [x.shape[0] for _, x in structs]
    aoff = np.concatenate([[0], np.cumsum(sizes)])
    rng = np.random.default_rng(a.seed)
    feats = torch.from_numpy(rng.normal(size=(sum(sizes), 92)).astype(np.float32)).to(dev)
    masses = rng.uniform(1.0, 200.0, sum(sizes))
    torch.manual_seed(1)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                               atom_input_features=92, gradwise_weight=1.0, stresswise_weight=0.0)
    model = ALIGNNAtomWise(cfg).to(dev).eval()
    N, delta, kpts, npts, width = (2, 2, 2), 0.01, (20, 20, 20), 100, 1e-3
    q = [qpath(100) for _ in structs]
    Nc = int(np.prod(N))

    def batched(max_batch_atoms=DEFAULT_MAX_BATCH_ATOMS):
        r = phonons(model, structs, feats, masses, supercell=N, delta=delta, qpoints=q, dos_kpts=kpts, dos_npts=npts,
                    dos_width=width, max_batch_atoms=max_batch_atoms)
        torch.cuda.synchronize()
        return r

    def per_crystal():
        out = []
        for b, (lat, X) in enumerate(structs):
            sl = slice(aoff[b], aoff[b + 1])
            tiled = feats[sl].cpu().repeat(Nc, 1)
            latN, disp = displaced_supercells(lat, X, N, delta)
            lat_t = torch.tensor(latN, dtype=torch.float32).view(1, 3, 3).to(dev)
            x0 = PO.supercell(lat, X, N)[1]
            forces = []
            for x in [x0] + list(disp):                           # ASE evaluates the undisplaced supercell too
                g, lg = neighbors.crystal_graph(latN, x, tiled, cutoff=8.0, neighbor_strategy="k-nearest",
                                                max_neighbors=12)
                res = model((g.to(dev), lg.to(dev), lat_t))
                forces.append(scaled_forces(res["grad"].detach().reshape(-1, 3).cpu().numpy(), 1.0))
            f = np.stack(forces[1:]).astype(np.float64)
            out.append(PO.postprocess(f, masses[sl], N, delta, qpoints=q[b], dos_kpts=kpts, dos_npts=npts,
                                      dos_width=width))
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
    dC = max(float(np.abs(got.force_constants[b].cpu().numpy() - r["C_N"]).max() / np.abs(r["C_N"]).max())
             for b, r in enumerate(ref))
    dW = max(float(np.abs(np.sign(e) * (e / PO.EV_PER_SQRT_EV_A2_AMU) ** 2 - r["omega2"]).max()
                   / np.abs(r["omega2"]).max())
             for e, r in zip((x.cpu().numpy() for x in got.band_energies), ref))
    dD = max(float(np.abs(got.dos_weights[b].cpu().numpy() - r["dos_weights"]).max() / np.abs(r["dos_weights"]).max())
             for b, r in enumerate(ref))
    ops.TIMER = ops.KernelTimer()
    try:
        batched()
        summ = ops.TIMER.summary()
    finally:
        ops.TIMER = None
    split = {k[len("phonon_"):]: round(summ[k]["total_ms"], 1) for k in summ if k.startswith("phonon_")}
    sweep = {}
    for mba in sorted({4096, 8192, DEFAULT_MAX_BATCH_ATOMS, 32768}):
        torch.cuda.reset_peak_memory_stats()
        t = time.perf_counter()
        try:
            batched(mba)
        except torch.OutOfMemoryError:
            sweep[mba] = "out of memory"
            torch.cuda.empty_cache()
            continue
        sweep[mba] = dict(ms=round((time.perf_counter() - t) * 1e3, 1),
                          peak_allocated_GB=round(torch.cuda.max_memory_allocated() / 1e9, 2))
    med_b, med_p = statistics.median(ms["batched"]), statistics.median(ms["per_crystal"])
    supercells = sum(6 * n for n in sizes)
    out = dict(workload=f"{len(structs)} sample structures with <= {a.max_atoms} atoms ({sum(sizes)} atoms), supercell "
                        f"{N}, {supercells} displaced supercells ({sum(6 * n * Nc * n for n in sizes)} atoms), "
                        f"ALIGNNAtomWise 4+4 d=256, k-nearest 8 A / 12, 100 q-points per crystal, DOS {kpts} "
                        f"{npts} points width {width}",
               batched_ms=[round(v, 1) for v in ms["batched"]], batched_ms_median=round(med_b, 1),
               per_crystal_ms=[round(v, 1) for v in ms["per_crystal"]], per_crystal_ms_median=round(med_p, 1),
               speedup_median=round(med_p / med_b, 2), batched_span_ms=split,
               max_batch_atoms_sweep=sweep, default_max_batch_atoms=DEFAULT_MAX_BATCH_ATOMS,
               max_force_constant_difference_rel=dC, max_band_omega2_difference_rel=dW,
               max_dos_weight_difference_rel=dD,
               eigvalsh_kernels={"M=24 x 8100": eig_kernels(dev, 24, 8100), "M=36 x 64": eig_kernels(dev, 36, 64)},
               device=device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
