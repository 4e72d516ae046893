"""Authoring-time script: writes tests/golden/sample_structures.npz from the 70 POSCAR files of the reference's
`alignn/examples/sample_data/` (JARVIS-DFT structures, 1-64 atoms).  Run once by hand with the reference checkout:

    python oracle/make_sample_structures.py /path/to/alignn/alignn/examples/sample_data

The npz is data only (what the GPU tests and tools/bench_crystal_graphs.py read):
  ids [S] str, lattices [S,3,3] f64 (row vectors), atom_offsets [S+1] i64, cart_coords [N,3] f64 (= frac @ lattice, as
  jarvis' `Atoms.cart_coords` computes it for a "direct" POSCAR), frac_coords [N,3] f64, symbols [N] str.
"""
import glob
import os
import sys

import numpy as np


def read_poscar(path):
    lines = [ln.strip() for ln in open(path).read().splitlines()]
    scale = float(lines[1].split()[0])
    lat = np.array([[float(x) for x in lines[i].split()[:3]] for i in (2, 3, 4)]) * scale
    species = lines[5].split()
    counts = [int(x) for x in lines[6].split()]
    row = 7
    if lines[row][0] in "sS":                     # selective dynamics
        row += 1
    direct = lines[row][0] in "dD"
    row += 1
    n = sum(counts)
    xyz = np.array([[float(x) for x in lines[row + i].split()[:3]] for i in range(n)])
    frac = xyz if direct else (xyz * scale) @ np.linalg.inv(lat)
    symbols = [s for s, c in zip(species, counts) for _ in range(c)]
    return lat, frac, symbols


def main(src):
    paths = sorted(glob.glob(os.path.join(src, "POSCAR-*.vasp")))
    ids, lats, fracs, syms = [], [], [], []
    for p in paths:
        lat, frac, s = read_poscar(p)
        ids.append(os.path.basename(p)[len("POSCAR-"):-len(".vasp")])
        lats.append(lat)
        fracs.append(frac)
        syms += s
    frac = np.concatenate(fracs)
    offsets = np.zeros(len(paths) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([f.shape[0] for f in fracs])
    cart = np.concatenate([f @ lat for f, lat in zip(fracs, lats)])
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sample_structures.npz")
    np.savez_compressed(out, ids=np.array(ids), lattices=np.stack(lats), atom_offsets=offsets, cart_coords=cart,
                        frac_coords=frac, symbols=np.array(syms))
    sizes = np.diff(offsets)
    print(f"{out}: {len(paths)} structures, {sizes.min()}-{sizes.max()} atoms (mean {sizes.mean():.1f})")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "alignn/examples/sample_data")
