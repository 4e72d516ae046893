"""CPU: the ExpCellFilter restatement `oracle/cell_filter_oracle.py` -- its coordinate round trip, its forces against
finite differences of the energy at F = I on a periodic Morse pair potential (which also pins the stress sign and the
calculator's 160.21766208 conversion), both branches of its cell-force choice, a physical fixed point reached by FIRE
on the filter, the batched driver against one-by-one runs, and the C layout of the cell step's parameter struct."""
import ctypes
import os
import subprocess

import numpy as np
from scipy.linalg import expm

from alignn_b200 import _lib
from oracle import cell_filter_oracle as CF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pair_model(phi, dphi, cutoff):
    """E = 1/2 sum over atoms i, j and lattice translations R of phi(|x_j + R - x_i|) below the cutoff; returns
    evaluate(cell, X) -> (E, forces as fp32 "grad", the model's stress 160.21766208 * (1/V) dE/d(strain), fp32)."""
    def evaluate(cell, X):
        cell, X = np.asarray(cell, dtype=np.float64), np.asarray(X, dtype=np.float64)
        rec = np.linalg.inv(cell).T
        reach = [int(np.ceil(cutoff * np.linalg.norm(rec[a]))) + 1 for a in range(3)]
        shifts = np.array([(i, j, k) for i in range(-reach[0], reach[0] + 1) for j in range(-reach[1], reach[1] + 1)
                           for k in range(-reach[2], reach[2] + 1)], dtype=np.float64) @ cell
        E, F, S = 0.0, np.zeros_like(X), np.zeros((3, 3))
        for i in range(len(X)):
            d = X[None, :, :] + shifts[:, None, :] - X[i]           # [R, j, 3]
            d = d.reshape(-1, 3)
            r = np.linalg.norm(d, axis=1)
            keep = (r > 1e-9) & (r < cutoff)
            d, r = d[keep], r[keep]
            E += 0.5 * phi(r).sum()
            w = dphi(r) / r
            F[i] += (w[:, None] * d).sum(0)
            S += 0.5 * (w[:, None, None] * d[:, :, None] * d[:, None, :]).sum(0)
        V = abs(np.linalg.det(cell))
        return E, F.astype(np.float32), (CF.EV_A3_PER_GPA * S / V).astype(np.float32)
    return evaluate


def _morse(D=0.5, a=1.3, r0=2.4, cutoff=5.3):
    e = lambda r: np.exp(-a * (r - r0))                              # noqa: E731
    return _pair_model(lambda r: D * (1 - e(r)) ** 2 - D, lambda r: 2 * D * a * (1 - e(r)) * e(r), cutoff)


def _morse_crystal(seed=0, n=3):
    rng = np.random.default_rng(seed)
    cell = np.diag([3.6, 3.9, 4.2]) + rng.normal(scale=0.2, size=(3, 3))
    X = rng.random((n, 3)) @ cell
    return cell, X


def _fcc_springs(r0=2.5, k=1.0):
    return _pair_model(lambda r: 0.5 * k * (r - r0) ** 2, lambda r: k * (r - r0), 1.2 * r0)


def _fcc_cell(r0, strain):
    a = r0 * np.sqrt(2.0)
    return 0.5 * a * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]]) @ np.asarray(strain).T


def test_round_trip():
    rng = np.random.default_rng(1)
    cell, X = _morse_crystal()
    f = CF.ExpCellFilter(cell, X)
    f.C = cell @ expm(0.1 * rng.normal(size=(3, 3))).T              # some deformation away from C0
    f.X = X @ expm(0.05 * rng.normal(size=(3, 3))).T
    C, Xc = f.C.copy(), f.X.copy()
    f.set_positions(f.get_positions())
    assert np.abs(f.C - C).max() <= 1e-12 * np.abs(C).max()
    assert np.abs(f.X - Xc).max() <= 1e-12 * np.abs(Xc).max()


def test_forces_are_energy_derivatives_at_identity():
    evaluate = _morse()
    cell, X = _morse_crystal()
    n = len(X)
    E0, f, s = evaluate(cell, X)
    filt = CF.ExpCellFilter(cell, X)
    rows = filt.get_forces(f, CF.calculator_stress(s))
    assert filt.exact                                               # at F = I the exact direction is W itself

    def energy(u, L):
        Fn = expm(L)
        return evaluate(cell @ Fn.T, (X + u) @ Fn.T)[0]
    h = 1e-5
    fd = np.zeros((n + 3, 3))
    for i in range(n + 3):
        for k in range(3):
            u, L = np.zeros((n, 3)), np.zeros((3, 3))
            (u if i < n else L)[i if i < n else i - n, k] = h
            fd[i, k] = -(energy(u, L) - energy(-u, -L)) / (2 * h)
    scale = np.abs(fd).max()
    assert np.abs(rows[:n] - fd[:n]).max() <= 1e-6 * scale, (rows[:n], fd[:n])
    assert np.abs(rows[n:] - fd[n:]).max() <= 1e-6 * np.abs(fd[n:]).max(), (rows[n:], fd[n:])
    # the conversion: without the calculator's / 160.21766208 the cell rows would be that much too large
    assert np.abs(rows[n:]).max() > 0.1 * np.abs(fd[n:]).max() and np.abs(rows[n:]).max() < 10 * np.abs(fd[n:]).max()


def test_calculator_stress_is_fp32_left_to_right():
    s = np.arange(9, dtype=np.float32).reshape(3, 3) * np.float32(1.37) - np.float32(3.1)
    got = CF.calculator_stress(s, 0.7)
    assert got.dtype == np.float32
    v = np.array([s[0, 0], s[1, 1], s[2, 2], (s[1, 2] + s[2, 1]) / np.float32(2), (s[0, 2] + s[2, 0]) / np.float32(2),
                  (s[0, 1] + s[1, 0]) / np.float32(2)], dtype=np.float32)
    want = (v * np.float32(0.7)) / np.float32(160.21766208)
    assert np.array_equal(got, want)


def test_cell_force_branches():
    stress = np.array([0.02, -0.01, 0.015, 0.004, -0.006, 0.003])
    C0 = np.diag([4.0, 4.5, 5.0])
    near = expm(np.diag([0.01, -0.02, 0.015]))
    G, exact = CF.cell_forces(near, C0 @ near.T, stress)
    assert exact
    # a large preloaded shear: the exact direction turns away from the naive one and the filter falls back to W
    F = expm(np.array([[0.0, 2.5, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]]))
    G, exact = CF.cell_forces(F, C0 @ F.T, stress)
    assert not exact
    W = np.linalg.solve(F, (-abs(np.linalg.det(C0 @ F.T)) * CF.voigt_6_to_full_3x3(stress)).T).T
    assert np.array_equal(G, W)


def test_fcc_springs_relax_to_the_ideal_cell():
    """One atom in an FCC primitive cell, nearest-neighbour harmonic springs of rest length r0: from a strained and
    sheared cell the filtered FIRE ends at the ideal cell, 12 neighbours at r0 and volume r0^3 / sqrt(2), up to a free
    rotation."""
    r0 = 2.5
    evaluate = _fcc_springs(r0)
    cell = _fcc_cell(r0, [[1.04, 0.03, 0.0], [0.0, 1.04, -0.02], [0.01, 0.0, 1.04]])
    fmax = 1e-6
    res = CF.relax(evaluate, cell, np.zeros((1, 3)), fmax=fmax, steps=3000)
    assert res["converged"], res["nsteps"]
    C = res["cell"]
    nbr = [C[0], C[1], C[2], C[0] - C[1], C[0] - C[2], C[1] - C[2]]
    d = np.array([np.linalg.norm(v) for v in nbr])
    assert np.abs(d - r0).max() <= 1e-5, d
    assert abs(abs(np.linalg.det(C)) - r0 ** 3 / np.sqrt(2.0)) <= 1e-5 * r0 ** 3, np.linalg.det(C)
    assert abs(abs(np.linalg.det(cell)) - r0 ** 3 / np.sqrt(2.0)) > 0.05 * r0 ** 3   # it did move


def test_batched_oracle_equals_one_by_one_bitwise():
    """Springs crystals that converge at different steps and Morse crystals that run to the step limit."""
    springs, morse = _fcc_springs(), _morse()
    crystals = [(_fcc_cell(2.5, np.diag([1.04, 1.0, 0.98]) + 0.02), np.zeros((1, 3)), springs),
                _morse_crystal(seed=1, n=3) + (morse,),
                (_fcc_cell(2.5, np.eye(3) * 1.08), np.zeros((1, 3)), springs),
                _morse_crystal(seed=2, n=2) + (morse,)]
    fmax, steps, mult = 0.02, 40, 1.5
    alone = [CF.relax(ev, c, x, fmax=fmax, steps=steps, force_multiplier=mult, stress_wt=0.9) for c, x, ev in crystals]
    assert len({r["nsteps"] for r in alone}) > 2 and any(r["converged"] for r in alone)

    def evaluate_batch(ids, cx):
        return [crystals[b][2](c, x) for b, (c, x) in zip(ids, cx)]
    bat = CF.relax_batch(evaluate_batch, [(c, x) for c, x, _ in crystals], fmax=fmax, steps=steps, force_multiplier=mult,
                         stress_wt=0.9)
    for b, r in enumerate(alone):
        assert bat["nsteps"][b] == r["nsteps"] and bat["converged"][b] == r["converged"]
        assert bat["evaluations"][b] == r["evaluations"]
        assert np.array_equal(bat["positions"][b], r["positions"]) and np.array_equal(bat["cell"][b], r["cell"])
        assert np.array_equal(bat["forces"][b], r["forces"]) and np.array_equal(bat["stress"][b], r["stress"])
        assert bat["energy"][b] == r["energy"]
        assert np.array_equal(bat["fire"][b].v, r["fire"].v)
    assert any(np.abs(r["cell"] - c).max() > 1e-2 for r, (c, _, _) in zip(alone, crystals))


def test_fire_cell_params_struct_matches_c_layout(tmp_path):
    fire = [f for f, _ in _lib.FireParams._fields_]
    src = tmp_path / "fp.c"
    offs = ["offsetof(alignn_b200_fire_cell_params, stress_wt)"] + [f"offsetof(alignn_b200_fire_cell_params, fire.{f})"
                                                                      for f in fire]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\nint main(){printf("%zu'
                   + " %zu" * len(offs) + '\\n", sizeof(alignn_b200_fire_cell_params), ' + ", ".join(offs)
                   + ");return 0;}\n")
    exe = tmp_path / "fp"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    base = _lib.FireCellParams.fire.offset
    want = [ctypes.sizeof(_lib.FireCellParams), _lib.FireCellParams.stress_wt.offset]
    want += [base + getattr(_lib.FireParams, f).offset for f in fire]
    assert got == want


def test_knn_cut_tie_detection():
    """A simple cubic cell: 6 first neighbours at a, 12 second at a sqrt(2); the cut after 4 neighbours splits the first
    shell (a tie), the cuts after 6 and 18 fall between shells."""
    from alignn_b200 import neighbors
    lat, X = np.eye(3) * 3.0, np.zeros((1, 3))
    assert neighbors.knn_cut_is_tied(lat, X, max_neighbors=4)
    assert not neighbors.knn_cut_is_tied(lat, X, max_neighbors=6)
    assert not neighbors.knn_cut_is_tied(lat, X, max_neighbors=18)
    assert neighbors.knn_cut_is_tied(lat, X, max_neighbors=12)
    # an oblique cell: the images x + R and x - R still tie wherever the cut splits them
    rng = np.random.default_rng(0)
    lat = np.eye(3) * 3.0 + rng.normal(scale=0.3, size=(3, 3))
    assert neighbors.knn_cut_is_tied(lat, X, max_neighbors=1)
    assert not neighbors.knn_cut_is_tied(lat, X, max_neighbors=2)
