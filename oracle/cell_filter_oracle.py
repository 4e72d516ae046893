"""numpy/scipy restatement of the reference's default relaxation, `ForceField.optimize_atoms(optimizer="FIRE",
optimize_lattice=True)` (alignn/ff/ff.py:373-417): ASE 3.22.1's `ExpCellFilter` around the atoms (ff.py:400-401),
FIRE run on the filter, the calculator's forces and Voigt stress (alignn/ff/calculators.py:309-311, 328-346).  The
specification `alignn_b200.relax_structures(optimize_lattice=True)` and the kernel `alignn_b200_fire_cell_step` are
tested against.

ASE sources restated (ase 3.22.1, ase/constraints.py), with the defaults the reference passes (mask all ones, no
hydrostatic strain, no constant volume, scalar_pressure = 0; ExpCellFilter forces cell_factor = 1.0, with which
expm of the cell rows is the deformation gradient):
  UnitCellFilter.deform_grad     F = solve(C0, C).T                      (C0 the cell when the filter was made)
  ExpCellFilter.get_positions    rows [:n] = solve(F, X.T).T, rows [n:] = logm(F)
  ExpCellFilter.set_positions    Fn = expm(P[n:]); cell = C0 @ Fn.T; X = P[:n] @ Fn.T
  ExpCellFilter.get_forces       W = -V voigt_6_to_full_3x3(s); W = solve(F, W.T).T; atom rows f @ F; cell rows the
                                 symmetrised -expm(Y)[0:3, 3:6], Y = [[L, -W expm(-L)], [0, L]], or W itself (the
                                 "naive" direction) when the two are neither all close nor aligned (cosine > 0.8)
  Optimizer.converged            max over all n + 3 rows of |row|^2 < fmax^2
This file was written from those sources; the block above is what tests/test_cell_filter_oracle.py checks
independently (round trip, finite differences of the energy at F = I, a physical fixed point).

The cell rows are ASE's search direction: they equal the exact gradient -dE/dlog F only at F = I.

Conventions, beyond those of oracle/fire_oracle.py:
  * the calculator's stress is full_3x3_to_voigt_6_stress of the model's fp32 [3,3] stress, times stress_wt, divided
    by 160.21766208, all in fp32 left to right (calculator_stress); the filter widens it to float64.  ASE under numpy
    1.x rounds `-volume * stress` to float32; that is not reproduced (like the fp32 roundings of fire_oracle.py).
  * the reference's `example_print` replaces `self.atoms` with the unwrapped atoms every step, so what it returns is
    the final cell, Cartesian positions, energy and the plain Cartesian forces f -- not the filter's rows.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import expm, logm

from . import fire_oracle as FO

EV_A3_PER_GPA = 160.21766208   # the calculator's conversion of the model's stress (calculators.py:340)


def calculator_stress(model_stress, stress_wt: float = 1.0) -> np.ndarray:
    """calculators.py:328-346: fp32 Voigt (xx, yy, zz, yz, xz, xy) of the model's [3,3] stress, * stress_wt /
    160.21766208, in fp32 left to right."""
    s = np.asarray(model_stress, dtype=np.float32).reshape(3, 3)
    v = np.array([s[0, 0], s[1, 1], s[2, 2], (s[1, 2] + s[2, 1]) / np.float32(2), (s[0, 2] + s[2, 0]) / np.float32(2),
                  (s[0, 1] + s[1, 0]) / np.float32(2)], dtype=np.float32)
    return v * np.float32(stress_wt) / np.float32(EV_A3_PER_GPA)


def voigt_6_to_full_3x3(s) -> np.ndarray:
    xx, yy, zz, yz, xz, xy = np.asarray(s, dtype=np.float64)
    return np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]])


def cell_forces(F, C, stress) -> tuple[np.ndarray, bool]:
    """ExpCellFilter.get_forces, cell rows: (G or W, True when the exact direction G is taken)."""
    V = abs(np.linalg.det(C))
    W = -V * voigt_6_to_full_3x3(stress)
    W = np.linalg.solve(F, W.T).T
    L = logm(F)
    Y = np.zeros((6, 6))
    Y[0:3, 0:3] = L
    Y[3:6, 3:6] = L
    Y[0:3, 3:6] = -W @ expm(-L)
    G = -expm(Y)[0:3, 3:6]
    for i, j in ((0, 1), (0, 2), (1, 2)):
        G[i, j] = G[j, i] = 0.5 * (G[i, j] + G[j, i])
    with np.errstate(invalid="ignore", divide="ignore"):
        cos = np.sum(G * W) / np.sqrt(np.sum(G ** 2) * np.sum(W ** 2))
    exact = bool(np.all(np.isclose(G, W)) or cos > 0.8)
    return (G if exact else W), exact


class ExpCellFilter:
    """The filter's state: the atoms' Cartesian positions X [n,3] and cell C [3,3] (rows are lattice vectors), and the
    cell C0 it was made with."""

    def __init__(self, cell, positions):
        self.C0 = np.array(cell, dtype=np.float64).reshape(3, 3)
        self.C = self.C0.copy()
        self.X = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.exact = None                      # the branch of the last get_forces

    def deform_grad(self) -> np.ndarray:
        return np.linalg.solve(self.C0, self.C).T

    def get_positions(self) -> np.ndarray:
        F = self.deform_grad()
        return np.concatenate([np.linalg.solve(F, self.X.T).T, np.real(logm(F))])

    def set_positions(self, P) -> None:
        n = len(self.X)
        Fn = expm(P[n:])
        self.C = self.C0 @ Fn.T
        self.X = P[:n] @ Fn.T

    def get_forces(self, forces, stress) -> np.ndarray:
        """forces: the calculator's fp32 Cartesian forces [n,3]; stress: its Voigt stress (eV/A^3)."""
        F = self.deform_grad()
        G, self.exact = cell_forces(F, self.C, stress)
        return np.concatenate([np.asarray(forces, dtype=np.float64) @ F, G])


def relax(evaluate, cell, positions, *, fmax: float = 0.1, steps: int = 100, force_multiplier: float = 1.0,
          stress_wt: float = 1.0, **params):
    """One crystal: FIRE on the filter (Dynamics.irun).  `evaluate(cell, x) -> (energy, grad, model_stress [3,3])` is
    the model at cell and Cartesian positions x.  Returns a dict with cell, positions, energy, forces (fp32,
    Cartesian), stress (fp32 Voigt, eV/A^3), rows (the filter's forces), nsteps, converged, evaluations, the Fire
    object and the filter."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    filt = ExpCellFilter(cell, positions)
    opt = FO.Fire(filt.get_positions(), **params)

    def ev():
        e, g, s = evaluate(filt.C.copy(), filt.X.copy())
        f, sv = FO.scaled_forces(g, force_multiplier), calculator_stress(s, stress_wt)
        return e, f, sv, filt.get_forces(f, sv)
    energy, f, sv, rows = ev()
    nsteps, evals = 0, 1
    while not FO.converged(rows, fmax) and nsteps < steps:
        opt.x = filt.get_positions()           # FIRE.step: r = atoms.get_positions() every step
        opt.step(rows)
        filt.set_positions(opt.x)
        nsteps += 1
        energy, f, sv, rows = ev()
        evals += 1
    return dict(cell=filt.C, positions=filt.X, energy=energy, forces=f, stress=sv, rows=rows, nsteps=nsteps,
                converged=FO.converged(rows, fmax), evaluations=evals, fire=opt, filter=filt)


def relax_batch(evaluate_batch, structures, *, fmax: float = 0.1, steps: int = 100, force_multiplier: float = 1.0,
                stress_wt: float = 1.0, **params):
    """B independent runs of `relax`, advanced together: each round evaluates the crystals still running (ascending
    id) with `evaluate_batch(ids, [(cell_b, x_b)]) -> [(energy_b, grad_b, model_stress_b)]`, then each takes its own
    decision.  A converged or exhausted crystal is frozen and left out of later evaluations."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    B = len(structures)
    filts = [ExpCellFilter(c, x) for c, x in structures]
    opts = [FO.Fire(f.get_positions(), **params) for f in filts]
    status = [FO.RUNNING] * B
    nsteps, evals = [0] * B, [0] * B
    energy, forces, stress, rows = [None] * B, [None] * B, [None] * B, [None] * B
    while True:
        ids = [b for b in range(B) if status[b] == FO.RUNNING]
        if not ids:
            break
        for b, (e, g, s) in zip(ids, evaluate_batch(ids, [(filts[b].C.copy(), filts[b].X.copy()) for b in ids])):
            energy[b], forces[b] = e, FO.scaled_forces(g, force_multiplier)
            stress[b] = calculator_stress(s, stress_wt)
            rows[b] = filts[b].get_forces(forces[b], stress[b])
            evals[b] += 1
            if FO.converged(rows[b], fmax):
                status[b] = FO.CONVERGED
            elif nsteps[b] >= steps:
                status[b] = FO.STEP_LIMIT
            else:
                opts[b].x = filts[b].get_positions()
                opts[b].step(rows[b])
                filts[b].set_positions(opts[b].x)
                nsteps[b] += 1
    return dict(cell=[f.C for f in filts], positions=[f.X for f in filts], energy=energy, forces=forces, stress=stress,
                rows=rows, nsteps=nsteps, converged=[s == FO.CONVERGED for s in status], evaluations=evals, fire=opts,
                filter=filts)
