"""numpy restatement of the reference's quasi-Newton relaxations, `ForceField.optimize_atoms(optimizer="LBFGS" or
"BFGS", optimize_lattice=False or True)` (alignn/ff/ff.py:385-412), with ASE 3.22.1: the specification
`alignn_b200.relax_structures(optimizer=...)` and the kernels of csrc/qn_device.cu are tested against.

ASE sources restated (ase 3.22.1, ase/optimize/lbfgs.py, ase/optimize/bfgs.py, ase/optimize/optimize.py):

The driver is `Dynamics.irun`, exactly as for FIRE. It evaluates, then tests `Optimizer.converged`, which is
`max_row |f|^2 < fmax^2` over n rows, or n + 3 rows under the filter. While the test fails and `nsteps < steps`, it
steps and evaluates again.

Under the filter, `r` and `f` are the filter's `get_positions()` and `get_forces()`. Those are m = n + 3 rows, and
`len(filter) = n + 3`. Without the filter they are the Cartesian positions and the fp32 forces widened to float64, and
m = n.

    Optimizer.defaults: maxstep = 0.2

    LBFGS(maxstep=0.2, memory=100, damping=1.0, alpha=70.0, use_line_search=False); H0 = 1/alpha (never changed)
      initialize: iteration = 0; s = y = rho = []; r0 = f0 = None
      step(f):
        r = get_positions()
        update(r, f, r0, f0):
          if iteration > 0:
            s.append(r.ravel() - r0.ravel()); y.append(f0.ravel() - f.ravel()); rho.append(1.0 / dot(y[-1], s[-1]))
          if iteration > memory: s.pop(0); y.pop(0); rho.pop(0)
        loopmax = min(memory, iteration)
        q = -f.ravel()
        for i = loopmax-1 .. 0:  a[i] = rho[i] * dot(s[i], q);  q -= a[i] * y[i]
        z = H0 * q
        for i = 0 .. loopmax-1:  b = rho[i] * dot(y[i], z);  z += s[i] * (a[i] - b)
        p = -z.reshape(-1, 3)
        dr = determine_step(p) * damping       # lengths per row; longest >= maxstep -> dr *= maxstep / longest
        set_positions(r + dr); iteration += 1; r0 = r; f0 = f

    BFGS(maxstep=0.2, alpha=70.0)
      initialize: H0 = eye(3 * len(atoms)) * alpha; H = r0 = f0 = None
      step(f):
        r = get_positions(); f = f.ravel()
        update(r.flat, f, r0, f0):
          if H is None: H = H0; return
          dr = r - r0
          if abs(dr).max() < 1e-7: return                    # same configuration again
          df = f - f0; a = dot(dr, df); dg = H @ dr; b = dot(dr, dg)
          H -= outer(df, df) / a + outer(dg, dg) / b
        omega, V = eigh(H)
        dr = (V @ ((f @ V) / abs(omega))).reshape(-1, 3)
        steplengths = sqrt((dr**2).sum(1)); if max(steplengths) >= maxstep: dr *= maxstep / max(steplengths)
        set_positions(r + dr); r0 = r.flat.copy(); f0 = f.copy()

Points kept: both optimizers cap the longest row, with >= (FIRE caps the whole-vector norm, with >); the direction
|H|^-1 f is a matrix function, so eigenvector signs and bases of degenerate eigenspaces do not change it.  The
conventions of fire_oracle.py and cell_filter_oracle.py carry over unchanged: fp32 forces grad * fp32(force_multiplier),
energy out * natoms without the penalty, the calculator's fp32 Voigt stress, and the filter's L = log F carried from
the last set_positions, not re-derived with logm (`filter_positions`): the quasi-Newton updates difference the
positions of consecutive steps, and logm's rounding would swamp those differences near convergence.

Deliberate difference: where ASE carries on with inf or NaN positions (y.s, a or b zero or not finite, or a step
that is not finite), `step` raises `Breakdown` and leaves the optimizer and the positions as they were.
"""
from __future__ import annotations

import numpy as np

from . import cell_filter_oracle as CF
from . import fire_oracle as FO

LBFGS_DEFAULTS = dict(maxstep=0.2, memory=100, damping=1.0, alpha=70.0)
BFGS_DEFAULTS = dict(maxstep=0.2, alpha=70.0)


class Breakdown(ArithmeticError):
    """The update or the step of a quasi-Newton optimizer is not finite."""


def determine_step(dr, maxstep: float) -> np.ndarray:
    """The longest row of dr capped at maxstep, with >=; the scale taken once, as ASE's `dr *= maxstep / longest`."""
    longest = np.sqrt((dr ** 2).sum(1)).max()
    if not np.isfinite(longest):
        raise Breakdown("the step is not finite")
    if longest >= maxstep:
        dr = dr * (maxstep / longest)
    return dr


class LBFGS:
    """LBFGS's state for one crystal and its `step(r, f) -> r + dr`: r and f the m x 3 rows of this evaluation."""

    def __init__(self, **params):
        p = dict(LBFGS_DEFAULTS, **params)
        self.maxstep, self.memory, self.damping, self.H0 = p["maxstep"], p["memory"], p["damping"], 1.0 / p["alpha"]
        self.iteration = 0
        self.s, self.y, self.rho = [], [], []
        self.r0 = self.f0 = None

    def step(self, r, f) -> np.ndarray:
        r, f = np.asarray(r, dtype=np.float64), np.asarray(f, dtype=np.float64)
        if self.iteration > 0:
            s0, y0 = r.ravel() - self.r0.ravel(), self.f0.ravel() - f.ravel()
            ys = np.dot(y0, s0)
            with np.errstate(divide="ignore", over="ignore"):
                rh = 1.0 / ys
            if not (np.isfinite(ys) and ys != 0.0 and np.isfinite(rh)):
                raise Breakdown("y.s is zero or not finite")
            self.s.append(s0)
            self.y.append(y0)
            self.rho.append(rh)
        if self.iteration > self.memory:
            self.s.pop(0)
            self.y.pop(0)
            self.rho.pop(0)
        loopmax = min(self.memory, self.iteration)
        a = np.empty(loopmax)
        q = -f.ravel()
        for i in range(loopmax - 1, -1, -1):
            a[i] = self.rho[i] * np.dot(self.s[i], q)
            q = q - a[i] * self.y[i]
        z = self.H0 * q
        for i in range(loopmax):
            b = self.rho[i] * np.dot(self.y[i], z)
            z = z + self.s[i] * (a[i] - b)
        dr = determine_step(-z.reshape(-1, 3), self.maxstep) * self.damping
        self.iteration += 1
        self.r0, self.f0 = r.copy(), f.copy()
        return r + dr


class BFGS:
    """BFGS's state for one crystal and its `step(r, f) -> r + dr`."""

    def __init__(self, m: int, **params):
        p = dict(BFGS_DEFAULTS, **params)
        self.maxstep = p["maxstep"]
        self.H0 = np.eye(3 * m) * p["alpha"]
        self.H = self.r0 = self.f0 = None

    def update(self, r, f) -> None:
        if self.H is None:
            self.H = self.H0.copy()
            return
        dr = r - self.r0
        if np.abs(dr).max() < 1e-7:
            return
        df = f - self.f0
        a = np.dot(dr, df)
        dg = self.H @ dr
        b = np.dot(dr, dg)
        if not (np.isfinite(a) and a != 0.0 and np.isfinite(b) and b != 0.0):
            raise Breakdown("a or b is zero or not finite")
        self.H = self.H - (np.outer(df, df) / a + np.outer(dg, dg) / b)

    def step(self, r, f) -> np.ndarray:
        r, f = np.asarray(r, dtype=np.float64).ravel(), np.asarray(f, dtype=np.float64).ravel()
        H = self.H
        self.update(r, f)
        omega, V = np.linalg.eigh(self.H)
        with np.errstate(divide="ignore", invalid="ignore"):
            dr = (V @ ((f @ V) / np.abs(omega))).reshape(-1, 3)
        try:
            dr = determine_step(dr, self.maxstep)
        except Breakdown:
            self.H = H
            raise
        self.r0, self.f0 = r.copy(), f.copy()
        return r.reshape(-1, 3) + dr


def filter_positions(filt, L) -> np.ndarray:
    """ExpCellFilter.get_positions with the carried log-deformation L (zero before the first step)."""
    F = filt.deform_grad()
    return np.concatenate([np.linalg.solve(F, filt.X.T).T, L])


def _filter_step(opt, filt, L, rows) -> np.ndarray:
    """One optimizer step on the filter; returns the new L."""
    P = opt.step(filter_positions(filt, L), rows)
    filt.set_positions(P)
    return P[len(filt.X):].copy()


def make(optimizer: str, m: int, **params):
    if optimizer == "LBFGS":
        return LBFGS(**params)
    if optimizer == "BFGS":
        return BFGS(m, **params)
    raise ValueError(f"optimizer must be 'LBFGS' or 'BFGS', got {optimizer!r}")


def relax(optimizer: str, evaluate, positions, *, fmax: float = 0.1, steps: int = 100, force_multiplier: float = 1.0,
          **params):
    """One crystal, cell fixed: Dynamics.irun.  `evaluate(x) -> (energy, grad)`.  Returns a dict with positions,
    energy, forces (fp32), nsteps, converged, evaluations and the optimizer."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    x = np.array(positions, dtype=np.float64).reshape(-1, 3)
    opt = make(optimizer, len(x), **params)
    energy, grad = evaluate(x)
    f = FO.scaled_forces(grad, force_multiplier)
    nsteps, evals = 0, 1
    while not FO.converged(f, fmax) and nsteps < steps:
        x = opt.step(x, f)
        nsteps += 1
        energy, grad = evaluate(x)
        f = FO.scaled_forces(grad, force_multiplier)
        evals += 1
    return dict(positions=x, energy=energy, forces=f, nsteps=nsteps, converged=FO.converged(f, fmax), evaluations=evals,
                optimizer=opt)


def relax_cell(optimizer: str, evaluate, cell, positions, *, fmax: float = 0.1, steps: int = 100,
               force_multiplier: float = 1.0, stress_wt: float = 1.0, **params):
    """One crystal on ExpCellFilter: `evaluate(cell, x) -> (energy, grad, model_stress [3,3])`.  Returns a dict as
    cell_filter_oracle.relax, with the optimizer."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    filt = CF.ExpCellFilter(cell, positions)
    opt = make(optimizer, len(filt.X) + 3, **params)

    def ev():
        e, g, s = evaluate(filt.C.copy(), filt.X.copy())
        f, sv = FO.scaled_forces(g, force_multiplier), CF.calculator_stress(s, stress_wt)
        return e, f, sv, filt.get_forces(f, sv)
    energy, f, sv, rows = ev()
    nsteps, evals, L = 0, 1, np.zeros((3, 3))
    while not FO.converged(rows, fmax) and nsteps < steps:
        L = _filter_step(opt, filt, L, rows)
        nsteps += 1
        energy, f, sv, rows = ev()
        evals += 1
    return dict(cell=filt.C, positions=filt.X, energy=energy, forces=f, stress=sv, rows=rows, nsteps=nsteps,
                converged=FO.converged(rows, fmax), evaluations=evals, optimizer=opt, filter=filt)


def relax_batch(optimizer: str, evaluate_batch, structures, *, optimize_lattice: bool = False, fmax: float = 0.1,
                steps: int = 100, force_multiplier: float = 1.0, stress_wt: float = 1.0, **params):
    """B independent runs of `relax` (structures: positions) or `relax_cell` (structures: (cell, positions)), advanced
    together: each round evaluates the crystals still running (ascending id) with `evaluate_batch(ids, structs)`, which
    returns (energy, grad) or (energy, grad, model_stress) per crystal, then each takes its own decision."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    B = len(structures)
    if optimize_lattice:
        filts = [CF.ExpCellFilter(c, x) for c, x in structures]
        opts = [make(optimizer, len(fl.X) + 3, **params) for fl in filts]
        Ls = [np.zeros((3, 3)) for _ in filts]
        xs = None
    else:
        xs = [np.array(x, dtype=np.float64).reshape(-1, 3) for x in structures]
        opts = [make(optimizer, len(x), **params) for x in xs]
    status = [FO.RUNNING] * B
    nsteps, evals = [0] * B, [0] * B
    energy, forces, stress, rows = [None] * B, [None] * B, [None] * B, [None] * B
    while True:
        ids = [b for b in range(B) if status[b] == FO.RUNNING]
        if not ids:
            break
        arg = [(filts[b].C.copy(), filts[b].X.copy()) for b in ids] if optimize_lattice else [xs[b] for b in ids]
        for b, res in zip(ids, evaluate_batch(ids, arg)):
            energy[b], forces[b] = res[0], FO.scaled_forces(res[1], force_multiplier)
            if optimize_lattice:
                stress[b] = CF.calculator_stress(res[2], stress_wt)
                rows[b] = filts[b].get_forces(forces[b], stress[b])
            else:
                rows[b] = forces[b]
            evals[b] += 1
            if FO.converged(rows[b], fmax):
                status[b] = FO.CONVERGED
            elif nsteps[b] >= steps:
                status[b] = FO.STEP_LIMIT
            else:
                if optimize_lattice:
                    Ls[b] = _filter_step(opts[b], filts[b], Ls[b], rows[b])
                else:
                    xs[b] = opts[b].step(xs[b], rows[b])
                nsteps[b] += 1
    out = dict(energy=energy, forces=forces, nsteps=nsteps, converged=[s == FO.CONVERGED for s in status],
               evaluations=evals, optimizer=opts)
    if optimize_lattice:
        out.update(cell=[fl.C for fl in filts], positions=[fl.X for fl in filts], stress=stress, rows=rows, filter=filts)
    else:
        out.update(positions=xs)
    return out
