"""numpy restatement of the reference's structure relaxation, `ForceField.optimize_atoms(optimizer="FIRE",
optimize_lattice=False)` (alignn/ff/ff.py:373-417), with ASE 3.22.1 (the version alignn's environment.yml pins):
the specification `alignn_b200.relax_structures` and the kernel `alignn_b200_fire_step` are tested against.

ASE sources restated (ase 3.22.1):
  ase/optimize/fire.py      FIRE.__init__ (defaults), FIRE.initialize (v = None), FIRE.step
  ase/optimize/optimize.py  Optimizer.run (`if steps: self.max_steps = steps`), Optimizer.converged,
                            Dynamics.irun (evaluate, test, then step / nsteps += 1 / evaluate while not converged and
                            nsteps < max_steps)
Reference call sites:
  alignn/ff/ff.py:404-412         optimizer(self.atoms, ...) with FIRE's defaults; self.dyn.run(fmax=fmax, steps=steps)
  alignn/ff/ff.py:378-379         steps=100, fmax=0.1
  alignn/ff/calculators.py:284-291  the graph of the current positions (atom_dgl_multigraph), every evaluation
  alignn/ff/calculators.py:309-311  forces = result["grad"] (fp32) * force_multiplier
  alignn/ff/calculators.py:357-365  energy = result["out"] * num_atoms (intensive); forces *= num_atoms
                                    (force_mult_natoms), forces *= config["batch_size"] (force_mult_batchsize)

Conventions kept here, and by the device path:
  * the calculator's force scaling is one fp32 product grad * fp32(force_multiplier), the multiplier being the
    calculator's force_multiplier times batch_size (force_mult_batchsize, its default) times natoms (force_mult_natoms);
  * energy = out * natoms, which leaves out the bond penalty `ALIGNNAtomWise` adds to the energy it differentiates
    (alignn_atomwise.py:495-510): the forces include the penalty's gradient, the reported energy does not;
  * FIRE state, positions and velocities are float64; forces are the fp32 product widened to float64, and the
    convergence test squares those.  ASE under numpy 1.x rounds `dt * f` and `a * f / |f| * |v|` (and the squares of
    the convergence test) to float32 when the forces are float32; that depends on numpy's casting rules, so it is not
    reproduced -- a known difference of the order of float32 rounding per step.
"""
from __future__ import annotations

import numpy as np

# FIRE.__init__ defaults (downhill_check=False, maxstep from Optimizer.defaults)
FIRE_DEFAULTS = dict(dt=0.1, maxstep=0.2, dtmax=1.0, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99, a=0.1)

RUNNING, CONVERGED, STEP_LIMIT = 0, 1, 2


def scaled_forces(grad, force_multiplier: float = 1.0) -> np.ndarray:
    """calculators.py:309-311, 362-365: the fp32 forces the calculator hands ASE, result["grad"] times the multiplier."""
    return np.asarray(grad, dtype=np.float32).reshape(-1, 3) * np.float32(force_multiplier)


def converged(forces, fmax: float) -> bool:
    """Optimizer.converged: max over atoms of |F_i|^2 < fmax^2, strict; the squares of the float64-widened forces."""
    f = np.asarray(forces, dtype=np.float64)
    return bool((f ** 2).sum(axis=1).max() < fmax ** 2)


class Fire:
    """FIRE's state for one crystal and its `step` (fire.py, FIRE.initialize / FIRE.step with downhill_check=False)."""

    def __init__(self, positions, **params):
        p = dict(FIRE_DEFAULTS, **params)
        self.maxstep, self.dtmax, self.Nmin = p["maxstep"], p["dtmax"], p["Nmin"]
        self.finc, self.fdec, self.astart, self.fa = p["finc"], p["fdec"], p["astart"], p["fa"]
        self.dt, self.a = p["dt"], p["a"]
        self.Nsteps = 0
        self.v = None                                                   # FIRE.initialize
        self.x = np.array(positions, dtype=np.float64).reshape(-1, 3)

    def step(self, f) -> None:
        f = np.asarray(f, dtype=np.float64)
        if self.v is None:                                              # first step: only v = 0, no mix, no reset
            self.v = np.zeros((len(self.x), 3))
        else:
            vf = np.vdot(f, self.v)
            if vf > 0.0:
                self.v = (1.0 - self.a) * self.v + self.a * f / np.sqrt(np.vdot(f, f)) * np.sqrt(np.vdot(self.v, self.v))
                if self.Nsteps > self.Nmin:
                    self.dt = min(self.dt * self.finc, self.dtmax)
                    self.a *= self.fa
                self.Nsteps += 1
            else:
                self.v[:] *= 0.0
                self.a = self.astart
                self.dt *= self.fdec
                self.Nsteps = 0
        self.v += self.dt * f
        dr = self.dt * self.v
        normdr = np.sqrt(np.vdot(dr, dr))                               # the norm over the whole crystal
        if normdr > self.maxstep:
            dr = self.maxstep * dr / normdr
        self.x = self.x + dr


def relax(evaluate, positions, *, fmax: float = 0.1, steps: int = 100, force_multiplier: float = 1.0, **params):
    """One crystal: Dynamics.irun.  `evaluate(x) -> (energy, grad)` is the model at positions x.  At most steps + 1
    evaluations; energy and forces are those at the final positions.  Returns a dict with positions, energy, forces
    (fp32), nsteps, converged, evaluations and the Fire object."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    opt = Fire(positions, **params)
    energy, grad = evaluate(opt.x)
    f = scaled_forces(grad, force_multiplier)
    nsteps, evals = 0, 1
    while not converged(f, fmax) and nsteps < steps:
        opt.step(f)
        nsteps += 1
        energy, grad = evaluate(opt.x)
        f = scaled_forces(grad, force_multiplier)
        evals += 1
    return dict(positions=opt.x, energy=energy, forces=f, nsteps=nsteps, converged=converged(f, fmax), evaluations=evals,
                fire=opt)


def relax_batch(evaluate_batch, structures_positions, *, fmax: float = 0.1, steps: int = 100, force_multiplier: float = 1.0,
                **params):
    """B independent runs of `relax`, advanced together: each round evaluates the crystals still running (ascending id)
    with `evaluate_batch(ids, [x_b]) -> [(energy_b, grad_b)]`, then each takes its own decision.  A converged or
    exhausted crystal is frozen and left out of later evaluations."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    B = len(structures_positions)
    opts = [Fire(x, **params) for x in structures_positions]
    status = [RUNNING] * B
    nsteps, evals = [0] * B, [0] * B
    energy, forces = [None] * B, [None] * B
    while True:
        ids = [b for b in range(B) if status[b] == RUNNING]
        if not ids:
            break
        for b, (e, g) in zip(ids, evaluate_batch(ids, [opts[b].x for b in ids])):
            energy[b], forces[b] = e, scaled_forces(g, force_multiplier)
            evals[b] += 1
            if converged(forces[b], fmax):
                status[b] = CONVERGED
            elif nsteps[b] >= steps:
                status[b] = STEP_LIMIT
            else:
                opts[b].step(forces[b])
                nsteps[b] += 1
    return dict(positions=[o.x for o in opts], energy=energy, forces=forces, nsteps=nsteps,
                converged=[s == CONVERGED for s in status], evaluations=evals, fire=opts)
