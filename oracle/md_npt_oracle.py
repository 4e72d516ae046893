"""numpy restatement of the reference's constant-pressure molecular dynamics, `ForceField.run_npt_berendsen`
(alignn/ff/ff.py:545-582, the `npt_berendsen` task of alignn/run_alignn_ff.py:199-213), with ASE 3.22.1: the
specification `alignn_b200.run_md(ensemble="npt_berendsen")` and the kernel `alignn_b200_md_npt_step` are tested
against.

ASE sources restated (ase 3.22.1):
  ase/units.py                 Pascal = (1 / _e) / 1e30; bar = 1e5 * Pascal (CODATA 2014, as oracle/md_oracle.py)
  ase/md/nptberendsen.py       NPTBerendsen(atoms, timestep, temperature_K=T0, taut=taut, taup=taup, pressure=P,
                               compressibility=c, fixcm=True):
      __init__:                self.pressure = _process_pressure(pressure, pressure_au): exactly one of the two, else
                                   TypeError; pressure_au = pressure * (1e5 * units.Pascal)
                               compressibility_au = compressibility / (1e5 * units.Pascal); with compressibility=None
                                   it stays None and the first step fails on `taupscl * None` (TypeError)
      scale_positions_and_cell:
                               taupscl = self.dt / self.taup
                               stress = self.atoms.get_stress(voigt=False, include_ideal_gas=True)
                               old_pressure = -stress.trace() / 3
                               scl_pressure = (1.0 - taupscl * self.compressibility / 3.0 *
                                               (self.pressure - old_pressure))
                               cell = self.atoms.get_cell(); cell = scl_pressure * cell
                               self.atoms.set_cell(cell, scale_atoms=True)
      step:                    NVTBerendsen.scale_velocities(self); self.scale_positions_and_cell()
                               forces = atoms.get_forces(md=True)        (a new evaluation: the structure moved)
                               p = self.atoms.get_momenta(); p += 0.5 * self.dt * forces
                               fixcm: psum = p.sum(axis=0) / float(len(p)); p = p - psum
                               set_positions(get_positions() + self.dt * p / masses[:, np.newaxis]); set_momenta(p)
                               forces = get_forces(md=True); set_momenta(get_momenta() + 0.5 * self.dt * forces)
  ase/md/nvtberendsen.py       scale_velocities: oracle/md_oracle.py's berendsen_scale, p = s * p
  ase/atoms.py                 get_stress(voigt=False, include_ideal_gas=True): stress = the calculator's Voigt
                               stress (a copy); stresscomp = [[0, 5, 4], [5, 1, 3], [4, 3, 2]]; invmass = 1.0 / masses;
                               invvol = 1.0 / self.get_volume(); for alpha, beta >= alpha:
                               stress[stresscomp[alpha, beta]] -= (p[:, alpha] * p[:, beta] * invmass).sum() * invvol;
                               voigt_6_to_full_3x3_stress(stress).  get_volume = abs(np.linalg.det(cell)).
                               set_cell(cell, scale_atoms=True): M = np.linalg.solve(old_cell, cell);
                               positions[:] = np.dot(positions, M)
  ase/md/md.py                 MolecularDynamics.irun: evaluate, then `steps` times step and log (oracle/md_oracle.py)
Reference call sites:
  alignn/ff/ff.py:545-582      NPTBerendsen(atoms, timestep, temperature_K=300, taut=49.11347394232032,
                               taup=98.22694788464064, pressure=None, compressibility=None) -- 500 * fs and
                               1000 * fs bitwise; with both None the reference's own call cannot run (its test,
                               alignn/tests/test_alignn_ff.py:111, is commented out), so here both are required
  alignn/run_alignn_ff.py:199-213  the npt_berendsen task (passes neither)

One step after the logged evaluation that gave the forces f and the calculator's Voigt stress s (fp32):
  1. s_T = berendsen_scale(T(p), T0, dt, taut); p = s_T p
  2. the barostat on s less the ideal-gas term of these momenta; mu = 1 - (dt/taup) c / 3 (P0 - P); C = mu C;
     X = X @ solve(C_old, C)
  3. evaluation A at (C, X); only its forces fA are used
  4. p += 0.5 dt fA; p -= p.sum(0) / n; X += dt p / m
  5. evaluation B at (C, X) -- logged; p += 0.5 dt fB.  Its stress is the one the next step's barostat reads.
So a run of `steps` steps makes 2 steps + 1 evaluations, steps + 1 of them logged.

Conventions, beyond those of oracle/md_oracle.py and oracle/cell_filter_oracle.py (calculator_stress):
  * the ideal-gas subtraction is in place on the calculator's float32 Voigt array: each component is
    fp32(double(s_k) - term) (the float32 scalar minus a float64 scalar is float64 under numpy 1 and 2, and the store
    rounds it).  The trace of the float32 3 x 3 is a float32 sum, (s_xx + s_yy) + s_zz.
  * numpy 1.x, which the reference pins (numpy<2), promotes the float32 trace to float64 in `-trace / 3` (a scalar
    with a Python int); numpy 2 would keep float32.  The numpy 1 result is the one restated: old_pressure =
    -float64(trace) / 3.0 and the rest of the barostat in float64 (`pressure`).
  * the pressure logged with each evaluation is that same quantity with the momenta of the evaluation (before the next
    step's velocity scaling), in eV/A^3, ideal-gas term included.
  * temperatures in K, pressure in bar and compressibility in 1/bar as the reference's arguments; P0 and c travel in
    ASE units (pressure_au, compressibility_au).
The device path scales positions as X * mu (one rounding per coordinate) where ASE forms solve(C, mu C) = mu I up to
rounding; the two differ by about 1e-16 relative per step.  A cell whose volume or mu is not finite and > 0 stops the
device run for that crystal (status 4); ASE would carry on with a collapsed or inverted cell.  Not reproduced.
"""
from __future__ import annotations

import numpy as np

from .cell_filter_oracle import calculator_stress
from .fire_oracle import scaled_forces
from .md_oracle import _e, berendsen_scale, fs, kinetic_energy, temperature

Pascal = (1 / _e) / 1e30          # ase.units.Pascal
TAUT, TAUP = 49.11347394232032, 98.22694788464064   # ForceField.run_npt_berendsen's literals: 500 * fs, 1000 * fs
assert TAUT == 500 * fs and TAUP == 1000 * fs

_IDEAL = ((0, 0, 0), (0, 1, 5), (0, 2, 4), (1, 1, 1), (1, 2, 3), (2, 2, 2))   # (alpha, beta, Voigt index)


def pressure_au(pressure_bar: float) -> float:
    """NPTBerendsen._process_pressure: bar to eV/A^3."""
    return pressure_bar * (1e5 * Pascal)


def compressibility_au(compressibility_per_bar: float) -> float:
    """NPTBerendsen.__init__: 1/bar to A^3/eV."""
    return compressibility_per_bar / (1e5 * Pascal)


def volume(cell) -> float:
    return abs(np.linalg.det(np.asarray(cell, dtype=np.float64)))


def ideal_gas_stress(stress, p, masses, cell) -> np.ndarray:
    """Atoms.get_stress(include_ideal_gas=True) in Voigt order: the calculator's fp32 stress less
    (p_a p_b / m).sum() / V per component, in place on the fp32 array."""
    s = np.array(stress, dtype=np.float32).reshape(6)
    invmass = 1.0 / np.asarray(masses, dtype=np.float64)
    invvol = 1.0 / volume(cell)
    for a, b, k in _IDEAL:
        s[k] = np.float64(s[k]) - (p[:, a] * p[:, b] * invmass).sum() * invvol
    return s


def pressure(stress6) -> float:
    """-trace / 3 of the fp32 stress: the trace in fp32, the rest in float64 (numpy 1.x's scalar promotion)."""
    s = np.asarray(stress6, dtype=np.float32)
    trace = (s[0] + s[1]) + s[2]                   # np.float32
    return -np.float64(trace) / 3.0


def barostat_scale(stress6, P0_au: float, compressibility_au_: float, dt: float, taup: float) -> float:
    """scale_positions_and_cell's scl_pressure from the ideal-gas-corrected fp32 stress."""
    taupscl = dt / taup
    return 1.0 - taupscl * compressibility_au_ / 3.0 * (P0_au - pressure(stress6))


class NPT:
    """One crystal's NPTBerendsen state: cell C [3,3] (rows are lattice vectors), positions X and momenta p (float64),
    masses [n] amu; dt, taut, taup in ASE time units; P0 in eV/A^3, compressibility in A^3/eV."""

    def __init__(self, cell, positions, masses, *, dt: float, temperature_K: float, pressure_au_: float,
                 compressibility_au_: float, taut: float = TAUT, taup: float = TAUP, momenta=None):
        self.C = np.array(cell, dtype=np.float64).reshape(3, 3)
        self.x = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.m = np.asarray(masses, dtype=np.float64).reshape(-1)
        self.p = np.zeros_like(self.x) if momenta is None else np.array(momenta, dtype=np.float64).reshape(-1, 3)
        self.dt, self.T0, self.taut, self.taup = dt, temperature_K, taut, taup
        self.P0, self.c = pressure_au_, compressibility_au_
        self.mu = None                                 # the last barostat scale

    def first_half(self, sv) -> None:
        """Steps 1-2: velocity scaling, then the cell and positions scaled on the calculator stress sv of the last
        evaluation."""
        s = berendsen_scale(temperature(self.p, self.m), self.T0, self.dt, self.taut)
        self.p = s * self.p
        self.mu = barostat_scale(ideal_gas_stress(sv, self.p, self.m, self.C), self.P0, self.c, self.dt, self.taup)
        cell = self.mu * self.C
        M = np.linalg.solve(self.C, cell)
        self.x = np.dot(self.x, M)
        self.C = cell

    def middle(self, fA) -> None:
        """Step 4, on the forces of evaluation A."""
        self.p += 0.5 * self.dt * fA
        psum = self.p.sum(axis=0) / float(len(self.p))
        self.p = self.p - psum
        self.x = self.x + self.dt * self.p / self.m[:, np.newaxis]

    def second_half(self, fB) -> None:
        self.p = self.p + 0.5 * self.dt * fB


def _check(pressure_bar, compressibility):
    if pressure_bar is None:                           # NPTBerendsen._process_pressure
        raise TypeError("Exactly one of the parameters 'pressure', and 'pressure_au' must be given")
    if compressibility is None:                        # ASE: the first step's taupscl * None
        raise TypeError("unsupported operand type(s) for *: 'float' and 'NoneType' (compressibility=None)")


def _new_rec():
    return dict(energy=[], kinetic_energy=[], temperature=[], pressure=[], stress=[], cells=[], forces=None)


def _log(rec, md, energy, f, sv):
    rec["energy"].append(energy)
    rec["kinetic_energy"].append(kinetic_energy(md.p, md.m))
    rec["temperature"].append(temperature(md.p, md.m))
    rec["stress"].append(sv)
    rec["pressure"].append(pressure(ideal_gas_stress(sv, md.p, md.m, md.C)))
    rec["cells"].append(md.C.copy())
    rec["forces"] = f


def _result(md, rec, traj, steps):
    return dict(positions=md.x, momenta=md.p, cell=md.C, forces=rec["forces"], energy=rec["energy"],
                kinetic_energy=rec["kinetic_energy"], temperature=rec["temperature"], pressure=rec["pressure"],
                stress=rec["stress"], cells=rec["cells"], evaluations=2 * steps + 1, trajectory=traj, md=md)


def run(evaluate, cell, positions, masses, *, steps: int, dt: float, temperature_K: float, pressure=None,
        compressibility=None, taut: float = TAUT, taup: float = TAUP, momenta=None, force_multiplier: float = 1.0,
        stress_wt: float = 1.0, trajectory_interval: int = None):
    """One crystal: NPTBerendsen under MolecularDynamics.irun.  `evaluate(cell, x) -> (energy, grad, model_stress
    [3,3])` is the model at cell and Cartesian positions x.  pressure in bar, compressibility in 1/bar (both required,
    see _check).  Returns a dict with positions, momenta, cell, forces (fp32, of the last evaluation), the per-logged-
    evaluation lists energy, kinetic_energy, temperature, pressure (eV/A^3), stress (fp32 Voigt, eV/A^3) and cells, the
    number of evaluations (2 steps + 1), the trajectory (positions at logged evaluations 0, k, 2k, ...) and the NPT."""
    _check(pressure, compressibility)
    if steps < 1:
        raise ValueError("steps must be >= 1")
    return run_batch(lambda cx: [evaluate(c, x) for c, x in cx], [cell], [positions], [masses], steps=steps, dt=dt,
                     temperature_K=[temperature_K], pressure=[pressure], compressibility=[compressibility], taut=taut,
                     taup=taup, momenta=[momenta], force_multiplier=force_multiplier, stress_wt=stress_wt,
                     trajectory_interval=trajectory_interval)[0]


def run_batch(evaluate_batch, cells, positions, masses, *, steps: int, dt: float, temperature_K, pressure=None,
              compressibility=None, taut: float = TAUT, taup: float = TAUP, momenta=None, force_multiplier: float = 1.0,
              stress_wt: float = 1.0, trajectory_interval: int = None):
    """B independent runs of `run`, advanced in lockstep: each of the 2 steps + 1 rounds evaluates every crystal with
    `evaluate_batch([(cell_b, x_b)]) -> [(energy_b, grad_b, model_stress_b)]`.  temperature_K, pressure and
    compressibility are one value or one per crystal; momenta is None or one [n_b,3] array (or None) per crystal."""
    B = len(positions)
    per = lambda v: list(v) if np.ndim(v) == 1 else [v] * B      # noqa: E731
    T0, P, c = per(temperature_K), per(pressure), per(compressibility)
    for b in range(B):
        _check(P[b], c[b])
    if steps < 1:
        raise ValueError("steps must be >= 1")
    mom = [None] * B if momenta is None else list(momenta)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        mds = [NPT(cells[b], positions[b], masses[b], dt=dt, temperature_K=T0[b], pressure_au_=pressure_au(P[b]),
                   compressibility_au_=compressibility_au(c[b]), taut=taut, taup=taup, momenta=mom[b]) for b in range(B)]
        recs = [_new_rec() for _ in range(B)]
        trajs = [[] if trajectory_interval else None for _ in range(B)]

        def evaluate():
            out = evaluate_batch([(md.C.copy(), md.x.copy()) for md in mds])
            return [(e, scaled_forces(g, force_multiplier), calculator_stress(s, stress_wt)) for e, g, s in out]
        for e in range(steps + 1):
            if trajectory_interval and e % trajectory_interval == 0:
                for b in range(B):
                    trajs[b].append(mds[b].x.copy())
            for b, (energy, f, sv) in enumerate(evaluate()):          # the logged evaluation e (B of step e)
                md = mds[b]
                if e >= 1:
                    md.second_half(f.astype(np.float64))
                _log(recs[b], md, energy, f, sv)
                if e < steps:
                    md.first_half(sv)
            if e == steps:
                break
            for b, (_, fA, _) in enumerate(evaluate()):                # evaluation A of step e + 1
                mds[b].middle(fA.astype(np.float64))
    return [_result(md, r, t, steps) for md, r, t in zip(mds, recs, trajs)]
