"""numpy restatement of the reference's Nose-Hoover / Parrinello-Rahman molecular dynamics,
`ForceField.run_npt_nose_hoover` (alignn/ff/ff.py:584-617, the `npt` task of alignn/run_alignn_ff.py:243-256), with
ASE 3.22.1's `NPT`: the specification `alignn_b200.run_md(ensemble="npt_nose_hoover")` and the kernel
`alignn_b200_md_nose_hoover_step` are tested against.

ASE sources restated (ase 3.22.1, ase/md/npt.py: Melchionna's combined Nose-Hoover thermostat and Parrinello-Rahman
barostat), as NPT(atoms, dt, temperature_K=T0, externalstress=s_ext, ttime=ttime, pfactor=pfactor) with mask=None (all
ones) and frac_traceless = 1:
  __init__:            raises TypeError for pfactor without externalstress; zero_center_of_mass_momentum:
                       p = p - p.sum(0) / n (not mass-weighted); self.temperature = units.kB * T0 (kT, eV);
                       set_stress(externalstress); eta = zeros((3, 3)), zeta = 0.0; _calculateconstants
  set_stress:          a scalar s -> [-s, -s, -s, 0, 0, 0]; a 3 x 3 must be symmetric ((m - m.T) below 1e-10, else
                       ValueError) -> (xx, yy, zz, yz, xz, xy); a 6-vector as is; any other shape ValueError
  _calculateconstants: tfact = 2.0 / (3 * n * kT * ttime * ttime), 0.0 for ttime None;
                       pfact = 1.0 / (pfactor * linalg.det(h)), 0.0 for pfactor None -- frozen at the initial cell;
                       desiredEkin = 1.5 * (n - 1) * kT
  initialize:          (at the first run) h upper triangular (h[1,0] == h[2,0] == h[2,1] == 0, rows the lattice
                       vectors) or NotImplementedError; inv_h = inv(h); q = r inv_h - 0.5;
                       h_past = h - dt * dot(h, eta);
                       deltaeta = -dt * pfact * det(h) * (stress - externalstress), zeros for pfactor None;
                       eta_past = eta - mask * U(deltaeta);
                       zeta_past = zeta - dt * tfact * (get_kinetic_energy() - desiredEkin);
                       _calculate_q_past_and_future
  _calculate_q_past_and_future:
                       p0 = the momenta; p = p0; twice: q_past = q - dt * dot(p / m, inv_h); q_future from the forces;
                       p = dot(q_future - q_past, h / (2 * dt)) * m; if 0.5 * sum(sum(p * p, -1) / m) / n < 1e-5:
                       return; p = (p0 - p) + p0.  The atoms keep p0.
  _calculate_q_future: alpha = (dt * dt) * dot(F / m, inv_h); beta = dt * dot(h, dot(eta + 0.5 * zeta * I, inv_h));
                       q_future = dot(2 * q + dot(q_past, beta - I) + alpha, inv(beta + I))
  step:                h_future = h_past + 2 * dt * dot(h, eta);
                       deltaeta = -2 * dt * (pfact * det(h) * (stress - externalstress)), zeros for pfactor None;
                       eta_future = eta_past + mask * U(deltaeta);
                       zeta_future = zeta_past + 2 * dt * tfact * (get_kinetic_energy() - desiredEkin);
                       h_past, h = h, h_future; inv_h = inv(h); q_past, q = q, q_future; set_cell(h) and
                       r = dot(q + 0.5, h); eta_past, eta = eta, eta_future; zeta_past, zeta = zeta, zeta_future;
                       F = get_forces() (a new evaluation); q_future from F; p = dot(q_future - q_past, h / (2 dt)) * m
  U(v) = [[v0, v5, v4], [0, v1, v3], [0, 0, v2]] (_makeuppertriangular); stress = get_stress(include_ideal_gas=True),
  the calculator's fp32 Voigt stress less the ideal-gas term of the current momenta (oracle/md_npt_oracle.py), read
  only when pfactor is given.  zeta_integrated (the conserved quantity's bookkeeping) feeds no output and is not kept.
Reference call sites:
  alignn/ff/ff.py:584-617     NPT(atoms, timestep, temperature_K=300, externalstress=0.0): neither ttime nor pfactor,
                              so thermostat and barostat are both off (tfact = pfact = 0); its `taut` is computed and
                              never passed
  alignn/run_alignn_ff.py:243-256  the npt task

One model evaluation per step: the stress step k + 1 reads is the one of step k's evaluation at the same structure (the
calculator's cache), and the forces of the first evaluation serve both initialisation passes.  So `steps` steps make
steps + 1 evaluations, all logged as md_npt_oracle logs them (energy, ekin and T, the calculator's stress, the pressure
with the ideal-gas term, the cell); row 0 is the state initialize() leaves, with the centre-of-mass momentum removed.

Conventions, beyond those of oracle/md_oracle.py and oracle/md_npt_oracle.py: forces are the calculator's fp32 array
widened to float64; the stress in `stress - externalstress` is the ideal-gas-corrected fp32 Voigt array widened to
float64; matrices are float64 with numpy's np.dot and np.linalg.inv / det, which the device path replaces by fixed-order
products and closed-form 3 x 3 inverses and determinants (differences of a few ulps per step).
Derived facts (tests/test_md_nose_hoover_oracle.py): with ttime = pfactor = None and a mean kinetic energy at or above
1e-5 eV per atom this is velocity Verlet (the second initialisation pass makes r1 = r0 + dt p0/m + dt^2 F0/(2m), and
the central difference p_k = (r_{k+1} - r_{k-1}) m / (2 dt) is Verlet's p_k), with h, eta and zeta constant; a crystal
at rest leaves the initialisation after its first pass, so its first step is r1 = r0 + dt^2 F0/m.
"""
from __future__ import annotations

import numpy as np

from .cell_filter_oracle import calculator_stress
from .fire_oracle import scaled_forces
from .md_npt_oracle import ideal_gas_stress, pressure
from .md_oracle import kB, kinetic_energy, temperature


def external_stress(s) -> np.ndarray:
    """NPT.set_stress: [6] float64 Voigt (xx yy zz yz xz xy), eV/A^3."""
    if np.isscalar(s):
        return np.array([-s, -s, -s, 0.0, 0.0, 0.0])
    s = np.array(s)
    if s.shape == (3, 3):
        if not (s - np.transpose(s)).max() < 1e-10:
            raise ValueError("The external stress must be a symmetric tensor.")
        return np.array((s[0, 0], s[1, 1], s[2, 2], s[1, 2], s[0, 2], s[0, 1]))
    if s.shape != (6,):
        raise ValueError("The external stress has the wrong shape.")
    return s


def constants(n: int, kT: float, ttime, pfactor, h):
    """NPT._calculateconstants: (tfact, pfact, desiredEkin); ttime in ASE time units, pfactor in ASE units."""
    tfact = 0.0 if ttime is None else 2.0 / (3 * n * kT * ttime * ttime)
    pfact = 0.0 if pfactor is None else 1.0 / (pfactor * np.linalg.det(h))
    return tfact, pfact, 1.5 * (n - 1) * kT


def upper(v) -> np.ndarray:
    """NPT._makeuppertriangular."""
    return np.array(((v[0], v[5], v[4]), (0, v[1], v[3]), (0, 0, v[2])))


def _is_upper_triangular(h) -> bool:
    return h[1, 0] == h[2, 0] == h[2, 1] == 0.0


class NPT:
    """One crystal's NPT state: cell h [3,3] (rows are lattice vectors), positions x and momenta p (float64), masses [n]
    amu; dt and ttime in ASE time units, pfactor in ASE units, externalstress as NPT takes it (eV/A^3)."""

    def __init__(self, cell, positions, masses, *, dt: float, temperature_K=None, externalstress=0.0, ttime=None,
                 pfactor=None, momenta=None):
        if temperature_K is None:                                   # MolecularDynamics._process_temperature
            raise TypeError("Missing 'temperature_K' argument")
        if externalstress is None and pfactor is not None:
            raise TypeError("Missing 'externalstress' argument.")
        self.h = np.array(cell, dtype=np.float64).reshape(3, 3)
        self.x = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.m = np.asarray(masses, dtype=np.float64).reshape(-1)
        n = len(self.m)
        p = np.zeros_like(self.x) if momenta is None else np.array(momenta, dtype=np.float64).reshape(-1, 3)
        self.p = p - p.sum(0) / n                                   # zero_center_of_mass_momentum
        self.dt, self.kT = dt, kB * temperature_K
        self.s_ext = None if externalstress is None else external_stress(externalstress)
        self.barostat = pfactor is not None
        self.eta, self.zeta = np.zeros((3, 3)), 0.0
        self.tfact, self.pfact, self.desiredEkin = constants(n, self.kT, ttime, pfactor, self.h)
        self.passes = None                                          # initialisation passes run (1 or 2)

    def _stress(self, sv):
        return ideal_gas_stress(sv, self.p, self.m, self.h)

    def _q_future(self, f):
        dt, I = self.dt, np.identity(3)
        alpha = (dt * dt) * np.dot(f / self.m[:, None], self.inv_h)
        beta = dt * np.dot(self.h, np.dot(self.eta + 0.5 * self.zeta * I, self.inv_h))
        inv_b = np.linalg.inv(beta + I)
        self.q_future = np.dot(2 * self.q + np.dot(self.q_past, beta - I) + alpha, inv_b)

    def initialize(self, f, sv) -> None:
        """NPT.initialize at the first evaluation: forces f (float64) and the calculator's fp32 Voigt stress sv."""
        dt, h = self.dt, self.h
        if not _is_upper_triangular(h):
            raise NotImplementedError("Can (so far) only operate on lists of atoms where the computational box is an "
                                      "upper triangular matrix.")
        self.inv_h = np.linalg.inv(h)
        self.q = np.dot(self.x, self.inv_h) - 0.5
        self.h_past = h - dt * np.dot(h, self.eta)
        deltaeta = (-dt * self.pfact * np.linalg.det(h) * (self._stress(sv) - self.s_ext) if self.barostat
                    else np.zeros(6))
        self.eta_past = self.eta - upper(deltaeta)
        self.zeta_past = self.zeta - dt * self.tfact * (kinetic_energy(self.p, self.m) - self.desiredEkin)
        p0, m = self.p, self.m[:, None]
        p = np.array(p0, copy=True)
        for i in range(2):
            self.passes = i + 1
            self.q_past = self.q - dt * np.dot(p / m, self.inv_h)
            self._q_future(f)
            p = np.dot(self.q_future - self.q_past, h / (2 * dt)) * m
            if 0.5 * np.sum(np.sum(p * p, -1) / self.m) / len(self.m) < 1e-5:
                return
            p = (p0 - p) + p0

    def begin_step(self, sv) -> None:
        """NPT.step up to the evaluation, on the stress sv cached from the last evaluation."""
        dt = self.dt
        h_future = self.h_past + 2 * dt * np.dot(self.h, self.eta)
        deltaeta = (-2 * dt * (self.pfact * np.linalg.det(self.h) * (self._stress(sv) - self.s_ext)) if self.barostat
                    else np.zeros(6))
        eta_future = self.eta_past + upper(deltaeta)
        zeta_future = self.zeta_past + 2 * dt * self.tfact * (kinetic_energy(self.p, self.m) - self.desiredEkin)
        self.h_past, self.h = self.h, h_future
        self.inv_h = np.linalg.inv(self.h)
        self.q_past, self.q = self.q, self.q_future
        self.x = np.dot(self.q + 0.5, self.h)
        self.eta_past, self.eta = self.eta, eta_future
        self.zeta_past, self.zeta = self.zeta, zeta_future

    def finish_step(self, f) -> None:
        """NPT.step after the evaluation, on its forces f (float64)."""
        self._q_future(f)
        self.p = np.dot(self.q_future - self.q_past, self.h / (2 * self.dt)) * self.m[:, None]


def _log(rec, md, energy, f, sv):
    rec["energy"].append(energy)
    rec["kinetic_energy"].append(kinetic_energy(md.p, md.m))
    rec["temperature"].append(temperature(md.p, md.m))
    rec["stress"].append(sv)
    rec["pressure"].append(pressure(ideal_gas_stress(sv, md.p, md.m, md.h)))
    rec["cells"].append(md.h.copy())
    rec["forces"] = f


def run(evaluate, cell, positions, masses, *, steps: int, dt: float, temperature_K=None, externalstress=0.0,
        ttime=None, pfactor=None, momenta=None, force_multiplier: float = 1.0, stress_wt: float = 1.0,
        trajectory_interval: int = None):
    """One crystal: NPT.run(steps) with the observers after every evaluation.  `evaluate(cell, x) -> (energy, grad,
    model_stress [3,3])` is the model at cell and Cartesian positions x.  ttime in ASE time units, pfactor in ASE units
    (amu/A), both None by default as in the reference's call.  Returns a dict with positions, momenta, cell, forces (fp32,
    of the last evaluation), the per-evaluation lists energy, kinetic_energy, temperature, pressure (eV/A^3), stress
    (fp32 Voigt, eV/A^3) and cells, evaluations (steps + 1), the trajectory (positions at evaluations 0, k, 2k, ...) and
    the NPT."""
    return run_batch(lambda cx: [evaluate(c, x) for c, x in cx], [cell], [positions], [masses], steps=steps, dt=dt,
                     temperature_K=[temperature_K], externalstress=[externalstress], ttime=ttime, pfactor=pfactor,
                     momenta=[momenta], force_multiplier=force_multiplier, stress_wt=stress_wt,
                     trajectory_interval=trajectory_interval)[0]


def run_batch(evaluate_batch, cells, positions, masses, *, steps: int, dt: float, temperature_K, externalstress=0.0,
              ttime=None, pfactor=None, momenta=None, force_multiplier: float = 1.0, stress_wt: float = 1.0,
              trajectory_interval: int = None):
    """B independent runs of `run`, advanced in lockstep: each of the steps + 1 rounds evaluates every crystal with
    `evaluate_batch([(cell_b, x_b)]) -> [(energy_b, grad_b, model_stress_b)]`.  temperature_K is one value or one per
    crystal; externalstress is one value for all or a list with one per crystal; momenta is None or one [n_b,3] array
    (or None) per crystal."""
    B = len(positions)
    T0 = list(temperature_K) if np.ndim(temperature_K) == 1 else [temperature_K] * B
    ext = list(externalstress) if isinstance(externalstress, list) else [externalstress] * B
    if steps < 1:
        raise ValueError("steps must be >= 1")
    mom = [None] * B if momenta is None else list(momenta)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        mds = [NPT(cells[b], positions[b], masses[b], dt=dt, temperature_K=T0[b], externalstress=ext[b], ttime=ttime,
                   pfactor=pfactor, momenta=mom[b]) for b in range(B)]
        recs = [dict(energy=[], kinetic_energy=[], temperature=[], pressure=[], stress=[], cells=[], forces=None)
                for _ in range(B)]
        trajs = [[] if trajectory_interval else None for _ in range(B)]
        for e in range(steps + 1):
            if trajectory_interval and e % trajectory_interval == 0:
                for b in range(B):
                    trajs[b].append(mds[b].x.copy())
            out = evaluate_batch([(md.h.copy(), md.x.copy()) for md in mds])
            for b, (energy, grad, S) in enumerate(out):
                md, f, sv = mds[b], scaled_forces(grad, force_multiplier), calculator_stress(S, stress_wt)
                if e == 0:
                    md.initialize(f.astype(np.float64), sv)
                else:
                    md.finish_step(f.astype(np.float64))
                _log(recs[b], md, energy, f, sv)
                if e < steps:
                    md.begin_step(sv)
    return [dict(positions=md.x, momenta=md.p, cell=md.h, forces=r["forces"], energy=r["energy"],
                 kinetic_energy=r["kinetic_energy"], temperature=r["temperature"], pressure=r["pressure"],
                 stress=r["stress"], cells=r["cells"], evaluations=steps + 1, trajectory=t, md=md)
            for md, r, t in zip(mds, recs, trajs)]
