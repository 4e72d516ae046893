"""Molecular dynamics for a batch of crystals with ALIGNN-FF on the GPU: NVE velocity Verlet, NVT Berendsen, NVT Langevin,
NVT Andersen and NPT Berendsen.

The reference runs MD one structure at a time: `ForceField.run_nve_velocity_verlet` and `run_nvt_berendsen`
(alignn/ff/ff.py:419-443, 510-543) drive ASE's integrators, and every step its calculator (alignn/ff/calculators.py:
280-372) builds g and L(g) on the CPU, copies them to the GPU, runs the model and copies the forces back for numpy to
integrate.  Here all crystals advance in lockstep: per evaluation one device graph build
(`neighbors.crystal_graphs_device`), one model call and one integrator launch (`ops.md_step`, csrc/md_device.cu) that
also writes each crystal's kinetic energy and temperature.  Each crystal follows the trajectory it would follow run
alone; `oracle/md_oracle.py` is the specification (ASE 3.22.1 semantics, float64 state).  The stochastic thermostats
(`ForceField.run_nvt_langevin` / `run_nvt_andersen`, alignn/ff/ff.py:444-508) launch `ops.md_thermostat_step` instead
and draw their noise from a counter-based stream keyed by each crystal's seed (csrc/md_noise.cuh) rather than numpy's
global RNG; `oracle/md_thermostat_oracle.py` is their specification.  NPT Berendsen (`ForceField.run_npt_berendsen`,
alignn/ff/ff.py:545-582) moves the cells too: every step rebuilds the graphs from the rescaled cells, evaluates the
model twice and launches `ops.md_npt_step` after each evaluation; `oracle/md_npt_oracle.py` is its specification.
ASE's NPT (Nose-Hoover thermostat and Parrinello-Rahman barostat, `ForceField.run_npt_nose_hoover`, alignn/ff/ff.py:
584-617) integrates in fractional coordinates with one model call and one `ops.md_nose_hoover_step` launch per step;
`oracle/md_nose_hoover_oracle.py` is its specification, and `upper_triangular` rotates structures into the cell form it
needs.
"""
from __future__ import annotations

import math
import numbers
from typing import Callable, NamedTuple, Optional

import numpy as np
import torch

from . import calculator, neighbors, ops

# ase.units (ASE 3.22.1, CODATA 2014): the femtosecond in ASE time units and the Boltzmann constant in eV/K
_e, _amu, _k = 1.6021766208e-19, 1.660539040e-27, 1.38064852e-23
FS = 1e-15 * (1e10 * math.sqrt(_e / _amu))     # 0.09822694788464063
KB = _k / _e                                   # 8.617330337217213e-05
BAR = 1e5 * ((1 / _e) / 1e30)                  # ase.units: 1e5 * Pascal, the bar in eV/A^3

ENSEMBLES = {"nve_velocity_verlet": ops.MD_NVE, "nvt_berendsen": ops.MD_NVT_BERENDSEN,
             "nvt_langevin": ops.MD_NVT_LANGEVIN, "nvt_andersen": ops.MD_NVT_ANDERSEN,
             "npt_berendsen": ops.MD_NPT_BERENDSEN, "npt_nose_hoover": ops.MD_NPT_NOSE_HOOVER}
STOCHASTIC = (ops.MD_NVT_LANGEVIN, ops.MD_NVT_ANDERSEN)
LANGEVIN_FRICTION = 1e-4      # ForceField.run_nvt_langevin's default friction, in 1 / ASE time unit
NPT_TAUT = 49.11347394232032  # ForceField.run_npt_berendsen's taut literal: 500 fs in ASE units, bitwise


class MDResult(NamedTuple):
    positions: torch.Tensor       # [N,3] float64 final Cartesian positions (not wrapped into the cell)
    momenta: torch.Tensor         # [N,3] float64 final momenta (ASE units: amu * A / ASE time)
    forces: torch.Tensor          # [N,3] fp32 forces of the last evaluation, grad * force_multiplier
    energy: torch.Tensor          # [steps+1,B] fp32 potential energy per evaluation, out * natoms (no bond penalty)
    kinetic_energy: torch.Tensor  # [steps+1,B] float64 kinetic energy per evaluation (eV)
    temperature: torch.Tensor     # [steps+1,B] float64 temperature per evaluation (K)
    atom_offsets: torch.Tensor    # [B+1] int64: atoms of crystal b are rows atom_offsets[b]:atom_offsets[b+1]
    trajectory: Optional[torch.Tensor]   # [T,N,3] float64 positions at evaluations 0, k, 2k, ... <= steps, or None


class NPTResult(NamedTuple):
    positions: torch.Tensor       # [N,3] float64 final Cartesian positions (not wrapped into the cell)
    momenta: torch.Tensor         # [N,3] float64 final momenta (ASE units: amu * A / ASE time)
    forces: torch.Tensor          # [N,3] fp32 forces of the last logged evaluation, grad * force_multiplier
    energy: torch.Tensor          # [steps+1,B] fp32 potential energy per logged evaluation, out * natoms
    kinetic_energy: torch.Tensor  # [steps+1,B] float64 kinetic energy per logged evaluation (eV)
    temperature: torch.Tensor     # [steps+1,B] float64 temperature per logged evaluation (K)
    atom_offsets: torch.Tensor    # [B+1] int64: atoms of crystal b are rows atom_offsets[b]:atom_offsets[b+1]
    trajectory: Optional[torch.Tensor]   # [T,N,3] float64 positions at logged evaluations 0, k, 2k, ..., or None
    cells: torch.Tensor           # [steps+1,B,3,3] float64 the cell of each logged evaluation (rows: lattice vectors)
    stress: torch.Tensor          # [steps+1,B,6] fp32 the calculator's Voigt stress (eV/A^3; xx yy zz yz xz xy)
    pressure: torch.Tensor        # [steps+1,B] float64 -trace/3 of that stress less the ideal-gas term (eV/A^3)


def maxwell_boltzmann_momenta(masses, temperature_K: float, rng=None) -> np.ndarray:
    """Momenta drawn from the Maxwell-Boltzmann distribution at temperature_K, as ASE 3.22.1's
    `MaxwellBoltzmannDistribution(atoms, temperature_K=...)` (what `ForceField.set_momentum_maxwell_boltzmann` calls)
    draws them: xi = rng.standard_normal((n, 3)), p = xi * sqrt(masses * kB*T)[:, None].  masses [n] in amu; rng is a
    numpy Generator or RandomState, or None for the np.random module.  Returns [n,3] float64 for `run_md(momenta=...)`."""
    if rng is None:
        rng = np.random
    masses = np.asarray(masses, dtype=np.float64)
    xi = rng.standard_normal((len(masses), 3))
    return xi * np.sqrt(masses * (KB * temperature_K))[:, np.newaxis]


def _seeds(seed, B: int) -> np.ndarray:
    """[B] uint64: seed + b for one int in [0, 2^63), or B ints in [0, 2^64)."""
    def ok(v, hi):
        return not isinstance(v, (bool, np.bool_)) and isinstance(v, numbers.Integral) and 0 <= int(v) < hi
    if seed is None:
        raise ValueError("nvt_langevin and nvt_andersen need a seed: an int in [0, 2^63) or one int per crystal")
    if np.ndim(seed) == 0:
        if not ok(seed, 2 ** 63):
            raise ValueError(f"seed must be an int in [0, 2^63) or {B} ints in [0, 2^64), got {seed!r}")
        return np.array([int(seed) + b for b in range(B)], dtype=np.uint64)
    s = list(seed)
    if len(s) != B or not all(ok(v, 2 ** 64) for v in s):
        raise ValueError(f"seed must be an int in [0, 2^63) or {B} ints in [0, 2^64), got {seed!r}")
    return np.array([int(v) for v in s], dtype=np.uint64)


def run_md(model, structures, atom_features: torch.Tensor, masses, *, ensemble: str = "nve_velocity_verlet",
           steps: int = 1000, timestep: float = 0.01, temperature_K=300.0, taut: Optional[float] = None, momenta=None,
           trajectory_interval: Optional[int] = None, neighbor_strategy: str = "k-nearest", cutoff: float = 8.0,
           max_neighbors: int = 12, cutoff_extra: float = 3.5, force_multiplier: float = 1.0,
           friction: Optional[float] = None, andersen_prob: float = 0.1, seed=None, pressure=None,
           compressibility=None, taup: float = 1000.0, stress_wt: float = 1.0, externalstress=0.0,
           ttime: Optional[float] = None, pfactor: Optional[float] = None):
    """Run `steps` steps of molecular dynamics on a batch of crystals, the cells fixed: a batched
    `ForceField.run_nve_velocity_verlet(steps=steps)` (ensemble="nve_velocity_verlet", ASE's VelocityVerlet) or
    `run_nvt_berendsen(temperature_K=..., taut=..., steps=steps)` (ensemble="nvt_berendsen", ASE's NVTBerendsen with
    fixcm=True), `run_nvt_langevin(temperature_K=..., friction=...)` (ensemble="nvt_langevin", ASE's Langevin with
    fixcm=True) or `run_nvt_andersen(temperature_K=..., andersen_prob=...)` (ensemble="nvt_andersen", ASE's Andersen
    with fixcm=True).  Returns an `MDResult`.

    model: an `ALIGNNAtomWise` or `eALIGNNAtomWise` in eval mode on a CUDA device, with calculate_gradient=True and
    output_features=1; each crystal gets what it would get run alone.
    structures: sequence of (lattice [3,3], cart_coords [n,3]), as for `neighbors.crystal_graphs_device`;
    atom_features: [sum n, F] on the model's device, in the same atom order; masses: [sum n] in amu, all > 0.
    timestep in fs (the reference's default 0.01); taut in fs, default 100 * timestep (taken as 100 times the
    converted timestep, as ForceField does), and not below timestep; temperature_K: the thermostat's target in K, one
    value or one per crystal (unused by NVE).  momenta: [sum n, 3] in ASE units (amu * A / ASE time), default zero --
    `maxwell_boltzmann_momenta` draws them as `set_momentum_maxwell_boltzmann` does.  Graph options are those of
    `crystal_graphs_device`; force_multiplier as for `relax_structures`.

    MolecularDynamics.irun: evaluate, then `steps` times step and evaluate -- steps + 1 evaluations, and energy, kinetic
    energy and temperature are logged after each.  trajectory_interval=k keeps the positions of evaluations 0, k, 2k,
    ....  Positions are not wrapped into the cell.  A crystal whose positions stop being finite raises RuntimeError
    naming it and the step.

    Langevin and Andersen: friction in 1/fs, finite and >= 0, None for ForceField's 1e-4 in ASE units (exactly);
    andersen_prob in [0, 1] per component and step (ForceField's 0.1).  seed is required: an int in [0, 2^63), crystal
    b drawing the stream of seed + b, or B ints in [0, 2^64), one per crystal.  Nothing is drawn from global state: a
    crystal's trajectory is a function of the arguments and of its own seed, so run alone with that seed it repeats
    its trajectory in the batch bit for bit.  Langevin (fixcm) divides by n - 1 and rejects one-atom crystals.

    NPT Berendsen (ensemble="npt_berendsen"): `run_npt_berendsen(temperature_K=..., taut=..., taup=..., pressure=...,
    compressibility=...)`, ASE's NPTBerendsen with fixcm=True -- the Berendsen thermostat, then the cell and positions
    scaled by mu = 1 - (dt/taup) compressibility / 3 (pressure - P) every step, P the pressure of the calculator's
    stress s = fp32(voigt(stress) * stress_wt / 160.21766208) with the ideal-gas term of the momenta.  pressure in bar
    (any sign) and compressibility in 1/bar (>= 0; 0 switches the barostat off) are required, one value or one per
    crystal; taup in fs (ForceField's 1000 fs); taut None means ForceField's 500 fs here.  The model must compute stress
    (stresswise_weight != 0).  Each step evaluates twice, at the rescaled structure (its forces drive the half-kick)
    and after the drift (logged), so steps + 1 of the 2 steps + 1 evaluations are logged.  Returns an `NPTResult`: the
    MDResult fields plus the cell, the calculator's stress and the pressure of every logged evaluation.  A cell whose
    volume or scale factor stops being finite and > 0 raises RuntimeError naming the crystal and the step.  The
    pressure keywords are ignored by the other ensembles.

    NPT Nose-Hoover (ensemble="npt_nose_hoover"): `run_npt_nose_hoover(temperature_K=..., externalstress=...)`, ASE's
    NPT -- Melchionna's Nose-Hoover thermostat with a Parrinello-Rahman barostat, a central difference in fractional
    coordinates of the cell.  externalstress in eV/A^3 as ASE takes it (ForceField's 0.0): a number s (the stress
    [-s, -s, -s, 0, 0, 0], i.e. a pressure s), a Voigt [6] (xx yy zz yz xz xy) or a symmetric [3,3] for every crystal,
    or [B,6] / [B,3,3] per crystal.  ttime in fs and pfactor in ASE units (amu/A) switch on the thermostat and the
    barostat; both default to None, which is the reference's call (it passes neither), so by default the thermostat and
    barostat are off and the cells do not move.  ASE suggests ttime around 25 fs and pfactor = (ptime * FS)^2 * B, ptime
    in fs (about 75 fs) and B the bulk modulus in eV/A^3.  taut is ignored here: ForceField computes it and never passes
    it.  The model must compute stress.  ASE's NPT needs upper triangular cells (rows a, b, c with b in the yz-plane and
    c along z): another cell raises ValueError naming the crystal; `upper_triangular` rotates structures into that form.
    One model evaluation per step, all steps + 1 logged; returns an `NPTResult`.  A cell, or the matrix beta + I of the
    update, that becomes singular or not finite raises RuntimeError naming the crystal and the step.  The other
    ensembles ignore externalstress, ttime and pfactor."""
    calculator.check_model("run_md", model)
    if ensemble not in ENSEMBLES:
        raise ValueError(f"ensemble must be one of {sorted(ENSEMBLES)}, got {ensemble!r}")
    calculator.check_steps(steps)
    calculator.check_positive("timestep", timestep, "fs")
    if trajectory_interval is not None and (not calculator.integer(trajectory_interval) or trajectory_interval < 1):
        raise ValueError(f"trajectory_interval must be None or an integer >= 1, got {trajectory_interval!r}")
    lats, Xs, dev = calculator.check_batch("run_md", model, structures, atom_features, neighbor_strategy, max_neighbors)
    B = len(Xs)
    sizes = [x.shape[0] for x in Xs]
    aoff = neighbors.ragged_offsets(sizes)
    N = int(aoff[-1])
    m = calculator.host_masses(masses, N)
    p0 = np.zeros((N, 3)) if momenta is None else calculator.host_array(momenta, "momenta", (N, 3))
    dt = float(timestep) * FS
    kind = ENSEMBLES[ensemble]
    T0, taut_ase = None, 0.0
    if kind != ops.MD_NVE:
        t = [temperature_K] * B if np.ndim(temperature_K) == 0 else list(temperature_K)
        if len(t) != B or not all(calculator.real(v) and v > 0 for v in t):
            raise ValueError(f"temperature_K must be a finite number > 0 or {B} of them, got {temperature_K!r}")
        T0 = torch.tensor([float(v) for v in t], dtype=torch.float64, device=dev)
    if kind in (ops.MD_NVT_BERENDSEN, ops.MD_NPT_BERENDSEN):
        if taut is None:                                # ForceField: taut = 100 * self.timestep, in ASE units (NVT)
            taut_ase = NPT_TAUT if kind == ops.MD_NPT_BERENDSEN else 100 * dt
        elif not calculator.real(taut):
            raise ValueError(f"taut must be a finite number (fs), got {taut!r}")
        else:
            taut_ase = float(taut) * FS
        if not taut_ase >= dt:
            raise ValueError(f"taut must not be smaller than timestep, got taut={taut!r} and timestep={timestep!r}")
    if kind in STOCHASTIC:
        seeds = _seeds(seed, B)
        if friction is None:
            fr_ase = LANGEVIN_FRICTION
        elif not calculator.real(friction) or not friction >= 0:
            raise ValueError(f"friction must be a finite number >= 0 (1/fs) or None, got {friction!r}")
        else:
            fr_ase = float(friction) / FS
        if not calculator.real(andersen_prob) or not 0.0 <= andersen_prob <= 1.0:
            raise ValueError(f"andersen_prob must be a number in [0, 1], got {andersen_prob!r}")
        if kind == ops.MD_NVT_LANGEVIN and min(sizes) < 2:
            raise ValueError(f"nvt_langevin needs at least 2 atoms per crystal (fixcm divides by n - 1); crystal "
                             f"{sizes.index(min(sizes))} has 1")
        seeds_d = torch.from_numpy(seeds.view(np.int64)).to(dev)
        vel = torch.zeros(N, 3, device=dev, dtype=torch.float64)
        rnd_vel = torch.zeros(N, 3, device=dev, dtype=torch.float64)

    pos = torch.from_numpy(np.ascontiguousarray(np.concatenate(Xs))).to(dev)
    mom = torch.from_numpy(np.ascontiguousarray(p0)).to(dev)
    m_d = torch.from_numpy(np.ascontiguousarray(m)).to(dev)
    forces = torch.zeros(N, 3, device=dev, dtype=torch.float32)
    status = torch.zeros(B, device=dev, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(dev)
    npt = kind in (ops.MD_NPT_BERENDSEN, ops.MD_NPT_NOSE_HOOVER)
    f64 = dict(dtype=torch.float64, device=dev)
    log = _Log(torch.zeros(steps + 1, B, device=dev, dtype=torch.float32), torch.zeros(steps + 1, B, **f64),
               torch.zeros(steps + 1, B, **f64), torch.zeros(steps + 1, B, 3, 3, **f64) if npt else None,
               torch.zeros(steps + 1, B, 6, device=dev, dtype=torch.float32) if npt else None,
               torch.zeros(steps + 1, B, **f64) if npt else None)
    run = (aoff_d, m_d, T0, pos, mom, forces, status, log)
    kw = dict(steps=int(steps), dt=dt, kB=KB, force_multiplier=float(force_multiplier))
    if kind == ops.MD_NPT_BERENDSEN:
        ens = _npt_berendsen(model, lats, run, taut=taut_ase, pressure=pressure, compressibility=compressibility,
                             taup=taup, stress_wt=stress_wt, **kw)
    elif kind == ops.MD_NPT_NOSE_HOOVER:
        ens = _nose_hoover(model, lats, sizes, run, externalstress=externalstress, ttime=ttime, pfactor=pfactor,
                           stress_wt=stress_wt, **kw)
    elif kind in STOCHASTIC:
        ens = _Ensemble(lambda e, phase, grad, stress: ops.md_thermostat_step(
            grad, aoff_d, m_d, T0, seeds_d, pos, mom, vel, rnd_vel, forces, log.kinetic_energy[e], log.temperature[e],
            status, evaluation=e, ensemble=kind, friction=fr_ase, andersen_prob=float(andersen_prob), **kw),
            False, None, 1, "md_step", None)
    else:
        ens = _Ensemble(lambda e, phase, grad, stress: ops.md_step(
            grad, aoff_d, m_d, T0, pos, mom, forces, log.kinetic_energy[e], log.temperature[e], status, evaluation=e,
            ensemble=kind, taut=taut_ase, **kw), False, None, 1, "md_step", None)
    graph = dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                 cutoff_extra=cutoff_extra)
    traj = _run(model, lats, Xs, atom_features, dev, graph, ens, pos, status, log, int(steps), trajectory_interval)
    base = (pos, mom, forces, log.energy, log.kinetic_energy, log.temperature, aoff_d, traj)
    return MDResult(*base) if ens.cells is None else NPTResult(*base, log.cells, log.stress, log.pressure)


class _Log(NamedTuple):
    """run_md's per-evaluation log, [steps+1, B, ...]: the last three only when the cells move."""
    energy: torch.Tensor
    kinetic_energy: torch.Tensor
    temperature: torch.Tensor
    cells: Optional[torch.Tensor]
    stress: Optional[torch.Tensor]
    pressure: Optional[torch.Tensor]


class _Ensemble(NamedTuple):
    """What run_md's loop needs of an ensemble."""
    launch: Callable          # launch(e, phase, grad, stress): the step kernel after evaluation e (or its phase 1)
    stress: bool              # the logged evaluations need the model's stress
    cells: Optional[torch.Tensor]   # [B,3,3] float64 cells the launches move, or None for fixed cells
    phases: int               # 2: each step also evaluates, unlogged, at the rescaled structure (NPT Berendsen)
    kernel: str               # the kernel the MD_BAD_INPUT message names
    degenerate: Optional[str]   # why a cell is MD_CELL_DEGENERATE, or None where the ensemble has no such status


def _run(model, lats, Xs, atom_features, dev, graph, ens: _Ensemble, pos, status, log: _Log, steps: int,
         trajectory_interval) -> Optional[torch.Tensor]:
    """run_md's loop for every ensemble: per evaluation e one graph build on the current cells and positions, the model
    and the ensemble's launch, then one read-back of the statuses and, unless e == steps, the cells and positions of
    the next evaluation (with `ens.phases` == 2 the step's unlogged evaluation and launch follow, and a second
    read-back).  Returns the trajectory, or None."""
    B = len(Xs)
    sizes = [x.shape[0] for x in Xs]
    host_cells, host_pos = [np.array(c, dtype=np.float64) for c in lats], [x.copy() for x in Xs]
    traj = []
    for e in range(steps + 1):
        log.energy[e], grad, stress, _ = calculator.evaluate(model, list(zip(host_cells, host_pos)), atom_features, dev,
                                                             graph, span="md", stress=ens.stress)
        if trajectory_interval is not None and e % trajectory_interval == 0:
            traj.append(pos.clone())                                         # the positions of evaluation e
        if ens.cells is not None:
            log.cells[e] = ens.cells
        for phase in range(ens.phases if e < steps else 1):
            if phase == 1:                                                   # evaluation A of step e + 1
                _, grad, _, _ = calculator.evaluate(model, list(zip(host_cells, host_pos)), atom_features, dev, graph,
                                                    span="md")
            with ops._span("md_step", 0):
                ens.launch(e, phase, grad, stress)
            # one copy: the statuses and, unless this was the last evaluation, the (cells and) positions of the next
            st = calculator.read_back("md_readback", status, range(B), sizes, host_pos, pos if e < steps else None,
                                      host_cells, ens.cells if phase == 0 and e < steps else None)
            if (st == ops.MD_BAD_INPUT).any():
                raise RuntimeError(f"alignn_b200_{ens.kernel}: the model's forces do not match the crystals' atom counts")
            bad = np.flatnonzero(st == ops.MD_CELL_DEGENERATE)
            if ens.degenerate is not None and bad.size:
                raise RuntimeError(f"run_md: the cell of crystal {int(bad[0])} became degenerate in step {e + 1} "
                                   f"({ens.degenerate})")
            if (st != 0).any():
                raise RuntimeError(f"run_md: the MD kernel reported statuses {st.astype(int).tolist()}")
        if e == steps:
            break
        for b in range(B):
            if not np.isfinite(host_pos[b]).all():
                raise RuntimeError(f"run_md: the positions of crystal {b} are not finite after step {e + 1}")
    return torch.stack(traj) if traj else None


def _per_crystal(v, B: int, name: str, unit: str, ok) -> list:
    vals = [v] * B if np.ndim(v) == 0 else list(v)
    if v is None or len(vals) != B or not all(calculator.real(x) and ok(x) for x in vals):
        raise ValueError(f"npt_berendsen needs {name} ({unit}): a finite number{'' if name == 'pressure' else ' >= 0'} "
                         f"or {B} of them, got {v!r}")
    return [float(x) for x in vals]


def _npt_berendsen(model, lats, run, *, taut, pressure, compressibility, taup, stress_wt, **kw) -> _Ensemble:
    """run_md's NPT Berendsen: per step, phase 0 after the logged evaluation, then evaluation A at the rescaled
    structure and phase 1 (see csrc/md_device.cu)."""
    aoff_d, m_d, T0, pos, mom, forces, status, log = run
    B, dev = len(lats), pos.device
    if model.config.stresswise_weight == 0:
        raise ValueError("run_md(ensemble='npt_berendsen') needs a model that computes stress (stresswise_weight != 0)")
    P0 = _per_crystal(pressure, B, "pressure", "bar", lambda x: True)
    comp = _per_crystal(compressibility, B, "compressibility", "1/bar", lambda x: x >= 0)
    calculator.check_positive("taup", taup, "fs")
    calculator.check_real("stress_wt", stress_wt)
    f64 = dict(dtype=torch.float64, device=dev)
    P0_d = torch.tensor([v * BAR for v in P0], **f64)          # NPTBerendsen: pressure * (1e5 * units.Pascal)
    comp_d = torch.tensor([v / BAR for v in comp], **f64)      # compressibility / (1e5 * units.Pascal)
    cells = torch.from_numpy(np.ascontiguousarray(np.stack(lats))).to(dev)
    kw.update(taut=taut, taup=float(taup) * FS, stress_wt=float(stress_wt))

    def launch(e, phase, grad, stress):
        ops.md_npt_step(grad, stress, aoff_d, m_d, T0, P0_d, comp_d, cells, pos, mom, forces, log.stress[e],
                        log.kinetic_energy[e], log.temperature[e], log.pressure[e], status, evaluation=e, phase=phase,
                        **kw)
    return _Ensemble(launch, True, cells, 2, "md_npt_step",
                     "its volume or the barostat's scale factor is not finite and positive")


def upper_triangular(structures):
    """Rotate each (lattice [3,3], cart_coords [n,3]) rigidly into the cell form ASE's NPT needs: rows a, b, c with c
    along +z, b in the yz-plane (y > 0) and a free, so lattice[1,0] = lattice[2,0] = lattice[2,1] = 0 exactly.  Returns
    (structures, rotations): the rotated (lattice @ R.T, cart_coords @ R.T) pairs and R [B,3,3], each a proper rotation
    (orthogonal, det +1), so distances, angles and the energy are unchanged and forces and stresses rotate with R.
    A cell that is already in this form comes back unchanged (R = I exactly)."""
    out, rots = [], []
    for b, (lat, X) in enumerate(structures):
        L = np.asarray(lat, dtype=np.float64).reshape(3, 3)
        X = np.asarray(X, dtype=np.float64).reshape(-1, 3)
        with np.errstate(divide="ignore", invalid="ignore"):
            ez = L[2] / np.linalg.norm(L[2])
            yb = L[1] - np.dot(L[1], ez) * ez
            ey = yb / np.linalg.norm(yb)
        R = np.stack([np.cross(ey, ez), ey, ez])
        if not np.isfinite(R).all():
            raise ValueError(f"upper_triangular: the lattice vectors b and c of crystal {b} are zero or parallel")
        Lr = L @ R.T
        Lr[1, 0] = Lr[2, 0] = Lr[2, 1] = 0.0
        out.append((Lr, X @ R.T))
        rots.append(R)
    return out, np.stack(rots)


def _external_stress(v, B: int) -> np.ndarray:
    """ASE's NPT.set_stress for every crystal: [B,6] float64 Voigt (xx yy zz yz xz xy), eV/A^3."""
    a = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v
    try:
        a = np.asarray(a, dtype=np.float64)
    except (TypeError, ValueError):
        a = None
    if a is None or not np.isfinite(a).all() or a.shape not in ((), (6,), (3, 3), (B, 6), (B, 3, 3)):
        raise ValueError(f"externalstress must be a finite number, a [6] or symmetric [3,3] array, or [{B},6] / "
                         f"[{B},3,3] per crystal (eV/A^3), got {v!r}")
    if a.ndim == 0:
        s = float(a)
        return np.tile(np.array([-s, -s, -s, 0.0, 0.0, 0.0]), (B, 1))
    if a.shape[-2:] == (3, 3):
        m = a.reshape(-1, 3, 3)
        if not all((x - x.T).max() < 1e-10 for x in m):
            raise ValueError("externalstress: the external stress must be a symmetric tensor")
        a = np.stack([m[:, 0, 0], m[:, 1, 1], m[:, 2, 2], m[:, 1, 2], m[:, 0, 2], m[:, 0, 1]], axis=1)
    return np.array(np.broadcast_to(a.reshape(-1, 6), (B, 6)), order="C")


def _nose_hoover_constants(sizes, T0, ttime, pfactor, cells):
    """ASE's NPT._calculateconstants per crystal, in numpy as ASE computes them: (tfact, pfact, desiredEkin) lists for n
    atoms, kT = kB T0, ttime in ASE time units and pfactor in ASE units (None: 0), pfact frozen at the initial cell."""
    tf, pf, de = [], [], []
    for n, t, h in zip(sizes, T0, cells):
        n, kT = int(n), KB * float(t)
        tf.append(0.0 if ttime is None else 2.0 / (3 * n * kT * ttime * ttime))
        pf.append(0.0 if pfactor is None else 1.0 / (pfactor * np.linalg.det(np.asarray(h, dtype=np.float64))))
        de.append(1.5 * (n - 1) * kT)
    return tf, pf, de


def _nose_hoover(model, lats, sizes, run, *, externalstress, ttime, pfactor, stress_wt, **kw) -> _Ensemble:
    """run_md's ASE NPT: per evaluation e one `md_nose_hoover_step` launch on the model's forces and stress (see
    csrc/md_device.cu)."""
    aoff_d, m_d, T0, pos, mom, forces, status, log = run
    B, N, dev = len(lats), pos.shape[0], pos.device
    if model.config.stresswise_weight == 0:
        raise ValueError("run_md(ensemble='npt_nose_hoover') needs a model that computes stress (stresswise_weight != 0)")
    for b, lat in enumerate(lats):
        if not lat[1, 0] == lat[2, 0] == lat[2, 1] == 0.0:
            raise ValueError(f"run_md(ensemble='npt_nose_hoover'): the cell of crystal {b} is not upper triangular; ASE's "
                             "NPT needs lattice rows a, b, c with b in the yz-plane and c along z "
                             "(alignn_b200.upper_triangular rotates structures into that form)")
    if ttime is not None and not (calculator.real(ttime) and ttime > 0):
        raise ValueError(f"ttime must be None or a finite number > 0 (fs), got {ttime!r}")
    if pfactor is not None and not (calculator.real(pfactor) and pfactor > 0):
        raise ValueError(f"pfactor must be None or a finite number > 0 (ASE units, amu/A), got {pfactor!r}")
    calculator.check_real("stress_wt", stress_wt)
    if externalstress is None and pfactor is not None:
        raise ValueError("run_md(ensemble='npt_nose_hoover'): pfactor needs an externalstress")
    ext = _external_stress(0.0 if externalstress is None else externalstress, B)
    tf, pf, de = _nose_hoover_constants(sizes, T0.cpu().tolist(), None if ttime is None else float(ttime) * FS,
                                        None if pfactor is None else float(pfactor), lats)
    f64 = dict(dtype=torch.float64, device=dev)
    tf_d, pf_d, de_d = (torch.tensor(v, **f64) for v in (tf, pf, de))
    ext_d = torch.from_numpy(ext).to(dev)
    cells = torch.from_numpy(np.ascontiguousarray(np.stack(lats))).to(dev)
    state = torch.zeros(B, ops.MD_NH_STATE, **f64)
    q, q_future = torch.zeros(N, 3, **f64), torch.zeros(N, 3, **f64)
    kw.update(stress_wt=float(stress_wt))

    def launch(e, phase, grad, stress):
        ops.md_nose_hoover_step(grad, stress, aoff_d, m_d, tf_d, pf_d, de_d, ext_d, cells, state, pos, mom, q, q_future,
                                forces, log.stress[e], log.kinetic_energy[e], log.temperature[e], log.pressure[e],
                                status, evaluation=e, **kw)
    return _Ensemble(launch, True, cells, 1, "md_nose_hoover_step",
                     "its determinant, or that of the update's beta + I, is not finite and nonzero")
