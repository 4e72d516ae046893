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
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import neighbors, ops
from .relax import _check_batch, _check_model, _evaluate, _forces_and_stress_as_alone, _forces_as_alone, _graphs

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


def _real(x) -> bool:
    return not isinstance(x, bool) and isinstance(x, numbers.Real) and math.isfinite(x)


def _host_array(x, name: str, shape) -> np.ndarray:
    a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x
    try:
        a = np.asarray(a, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a real array of shape {list(shape)}") from None
    if a.shape != tuple(shape) or not np.isfinite(a).all():
        raise ValueError(f"{name} must be a finite array of shape {list(shape)}, got shape {list(a.shape)}")
    return a


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
    _check_model("run_md", model)
    if ensemble not in ENSEMBLES:
        raise ValueError(f"ensemble must be one of {sorted(ENSEMBLES)}, got {ensemble!r}")
    if isinstance(steps, bool) or not isinstance(steps, numbers.Integral) or not 1 <= steps <= ops.FIRE_MAX_STEPS:
        raise ValueError(f"steps must be an integer in [1, {ops.FIRE_MAX_STEPS}], got {steps!r}")
    if not _real(timestep) or not timestep > 0:
        raise ValueError(f"timestep must be a finite number > 0 (fs), got {timestep!r}")
    if trajectory_interval is not None and (isinstance(trajectory_interval, bool) or
                                            not isinstance(trajectory_interval, numbers.Integral) or
                                            trajectory_interval < 1):
        raise ValueError(f"trajectory_interval must be None or an integer >= 1, got {trajectory_interval!r}")
    lats, Xs, dev = _check_batch("run_md", model, structures, atom_features, neighbor_strategy, max_neighbors)
    B = len(Xs)
    sizes = [x.shape[0] for x in Xs]
    aoff = neighbors.ragged_offsets(sizes)
    N = int(aoff[-1])
    m = _host_array(masses, "masses", (N,))
    if not (m > 0).all():
        raise ValueError("masses must all be > 0 (amu)")
    p0 = np.zeros((N, 3)) if momenta is None else _host_array(momenta, "momenta", (N, 3))
    dt = float(timestep) * FS
    kind = ENSEMBLES[ensemble]
    T0, taut_ase = None, 0.0
    if kind != ops.MD_NVE:
        t = [temperature_K] * B if np.ndim(temperature_K) == 0 else list(temperature_K)
        if len(t) != B or not all(_real(v) and v > 0 for v in t):
            raise ValueError(f"temperature_K must be a finite number > 0 or {B} of them, got {temperature_K!r}")
        T0 = torch.tensor([float(v) for v in t], dtype=torch.float64, device=dev)
    if kind in (ops.MD_NVT_BERENDSEN, ops.MD_NPT_BERENDSEN):
        if taut is None:                                # ForceField: taut = 100 * self.timestep, in ASE units (NVT)
            taut_ase = NPT_TAUT if kind == ops.MD_NPT_BERENDSEN else 100 * dt
        elif not _real(taut):
            raise ValueError(f"taut must be a finite number (fs), got {taut!r}")
        else:
            taut_ase = float(taut) * FS
        if not taut_ase >= dt:
            raise ValueError(f"taut must not be smaller than timestep, got taut={taut!r} and timestep={timestep!r}")
    if kind in STOCHASTIC:
        seeds = _seeds(seed, B)
        if friction is None:
            fr_ase = LANGEVIN_FRICTION
        elif not _real(friction) or not friction >= 0:
            raise ValueError(f"friction must be a finite number >= 0 (1/fs) or None, got {friction!r}")
        else:
            fr_ase = float(friction) / FS
        if not _real(andersen_prob) or not 0.0 <= andersen_prob <= 1.0:
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
    if kind == ops.MD_NPT_BERENDSEN:
        return _run_npt(model, lats, Xs, atom_features, aoff, pos, mom, m_d, T0, dev, steps=int(steps), dt=dt,
                        taut=taut_ase, pressure=pressure, compressibility=compressibility, taup=taup,
                        stress_wt=stress_wt, trajectory_interval=trajectory_interval,
                        graph=dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                                   cutoff_extra=cutoff_extra),
                        force_multiplier=float(force_multiplier))
    if kind == ops.MD_NPT_NOSE_HOOVER:
        return _run_nose_hoover(model, lats, Xs, atom_features, aoff, pos, mom, m_d, T0, dev, steps=int(steps), dt=dt,
                                externalstress=externalstress, ttime=ttime, pfactor=pfactor, stress_wt=stress_wt,
                                trajectory_interval=trajectory_interval,
                                graph=dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff,
                                           max_neighbors=max_neighbors, cutoff_extra=cutoff_extra),
                                force_multiplier=float(force_multiplier))
    forces = torch.zeros(N, 3, device=dev, dtype=torch.float32)
    energy = torch.zeros(steps + 1, B, device=dev, dtype=torch.float32)
    ekin = torch.zeros(steps + 1, B, device=dev, dtype=torch.float64)
    temp = torch.zeros(steps + 1, B, device=dev, dtype=torch.float64)
    status = torch.zeros(B, device=dev, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(dev)
    host_pos = [x.copy() for x in Xs]
    traj = []
    for e in range(steps + 1):
        with ops._span("md_build", 0):
            g, lg, lat = _graphs(model, list(zip(lats, host_pos)), atom_features, dev,
                                 neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                                 cutoff_extra=cutoff_extra)
        with ops._span("md_model", 0):
            with torch.enable_grad():
                res = _evaluate(model, g, lg, lat)
                grad = _forces_as_alone(model, g, res, B)
            out = res["out"].detach().reshape(-1)                            # 0-d for a one-crystal batch
            energy[e] = out * g.batch_num_nodes_on_device().to(out.dtype)
        if trajectory_interval is not None and e % trajectory_interval == 0:
            traj.append(pos.clone())                                         # the positions of evaluation e
        with ops._span("md_step", 0):
            if kind in STOCHASTIC:
                ops.md_thermostat_step(grad, aoff_d, m_d, T0, seeds_d, pos, mom, vel, rnd_vel, forces, ekin[e], temp[e],
                                       status, evaluation=e, steps=int(steps), dt=dt, kB=KB, ensemble=kind,
                                       friction=fr_ase, andersen_prob=float(andersen_prob),
                                       force_multiplier=float(force_multiplier))
            else:
                ops.md_step(grad, aoff_d, m_d, T0, pos, mom, forces, ekin[e], temp[e], status, evaluation=e,
                            steps=int(steps), dt=dt, kB=KB, ensemble=kind, taut=taut_ase,
                            force_multiplier=float(force_multiplier))
        with ops._span("md_readback", 0):
            # one copy: the statuses and, unless this was the last evaluation, the positions of the next one
            back = torch.cat([status.to(torch.float64)] + ([pos.reshape(-1)] if e < steps else [])).cpu().numpy()
        if (back[:B] == ops.MD_BAD_INPUT).any():
            raise RuntimeError("alignn_b200_md_step: the model's forces do not match the crystals' atom counts")
        if (back[:B] != 0).any():
            raise RuntimeError(f"run_md: the MD kernel reported statuses {back[:B].astype(int).tolist()}")
        if e == steps:
            break
        new_pos = back[B:].reshape(-1, 3)
        for b in range(B):
            host_pos[b] = new_pos[aoff[b]:aoff[b + 1]]
            if not np.isfinite(host_pos[b]).all():
                raise RuntimeError(f"run_md: the positions of crystal {b} are not finite after step {e + 1}")
    return MDResult(pos, mom, forces, energy, ekin, temp, aoff_d, torch.stack(traj) if traj else None)


def _per_crystal(v, B: int, name: str, unit: str, ok) -> list:
    vals = [v] * B if np.ndim(v) == 0 else list(v)
    if v is None or len(vals) != B or not all(_real(x) and ok(x) for x in vals):
        raise ValueError(f"npt_berendsen needs {name} ({unit}): a finite number{'' if name == 'pressure' else ' >= 0'} "
                         f"or {B} of them, got {v!r}")
    return [float(x) for x in vals]


def _run_npt(model, lats, Xs, atom_features, aoff, pos, mom, m_d, T0, dev, *, steps, dt, taut, pressure,
             compressibility, taup, stress_wt, trajectory_interval, graph, force_multiplier) -> NPTResult:
    """run_md's NPT Berendsen loop: per step, phase 0 after the logged evaluation, then evaluation A at the rescaled
    structure and phase 1 (see csrc/md_device.cu)."""
    B, N = len(Xs), int(aoff[-1])
    if model.config.stresswise_weight == 0:
        raise ValueError("run_md(ensemble='npt_berendsen') needs a model that computes stress (stresswise_weight != 0)")
    P0 = _per_crystal(pressure, B, "pressure", "bar", lambda x: True)
    comp = _per_crystal(compressibility, B, "compressibility", "1/bar", lambda x: x >= 0)
    if not _real(taup) or not taup > 0:
        raise ValueError(f"taup must be a finite number > 0 (fs), got {taup!r}")
    if not _real(stress_wt):
        raise ValueError(f"stress_wt must be a finite real number, got {stress_wt!r}")
    f64 = dict(dtype=torch.float64, device=dev)
    P0_d = torch.tensor([v * BAR for v in P0], **f64)          # NPTBerendsen: pressure * (1e5 * units.Pascal)
    comp_d = torch.tensor([v / BAR for v in comp], **f64)      # compressibility / (1e5 * units.Pascal)
    cells = torch.from_numpy(np.ascontiguousarray(np.stack(lats))).to(dev)
    forces = torch.zeros(N, 3, device=dev, dtype=torch.float32)
    energy = torch.zeros(steps + 1, B, device=dev, dtype=torch.float32)
    ekin, temp, press = (torch.zeros(steps + 1, B, **f64) for _ in range(3))
    cell_log = torch.zeros(steps + 1, B, 3, 3, **f64)
    stress_log = torch.zeros(steps + 1, B, 6, device=dev, dtype=torch.float32)
    status = torch.zeros(B, device=dev, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(dev)
    host_cells, host_pos = [np.array(c, dtype=np.float64) for c in lats], [x.copy() for x in Xs]
    kw = dict(steps=steps, dt=dt, kB=KB, taut=taut, taup=float(taup) * FS, force_multiplier=force_multiplier,
              stress_wt=float(stress_wt))
    traj = []

    def evaluate(with_stress):
        with ops._span("md_build", 0):
            g, lg, lat = _graphs(model, list(zip(host_cells, host_pos)), atom_features, dev, **graph)
        with ops._span("md_model", 0):
            with torch.enable_grad():
                res = _evaluate(model, g, lg, lat)
                if with_stress:
                    return g, res, _forces_and_stress_as_alone(model, g, res, B)
                return g, res, (_forces_as_alone(model, g, res, B), None)

    def read_back(e, phase, with_cells):
        with ops._span("md_readback", 0):
            # one copy: the statuses, then (the cells and) the positions the next graph build needs
            back = torch.cat([status.to(torch.float64)] + ([cells.reshape(-1)] if with_cells else []) +
                             [pos.reshape(-1)]).cpu().numpy()
        st = back[:B]
        if (st == ops.MD_BAD_INPUT).any():
            raise RuntimeError("alignn_b200_md_npt_step: the model's forces do not match the crystals' atom counts")
        bad = np.flatnonzero(st == ops.MD_CELL_DEGENERATE)
        if bad.size:
            raise RuntimeError(f"run_md: the cell of crystal {int(bad[0])} became degenerate in step {e + 1} (its volume "
                               "or the barostat's scale factor is not finite and positive)")
        if (st != 0).any():
            raise RuntimeError(f"run_md: the MD kernel reported statuses {st.astype(int).tolist()}")
        o = B
        if with_cells:
            new_cells = back[B:B + 9 * B].reshape(B, 3, 3)
            o += 9 * B
            for b in range(B):
                host_cells[b] = new_cells[b]
        new_pos = back[o:].reshape(-1, 3)
        for b in range(B):
            host_pos[b] = new_pos[aoff[b]:aoff[b + 1]]
            if phase == 1 and not np.isfinite(host_pos[b]).all():
                raise RuntimeError(f"run_md: the positions of crystal {b} are not finite after step {e + 1}")

    for e in range(steps + 1):
        g, res, (grad, stress) = evaluate(True)                     # logged evaluation e (B of step e)
        out = res["out"].detach().reshape(-1)
        energy[e] = out * g.batch_num_nodes_on_device().to(out.dtype)
        if trajectory_interval is not None and e % trajectory_interval == 0:
            traj.append(pos.clone())
        cell_log[e] = cells
        with ops._span("md_step", 0):
            ops.md_npt_step(grad, stress, aoff_d, m_d, T0, P0_d, comp_d, cells, pos, mom, forces, stress_log[e], ekin[e],
                            temp[e], press[e], status, evaluation=e, phase=0, **kw)
        read_back(e, 0, e < steps)
        if e == steps:
            break
        _, _, (grad, _) = evaluate(False)                           # evaluation A of step e + 1
        with ops._span("md_step", 0):
            ops.md_npt_step(grad, stress, aoff_d, m_d, T0, P0_d, comp_d, cells, pos, mom, forces, stress_log[e], ekin[e],
                            temp[e], press[e], status, evaluation=e, phase=1, **kw)
        read_back(e, 1, False)
    return NPTResult(pos, mom, forces, energy, ekin, temp, aoff_d, torch.stack(traj) if traj else None, cell_log,
                     stress_log, press)


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


def _run_nose_hoover(model, lats, Xs, atom_features, aoff, pos, mom, m_d, T0, dev, *, steps, dt, externalstress,
                     ttime, pfactor, stress_wt, trajectory_interval, graph, force_multiplier) -> NPTResult:
    """run_md's loop for ASE's NPT: per evaluation e one graph build on the current cells, the model with stress and one
    `md_nose_hoover_step` launch (see csrc/md_device.cu)."""
    B, N = len(Xs), int(aoff[-1])
    if model.config.stresswise_weight == 0:
        raise ValueError("run_md(ensemble='npt_nose_hoover') needs a model that computes stress (stresswise_weight != 0)")
    for b, lat in enumerate(lats):
        if not lat[1, 0] == lat[2, 0] == lat[2, 1] == 0.0:
            raise ValueError(f"run_md(ensemble='npt_nose_hoover'): the cell of crystal {b} is not upper triangular; ASE's "
                             "NPT needs lattice rows a, b, c with b in the yz-plane and c along z "
                             "(alignn_b200.upper_triangular rotates structures into that form)")
    if ttime is not None and not (_real(ttime) and ttime > 0):
        raise ValueError(f"ttime must be None or a finite number > 0 (fs), got {ttime!r}")
    if pfactor is not None and not (_real(pfactor) and pfactor > 0):
        raise ValueError(f"pfactor must be None or a finite number > 0 (ASE units, amu/A), got {pfactor!r}")
    if not _real(stress_wt):
        raise ValueError(f"stress_wt must be a finite real number, got {stress_wt!r}")
    if externalstress is None and pfactor is not None:
        raise ValueError("run_md(ensemble='npt_nose_hoover'): pfactor needs an externalstress")
    ext = _external_stress(0.0 if externalstress is None else externalstress, B)
    tf, pf, de = _nose_hoover_constants(np.diff(aoff), T0.cpu().tolist(), None if ttime is None else float(ttime) * FS,
                                        None if pfactor is None else float(pfactor), lats)
    f64 = dict(dtype=torch.float64, device=dev)
    tf_d, pf_d, de_d = (torch.tensor(v, **f64) for v in (tf, pf, de))
    ext_d = torch.from_numpy(ext).to(dev)
    cells = torch.from_numpy(np.ascontiguousarray(np.stack(lats))).to(dev)
    state = torch.zeros(B, ops.MD_NH_STATE, **f64)
    q, q_future = torch.zeros(N, 3, **f64), torch.zeros(N, 3, **f64)
    forces = torch.zeros(N, 3, device=dev, dtype=torch.float32)
    energy = torch.zeros(steps + 1, B, device=dev, dtype=torch.float32)
    ekin, temp, press = (torch.zeros(steps + 1, B, **f64) for _ in range(3))
    cell_log = torch.zeros(steps + 1, B, 3, 3, **f64)
    stress_log = torch.zeros(steps + 1, B, 6, device=dev, dtype=torch.float32)
    status = torch.zeros(B, device=dev, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(dev)
    host_cells, host_pos = [np.array(c, dtype=np.float64) for c in lats], [x.copy() for x in Xs]
    traj = []
    for e in range(steps + 1):
        with ops._span("md_build", 0):
            g, lg, lat = _graphs(model, list(zip(host_cells, host_pos)), atom_features, dev, **graph)
        with ops._span("md_model", 0):
            with torch.enable_grad():
                res = _evaluate(model, g, lg, lat)
                grad, stress = _forces_and_stress_as_alone(model, g, res, B)
            out = res["out"].detach().reshape(-1)
            energy[e] = out * g.batch_num_nodes_on_device().to(out.dtype)
        if trajectory_interval is not None and e % trajectory_interval == 0:
            traj.append(pos.clone())
        cell_log[e] = cells
        with ops._span("md_step", 0):
            ops.md_nose_hoover_step(grad, stress, aoff_d, m_d, tf_d, pf_d, de_d, ext_d, cells, state, pos, mom, q,
                                    q_future, forces, stress_log[e], ekin[e], temp[e], press[e], status, evaluation=e,
                                    steps=steps, dt=dt, kB=KB, force_multiplier=force_multiplier,
                                    stress_wt=float(stress_wt))
        with ops._span("md_readback", 0):
            # one copy: the statuses and, unless this was the last evaluation, the next cells and positions
            back = torch.cat([status.to(torch.float64)] +
                             ([cells.reshape(-1), pos.reshape(-1)] if e < steps else [])).cpu().numpy()
        st = back[:B]
        if (st == ops.MD_BAD_INPUT).any():
            raise RuntimeError("alignn_b200_md_nose_hoover_step: the model's forces do not match the crystals' atom "
                               "counts")
        bad = np.flatnonzero(st == ops.MD_CELL_DEGENERATE)
        if bad.size:
            raise RuntimeError(f"run_md: the cell of crystal {int(bad[0])} became degenerate in step {e + 1} (its "
                               "determinant, or that of the update's beta + I, is not finite and nonzero)")
        if (st != 0).any():
            raise RuntimeError(f"run_md: the MD kernel reported statuses {st.astype(int).tolist()}")
        if e == steps:
            break
        new_cells, new_pos = back[B:10 * B].reshape(B, 3, 3), back[10 * B:].reshape(-1, 3)
        for b in range(B):
            host_cells[b], host_pos[b] = new_cells[b], new_pos[aoff[b]:aoff[b + 1]]
            if not np.isfinite(host_pos[b]).all():
                raise RuntimeError(f"run_md: the positions of crystal {b} are not finite after step {e + 1}")
    return NPTResult(pos, mom, forces, energy, ekin, temp, aoff_d, torch.stack(traj) if traj else None, cell_log,
                     stress_log, press)
