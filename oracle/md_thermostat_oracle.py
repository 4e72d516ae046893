"""numpy restatement of the reference's stochastic thermostats, `ForceField.run_nvt_langevin` and
`ForceField.run_nvt_andersen` (alignn/ff/ff.py:444-508), with ASE 3.22.1 and the counter-based noise stream of
csrc/md_noise.cuh: the specification `alignn_b200.run_md(ensemble="nvt_langevin" | "nvt_andersen")` and the kernel
`alignn_b200_md_thermostat_step` are tested against.

ASE sources restated (ase 3.22.1), for one crystal with masses m [n,1] and kT = units.kB * temperature_K:
  ase/md/langevin.py   Langevin(atoms, dt, temperature_K=T, friction=fr, fixcm=True)
      updatevars:  sigma = np.sqrt(2 * T * fr / masses); c1 = dt / 2. - dt * dt * fr / 8.;
                   c2 = dt * fr / 2 - dt * dt * fr * fr / 8.; c3 = np.sqrt(dt) * sigma / 2. - dt**1.5 * fr * sigma / 8.;
                   c5 = dt**1.5 * sigma / (2 * np.sqrt(3)); c4 = fr / 2. * c5
      step:        v = atoms.get_velocities() (p / m); xi = standard_normal((n, 3)); eta = standard_normal((n, 3));
                   rnd_pos = c5 * eta; rnd_vel = c3 * xi - c4 * eta;
                   fixcm: rnd_pos -= rnd_pos.sum(axis=0) / n; rnd_vel -= (rnd_vel * masses).sum(axis=0) / (masses * n);
                          factor = np.sqrt(n / (n - 1.0)); rnd_pos *= factor; rnd_vel *= factor
                   v += c1 * forces / masses - c2 * v + rnd_vel; x = positions;
                   set_positions(x + dt * v + rnd_pos); v = (positions - x - rnd_pos) / dt;
                   forces = get_forces(); v += c1 * forces / masses - c2 * v + rnd_vel; set_momenta(v * masses)
      A one-atom crystal divides by n - 1.0 = 0 (ZeroDivisionError in the reference): rejected here.
  ase/md/andersen.py   Andersen(atoms, dt, temperature_K=T, andersen_prob=prob, fixcm=True)
      boltzmann_random(width, size): x = uniform(size); y = uniform(size);
                   width * np.cos(2 * np.pi * x) * (-2 * np.log(1 - y))**0.5
      step:        v = p / m; fixcm: v += ones * boltzmann_random((kT / sum(masses))**0.5, 3);
                   v += 0.5 * forces / masses * dt;
                   random_velocity = boltzmann_random((kT / masses)**0.5, (n, 3)); chance = random((n, 3));
                   v[chance <= prob] = random_velocity[chance <= prob]; x = positions;
                   fixcm: old_com = get_center_of_mass() ((m @ x) / M); v -= (m . v) / M;
                   set_positions(x + v * dt); fixcm: set_center_of_mass(old_com) (x_new -= com(x_new) - old_com);
                   v = (positions - x) / dt; forces = get_forces(); v += 0.5 * forces / masses * dt;
                   fixcm: v -= (m . v) / M; set_momenta(v * masses)
  ase/md/md.py         MolecularDynamics.irun: evaluate, then `steps` times step and evaluate (oracle/md_oracle.py).
Reference call sites:
  alignn/ff/ff.py:444-475      Langevin(atoms, timestep, temperature_K=300, friction=1e-4): friction in 1 / ASE time
  alignn/ff/ff.py:477-508      Andersen(atoms, timestep, temperature_K=300, andersen_prob=0.1)
  alignn/run_alignn_ff.py:214-228  the nvt_lagevin task

Noise.  ASE draws from numpy's global RNG, which a device cannot reproduce.  Both integrators here take a noise
source instead: `PhiloxNoise(seed)` restates csrc/md_noise.cuh (the stream the kernel draws, keyed by the crystal's seed
and indexed by atom, step, block and thermostat), and `NumpyNoise(rng)` makes ASE's own calls on a numpy Generator or
RandomState in ASE's order.  With PhiloxNoise the normals go through numpy's log / cos / sin rather than CUDA's, so the
device agrees with this restatement to a few ulp per draw, not bitwise.

Conventions and the known difference (forces are fp32 widened to float64 before any product; numpy 1.x would round
`c1 * forces` and `0.5 * forces` to float32) are those of oracle/md_oracle.py.
"""
from __future__ import annotations

import numpy as np

from .fire_oracle import scaled_forces
from .md_oracle import kB, kinetic_energy, temperature

LANGEVIN, ANDERSEN = "nvt_langevin", "nvt_andersen"
TAG = {LANGEVIN: 2, ANDERSEN: 3}          # the counter's thermostat word (the kernel's ensemble codes)
COM_ATOM = 0xFFFFFFFF                     # the atom word of Andersen's per-crystal centre-of-mass draws

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key) -> np.ndarray:
    """Philox4x32-10 (Salmon et al., SC'11; Random123's constants).  counter [..., 4] and key [..., 2] (or [2]), any
    unsigned integers below 2^32; returns [..., 4] uint32."""
    c = [np.asarray(counter, dtype=np.uint64)[..., i] for i in range(4)]
    key = np.asarray(key, dtype=np.uint64)
    k0, k1 = key[..., 0], key[..., 1]
    for r in range(10):
        if r > 0:
            k0 = (k0 + np.uint64(_W0)) & _MASK
            k1 = (k1 + np.uint64(_W1)) & _MASK
        p0 = _M0 * c[0]
        p1 = _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return np.stack(c, axis=-1).astype(np.uint32)


def unit_uniform(hi, lo) -> np.ndarray:
    """(k + 0.5) * 2^-52, k = (hi << 20) | (lo >> 12): exact, strictly inside (0, 1)."""
    k = (np.asarray(hi, dtype=np.uint64) << np.uint64(20)) | (np.asarray(lo, dtype=np.uint64) >> np.uint64(12))
    return (k.astype(np.float64) + 0.5) * 2.0 ** -52


def box_muller(u1, u2):
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2 * np.pi * u2), r * np.sin(2 * np.pi * u2)


def noise_blocks(seed: int, atoms, step: int, blocks: int, tag: int):
    """Blocks 0..blocks-1 of the given atom indices at (seed, step, tag): (words [A, blocks, 4] uint32, uniforms
    [A, blocks, 2], normals [A, blocks, 2])."""
    atoms = np.asarray(atoms, dtype=np.uint64).reshape(-1)
    A = atoms.shape[0]
    ctr = np.empty((A, blocks, 4), dtype=np.uint64)
    ctr[..., 0] = atoms[:, None]
    ctr[..., 1] = step
    ctr[..., 2] = np.arange(blocks, dtype=np.uint64)[None, :]
    ctr[..., 3] = tag
    seed = int(seed)
    w = philox4x32_10(ctr, [seed & 0xFFFFFFFF, seed >> 32])
    u = np.stack([unit_uniform(w[..., 0], w[..., 1]), unit_uniform(w[..., 2], w[..., 3])], axis=-1)
    z = np.stack(box_muller(u[..., 0], u[..., 1]), axis=-1)
    return w, u, z


class PhiloxNoise:
    """The device stream of one crystal (csrc/md_noise.cuh), indexed by the step s (the step that follows
    evaluation s)."""

    def __init__(self, seed: int):
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError("seed must be in [0, 2^64)")
        self.seed = int(seed)

    def langevin(self, step: int, n: int):
        """xi, eta [n,3]: normals 0..2 and 3..5 of each atom."""
        _, _, z = noise_blocks(self.seed, np.arange(n), step, 3, TAG[LANGEVIN])
        z = z.reshape(n, 6)
        return z[:, 0:3], z[:, 3:6]

    def andersen(self, step: int, n: int):
        """(com_x [3], com_y [3]) of the centre-of-mass kick, then per atom x, y, chance [n,3]: uniforms 0..2, 3..5
        and 6..8."""
        _, uc, _ = noise_blocks(self.seed, [COM_ATOM], step, 3, TAG[ANDERSEN])
        uc = uc.reshape(6)
        _, u, _ = noise_blocks(self.seed, np.arange(n), step, 5, TAG[ANDERSEN])
        u = u.reshape(n, 10)
        return uc[0:3], uc[3:6], u[:, 0:3], u[:, 3:6], u[:, 6:9]


class NumpyNoise:
    """ASE's own draws on a numpy Generator or RandomState (or the np.random module), in ASE's order."""

    def __init__(self, rng=None):
        self.rng = np.random if rng is None else rng

    def langevin(self, step: int, n: int):
        xi = self.rng.standard_normal(size=(n, 3))
        eta = self.rng.standard_normal(size=(n, 3))
        return xi, eta

    def andersen(self, step: int, n: int):
        cx = self.rng.uniform(size=3)
        cy = self.rng.uniform(size=3)
        x = self.rng.uniform(size=(n, 3))
        y = self.rng.uniform(size=(n, 3))
        chance = self.rng.random(size=(n, 3))
        return cx, cy, x, y, chance


def boltzmann_random(width, x, y):
    """Andersen.boltzmann_random on the uniforms x, y."""
    return width * np.cos(2 * np.pi * x) * (-2 * np.log(1 - y)) ** 0.5


class Thermostat:
    """One crystal's state: positions and momenta [n,3] float64, masses [n,1] amu, dt in ASE time units, friction in
    1 / ASE time unit; `noise` is a PhiloxNoise or NumpyNoise.  first_half(f) is everything of `step` before the
    evaluation (step index self.step, then incremented), second_half(f) what follows it."""

    def __init__(self, positions, masses, *, ensemble: str, dt: float, temperature_K: float, noise,
                 friction: float = None, andersen_prob: float = None, momenta=None):
        if ensemble not in (LANGEVIN, ANDERSEN):
            raise ValueError(f"unknown ensemble {ensemble!r}")
        self.x = np.array(positions, dtype=np.float64).reshape(-1, 3)
        self.m = np.asarray(masses, dtype=np.float64).reshape(-1, 1)
        if ensemble == LANGEVIN and len(self.x) < 2:
            raise ValueError("Langevin with fixcm divides by n - 1: a crystal needs two atoms")
        self.p = np.zeros_like(self.x) if momenta is None else np.array(momenta, dtype=np.float64).reshape(-1, 3)
        self.ensemble, self.dt, self.noise = ensemble, dt, noise
        self.temp = kB * temperature_K
        self.fr, self.prob = friction, andersen_prob
        self.step = 0
        self.reassigned = 0                 # Andersen: components reassigned so far
        self.v = self.rnd_vel = None
        if ensemble == LANGEVIN:
            self._updatevars()

    def _updatevars(self):
        dt, T, fr, masses = self.dt, self.temp, self.fr, self.m
        sigma = np.sqrt(2 * T * fr / masses)
        self.c1 = dt / 2. - dt * dt * fr / 8.
        self.c2 = dt * fr / 2 - dt * dt * fr * fr / 8.
        self.c3 = np.sqrt(dt) * sigma / 2. - dt**1.5 * fr * sigma / 8.
        self.c5 = dt**1.5 * sigma / (2 * np.sqrt(3))
        self.c4 = fr / 2. * self.c5

    def first_half(self, f) -> None:
        n = len(self.x)
        self.v = self.p / self.m
        if self.ensemble == LANGEVIN:
            xi, eta = self.noise.langevin(self.step, n)
            rnd_pos = self.c5 * eta
            rnd_vel = self.c3 * xi - self.c4 * eta
            rnd_pos -= rnd_pos.sum(axis=0) / n
            rnd_vel -= (rnd_vel * self.m).sum(axis=0) / (self.m * n)
            factor = np.sqrt(n / (n - 1.0))
            rnd_pos *= factor
            rnd_vel *= factor
            self.rnd_vel = rnd_vel
            self.v += self.c1 * f / self.m - self.c2 * self.v + rnd_vel
            x = self.x
            self.x = x + self.dt * self.v + rnd_pos
            self.v = (self.x - x - rnd_pos) / self.dt
        else:
            cx, cy, ux, uy, chance = self.noise.andersen(self.step, n)
            M = self.m.sum()
            self.v += np.ones(self.v.shape) * boltzmann_random((self.temp / M) ** 0.5, cx, cy)
            self.v += 0.5 * f / self.m * self.dt
            random_velocity = boltzmann_random((self.temp / np.repeat(self.m, 3, axis=1)) ** 0.5, ux, uy)
            hit = chance <= self.prob
            self.v[hit] = random_velocity[hit]
            self.reassigned += int(hit.sum())
            x = self.x
            old_com = self.m.ravel() @ x / M
            self.v -= np.dot(self.m.ravel(), self.v) / M
            xn = x + self.v * self.dt
            xn = xn - (self.m.ravel() @ xn / M - old_com)
            self.x = xn
            self.v = (xn - x) / self.dt
        self.step += 1

    def second_half(self, f) -> None:
        if self.ensemble == LANGEVIN:
            self.v += self.c1 * f / self.m - self.c2 * self.v + self.rnd_vel
        else:
            self.v += 0.5 * f / self.m * self.dt
            self.v -= np.dot(self.m.ravel(), self.v) / self.m.sum()
        self.p = self.v * self.m


def _advance(md, rec, e, steps, energy, grad, force_multiplier):
    f = scaled_forces(grad, force_multiplier)
    if e >= 1:
        md.second_half(f.astype(np.float64))
    rec["energy"].append(energy)
    rec["kinetic_energy"].append(kinetic_energy(md.p, md.m.ravel()))
    rec["temperature"].append(temperature(md.p, md.m.ravel()))
    rec["forces"] = f
    if e < steps:
        md.first_half(f.astype(np.float64))


def _result(md, rec, traj, steps):
    return dict(positions=md.x, momenta=md.p, forces=rec["forces"], energy=rec["energy"],
                kinetic_energy=rec["kinetic_energy"], temperature=rec["temperature"], evaluations=steps + 1,
                trajectory=traj, md=md)


def run(evaluate, positions, masses, *, ensemble: str, steps: int, dt: float, temperature_K: float, noise,
        friction: float = None, andersen_prob: float = None, momenta=None, force_multiplier: float = 1.0,
        trajectory_interval: int = None):
    """One crystal: MolecularDynamics.irun, as md_oracle.run.  `evaluate(x) -> (energy, grad)`; `noise` a PhiloxNoise
    (the device's stream) or NumpyNoise.  Returns md_oracle.run's dict; md.reassigned counts Andersen's
    reassignments."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        md = Thermostat(positions, masses, ensemble=ensemble, dt=dt, temperature_K=temperature_K, noise=noise,
                        friction=friction, andersen_prob=andersen_prob, momenta=momenta)
        rec = dict(energy=[], kinetic_energy=[], temperature=[], forces=None)
        traj = [] if trajectory_interval else None
        for e in range(steps + 1):
            if traj is not None and e % trajectory_interval == 0:
                traj.append(md.x.copy())
            energy, grad = evaluate(md.x)
            _advance(md, rec, e, steps, energy, grad, force_multiplier)
    return _result(md, rec, traj, steps)


def run_batch(evaluate_batch, positions, masses, *, ensemble: str, steps: int, dt: float, temperature_K, noises,
              friction: float = None, andersen_prob: float = None, momenta=None, force_multiplier: float = 1.0,
              trajectory_interval: int = None):
    """B independent runs of `run` in lockstep (as md_oracle.run_batch); temperature_K one value or one per crystal,
    noises one source per crystal."""
    if steps < 1:
        raise ValueError("steps must be >= 1")
    B = len(positions)
    T0 = list(temperature_K) if np.ndim(temperature_K) == 1 else [temperature_K] * B
    mom = [None] * B if momenta is None else list(momenta)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        mds = [Thermostat(positions[b], masses[b], ensemble=ensemble, dt=dt, temperature_K=T0[b], noise=noises[b],
                          friction=friction, andersen_prob=andersen_prob, momenta=mom[b]) for b in range(B)]
        recs = [dict(energy=[], kinetic_energy=[], temperature=[], forces=None) for _ in range(B)]
        trajs = [[] if trajectory_interval else None for _ in range(B)]
        for e in range(steps + 1):
            if trajectory_interval and e % trajectory_interval == 0:
                for b in range(B):
                    trajs[b].append(mds[b].x.copy())
            for b, (energy, grad) in enumerate(evaluate_batch([md.x for md in mds])):
                _advance(mds[b], recs[b], e, steps, energy, grad, force_multiplier)
    return [_result(md, r, t, steps) for md, r, t in zip(mds, recs, trajs)]
