"""numpy restatement of the reference's finite-displacement phonons, `ase_phonon` (alignn/ff/ff.py:1337-1430), with ASE
3.22.1's `Phonons` (the version alignn's environment.yml pins): the specification `alignn_b200.phonons` and the kernels
`alignn_b200_phonon_force_constants` / `alignn_b200_phonon_dynamical_matrix` are tested against.

ASE sources restated (ase 3.22.1):
  ase/atoms.py       Atoms.__mul__ / repeat: cell c = (m0, m1, m2), m0 outermost and m2 innermost, holds a contiguous
                     block of n atoms at x + (m0, m1, m2) @ cell; the supercell lattice has rows N_i * cell_i
  ase/phonons.py     Displacement.run with center_refcell=False (offset 0: the displaced atoms are rows 0..n-1): for atom
                     a, direction i in x, y, z, sign -1 then +1, positions[a, i] = pos[a, i] + sign * delta -- 6n
                     evaluations.  ASE also evaluates the undisplaced supercell first; `read` never uses that result,
                     so it is skipped here.
                     Phonons.read(acoustic=True) with its defaults method='frederiksen', symmetrize=3, cutoff=None:
                     f[a] -= f.sum(0) on each displaced force set, C_av = (f_minus - f_plus) / (2 delta), reshaped to
                     C_N [N_cells, 3n, 3n] (unit-cell index first), then three rounds of symmetrize and acoustic, and
                     D_N = C_N * outer(m^-1/2, m^-1/2) with each mass repeated three times.
                     Phonons.symmetrize: fftshift over the cell axes, i, j, k = 1 - N % 2, C[i:, j:, k:] *= 0.5 and
                     += its reversed-and-transposed copy, ifftshift (for even N the first slab is left out).
                     Phonons.acoustic: from a copy of C_N, subtract the sum over all cells and all a' of block (a, a')
                     from the (offset, a, a) diagonal block.
                     Phonons.lattice_vectors: R = indices(N).reshape(3, -1), (R + N // 2) % N - N // 2 (so for N = 2
                     cell 1 sits at R = -1).
                     Phonons.band_structure(path_kc, modes=False): D(q) = sum_R exp(-2 pi i q.R) D_N[R],
                     eigvalsh(D(q), UPLO='U'), sorted; a negative omega^2 becomes -sqrt(|omega^2|); times
                     s = _hbar * 1e10 / sqrt(_e * _amu) for eV.  q is fractional, in the reciprocal basis of the unit
                     cell (ASE's path.kpts).
                     Phonons.get_dos(kpts): the band energies on monkhorst_pack(kpts), every one with weight 1.
  ase/dft/kpoints.py monkhorst_pack(size) = (indices(size) + 0.5) / size - 0.5, in C order.
  ase/dft/dos.py     RawDOSData.sample_grid(npts, width) (padding 3, smearing 'Gauss'): grid linspace(min - 3w,
                     max + 3w, npts), each energy adding exp(-0.5 ((x - e) / w)^2) / (sqrt(2 pi) w) times its weight.
  ase/units.py       CODATA 2014: _hbar = 6.626070040e-34 / (2 pi), _e = 1.6021766208e-19, _amu = 1.660539040e-27.
Reference call sites:
  alignn/ff/ff.py:1337-1352  ase_phonon(N=2, npoints=100, delta=0.01, use_cvn=True, force_multiplier=1)
  alignn/ff/ff.py:1388-1396  Phonons(atoms, calc, supercell=(N, N, N), delta=delta); run(); read(acoustic=True);
                             get_band_structure(path); get_dos(kpts=(20, 20, 20)).sample_grid(npts=npoints, width=1e-3)

Conventions kept here, and by the device path (those of oracle/fire_oracle.py and oracle/md_oracle.py):
  * forces are the calculator's fp32 product grad * fp32(force_multiplier), widened to float64 -- the force function
    given to `run` returns them; analytic force fields return float64 directly;
  * masses are in amu, force constants in eV/A^2, band energies in eV.
Known difference: ASE's JSON cache keeps the calculator's float32 force arrays, so the reference takes the Frederiksen
sum and the central difference in float32.  As the half-kick rounding in md_oracle, that is not reproduced: both are
float64 here.
"""
from __future__ import annotations

import math

import numpy as np

# ase.units, CODATA 2014 (ASE 3.22.1's default)
_hplanck = 6.626070040e-34
_hbar = _hplanck / (2 * math.pi)
_e = 1.6021766208e-19
_amu = 1.660539040e-27
EV_PER_SQRT_EV_A2_AMU = _hbar * 1e10 / math.sqrt(_e * _amu)   # Phonons.band_structure's s: sqrt(eV/A^2/amu) -> eV

NUM_ROUNDS = 3                                                # read(symmetrize=3)


def supercell(lattice, positions, N):
    """`atoms * N`: (lattice [3,3] with rows N_i * cell_i, positions [Nc * n, 3]), cell c = (m0, m1, m2) in C order
    holding the block of n atoms at x + (m0, m1, m2) @ cell."""
    lat = np.asarray(lattice, dtype=np.float64).reshape(3, 3)
    x = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
    n = x.shape[0]
    M = int(np.prod(N))
    pos = np.tile(x, (M, 1))
    i0 = 0
    for m0 in range(N[0]):
        for m1 in range(N[1]):
            for m2 in range(N[2]):
                pos[i0:i0 + n] += np.dot((m0, m1, m2), lat)
                i0 += n
    return np.array([N[c] * lat[c] for c in range(3)]), pos


def displacements(n):
    """The order Displacement.run evaluates: (a, i, sign) for atom a, direction i, sign -1 then +1."""
    return [(a, i, s) for a in range(n) for i in range(3) for s in (-1, 1)]


def displaced_supercells(lattice, positions, N, delta):
    """(supercell lattice, [6n, Nc * n, 3] positions): the supercell with atom a of the reference cell (rows 0..n-1)
    moved by sign * delta along i, in `displacements` order."""
    latN, pos = supercell(lattice, positions, N)
    n = np.asarray(positions).reshape(-1, 3).shape[0]
    out = np.empty((6 * n,) + pos.shape)
    for k, (a, i, s) in enumerate(displacements(n)):
        out[k] = pos
        out[k, a, i] = pos[a, i] + s * delta
    return latN, out


def lattice_vectors(N):
    """Phonons.lattice_vectors with offset 0: [3, Nc] integer cell vectors in cell order."""
    R = np.indices(N).reshape(3, -1)
    Nc = np.array(N)[:, np.newaxis]
    R += Nc // 2
    R %= Nc
    R -= Nc // 2
    return R


def symmetrize(C_N, N):
    """Phonons.symmetrize with offset 0."""
    m = C_N.shape[1]
    C = C_N.reshape(tuple(N) + (m, m))
    C = np.fft.fftshift(C, axes=(0, 1, 2)).copy()
    i, j, k = 1 - np.asarray(N) % 2
    C[i:, j:, k:] *= 0.5
    C[i:, j:, k:] += C[i:, j:, k:][::-1, ::-1, ::-1].transpose(0, 1, 2, 4, 3).copy()
    C = np.fft.ifftshift(C, axes=(0, 1, 2)).copy()
    return C.reshape((-1, m, m))


def acoustic(C_N, n):
    """Phonons.acoustic with offset 0, in place."""
    C_N_temp = C_N.copy()
    for C in C_N_temp:
        for a in range(n):
            for a_ in range(n):
                C_N[0, 3 * a:3 * a + 3, 3 * a:3 * a + 3] -= C[3 * a:3 * a + 3, 3 * a_:3 * a_ + 3]


def force_constants(forces, masses, N, delta, rounds: int = NUM_ROUNDS):
    """Phonons.read(acoustic=True): forces [6n, Nc * n, 3] of the displaced supercells in `displacements` order (float64;
    not modified), masses [n] amu.  Returns (C_N, D_N), each [Nc, 3n, 3n] float64."""
    f_all = np.asarray(forces, dtype=np.float64)
    m = np.asarray(masses, dtype=np.float64).reshape(-1)
    n = m.shape[0]
    Nc = int(np.prod(N))
    assert f_all.shape == (6 * n, Nc * n, 3), f_all.shape
    C_xNav = np.empty((3 * n, Nc, n, 3))
    for a in range(n):
        for i in range(3):
            fminus = f_all[6 * a + 2 * i].copy()
            fplus = f_all[6 * a + 2 * i + 1].copy()
            fminus[a] -= fminus.sum(0)                              # method='frederiksen'
            fplus[a] -= fplus.sum(0)
            C_av = fminus - fplus
            C_av /= 2 * delta
            C_xNav[3 * a + i] = C_av.reshape((Nc, n, 3))
    C_N = C_xNav.swapaxes(0, 1).reshape((Nc, 3 * n, 3 * n))
    for _ in range(rounds):
        C_N = symmetrize(C_N, N)
        acoustic(C_N, n)
    D_N = C_N.copy()
    m_inv_x = np.repeat(m ** -0.5, 3)
    M_inv = np.outer(m_inv_x, m_inv_x)
    for D in D_N:
        D *= M_inv
    return C_N, D_N


def dynamical_matrix(D_N, N, q):
    """D(q) = sum_R exp(-2 pi i q.R) D_N[R] as band_structure forms it, complex128 [3n, 3n]."""
    phase_N = np.exp(-2.j * np.pi * np.dot(np.asarray(q, dtype=np.float64), lattice_vectors(N)))
    return np.sum(phase_N[:, np.newaxis, np.newaxis] * D_N, axis=0)


def omega2(D_N, N, qpoints):
    """[Q, 3n] sorted eigenvalues of D(q) (eigvalsh with UPLO='U'), in eV/A^2/amu."""
    return np.array([np.sort(np.linalg.eigvalsh(dynamical_matrix(D_N, N, q), UPLO="U"))
                     for q in np.asarray(qpoints, dtype=np.float64).reshape(-1, 3)]).reshape(-1, D_N.shape[1])


def energies_from_omega2(w2):
    """Band energies in eV: sqrt(omega^2), -sqrt(|omega^2|) where omega^2 < 0, times s."""
    w2 = np.asarray(w2, dtype=np.float64)
    w = np.sqrt(w2.astype(complex))
    neg = w2 < 0
    w[neg] = -1 * np.sqrt(np.abs(w2[neg]))
    return (EV_PER_SQRT_EV_A2_AMU * w).real


def band_structure(D_N, N, qpoints):
    """Phonons.band_structure(qpoints): [Q, 3n] band energies in eV."""
    return energies_from_omega2(omega2(D_N, N, qpoints))


def monkhorst_pack(size):
    """ase.dft.kpoints.monkhorst_pack: [prod(size), 3] fractional k-points."""
    if np.less_equal(size, 0).any():
        raise ValueError(f"Illegal size: {list(size)}")
    kpts = np.indices(size).transpose((1, 2, 3, 0)).reshape((-1, 3))
    return (kpts + 0.5) / size - 0.5


def sample_grid(energies, npts: int, width: float, chunk: int = 16384):
    """RawDOSData(energies, ones).sample_grid(npts, width=width): (grid [npts], weights [npts]).  The per-energy sum runs
    in _sample's order, one energy after the other (chunked through np.add.reduce along the energy axis)."""
    e = np.asarray(energies, dtype=np.float64).ravel()
    grid = np.linspace(e.min() - 3 * width, e.max() + 3 * width, npts)
    w = np.zeros(npts)
    for s in range(0, e.size, chunk):
        x1 = -0.5 * ((grid[np.newaxis, :] - e[s:s + chunk, np.newaxis]) / width) ** 2
        delta = np.exp(x1) / (np.sqrt(2 * np.pi) * width)
        w = np.add.reduce(np.concatenate([w[np.newaxis], 1.0 * delta]), axis=0)
    return grid, w


def postprocess(forces, masses, N, delta, qpoints=None, dos_kpts=None, dos_npts: int = 100, dos_width: float = 1e-3):
    """Everything after the force evaluations for one crystal: a dict with C_N, D_N, band_energies (or None),
    omega2 (of the q-points, or None), dos_energies and dos_weights (or None)."""
    C_N, D_N = force_constants(forces, masses, N, delta)
    out = dict(C_N=C_N, D_N=D_N, omega2=None, band_energies=None, dos_energies=None, dos_weights=None)
    if qpoints is not None:
        out["omega2"] = omega2(D_N, N, qpoints)
        out["band_energies"] = energies_from_omega2(out["omega2"])
    if dos_kpts is not None:
        out["dos_energies"], out["dos_weights"] = sample_grid(band_structure(D_N, N, monkhorst_pack(dos_kpts)),
                                                              dos_npts, dos_width)
    return out


def run(forces_fn, lattice, positions, masses, *, N=(2, 2, 2), delta: float = 0.01, **post):
    """One crystal: Phonons.run then the post-processing.  `forces_fn(lattice_N, positions_N) -> [Nc * n, 3]` is the
    calculator on one displaced supercell.  `post` goes to `postprocess`."""
    latN, disp = displaced_supercells(lattice, positions, N, delta)
    forces = np.stack([np.asarray(forces_fn(latN, x), dtype=np.float64).reshape(-1, 3) for x in disp])
    return postprocess(forces, masses, N, delta, **post)


def run_batch(forces_batch_fn, lattices, positions, masses, *, N=(2, 2, 2), delta: float = 0.01, qpoints=None, **post):
    """B crystals: every displaced supercell of every crystal is evaluated in one call of
    `forces_batch_fn([(lattice_N, positions_N)]) -> [forces]`, then each crystal is post-processed on its own.
    qpoints is None or one [Q_b, 3] array per crystal."""
    sets = [displaced_supercells(lat, x, N, delta) for lat, x in zip(lattices, positions)]
    flat = [(latN, x) for latN, disp in sets for x in disp]
    got = forces_batch_fn(flat)
    out, k = [], 0
    for b, (latN, disp) in enumerate(sets):
        f = np.stack([np.asarray(g, dtype=np.float64).reshape(-1, 3) for g in got[k:k + len(disp)]])
        k += len(disp)
        out.append(postprocess(f, masses[b], N, delta, qpoints=None if qpoints is None else qpoints[b], **post))
    return out
