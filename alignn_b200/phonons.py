"""Finite-displacement phonons for a batch of crystals with ALIGNN-FF on the GPU: force constants, band energies, DOS.

The reference computes phonons one structure at a time: `ase_phonon` (alignn/ff/ff.py:1337-1430) runs ASE 3.22.1's
`Phonons` on an N x N x N supercell, evaluating its calculator (alignn/ff/calculators.py:280-372) on the 6n displaced
supercells one after the other -- each a host graph build, a copy to the GPU and a model call -- and then forms the
force constants, the dynamical matrices and their eigenvalues in numpy on the host.  Here every displaced supercell of
every crystal goes through the device graph builder and the model in chunks of at most `max_batch_atoms` atoms, one
launch (`ops.phonon_force_constants`, csrc/phonon_device.cu) turns all forces into force constants, and the q-points
of all crystals with the same number of modes run through `ops.phonon_dynamical_matrix` and `torch.linalg.eigvalsh` in
blocks.  Each crystal gets the result it would get run alone; `oracle/phonon_oracle.py` is the specification.
"""
from __future__ import annotations

import math
from typing import List, NamedTuple, Optional

import numpy as np
import torch

from . import calculator, neighbors, ops

# ase.units (ASE 3.22.1, CODATA 2014): Phonons.band_structure's s, sqrt(eV / A^2 / amu) -> eV
_hbar = 6.626070040e-34 / (2 * math.pi)
_e, _amu = 1.6021766208e-19, 1.660539040e-27
EV_PER_SQRT_EV_A2_AMU = _hbar * 1e10 / math.sqrt(_e * _amu)

DEFAULT_MAX_BATCH_ATOMS = 4096            # atoms per model call: 23 GB peak for the 4 + 4, d = 256 model (DESIGN 13)
EIG_BLOCK_BYTES = 1 << 28                 # D(q) workspace of one eigensolver block
EIG_BLOCK_MATRICES = 16384                # cusolverDnXsyevBatched rejects batches of 32768 3x3 to 24x24 matrices


class PhononResult(NamedTuple):
    force_constants: List[torch.Tensor]            # per crystal [Nc, 3n, 3n] float64, ASE's C_N (eV/A^2)
    dynamical_matrix: List[torch.Tensor]           # per crystal [Nc, 3n, 3n] float64, ASE's D_N (eV/A^2/amu)
    band_energies: Optional[List[torch.Tensor]]    # per crystal [Q_b, 3n] float64 in eV, or None without qpoints
    dos_energies: Optional[torch.Tensor]           # [B, dos_npts] float64 grid (eV), or None without dos_kpts
    dos_weights: Optional[torch.Tensor]            # [B, dos_npts] float64 Gaussian-smeared DOS, or None
    atom_offsets: torch.Tensor                     # [B+1] int64: unit-cell atoms of crystal b


def supercell_cells(supercell):
    """The cells of `atoms * supercell` in ASE's order: [(m0, m1, m2)], m0 outermost and m2 innermost."""
    return [(m0, m1, m2) for m0 in range(supercell[0]) for m1 in range(supercell[1]) for m2 in range(supercell[2])]


def displaced_supercells(lattice, positions, supercell, delta: float):
    """The supercells ASE's `Phonons.run` evaluates, on the host in float64: (lattice [3,3] with rows N_i * cell_i,
    positions [6n, Nc n, 3]).  Cell c holds the n atoms at x + (m0, m1, m2) @ cell; supercell k = 6a + 2i + (sign > 0)
    has atom a of cell 0 moved by sign * delta along direction i (sign -1 then +1).  The undisplaced supercell, which
    ASE also evaluates but never reads, is not built."""
    lat = np.asarray(lattice, dtype=np.float64).reshape(3, 3)
    x = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
    n = x.shape[0]
    cells = supercell_cells(supercell)
    base = np.tile(x, (len(cells), 1))
    for c, m in enumerate(cells):
        base[c * n:(c + 1) * n] += np.dot(m, lat)
    out = np.repeat(base[np.newaxis], 6 * n, axis=0)
    for a in range(n):
        for i in range(3):
            out[6 * a + 2 * i, a, i] = base[a, i] - delta
            out[6 * a + 2 * i + 1, a, i] = base[a, i] + delta
    return np.array([supercell[c] * lat[c] for c in range(3)]), out


def monkhorst_pack(size) -> np.ndarray:
    """ASE's monkhorst_pack: [prod(size), 3] fractional k-points (indices + 0.5) / size - 0.5 in C order."""
    kpts = np.indices(size).transpose((1, 2, 3, 0)).reshape((-1, 3))
    return (kpts + 0.5) / size - 0.5


def _int_triple(v, name):
    if (not isinstance(v, (tuple, list)) or len(v) != 3 or
            any(not calculator.integer(x) or x < 1 for x in v)):
        raise ValueError(f"{name} must be three integers >= 1, got {v!r}")
    return tuple(int(x) for x in v)


def _check(supercell, delta, qpoints, dos_kpts, dos_npts, dos_width, force_multiplier, max_batch_atoms, B):
    sc = _int_triple(supercell, "supercell")
    if int(np.prod(sc)) > ops.PHONON_MAX_CELLS:
        raise ValueError(f"supercell has {int(np.prod(sc))} cells, more than {ops.PHONON_MAX_CELLS}")
    calculator.check_positive("delta", delta, "A")
    calculator.check_real("force_multiplier", force_multiplier)
    kpts = None if dos_kpts is None else _int_triple(dos_kpts, "dos_kpts")
    if not calculator.integer(dos_npts) or dos_npts < 2:
        raise ValueError(f"dos_npts must be an integer >= 2, got {dos_npts!r}")
    calculator.check_positive("dos_width", dos_width, "eV")
    if not calculator.integer(max_batch_atoms):
        raise ValueError(f"max_batch_atoms must be an integer, got {max_batch_atoms!r}")
    qs = None
    if qpoints is not None:
        if isinstance(qpoints, (np.ndarray, torch.Tensor)) or len(qpoints) != B:
            raise ValueError(f"qpoints must be None or a list of {B} arrays of shape [Q_b, 3]")
        qs = []
        for b, q in enumerate(qpoints):
            a = q.detach().cpu().numpy() if isinstance(q, torch.Tensor) else q
            try:
                a = np.asarray(a, dtype=np.float64)
            except (TypeError, ValueError):
                raise ValueError(f"qpoints[{b}] must be a real array of shape [Q_b, 3]") from None
            if a.ndim != 2 or a.shape[1] != 3 or a.shape[0] < 1 or not np.isfinite(a).all():
                raise ValueError(f"qpoints[{b}] must be a finite array of shape [Q_b >= 1, 3], got shape {list(a.shape)}")
            qs.append(np.ascontiguousarray(a))
    return sc, kpts, qs


def _eigvalsh(D: torch.Tensor) -> torch.Tensor:
    """Sorted eigenvalues of a block of Hermitian matrices (upper triangle).  For 3n <= 32 and more than one matrix torch
    calls cuSOLVER's batched solver (cusolverDnXsyevBatched), whose result for a matrix does not depend on the others in
    the block; a single matrix would go to syevd instead, so a block of one is evaluated as two."""
    if D.shape[0] == 1:
        return torch.linalg.eigvalsh(D.expand(2, -1, -1), UPLO="U")[:1]
    return torch.linalg.eigvalsh(D, UPLO="U")


def _energies(w2: torch.Tensor) -> torch.Tensor:
    """-sqrt(|w2|) where w2 < 0, sqrt(w2) elsewhere, in eV."""
    w = torch.sqrt(w2.abs())
    return torch.where(w2 < 0, -w, w) * EV_PER_SQRT_EV_A2_AMU


def phonons(model, structures, atom_features: torch.Tensor, masses, *, supercell=(2, 2, 2), delta: float = 0.01,
            qpoints=None, dos_kpts=(20, 20, 20), dos_npts: int = 100, dos_width: float = 1e-3,
            neighbor_strategy: str = "k-nearest", cutoff: float = 8.0, max_neighbors: int = 12,
            cutoff_extra: float = 3.5, force_multiplier: float = 1.0,
            max_batch_atoms: int = DEFAULT_MAX_BATCH_ATOMS) -> PhononResult:
    """Finite-displacement phonons of a batch of crystals: a batched `ase_phonon` -- ASE 3.22.1's `Phonons(atoms, calc,
    supercell, delta)`, `run()`, `read(acoustic=True)`, `band_structure(q)` and `get_dos(kpts).sample_grid(npts,
    width)`.  Returns a `PhononResult`.

    model: an `ALIGNNAtomWise` or `eALIGNNAtomWise` in eval mode on a CUDA device, with calculate_gradient=True and
    output_features=1.
    structures: sequence of (lattice [3,3], cart_coords [n,3]) unit cells, as for `neighbors.crystal_graphs_device`;
    atom_features: [sum n, F] on the model's device, in the same atom order; masses: [sum n] in amu, all > 0.
    supercell: one (N0, N1, N2) for the batch, at most ops.PHONON_MAX_CELLS cells; delta: the displacement in A.
    qpoints: None, or one finite [Q_b, 3] array per crystal of fractional q-points in the reciprocal basis of its unit
    cell (ASE's `path.kpts`); band_energies[b] are then the sorted band energies there in eV, an imaginary frequency
    given as a negative energy.  dos_kpts: the Monkhorst-Pack mesh of the DOS, or None for no DOS; every band energy on
    it gets weight 1 and a Gaussian of width dos_width (eV) on dos_npts points from min - 3 width to max + 3 width.
    Graph options are those of `crystal_graphs_device`; force_multiplier as for `relax_structures`.
    max_batch_atoms: the most atoms one model call takes, at least the largest supercell (Nc n).

    A crystal whose forces are not finite raises RuntimeError naming it."""
    calculator.check_model("phonons", model)
    lats, Xs, dev = calculator.check_batch("phonons", model, structures, atom_features, neighbor_strategy, max_neighbors)
    B = len(Xs)
    sc, kpts, qs = _check(supercell, delta, qpoints, dos_kpts, dos_npts, dos_width, force_multiplier, max_batch_atoms, B)
    sizes = [x.shape[0] for x in Xs]
    aoff = neighbors.ragged_offsets(sizes)
    m = calculator.host_masses(masses, int(aoff[-1]))
    Nc = int(np.prod(sc))
    if max_batch_atoms < Nc * max(sizes):
        raise ValueError(f"max_batch_atoms must be at least the largest supercell, {Nc * max(sizes)} atoms, "
                         f"got {max_batch_atoms!r}")
    delta = float(delta)

    # ---- forces of every displaced supercell, in chunks of at most max_batch_atoms atoms
    with ops._span("phonon_build", 0):
        sets = [displaced_supercells(lat, x, sc, delta) for lat, x in zip(lats, Xs)]
        tiled = [atom_features[aoff[b]:aoff[b + 1]].repeat(Nc, 1) for b in range(B)]
    roff = neighbors.ragged_offsets([6 * n * Nc * n for n in sizes])
    jobs = [(b, k) for b in range(B) for k in range(6 * sizes[b])]
    graph = dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                 cutoff_extra=cutoff_extra)
    _, grad_all = calculator.evaluate_chunks(model, [(sets[b][0], sets[b][1][k]) for b, k in jobs],
                                             lambda j: tiled[jobs[j][0]], dev, graph, max_batch_atoms=max_batch_atoms,
                                             span="phonon")

    # ---- force constants: one launch
    foff = neighbors.ragged_offsets([Nc * 9 * n * n for n in sizes])
    C_all = torch.empty(int(foff[-1]), device=dev, dtype=torch.float64)
    D_all = torch.empty_like(C_all)
    status = torch.zeros(B, device=dev, dtype=torch.int32)
    aoff_d, foff_d = torch.from_numpy(aoff).to(dev), torch.from_numpy(foff).to(dev)
    with ops._span("phonon_fc", 0):
        ops.phonon_force_constants(grad_all, aoff_d, torch.from_numpy(roff).to(dev), foff_d,
                                   torch.from_numpy(np.ascontiguousarray(m)).to(dev), C_all, D_all, status,
                                   supercell=sc, delta=delta, force_multiplier=float(force_multiplier))
    st = status.cpu().numpy()
    for b in range(B):
        if st[b] == ops.PHONON_NON_FINITE:
            raise RuntimeError(f"phonons: the forces of crystal {b} are not finite")
        if st[b] != 0:
            raise RuntimeError("alignn_b200_phonon_force_constants: the force buffer does not match the crystals")
    shape = lambda b: (Nc, 3 * sizes[b], 3 * sizes[b])       # noqa: E731
    C_N = [C_all[foff[b]:foff[b + 1]].view(shape(b)) for b in range(B)]
    D_N = [D_all[foff[b]:foff[b + 1]].view(shape(b)) for b in range(B)]

    # ---- D(q) and its eigenvalues: the band q-points and the DOS mesh of all crystals with the same mode count
    mesh = None if kpts is None else monkhorst_pack(kpts)
    bands = [None] * B if qs is not None else None
    mesh_w2 = [None] * B
    for n in sorted(set(sizes)):
        M = 3 * n
        group = [b for b in range(B) if sizes[b] == n]
        parts, owners = [], []                                     # owners: (b, "band" | "mesh", count)
        for b in group:
            if qs is not None:
                parts.append(qs[b])
                owners.append((b, "band", qs[b].shape[0]))
            if mesh is not None:
                parts.append(mesh)
                owners.append((b, "mesh", mesh.shape[0]))
        if not parts:
            continue
        q_all = torch.from_numpy(np.ascontiguousarray(np.concatenate(parts))).to(dev)
        c_all = torch.from_numpy(np.concatenate([np.full(cnt, b, dtype=np.int32) for b, _, cnt in owners])).to(dev)
        P = q_all.shape[0]
        w2 = torch.empty(P, M, device=dev, dtype=torch.float64)
        blk = max(1, min(P, EIG_BLOCK_MATRICES, EIG_BLOCK_BYTES // (16 * M * M)))
        Dq = torch.empty(blk, M, M, device=dev, dtype=torch.complex128)
        for s in range(0, P, blk):
            e = min(P, s + blk)
            with ops._span("phonon_dynmat", 0):
                ops.phonon_dynamical_matrix(D_all, foff_d, c_all[s:e], q_all[s:e], Dq[:e - s], status, supercell=sc,
                                            modes=M)
            with ops._span("phonon_eig", 0):
                w2[s:e] = _eigvalsh(Dq[:e - s])
        o = 0
        for b, kind, cnt in owners:
            if kind == "band":
                bands[b] = _energies(w2[o:o + cnt])
            else:
                mesh_w2[b] = w2[o:o + cnt]
            o += cnt
    if (status != 0).any():
        raise RuntimeError("alignn_b200_phonon_dynamical_matrix: the dynamical matrices do not match the crystals")

    # ---- DOS: RawDOSData(energies, ones).sample_grid(dos_npts, width=dos_width), per crystal
    dos_e = dos_w = None
    if mesh is not None:
        dos_e = torch.empty(B, dos_npts, device=dev, dtype=torch.float64)
        dos_w = torch.zeros(B, dos_npts, device=dev, dtype=torch.float64)
        width = float(dos_width)
        norm = math.sqrt(2 * math.pi) * width
        ramp = torch.arange(dos_npts, device=dev, dtype=torch.float64)
        with ops._span("phonon_dos", 0):
            for b in range(B):
                en = _energies(mesh_w2[b]).reshape(-1)
                start, stop = en.min() - 3 * width, en.max() + 3 * width
                grid = ramp * ((stop - start) / (dos_npts - 1)) + start     # np.linspace's arithmetic
                grid[-1] = stop
                dos_e[b] = grid
                for s in range(0, en.numel(), 32768):
                    x1 = -0.5 * ((grid[None, :] - en[s:s + 32768, None]) / width) ** 2
                    dos_w[b] += (torch.exp(x1) / norm).sum(0)
    return PhononResult(C_N, D_N, bands, dos_e, dos_w, aoff_d)
