"""Equation of state and bulk modulus for a batch of crystals with ALIGNN-FF on the GPU.

The reference's `ev_curve` (alignn/ff/ff.py:762-805) works on one crystal at a time: it optionally relaxes it with
`ForceField.optimize_atoms()`, strains it isotropically for each `dx`, builds a new `ForceField` for each strained copy
and calls `unrelaxed_atoms()` (ff.py:365-371) -- a host graph build, a copy and a model call per structure -- then fits
ASE 3.22.1's `EquationOfState(vol, y, eos="murnaghan")` with scipy and reports kv = B / kJ * 1e24 in GPa.  Here all
strained copies of all crystals go through the device graph builder and the model in chunks of at most
`max_batch_atoms` atoms (`single_point`), and one launch of `ops.eos_fit` (csrc/eos_device.cu) fits every crystal's
curve (`fit_eos`).  `oracle/eos_oracle.py` is the specification of the fit.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import numpy as np
import torch

from . import calculator, neighbors, ops
from .phonons import DEFAULT_MAX_BATCH_ATOMS
from .relax import CellRelaxResult, relax_structures

# ase.units (ASE 3.22.1, CODATA 2014): the reference's kv = B / kJ * 1.0e24
_e = 1.6021766208e-19
J = 1 / _e
kJ = 1000 * J

DEFAULT_STRAINS = np.arange(-0.05, 0.05, 0.01)      # the reference's dx: 10 points


class EOSFit(NamedTuple):
    e0: torch.Tensor                 # [R] float64 E0 (eV)
    bulk_modulus: torch.Tensor       # [R] float64 B0 (eV/A^3)
    bp: torch.Tensor                 # [R] float64 B0'
    v0: torch.Tensor                 # [R] float64 V0 (A^3)
    bulk_modulus_gpa: torch.Tensor   # [R] float64 B0 / kJ * 1e24 (GPa)
    status: torch.Tensor             # [R] int32: 0 ok, 1 V0 outside the volumes, 2 no fit, 3 bad input


class SinglePointResult(NamedTuple):
    energy: torch.Tensor             # [B] fp32 out * natoms (without the bond penalty), as `unrelaxed_atoms`
    forces: torch.Tensor             # [N,3] fp32 grad * fp32(force_multiplier)
    atom_offsets: torch.Tensor       # [B+1] int64: atoms of structure b are rows atom_offsets[b]:atom_offsets[b+1]


class EVCurveResult(NamedTuple):
    strains: torch.Tensor            # [S] float64 the isotropic strains e: lattice and positions scaled by 1 + e
    volumes: torch.Tensor            # [B,S] float64 |(a x b) . c| of each strained lattice (A^3)
    energies: torch.Tensor           # [B,S] fp32 out * natoms of each strained copy (eV)
    e0: torch.Tensor                 # [B] float64 fitted E0 (eV)
    bulk_modulus: torch.Tensor       # [B] float64 fitted B0 (eV/A^3)
    bulk_modulus_gpa: torch.Tensor   # [B] float64 the reference's kv (GPa)
    bp: torch.Tensor                 # [B] float64 fitted B0'
    v0: torch.Tensor                 # [B] float64 fitted V0 (A^3)
    status: torch.Tensor             # [B] int32 as EOSFit.status (1: ASE's warning; 2: ASE's curve_fit would raise)
    relaxed: Optional[CellRelaxResult]   # the relaxation with on_relaxed_struct=True, else None


def _eos_form(eos) -> int:
    if not isinstance(eos, str) or eos not in ops.EOS_FORMS:
        raise ValueError(f"eos must be one of {sorted(ops.EOS_FORMS)}, got {eos!r}")
    return ops.EOS_FORMS[eos]


def fit_eos(volumes, energies, eos: str = "murnaghan") -> EOSFit:
    """ASE 3.22.1's `EquationOfState(v, e, eos).fit()` for every row of [R, S] volumes (A^3) and energies (eV), S >= 4,
    in one launch: the least-squares parabola's seed, then Levenberg-Marquardt to the least-squares optimum.  Arrays or
    tensors; CUDA tensors stay on their device, anything else goes to the current CUDA device.  eos: "murnaghan" (the
    reference's), "birchmurnaghan" or "vinet".  Returns an `EOSFit`; rows are not read back, so a bad row does not
    raise: its status says what happened (parameters NaN for statuses 2 and 3)."""
    form = _eos_form(eos)
    dev = None
    for x in (volumes, energies):
        if isinstance(x, torch.Tensor) and x.is_cuda:
            dev = x.device
            break
    if dev is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    v, e = (torch.as_tensor(x.detach() if isinstance(x, torch.Tensor) else np.asarray(x, dtype=np.float64))
            .to(device=dev, dtype=torch.float64).contiguous() for x in (volumes, energies))
    if v.dim() != 2 or v.shape != e.shape or not 4 <= v.shape[1] <= ops.EOS_MAX_POINTS:
        raise ValueError(f"volumes and energies must both be [R, S] with 4 <= S <= {ops.EOS_MAX_POINTS}, got "
                         f"{list(v.shape)} and {list(e.shape)}")
    R = v.shape[0]
    params = torch.empty(R, 4, device=dev, dtype=torch.float64)
    status = torch.empty(R, device=dev, dtype=torch.int32)
    with ops._span("eos_fit", 0):
        ops.eos_fit(v, e, params, status, form=form)
    B = params[:, 1]
    # B / kJ * 1.0e24 as numpy rounds it: a true division (torch divides by a Python number through its reciprocal)
    return EOSFit(params[:, 0], B, params[:, 2], params[:, 3], B / torch.full_like(B, kJ) * 1.0e24, status)


def _check_options(force_multiplier, max_batch_atoms):
    calculator.check_real("force_multiplier", force_multiplier)
    if not calculator.integer(max_batch_atoms) or max_batch_atoms < 1:
        raise ValueError(f"max_batch_atoms must be an integer >= 1, got {max_batch_atoms!r}")


def single_point(model, structures, atom_features: torch.Tensor, *, neighbor_strategy: str = "k-nearest",
                 cutoff: float = 8.0, max_neighbors: int = 12, cutoff_extra: float = 3.5, force_multiplier: float = 1.0,
                 max_batch_atoms: int = DEFAULT_MAX_BATCH_ATOMS) -> SinglePointResult:
    """Energy and forces of every structure of a batch, each as if evaluated alone: a batched
    `ForceField.unrelaxed_atoms()` (alignn/ff/ff.py:365-371).  Returns a `SinglePointResult`.

    model, structures, atom_features and the graph options as for `relax_structures`; force_multiplier as there.
    The structures are packed greedily, in order, into model calls of at most max_batch_atoms atoms, which must hold
    the largest structure.  energy is out * natoms without the bond penalty; the forces count the penalty once per
    structure."""
    calculator.check_model("single_point", model)
    lats, Xs, dev = calculator.check_batch("single_point", model, structures, atom_features, neighbor_strategy,
                                           max_neighbors)
    _check_options(force_multiplier, max_batch_atoms)
    sizes = [x.shape[0] for x in Xs]
    if max_batch_atoms < max(sizes):
        raise ValueError(f"max_batch_atoms must be at least the largest structure, {max(sizes)} atoms, "
                         f"got {max_batch_atoms!r}")
    aoff = neighbors.ragged_offsets(sizes)
    graph = dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                 cutoff_extra=cutoff_extra)
    energy, grad = calculator.evaluate_chunks(model, list(zip(lats, Xs)), lambda j: atom_features[aoff[j]:aoff[j + 1]],
                                              dev, graph, max_batch_atoms=max_batch_atoms, span="single_point")
    forces = grad * torch.tensor(float(force_multiplier), dtype=torch.float32, device=dev)
    return SinglePointResult(energy, forces, torch.from_numpy(aoff).to(dev))


def strained(lattice, positions, strain: float):
    """jarvis' `Atoms.strain_atoms(strain)` restated: the lattice scaled by (1 + strain), fractional coordinates kept,
    as ((1 + strain) * lattice, (1 + strain) * cart) in float64, and the strained lattice's volume |(a x b) . c|."""
    s = 1.0 + float(strain)
    lat = s * np.asarray(lattice, dtype=np.float64)
    return lat, s * np.asarray(positions, dtype=np.float64), abs(float(np.dot(np.cross(lat[0], lat[1]), lat[2])))


def _strains(strains) -> np.ndarray:
    a = strains.detach().cpu().numpy() if isinstance(strains, torch.Tensor) else strains
    try:
        a = np.asarray(a, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError("strains must be a real 1-d array") from None
    if a.ndim != 1 or a.shape[0] < 4 or not np.isfinite(a).all() or not (a > -1).all():
        raise ValueError(f"strains must be a 1-d array of at least 4 finite values > -1, got {strains!r}")
    return a


def ev_curve(model, structures, atom_features: torch.Tensor, *, strains=DEFAULT_STRAINS, eos: str = "murnaghan",
             on_relaxed_struct: bool = False, stress_wt: float = 1.0, fmax: float = 0.1, steps: int = 100,
             neighbor_strategy: str = "k-nearest", cutoff: float = 8.0, max_neighbors: int = 12,
             cutoff_extra: float = 3.5, force_multiplier: float = 1.0,
             max_batch_atoms: int = DEFAULT_MAX_BATCH_ATOMS) -> EVCurveResult:
    """E(V) curves, equation-of-state fits and bulk moduli of a batch of crystals: a batched `ev_curve`.  Returns an
    `EVCurveResult`.

    model, structures, atom_features and the graph options as for `relax_structures`.  strains: the reference's dx,
    at least 4 finite values > -1; copy k of a crystal is ((1 + e_k) * lattice, (1 + e_k) * cart).  eos as for
    `fit_eos`.  on_relaxed_struct=True first relaxes the crystals as the reference's `optimize_atoms()` does --
    `relax_structures(..., optimize_lattice=True, stress_wt=stress_wt, fmax=fmax, steps=steps)` -- and strains the
    relaxed cells and Cartesian positions.  Every strained copy goes through `single_point` (max_batch_atoms must hold
    the largest crystal), then all curves through one `fit_eos` launch.

    Non-finite energies raise RuntimeError naming the crystal.  A crystal whose fit has V0 outside its volumes
    (status 1) or no fit (status 2) does not stop the batch: its status says so."""
    _eos_form(eos)
    calculator.check_model("ev_curve", model)
    lats, Xs, dev = calculator.check_batch("ev_curve", model, structures, atom_features, neighbor_strategy, max_neighbors)
    _check_options(force_multiplier, max_batch_atoms)
    st = _strains(strains)
    calculator.check_bool("on_relaxed_struct", on_relaxed_struct)
    B, S = len(Xs), st.shape[0]
    sizes = [x.shape[0] for x in Xs]
    if max_batch_atoms < max(sizes):
        raise ValueError(f"max_batch_atoms must be at least the largest structure, {max(sizes)} atoms, "
                         f"got {max_batch_atoms!r}")
    graph = dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                 cutoff_extra=cutoff_extra, force_multiplier=force_multiplier)
    relaxed = None
    if on_relaxed_struct:
        relaxed = relax_structures(model, list(zip(lats, Xs)), atom_features, fmax=fmax, steps=steps,
                                   optimize_lattice=True, stress_wt=stress_wt, **graph)
        aoff = neighbors.ragged_offsets(sizes)
        pos = relaxed.positions.cpu().numpy()
        lats = list(relaxed.cells.cpu().numpy())
        Xs = [pos[aoff[b]:aoff[b + 1]] for b in range(B)]

    copies, vols = [], np.empty((B, S), dtype=np.float64)
    for b in range(B):
        for k in range(S):
            lat, x, vols[b, k] = strained(lats[b], Xs[b], st[k])
            copies.append((lat, x))
    aoff = neighbors.ragged_offsets(sizes)
    feats = torch.cat([atom_features[aoff[b]:aoff[b + 1]].repeat(S, 1) for b in range(B)])
    sp = single_point(model, copies, feats, max_batch_atoms=max_batch_atoms, **graph)
    energies = sp.energy.view(B, S)
    bad = (~torch.isfinite(energies)).any(1).nonzero().flatten().tolist()
    if bad:
        raise RuntimeError(f"ev_curve: the energies of crystal {bad[0]} are not finite")
    volumes = torch.from_numpy(vols).to(dev)
    fit = fit_eos(volumes, energies.to(torch.float64), eos)
    return EVCurveResult(torch.from_numpy(st.copy()).to(dev), volumes, energies, fit.e0, fit.bulk_modulus,
                         fit.bulk_modulus_gpa, fit.bp, fit.v0, fit.status, relaxed)
