"""Relax a batch of crystals with ALIGNN-FF on the GPU: FIRE on the atomic positions, the cells fixed or relaxed too.

The reference relaxes one structure at a time: `ForceField.optimize_atoms(optimizer="FIRE", optimize_lattice=False)`
(alignn/ff/ff.py:373-417) runs ASE's FIRE, and every step its calculator (alignn/ff/calculators.py:280-372) builds g and
L(g) on the CPU, copies them to the GPU, runs the model and copies the forces back for numpy to integrate.  Here all
crystals advance together: per step one device graph build (`neighbors.crystal_graphs_device`) and one model call for
the crystals still running, and one FIRE launch (`ops.fire_step`, csrc/fire_device.cu) that also takes each crystal's
convergence decision.  Each crystal follows the trajectory it would follow relaxed alone and stops on its own test;
`oracle/fire_oracle.py` is the specification (ASE 3.22.1 semantics, float64 state).

With `optimize_lattice=True` the cells relax with the atoms, as the reference's default `optimize_atoms(...,
optimize_lattice=True)` does with ASE's `ExpCellFilter`: each step builds the graphs from the current cells, and
`ops.fire_cell_step` (csrc/fire_cell_device.cu) moves atoms and cells on the forces and the calculator's Voigt stress;
`oracle/cell_filter_oracle.py` is its specification.
"""
from __future__ import annotations

import math
import numbers
from typing import NamedTuple

import numpy as np
import torch

from . import neighbors, ops
from .alignn_atomwise import ALIGNNAtomWise, bond_penalty, cutoff_function_based_edges


class RelaxResult(NamedTuple):
    positions: torch.Tensor      # [N,3] float64 final Cartesian positions (not wrapped into the cell)
    energy: torch.Tensor         # [B] fp32 energy at the final positions, out * natoms (without the bond penalty)
    forces: torch.Tensor         # [N,3] fp32 forces at the final positions, grad * force_multiplier
    nsteps: torch.Tensor         # [B] int32 FIRE steps taken
    converged: torch.Tensor      # [B] bool: max_i |F_i| < fmax at the final positions
    atom_offsets: torch.Tensor   # [B+1] int64: atoms of crystal b are rows atom_offsets[b]:atom_offsets[b+1]


class CellRelaxResult(NamedTuple):
    positions: torch.Tensor      # [N,3] float64 final Cartesian positions (not wrapped into the cell)
    energy: torch.Tensor         # [B] fp32 energy at the final structure, out * natoms (without the bond penalty)
    forces: torch.Tensor         # [N,3] fp32 Cartesian forces at the final structure, grad * force_multiplier
    nsteps: torch.Tensor         # [B] int32 FIRE steps taken
    converged: torch.Tensor      # [B] bool: the filter's test, max over atom and cell rows of |row| < fmax
    atom_offsets: torch.Tensor   # [B+1] int64: atoms of crystal b are rows atom_offsets[b]:atom_offsets[b+1]
    cells: torch.Tensor          # [B,3,3] float64 final lattices, rows are lattice vectors as given
    stress: torch.Tensor         # [B,6] fp32 the calculator's Voigt stress (eV/A^3; xx yy zz yz xz xy) at the end


def _check(model, structures, atom_features, fmax, steps, neighbor_strategy, max_neighbors):
    if not isinstance(model, ALIGNNAtomWise):
        raise ValueError("relax_structures takes an ALIGNNAtomWise model")
    c = model.config
    if model.training:
        raise ValueError("relax_structures needs the model in eval mode (model.eval())")
    if not c.calculate_gradient:
        raise ValueError("relax_structures needs forces: the model has calculate_gradient=False")
    if c.output_features != 1:
        raise ValueError(f"relax_structures needs one energy per crystal, got output_features={c.output_features}")
    if not c.energy_mult_natoms and c.use_penalty:
        # the model adds the whole batch's bond penalty to every crystal's `out` then (DESIGN section 8): a batched
        # energy would depend on the other crystals in the batch
        raise NotImplementedError("relax_structures: energy_mult_natoms=False with use_penalty=True mixes the batch's "
                                  "penalty into every crystal's energy")
    if c.force_mult_natoms:
        # the model multiplies the pair forces by the atoms of the whole batch (alignn_atomwise.py:530-539); the
        # calculator's natoms factor goes into force_multiplier instead
        raise NotImplementedError("relax_structures: force_mult_natoms=True scales forces by the batch's atom count; "
                                  "fold natoms into force_multiplier")
    if isinstance(fmax, bool) or not isinstance(fmax, numbers.Real) or not math.isfinite(fmax) or fmax < 0:
        raise ValueError(f"fmax must be a finite number >= 0, got {fmax!r}")
    if isinstance(steps, bool) or not isinstance(steps, numbers.Integral) or not 1 <= steps <= ops.FIRE_MAX_STEPS:
        raise ValueError(f"steps must be an integer in [1, {ops.FIRE_MAX_STEPS}], got {steps!r}")
    params = list(model.parameters())
    if not params or not all(p.is_cuda for p in params):
        raise ValueError("relax_structures needs the model on a CUDA device (model.to('cuda'))")
    dev = params[0].device
    if not isinstance(atom_features, torch.Tensor) or not atom_features.is_cuda or atom_features.device != dev:
        raise ValueError(f"atom_features must be a tensor on the model's device {dev}")
    lats, Xs = neighbors._checked_structures(structures, neighbor_strategy, max_neighbors)
    n = sum(x.shape[0] for x in Xs)
    if atom_features.dim() != 2 or atom_features.shape[0] != n:
        raise ValueError(f"atom_features has {atom_features.shape[0]} rows for {n} atoms")
    return lats, Xs, dev


def _penalty_pair_grad(model, r: torch.Tensor) -> torch.Tensor:
    """d(bond penalty)/dr per bond, the term `ALIGNNAtomWise` adds to every crystal's energy (alignn_atomwise.py:498-510),
    on the same (possibly enveloped) bond lengths.  Works inside torch.no_grad()."""
    c = model.config
    with torch.enable_grad():
        r = r.detach().requires_grad_(True)
        bl = torch.norm(r, dim=1)
        if c.use_cutoff_function and not c.multiply_cutoff:
            bl = cutoff_function_based_edges(bl, inner_cutoff=c.inner_cutoff, exponent=c.exponent)
        (d,) = torch.autograd.grad(bond_penalty(bl, c).sum(), r)
    return d


def _pair_forces_as_alone(model, g, res, A: int) -> torch.Tensor:
    """The model's pair forces with the bond penalty's gradient counted once per crystal (see `_forces_as_alone`)."""
    c = model.config
    d = _penalty_pair_grad(model, g.edata["r"])
    hit = d.abs().amax(1) > 0
    pf = res["pair_forces"].detach()
    return torch.where(hit.unsqueeze(1), pf - (c.grad_multiplier * (A - 1)) * d, pf).contiguous()


def _forces_as_alone(model, g, res, A: int) -> torch.Tensor:
    """The model's forces with the bond penalty counted once per crystal.  `ALIGNNAtomWise` adds the whole batch's
    penalty to each of the A energies it differentiates with ones, so in a batch every bond's penalty gradient enters
    A times; a crystal relaxed alone (the calculator) sees it once.  Bonds without a penalty keep their pair forces
    bit for bit.  No read-back: the correction and the scatter run whether or not any bond is penalised."""
    c = model.config
    grad = res["grad"].detach().reshape(-1, 3)
    if A == 1 or not c.use_penalty:
        return grad.contiguous()
    return ops.pair_force_scatter(_pair_forces_as_alone(model, g, res, A), g.index, c.add_reverse_forces)


def _forces_and_stress_as_alone(model, g, res, A: int):
    """`_forces_as_alone` and the stress of the same pair forces: with a penalty in a batch the model's stress counts
    it A times too, so the per-crystal virial (the model's own, `ops.virial_stress`) is taken again from the corrected
    pair forces.  Without one the model's `stresses` are used as they are."""
    c = model.config
    if A == 1 or not c.use_penalty:
        return res["grad"].detach().reshape(-1, 3).contiguous(), res["stresses"].detach().reshape(-1, 3, 3).contiguous()
    pf = _pair_forces_as_alone(model, g, res, A)
    grad = ops.pair_force_scatter(pf, g.index, c.add_reverse_forces)
    stress = ops.virial_stress(g.edata["r"].detach(), pf, g.edge_graph_offsets64(), g.node_graph_offsets().long(),
                               g.ndata["V"], c.stress_multiplier)
    return grad, stress


def relax_structures(model, structures, atom_features: torch.Tensor, *, fmax: float = 0.1, steps: int = 100,
                     neighbor_strategy: str = "k-nearest", cutoff: float = 8.0, max_neighbors: int = 12,
                     cutoff_extra: float = 3.5, force_multiplier: float = 1.0, optimize_lattice: bool = False,
                     stress_wt: float = 1.0):
    """Relax the atomic positions of a batch of crystals with FIRE (ASE 3.22.1 defaults), the cells fixed: a batched
    `optimize_atoms(optimizer="FIRE", optimize_lattice=False, fmax=fmax, steps=steps)`.  Returns a `RelaxResult`.
    With optimize_lattice=True the cells relax too (see below) and a `CellRelaxResult` is returned.

    model: an `ALIGNNAtomWise` in eval mode on a CUDA device, with calculate_gradient=True and output_features=1.
    structures: sequence of (lattice [3,3], cart_coords [n,3]), as for `neighbors.crystal_graphs_device`;
    atom_features: [sum n, F] on the model's device, in the same atom order.
    Graph options are those of `crystal_graphs_device` (defaults: the reference's k-nearest, 8 A, 12 neighbours).
    force_multiplier: the calculator's force scaling as one factor, force_multiplier x batch_size (its default
    force_mult_batchsize=True) x natoms (force_mult_natoms); forces are the fp32 product grad * fp32(force_multiplier).

    Per crystal: evaluate, stop if max_i |F_i|^2 < fmax^2 (converged) or after `steps` FIRE steps, else step and
    evaluate again -- at most steps + 1 evaluations.  energy and forces are those of the last evaluation; energy is
    out * natoms and, like the calculator's, does not include the bond penalty whose gradient the forces include.
    Crystals that stop drop out of later graph builds and model calls.  Positions are not wrapped into the cell.

    optimize_lattice=True: the reference's default `optimize_atoms(optimizer="FIRE", optimize_lattice=True)`, FIRE on
    ASE 3.22.1's `ExpCellFilter` -- atoms and cells move together on the forces and the calculator's Voigt stress
    s = fp32(voigt(stress) * stress_wt / 160.21766208) (eV/A^3), and a crystal converges when the largest row of the
    filter's forces (atom rows f_i F and the three cell rows) is below fmax.  The model must compute stress
    (stresswise_weight != 0); optimize_lattice must be a bool.  Every step builds the graphs from the current cells.  The returned forces stay
    Cartesian; `cells` and `stress` are the final lattices and the stress of the last evaluation.  A cell that loses
    its volume raises RuntimeError naming the crystal."""
    lats, Xs, dev = _check(model, structures, atom_features, fmax, steps, neighbor_strategy, max_neighbors)
    if not isinstance(optimize_lattice, (bool, np.bool_)):
        raise ValueError(f"optimize_lattice must be a bool, got {optimize_lattice!r}")
    if isinstance(stress_wt, bool) or not isinstance(stress_wt, numbers.Real) or not math.isfinite(stress_wt):
        raise ValueError(f"stress_wt must be a finite real number, got {stress_wt!r}")
    cell = bool(optimize_lattice)
    if cell and model.config.stresswise_weight == 0:
        # a model built without stress (the reference's calculator gives such a model a stresswise_weight of 0.1 when
        # it builds one itself, but one passed in directly would hand the filter no stress at all)
        raise ValueError("relax_structures(optimize_lattice=True) needs a model that computes stress "
                         "(stresswise_weight != 0)")
    B = len(Xs)
    sizes = [x.shape[0] for x in Xs]
    aoff = neighbors.ragged_offsets(sizes)
    N = int(aoff[-1])
    pos = torch.from_numpy(np.ascontiguousarray(np.concatenate(Xs))).to(dev)
    vel = torch.zeros_like(pos)
    forces = torch.zeros(N, 3, device=dev, dtype=torch.float32)
    energy = torch.zeros(B, device=dev, dtype=torch.float32)
    fstate = torch.tensor([[ops.FIRE_DT0, ops.FIRE_A0]] * B, device=dev, dtype=torch.float64)
    istate = torch.tensor([[0, 1, 0, 0]] * B, device=dev, dtype=torch.int32)   # Nsteps, v is None, steps, status
    aoff_d = torch.from_numpy(aoff).to(dev)
    host_pos = [x.copy() for x in Xs]
    host_cells = lats
    if cell:                                    # the filter's state per crystal: C0, L = 0, F = I, C = C0, cell velocity
        cells0 = torch.from_numpy(np.ascontiguousarray(np.stack(lats))).to(dev)
        cells, logdef = cells0.clone(), torch.zeros_like(cells0)
        defgrad = torch.eye(3, dtype=torch.float64, device=dev).repeat(B, 1, 1)
        cvel, cforces = torch.zeros_like(cells0), torch.zeros_like(cells0)
        stress_out = torch.zeros(B, 6, device=dev, dtype=torch.float32)
        host_cells = [lat.copy() for lat in lats]
    active = list(range(B))
    while active:
        A = len(active)
        rows = torch.from_numpy(np.concatenate([np.arange(aoff[b], aoff[b + 1]) for b in active])).to(dev)
        act = torch.tensor(active, dtype=torch.int32).to(dev)
        with ops._span("relax_build", 0):
            feats = atom_features if A == B else atom_features[rows]
            g, lg, lat = neighbors.crystal_graphs_device([(host_cells[b], host_pos[b]) for b in active], feats,
                                                         neighbor_strategy=neighbor_strategy, cutoff=cutoff,
                                                         max_neighbors=max_neighbors, cutoff_extra=cutoff_extra, device=dev)
        with ops._span("relax_model", 0):
            with torch.enable_grad():
                res = model((g, lg, lat))
                if cell:
                    grad, stress = _forces_and_stress_as_alone(model, g, res, A)
                else:
                    grad = _forces_as_alone(model, g, res, A)
            out = res["out"].detach().reshape(-1)                            # 0-d for a one-crystal batch
            energy[act.long()] = out * g.batch_num_nodes_on_device().to(out.dtype)
        with ops._span("relax_fire", 0):
            if cell:
                ops.fire_cell_step(grad, stress, act, g.node_graph_offsets(), aoff_d, pos, vel, forces, cells0, logdef,
                                   defgrad, cells, cvel, cforces, stress_out, fstate, istate, fmax=float(fmax),
                                   steps=int(steps), force_multiplier=float(force_multiplier), stress_wt=float(stress_wt))
            else:
                ops.fire_step(grad, act, g.node_graph_offsets(), aoff_d, pos, vel, forces, fstate, istate,
                              fmax=float(fmax), steps=int(steps), force_multiplier=float(force_multiplier))
        with ops._span("relax_readback", 0):
            # one copy: the running crystals' status, (their cells,) their positions
            parts = [istate[act.long(), 3].to(torch.float64)] + ([cells[act.long()].reshape(-1)] if cell else [])
            back = torch.cat(parts + [pos[rows].reshape(-1)]).cpu().numpy()
        status = back[:A]
        o = 10 * A if cell else A
        new_pos = back[o:].reshape(-1, 3)
        if cell:
            new_cells = back[A:o].reshape(-1, 3, 3)
            for j, b in enumerate(active):
                host_cells[b] = new_cells[j]
        o = 0
        for b in active:
            host_pos[b] = new_pos[o:o + sizes[b]]
            o += sizes[b]
        if (status == ops.FIRE_BAD_INPUT).any():
            raise RuntimeError(f"alignn_b200_{'fire_cell_step' if cell else 'fire_step'}: the model's forces do not match "
                               "the crystals' atom counts")
        bad = [b for b, s in zip(active, status) if s == ops.FIRE_CELL_DEGENERATE]
        if cell and bad:
            raise RuntimeError(f"relax_structures: the cell of crystal {bad[0]} became degenerate (its volume or "
                               "expm of its log-deformation is not finite and positive)")
        active = [b for b, s in zip(active, status) if s == 0]
    ist = istate.cpu()
    base = (pos, energy, forces, ist[:, 2].to(dev), (ist[:, 3] == 1).to(dev), aoff_d)
    return CellRelaxResult(*base, cells, stress_out) if cell else RelaxResult(*base)
