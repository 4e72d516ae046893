"""Evaluate a batch of crystals with ALIGNN-FF on the GPU, each crystal as if alone: the batched counterpart of the
reference's calculator (alignn/ff/calculators.py:280-372), shared by the relaxation, MD, phonon and equation-of-state
drivers.

The reference builds g and L(g) of one structure on the CPU, copies them to the GPU and runs the model.  Here one
device graph build (`neighbors.crystal_graphs_device`) and one model call cover a batch, and `evaluate` returns what
the calculator would return for every crystal alone.  The model is an `ALIGNNAtomWise` or an `eALIGNNAtomWise`: eALIGNN
is evaluated through its per-crystal mode (DESIGN section 19), ALIGNNAtomWise through its forward plus the bond-penalty
correction.  This module also holds the model, batch and argument checks the drivers share and their one read-back.
"""
from __future__ import annotations

import math
import numbers

import numpy as np
import torch

from . import neighbors, ops
from .alignn_atomwise import ALIGNNAtomWise, bond_penalty, cutoff_function_based_edges
from .ealignn_atomwise import eALIGNNAtomWise


def real(x) -> bool:
    """x is a finite real number (not a bool)."""
    return not isinstance(x, bool) and isinstance(x, numbers.Real) and math.isfinite(x)


def integer(x) -> bool:
    """x is an integer (not a bool)."""
    return not isinstance(x, bool) and isinstance(x, numbers.Integral)


def check_real(name: str, x) -> None:
    if not real(x):
        raise ValueError(f"{name} must be a finite real number, got {x!r}")


def check_positive(name: str, x, unit: str) -> None:
    if not real(x) or not x > 0:
        raise ValueError(f"{name} must be a finite number > 0 ({unit}), got {x!r}")


def check_bool(name: str, x) -> None:
    if not isinstance(x, (bool, np.bool_)):
        raise ValueError(f"{name} must be a bool, got {x!r}")


def check_steps(steps) -> None:
    if not integer(steps) or not 1 <= steps <= ops.FIRE_MAX_STEPS:
        raise ValueError(f"steps must be an integer in [1, {ops.FIRE_MAX_STEPS}], got {steps!r}")


def host_array(x, name: str, shape) -> np.ndarray:
    """x (an array-like or a tensor) as a finite float64 numpy array of the given shape."""
    a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x
    try:
        a = np.asarray(a, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a real array of shape {list(shape)}") from None
    if a.shape != tuple(shape) or not np.isfinite(a).all():
        raise ValueError(f"{name} must be a finite array of shape {list(shape)}, got shape {list(a.shape)}")
    return a


def host_masses(masses, n: int) -> np.ndarray:
    m = host_array(masses, "masses", (n,))
    if not (m > 0).all():
        raise ValueError("masses must all be > 0 (amu)")
    return m


def check_model(caller: str, model) -> None:
    """The model checks the batched drivers share; `caller` names the call in the messages."""
    if not isinstance(model, (ALIGNNAtomWise, eALIGNNAtomWise)):
        raise ValueError(f"{caller} takes an ALIGNNAtomWise or eALIGNNAtomWise model")
    c = model.config
    if model.training:
        raise ValueError(f"{caller} needs the model in eval mode (model.eval())")
    if not c.calculate_gradient:
        raise ValueError(f"{caller} needs forces: the model has calculate_gradient=False")
    if c.output_features != 1:
        raise ValueError(f"{caller} needs one energy per crystal, got output_features={c.output_features}")
    if not c.energy_mult_natoms and c.use_penalty:
        # the model adds the whole batch's bond penalty to every crystal's `out` then (DESIGN section 8): a batched
        # energy would depend on the other crystals in the batch
        raise NotImplementedError(f"{caller}: energy_mult_natoms=False with use_penalty=True mixes the batch's "
                                  "penalty into every crystal's energy")
    if isinstance(model, eALIGNNAtomWise):
        # eALIGNN ignores force_mult_natoms, as the reference does.  Without ALIGNN layers its torque removal reads
        # ndata["cart_coords"], which no graph builder provides (the reference calculator fails with a KeyError there)
        if c.alignn_layers == 0 and c.remove_torque:
            raise ValueError(f"{caller}: an eALIGNNAtomWise with alignn_layers=0 and remove_torque=True needs "
                             "ndata['cart_coords'], which the crystal graphs do not carry")
        return
    if c.force_mult_natoms:
        # the model multiplies the pair forces by the atoms of the whole batch (alignn_atomwise.py:530-539); the
        # calculator's natoms factor goes into force_multiplier instead
        raise NotImplementedError(f"{caller}: force_mult_natoms=True scales forces by the batch's atom count; "
                                  "fold natoms into force_multiplier")


def check_batch(caller: str, model, structures, atom_features, neighbor_strategy, max_neighbors):
    """The device and structure checks the batched drivers share.  Returns (lattices, positions, device)."""
    params = list(model.parameters())
    if not params or not all(p.is_cuda for p in params):
        raise ValueError(f"{caller} needs the model on a CUDA device (model.to('cuda'))")
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


def _forces_as_alone(model, g, res, A: int, stress: bool):
    """The model's forces (and with `stress` its [A,3,3] stress) with the bond penalty counted once per crystal.
    `ALIGNNAtomWise` adds the whole batch's penalty to each of the A energies it differentiates with ones, so in a batch
    every bond's penalty gradient enters A times; a crystal evaluated alone (the calculator) sees it once.  Bonds
    without a penalty keep their pair forces bit for bit, and the per-crystal virial (the model's own,
    `ops.virial_stress`) is taken again from the corrected pair forces.  Without a penalty in a batch the model's own
    forces and stresses are used as they are.  No read-back: the correction and the scatter run whether or not any
    bond is penalised."""
    c = model.config
    if A == 1 or not c.use_penalty or isinstance(model, eALIGNNAtomWise):     # eALIGNN: already per crystal
        grad = res["grad"].detach().reshape(-1, 3).contiguous()
        return grad, res["stresses"].detach().reshape(-1, 3, 3).contiguous() if stress else None
    d = _penalty_pair_grad(model, g.edata["r"])
    hit = d.abs().amax(1) > 0
    pf = res["pair_forces"].detach()
    pf = torch.where(hit.unsqueeze(1), pf - (c.grad_multiplier * (A - 1)) * d, pf).contiguous()
    grad = ops.pair_force_scatter(pf, g.index, c.add_reverse_forces)
    if not stress:
        return grad, None
    return grad, ops.virial_stress(g.edata["r"].detach(), pf, g.edge_graph_offsets64(), g.node_graph_offsets().long(),
                                   g.ndata["V"], c.stress_multiplier)


def evaluate(model, structures, feats, dev, graph: dict, *, span: str, stress: bool = False):
    """One model call over a batch of (lattice, cart_coords) structures, each crystal as if evaluated alone.  feats:
    their [sum n, F] atom features; graph: the options of `crystal_graphs_device`.  Returns (energy [A] fp32, out *
    natoms without the bond penalty; grad [sum n, 3] fp32, the forces with the penalty counted once per crystal; the
    stress [A,3,3] fp32 of the same pair forces with `stress`, else None; the graph's batch offsets [A+1] int32).
    The graph build and the model call run under the `ops._span`s span + "_build" and span + "_model"."""
    ealignn = isinstance(model, eALIGNNAtomWise)
    with ops._span(span + "_build", 0):
        # eALIGNN builds L(g) of its filtered graph itself, so the build skips L(g)
        g, lg, lat = neighbors.crystal_graphs_device(structures, feats, device=dev, line_graph=not ealignn, **graph)
    with ops._span(span + "_model", 0):
        with torch.enable_grad():
            res = model._forward((g, lat), False, per_crystal=True) if ealignn else model((g, lg, lat))
            grad, st = _forces_as_alone(model, g, res, len(structures), stress)
        out = res["out"].detach().reshape(-1)                            # 0-d for a one-crystal batch
        energy = out * g.batch_num_nodes_on_device().to(out.dtype)
    return energy, grad, st, g.node_graph_offsets()


def evaluate_chunks(model, structures, features, dev, graph: dict, *, max_batch_atoms: int, span: str):
    """`evaluate` of every structure, the structures packed greedily, in order, into model calls of at most
    max_batch_atoms atoms (every structure must fit in one).  features(j) is structure j's [n_j, F] atom features.
    Returns (energy [J] fp32, grad [sum n_j, 3] fp32 in structure order)."""
    sizes = [x.shape[0] for _, x in structures]
    grad_all = torch.empty(sum(sizes), 3, device=dev, dtype=torch.float32)
    energy = torch.empty(len(sizes), device=dev, dtype=torch.float32)
    row, j = 0, 0
    while j < len(sizes):
        j0, atoms = j, 0
        while j < len(sizes) and atoms + sizes[j] <= max_batch_atoms:
            atoms += sizes[j]
            j += 1
        feats = torch.cat([features(k) for k in range(j0, j)])
        energy[j0:j], grad_all[row:row + atoms], _, _ = evaluate(model, structures[j0:j], feats, dev, graph, span=span)
        row += atoms
    return energy, grad_all


def read_back(span: str, status: torch.Tensor, crystals, sizes, host_pos: list, pos=None, host_cells=None, cells=None):
    """One device-to-host copy of the statuses [A] of the listed crystals, their cells [A,3,3] when `cells` is given
    and their position rows (concatenated in order) when `pos` is given, under the `ops._span` `span`.  Updates
    host_cells[b] and host_pos[b] of every crystal b listed and returns the statuses (float64)."""
    with ops._span(span, 0):
        parts = [status.to(torch.float64)] + [t.reshape(-1) for t in (cells, pos) if t is not None]
        back = torch.cat(parts).cpu().numpy()
    A = len(crystals)
    o = A
    if cells is not None:
        for j, b in enumerate(crystals):
            host_cells[b] = back[o + 9 * j:o + 9 * j + 9].reshape(3, 3)
        o += 9 * A
    if pos is not None:
        for b in crystals:
            host_pos[b] = back[o:o + 3 * sizes[b]].reshape(-1, 3)
            o += 3 * sizes[b]
    return back[:A]
