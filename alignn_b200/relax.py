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

`optimizer="LBFGS"` or `"BFGS"` runs ASE's quasi-Newton optimizers instead, in either lattice mode, through the same
loop: only the optimizer state and the step enqueued differ (`ops.lbfgs_step`, or `ops.bfgs_update`, torch's batched
`eigh` of each crystal's H and `ops.bfgs_apply`; csrc/qn_device.cu).  `oracle/qn_oracle.py` is their specification.

The model is an `ALIGNNAtomWise` or an `eALIGNNAtomWise`, evaluated through `calculator.evaluate` (each crystal as if
alone), as in the other batched drivers.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch

from . import calculator, neighbors, ops


class RelaxResult(NamedTuple):
    positions: torch.Tensor      # [N,3] float64 final Cartesian positions (not wrapped into the cell)
    energy: torch.Tensor         # [B] fp32 energy at the final positions, out * natoms (without the bond penalty)
    forces: torch.Tensor         # [N,3] fp32 forces at the final positions, grad * force_multiplier
    nsteps: torch.Tensor         # [B] int32 steps taken by the optimizer that ran
    converged: torch.Tensor      # [B] bool: max_i |F_i| < fmax at the final positions
    atom_offsets: torch.Tensor   # [B+1] int64: atoms of crystal b are rows atom_offsets[b]:atom_offsets[b+1]


class CellRelaxResult(NamedTuple):
    positions: torch.Tensor      # [N,3] float64 final Cartesian positions (not wrapped into the cell)
    energy: torch.Tensor         # [B] fp32 energy at the final structure, out * natoms (without the bond penalty)
    forces: torch.Tensor         # [N,3] fp32 Cartesian forces at the final structure, grad * force_multiplier
    nsteps: torch.Tensor         # [B] int32 steps taken by the optimizer that ran
    converged: torch.Tensor      # [B] bool: the filter's test, max over atom and cell rows of |row| < fmax
    atom_offsets: torch.Tensor   # [B+1] int64: atoms of crystal b are rows atom_offsets[b]:atom_offsets[b+1]
    cells: torch.Tensor          # [B,3,3] float64 final lattices, rows are lattice vectors as given
    stress: torch.Tensor         # [B,6] fp32 the calculator's Voigt stress (eV/A^3; xx yy zz yz xz xy) at the end


def _check(model, structures, atom_features, fmax, steps, neighbor_strategy, max_neighbors):
    calculator.check_model("relax_structures", model)
    if not calculator.real(fmax) or fmax < 0:
        raise ValueError(f"fmax must be a finite number >= 0, got {fmax!r}")
    calculator.check_steps(steps)
    return calculator.check_batch("relax_structures", model, structures, atom_features, neighbor_strategy, max_neighbors)


OPTIMIZERS = ("FIRE", "LBFGS", "BFGS")
# the other optimizers `ForceField.optimize_atoms` accepts (alignn/ff/ff.py:385-398), which this package does not build
NOT_BUILT_OPTIMIZERS = ("MDMin", "GPMin", "LBFGSLineSearch", "BFGSLineSearch", "SciPyFminCG", "SciPyFminBFGS")


def _check_optimizer(optimizer) -> str:
    if not isinstance(optimizer, str) or optimizer not in OPTIMIZERS + NOT_BUILT_OPTIMIZERS:
        raise ValueError(f"optimizer must be one of {', '.join(OPTIMIZERS)}, got {optimizer!r}")
    if optimizer in NOT_BUILT_OPTIMIZERS:
        raise NotImplementedError(f"relax_structures: optimizer {optimizer!r} is not implemented; "
                                  f"use one of {', '.join(OPTIMIZERS)}")
    return optimizer


def _filter_state(lats, dev):
    """ExpCellFilter's state per crystal, the cell operands of every optimizer's step: (C0, L = 0, F = I, C = C0, the
    cell rows, the calculator's Voigt stress)."""
    cells0 = torch.from_numpy(np.ascontiguousarray(np.stack(lats))).to(dev)
    defgrad = torch.eye(3, dtype=torch.float64, device=dev).repeat(len(lats), 1, 1)
    return (cells0, torch.zeros_like(cells0), defgrad, cells0.clone(), torch.zeros_like(cells0),
            torch.zeros(len(lats), 6, device=dev, dtype=torch.float32))


class _Fire:
    """The optimizer state of a batched FIRE relaxation (csrc/fire_device.cu, and csrc/fire_cell_device.cu under the
    filter) and its step, as `_QuasiNewton`'s."""

    def __init__(self, B, N, cell, dev):
        self.cell, self.kernel = cell, "fire_cell_step" if cell else "fire_step"
        self.vel = torch.zeros(N, 3, device=dev, dtype=torch.float64)
        self.cvel = torch.zeros(B, 3, 3, device=dev, dtype=torch.float64) if cell else None
        self.fstate = torch.tensor([[ops.FIRE_DT0, ops.FIRE_A0]] * B, device=dev, dtype=torch.float64)
        self.istate = torch.tensor([[0, 1, 0, 0]] * B, device=dev, dtype=torch.int32)  # Nsteps, v is None, steps, status

    def step(self, grad, stress, act, active, batch_offsets, aoff_d, pos, forces, cell_ops, kw):
        if self.cell:
            cells0, logdef, defgrad, cells, cforces, stress_out = cell_ops
            ops.fire_cell_step(grad, stress, act, batch_offsets, aoff_d, pos, self.vel, forces, cells0, logdef, defgrad,
                               cells, self.cvel, cforces, stress_out, self.fstate, self.istate, **kw)
        else:
            ops.fire_step(grad, act, batch_offsets, aoff_d, pos, self.vel, forces, self.fstate, self.istate,
                          fmax=kw["fmax"], steps=kw["steps"], force_multiplier=kw["force_multiplier"])


class _QuasiNewton:
    """The optimizer state of a batched LBFGS or BFGS relaxation (csrc/qn_device.cu) and its step: the rows of crystal b
    start at row aoff[b] (+ 3b under the filter) of every per-row array."""

    def __init__(self, optimizer, sizes, aoff, steps, cell, dev):
        self.optimizer, self.cell, self.sizes = optimizer, cell, sizes
        self.kernel = "lbfgs_step" if optimizer == "LBFGS" else "bfgs_update"
        B = len(sizes)
        rows = int(aoff[-1]) + (3 * B if cell else 0)
        self.rows = rows
        f64 = dict(device=dev, dtype=torch.float64)
        self.r0, self.f0 = torch.zeros(rows, 3, **f64), torch.zeros(rows, 3, **f64)
        self.istate = torch.zeros(B, 4, device=dev, dtype=torch.int32)
        if optimizer == "LBFGS":
            slots = min(ops.LBFGS_DEFAULTS["memory"], int(steps))
            self.work = torch.zeros(rows, 3, **f64)
            self.s_ring, self.y_ring = torch.zeros(slots * rows * 3, **f64), torch.zeros(slots * rows * 3, **f64)
            self.history = torch.zeros(B, 2 * slots, **f64)
        else:
            self.dims = [3 * (n + 3 if cell else n) for n in sizes]
            self.h_off = np.concatenate([[0], np.cumsum([d * d for d in self.dims])]).astype(np.int64)
            self.h_off_d = torch.from_numpy(self.h_off).to(dev)
            H = torch.zeros(int(self.h_off[-1]), **f64)
            for b, d in enumerate(self.dims):                  # H0 = alpha I
                H[int(self.h_off[b]):int(self.h_off[b + 1])].view(d, d).diagonal().fill_(ops.BFGS_DEFAULTS["alpha"])
            self.H = H
            self.r, self.f = torch.zeros(rows, 3, **f64), torch.zeros(rows, 3, **f64)
            self.work = torch.zeros(3, rows, 3, **f64)

    def step(self, grad, stress, act, active, batch_offsets, aoff_d, pos, forces, cell_ops, kw):
        if self.optimizer == "LBFGS":
            ops.lbfgs_step(grad, stress, act, batch_offsets, aoff_d, pos, forces, *cell_ops, self.r0, self.f0, self.work,
                           self.s_ring, self.y_ring, self.history, self.istate, **kw)
            return
        max_dim = max(self.dims[b] for b in active)
        ops.bfgs_update(grad, stress, act, batch_offsets, aoff_d, pos, forces, *cell_ops, self.h_off_d, self.H, self.r0,
                        self.f0, self.r, self.f, self.work, self.istate, max_dim=max_dim, **kw)
        groups = {}
        for b in active:
            groups.setdefault(self.dims[b], []).append(b)
        dev = pos.device
        for d, ids in groups.items():                          # eigh of every running crystal's H, d x d at a time
            base = torch.from_numpy(self.h_off[ids]).to(dev)
            idx = base.unsqueeze(1) + torch.arange(d * d, device=dev).unsqueeze(0)
            omega, V = torch.linalg.eigh(self.H[idx].view(len(ids), d, d))
            ops.bfgs_apply(torch.tensor(ids, dtype=torch.int32).to(dev), omega.contiguous(), V.contiguous(), aoff_d, pos,
                           *cell_ops[:4], self.r0, self.f0, self.r, self.f, self.work, self.istate, cell=self.cell)


def relax_structures(model, structures, atom_features: torch.Tensor, *, fmax: float = 0.1, steps: int = 100,
                     neighbor_strategy: str = "k-nearest", cutoff: float = 8.0, max_neighbors: int = 12,
                     cutoff_extra: float = 3.5, force_multiplier: float = 1.0, optimize_lattice: bool = False,
                     stress_wt: float = 1.0, optimizer: str = "FIRE"):
    """Relax the atomic positions of a batch of crystals with FIRE (ASE 3.22.1 defaults), the cells fixed: a batched
    `optimize_atoms(optimizer="FIRE", optimize_lattice=False, fmax=fmax, steps=steps)`.  Returns a `RelaxResult`.
    With optimize_lattice=True the cells relax too (see below) and a `CellRelaxResult` is returned.

    model: an `ALIGNNAtomWise` or `eALIGNNAtomWise` in eval mode on a CUDA device, with calculate_gradient=True and
    output_features=1; each crystal gets what it would get relaxed alone.
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
    its volume raises RuntimeError naming the crystal.

    optimizer: "FIRE" (the default), "LBFGS" or "BFGS" -- ASE 3.22.1's optimizers with the defaults the reference passes
    (LBFGS: maxstep 0.2, memory 100, damping 1, alpha 70, no line search; BFGS: maxstep 0.2, alpha 70), with either
    value of optimize_lattice; oracle/qn_oracle.py is their specification.  nsteps counts the steps of the optimizer
    that ran.  The other names optimize_atoms accepts raise NotImplementedError, anything else ValueError.  Where ASE
    would carry on with positions that are not finite (a zero or non-finite curvature y.s, a or b, or a step that is
    not finite) a RuntimeError names the crystal and the optimizer."""
    optimizer = _check_optimizer(optimizer)
    lats, Xs, dev = _check(model, structures, atom_features, fmax, steps, neighbor_strategy, max_neighbors)
    calculator.check_bool("optimize_lattice", optimize_lattice)
    calculator.check_real("stress_wt", stress_wt)
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
    forces = torch.zeros(N, 3, device=dev, dtype=torch.float32)
    energy = torch.zeros(B, device=dev, dtype=torch.float32)
    aoff_d = torch.from_numpy(aoff).to(dev)
    host_pos = [x.copy() for x in Xs]
    host_cells = [lat.copy() for lat in lats]
    cell_ops = _filter_state(lats, dev) if cell else (None,) * 6
    opt = _Fire(B, N, cell, dev) if optimizer == "FIRE" else _QuasiNewton(optimizer, sizes, aoff, steps, cell, dev)
    graph = dict(neighbor_strategy=neighbor_strategy, cutoff=cutoff, max_neighbors=max_neighbors,
                 cutoff_extra=cutoff_extra)
    kw = dict(fmax=float(fmax), steps=int(steps), force_multiplier=float(force_multiplier), stress_wt=float(stress_wt))
    active = list(range(B))
    while active:
        A = len(active)
        rows = torch.from_numpy(np.concatenate([np.arange(aoff[b], aoff[b + 1]) for b in active])).to(dev)
        act = torch.tensor(active, dtype=torch.int32).to(dev)
        feats = atom_features if A == B else atom_features[rows]
        energy[act.long()], grad, stress, batch_offsets = calculator.evaluate(
            model, [(host_cells[b], host_pos[b]) for b in active], feats, dev, graph, span="relax", stress=cell)
        with ops._span("relax_" + optimizer.lower(), 0):
            opt.step(grad, stress, act, active, batch_offsets, aoff_d, pos, forces, cell_ops, kw)
        # one copy: the running crystals' status, (their cells,) their positions
        status = calculator.read_back("relax_readback", opt.istate[act.long(), 3], active, sizes, host_pos, pos[rows],
                                      host_cells, cell_ops[3][act.long()] if cell else None)
        if (status == ops.FIRE_BAD_INPUT).any():
            raise RuntimeError(f"alignn_b200_{opt.kernel}: the model's forces do not match the crystals' atom counts")
        broke = [b for b, s in zip(active, status) if s == ops.QN_BREAKDOWN]
        if broke:
            raise RuntimeError(f"relax_structures: {optimizer} broke down on crystal {broke[0]} (a curvature y.s, a or b "
                               "that is zero or not finite, or a step that is not finite)")
        bad = [b for b, s in zip(active, status) if s == ops.FIRE_CELL_DEGENERATE]
        if cell and bad:
            raise RuntimeError(f"relax_structures: the cell of crystal {bad[0]} became degenerate (its volume or "
                               "expm of its log-deformation is not finite and positive)")
        active = [b for b, s in zip(active, status) if s == 0]
    ist = opt.istate.cpu()
    base = (pos, energy, forces, ist[:, 2].to(dev), (ist[:, 3] == 1).to(dev), aoff_d)
    return CellRelaxResult(*base, cell_ops[3], cell_ops[5]) if cell else RelaxResult(*base)
