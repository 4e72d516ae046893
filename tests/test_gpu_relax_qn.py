"""GPU (-m gpu): batched LBFGS and BFGS relaxation.  The step kernels (`ops.lbfgs_step`, `ops.bfgs_update` /
`ops.bfgs_apply`, csrc/qn_device.cu) against `oracle/qn_oracle.py` on scripted forces and stresses, their statuses,
and `relax_structures(optimizer=...)` against a host loop that relaxes each crystal alone the reference's way."""
import numpy as np
import pytest
import torch

from alignn_b200 import neighbors, ops, relax_structures
from alignn_b200.relax import _QuasiNewton
from oracle import cell_filter_oracle as CF
from oracle import fire_oracle as FO
from oracle import qn_oracle as QN
from tests.test_gpu_relax_cell import _host_evaluator, _model, _structures, _with_short_bond

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SIZES = [1, 2, 30, 1000]
MULT, WT = 1.5, 0.8


class _Kernels:
    """The device state of `relax_structures` for scripted crystals, stepped with explicit grads and stresses."""

    def __init__(self, optimizer, cells, x0, cell, steps, **params):
        self.optimizer, self.cell, self.params = optimizer, cell, params
        self.aoff = neighbors.ragged_offsets(SIZES)
        B = len(SIZES)
        t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)   # noqa: E731
        self.pos = t64(x0.copy())
        self.forces = torch.zeros(len(x0), 3, device=DEV, dtype=torch.float32)
        self.aoff_d = t64(self.aoff)
        self.cell_ops = (None,) * 6
        if cell:
            C0 = t64(cells)
            self.cell_ops = (C0, torch.zeros_like(C0), torch.eye(3, dtype=torch.float64, device=DEV).repeat(B, 1, 1),
                             C0.clone(), torch.zeros_like(C0), torch.zeros(B, 6, device=DEV))
        self.qn = _QuasiNewton(optimizer, SIZES, self.aoff, steps, cell, DEV)
        if optimizer == "LBFGS" and "memory" in params:          # a small ring, so that it wraps
            slots = min(params["memory"], steps)
            rows = self.qn.rows
            self.qn.s_ring = torch.zeros(slots * rows * 3, dtype=torch.float64, device=DEV)
            self.qn.y_ring = torch.zeros_like(self.qn.s_ring)
            self.qn.history = torch.zeros(B, 2 * slots, dtype=torch.float64, device=DEV)
        self.steps = steps

    def step(self, active, grads, stresses, fmax):
        boff = torch.tensor(neighbors.ragged_offsets([SIZES[b] for b in active]), dtype=torch.int32).to(DEV)
        grad = torch.from_numpy(np.concatenate(grads)).to(DEV)
        stress = torch.from_numpy(np.stack(stresses)).to(DEV) if self.cell else None
        act = torch.tensor(active, dtype=torch.int32).to(DEV)
        kw = dict(fmax=fmax, steps=self.steps, force_multiplier=MULT, stress_wt=WT)
        if self.optimizer == "LBFGS":
            q = self.qn
            ops.lbfgs_step(grad, stress, act, boff, self.aoff_d, self.pos, self.forces, *self.cell_ops, q.r0, q.f0,
                           q.work, q.s_ring, q.y_ring, q.history, q.istate, **kw, **self.params)
        else:
            self.qn.step(grad, stress, act, active, boff, self.aoff_d, self.pos, self.forces, self.cell_ops, kw)

    def state(self):
        out = [self.pos, self.forces, self.qn.istate, self.qn.r0, self.qn.f0]
        return [t.clone() for t in out] + ([t.clone() for t in self.cell_ops] if self.cell else [])


def _scripted(optimizer, cell, steps=20, **params):
    """Crystals on an SPD quadratic (forces from the oracle's positions, fp32) that converge at different steps; under
    the filter a stress that pulls each cell towards a log-strain of its own, so that the cell rows too come from a
    convex energy (on a field that is not a gradient, y.s can come close to 0 and the two-loop amplifies rounding)."""
    rng = np.random.default_rng(7)
    B = len(SIZES)
    cells = np.stack([np.diag([4.0, 4.5, 5.0]) + 0.3 * rng.normal(size=(3, 3)) for _ in range(3)] + [np.diag([20., 21., 22.])])
    x0 = np.concatenate([rng.random((n, 3)) @ cells[b] for b, n in enumerate(SIZES)])
    aoff = neighbors.ragged_offsets(SIZES)
    targets = [x0[aoff[b]:aoff[b + 1]] + rng.normal(scale=0.15, size=(n, 3)) for b, n in enumerate(SIZES)]
    stiff = [0.5 + rng.random((n, 1)) for n in SIZES]
    Lt = [0.01 * (lambda M: M + M.T)(rng.normal(size=(3, 3))) for _ in range(B)]
    fmax = 0.02
    dev = _Kernels(optimizer, cells, x0, cell, steps, **params)
    if cell:
        filts = [CF.ExpCellFilter(cells[b], x0[aoff[b]:aoff[b + 1]]) for b in range(B)]
        opts = [QN.make(optimizer, n + 3, **params) for n in SIZES]
        Ls = [np.zeros((3, 3)) for _ in SIZES]
    else:
        xs = [x0[aoff[b]:aoff[b + 1]].copy() for b in range(B)]
        opts = [QN.make(optimizer, n, **params) for n in SIZES]
    status, nsteps = [0] * B, [0] * B
    worst = 0.0
    active, s = list(range(B)), 0
    while active:
        grads, stresses, rows = [], [], {}
        for b in active:
            X = filts[b].X if cell else xs[b]
            g = (-stiff[b] * (X - targets[b])).astype(np.float32)
            if cell:                                            # a restoring stress towards the log-strain Lt[b]
                L = 0.5 * (Ls[b] + Ls[b].T)
                V = abs(np.linalg.det(filts[b].C))
                st = (CF.EV_A3_PER_GPA / WT * 0.5 * (L - Lt[b]) / V * V ** (1 / 3)).astype(np.float32)
            else:
                st = np.zeros((3, 3), dtype=np.float32)
            grads.append(g)
            stresses.append(st)
            f = FO.scaled_forces(g, MULT)
            rows[b] = filts[b].get_forces(f, CF.calculator_stress(st, WT)) if cell else f
        dev.step(active, grads, stresses, fmax)
        for b in active:
            if FO.converged(rows[b], fmax):
                status[b] = FO.CONVERGED
            elif nsteps[b] >= steps:
                status[b] = FO.STEP_LIMIT
            else:
                if cell:
                    Ls[b] = QN._filter_step(opts[b], filts[b], Ls[b], rows[b])
                else:
                    xs[b] = opts[b].step(xs[b], rows[b])
                nsteps[b] += 1
        P, IS = dev.pos.cpu().numpy(), dev.qn.istate.cpu().numpy()
        for b in range(B):
            want = filts[b].X if cell else xs[b]
            d = float(np.abs(P[aoff[b]:aoff[b + 1]] - want).max()) / max(float(np.abs(want).max()), 1e-300)
            worst = max(worst, d)
            if cell:
                C = dev.cell_ops[3][b].cpu().numpy()
                worst = max(worst, float(np.abs(C - filts[b].C).max()) / float(np.abs(filts[b].C).max()))
        active = [b for b in active if IS[b][3] == 0]
        assert [int(IS[b][2]) for b in range(B)] == nsteps, (s, IS, nsteps)
        s += 1
    return dev, status, nsteps, worst


@pytest.mark.parametrize("cell", [False, True])
def test_lbfgs_kernel_matches_oracle_and_is_repeatable(cell):
    dev, status, nsteps, worst = _scripted("LBFGS", cell, memory=5)
    print(f"[lbfgs scripted cell={cell}] status {status} nsteps {nsteps} worst relative difference {worst:.3g}")
    assert FO.CONVERGED in status and max(nsteps) > 6                     # the ring of 5 wrapped
    # under the filter the oracle's cell forces go through scipy's logm and expm and the kernel's through its Pade
    # expm, and the two-loop recursion divides by the small curvatures y.s near convergence
    assert worst <= (1e-10 if cell else 1e-12)
    again = _scripted("LBFGS", cell, memory=5)[0]
    for a, b in zip(dev.state(), again.state()):
        assert torch.equal(a, b)                                                # bitwise repeatable


@pytest.mark.parametrize("cell", [False, True])
def test_bfgs_kernels_match_oracle(cell):
    dev, status, nsteps, worst = _scripted("BFGS", cell)
    print(f"[bfgs scripted cell={cell}] status {status} nsteps {nsteps} worst relative difference {worst:.3g}")
    assert FO.CONVERGED in status and max(nsteps) > 6
    assert worst <= 1e-9


@pytest.mark.parametrize("optimizer", ["LBFGS", "BFGS"])
def test_statuses(optimizer):
    # 5: the same forces twice on a crystal that moved (y = df = 0)
    q = _QuasiNewton(optimizer, [2], np.array([0, 2]), 5, False, DEV)
    pos = torch.zeros(2, 3, dtype=torch.float64, device=DEV)
    forces = torch.zeros(2, 3, device=DEV)
    aoff = torch.tensor([0, 2], dtype=torch.int64, device=DEV)
    boff = torch.tensor([0, 2], dtype=torch.int32, device=DEV)
    act = torch.tensor([0], dtype=torch.int32, device=DEV)
    g = torch.ones(2, 3, device=DEV)
    kw = dict(fmax=0.0, steps=5, force_multiplier=1.0, stress_wt=1.0)
    for _ in range(2):
        q.step(g, None, act, [0], boff, aoff, pos, forces, (None,) * 6, kw)
    assert q.istate[0, 3].item() == ops.QN_BREAKDOWN
    before = pos.clone()
    q.step(g, None, act, [0], boff, aoff, pos, forces, (None,) * 6, kw)          # frozen: untouched
    assert torch.equal(before, pos)
    # 3: a batch slice that is not the crystal's atoms
    q = _QuasiNewton(optimizer, [2], np.array([0, 2]), 5, False, DEV)
    q.step(g, None, act, [0], torch.tensor([0, 1], dtype=torch.int32, device=DEV), aoff, pos, forces, (None,) * 6, kw)
    assert q.istate[0, 3].item() == ops.FIRE_BAD_INPUT
    # 4: a cell without volume
    q = _QuasiNewton(optimizer, [2], np.array([0, 2]), 5, True, DEV)
    C0 = torch.zeros(1, 3, 3, dtype=torch.float64, device=DEV)
    cops = (C0, torch.zeros_like(C0), torch.eye(3, dtype=torch.float64, device=DEV).view(1, 3, 3).clone(), C0.clone(),
            torch.zeros_like(C0), torch.zeros(1, 6, device=DEV))
    q.step(g, torch.ones(1, 3, 3, device=DEV), act, [0], boff, aoff, pos, forces, cops, kw)
    assert q.istate[0, 3].item() == ops.FIRE_CELL_DEGENERATE


@pytest.mark.parametrize("optimizer", ["LBFGS", "BFGS"])
@pytest.mark.parametrize("cell", [False, True])
@pytest.mark.parametrize("strategy,cutoff", [("k-nearest", 8.0), ("radius_graph", 6.0)])
def test_relax_matches_host_loop(optimizer, cell, strategy, cutoff):
    model = _model()
    structs, feats = _structures(count=6)
    steps, mult, fmax = 8, 1.5, 0.05
    evs, o = [], 0
    for lat, X in structs:
        evs.append(_host_evaluator(model, feats[o:o + X.shape[0]], strategy, cutoff))
        o += X.shape[0]
    if cell:
        ref = [QN.relax_cell(optimizer, ev, lat, X, fmax=fmax, steps=steps, force_multiplier=mult)
               for (lat, X), ev in zip(structs, evs)]
    else:
        ref = [QN.relax(optimizer, lambda x, ev=ev, lat=lat: ev(lat, x)[:2], X, fmax=fmax, steps=steps,
                        force_multiplier=mult) for (lat, X), ev in zip(structs, evs)]
    got = relax_structures(model, structs, feats, fmax=fmax, steps=steps, neighbor_strategy=strategy, cutoff=cutoff,
                           force_multiplier=mult, optimize_lattice=cell, optimizer=optimizer)
    nst = got.nsteps.cpu().tolist()
    print(f"[relax {optimizer} cell={cell} {strategy}] nsteps {nst} converged {got.converged.cpu().tolist()}")
    assert nst == [r["nsteps"] for r in ref]
    assert got.converged.cpu().tolist() == [r["converged"] for r in ref]
    off = got.atom_offsets.cpu().tolist()
    P, F = got.positions.cpu().numpy(), got.forces.cpu().numpy()
    for b, r in enumerate(ref):
        sl = slice(off[b], off[b + 1])
        assert np.abs(P[sl] - r["positions"]).max() <= 1e-6, b
        # with a floor of 1e-6 eV/A: a converged crystal's last forces are near zero, and there fp32 rounding
        # of the model (host and device graphs order edges differently) is all that is left
        assert np.abs(F[sl] - r["forces"]).max() <= 1e-5 * max(np.abs(r["forces"]).max(), 1e-30) + 1e-6, b
        if cell:
            assert np.abs(got.cells[b].cpu().numpy() - r["cell"]).max() <= 1e-6, b


@pytest.mark.parametrize("optimizer", ["LBFGS", "BFGS"])
def test_bond_penalty_counted_once_and_no_grad(optimizer):
    model = _model()
    structs, feats = _structures(count=3)
    short, f_short = _with_short_bond(structs, feats)
    got = relax_structures(model, structs + [short], torch.cat([feats, f_short]), fmax=0.0, steps=3,
                           optimize_lattice=True, optimizer=optimizer)
    one = relax_structures(model, [short], f_short, fmax=0.0, steps=3, optimize_lattice=True, optimizer=optimizer)
    off = got.atom_offsets.cpu().tolist()
    sl = slice(off[-2], off[-1])
    F1, S1 = one.forces.cpu().numpy(), one.stress.cpu().numpy()[0]
    assert np.abs(got.forces[sl].cpu().numpy() - F1).max() <= 1e-5 * np.abs(F1).max() + 1e-6
    assert np.abs(got.stress[-1].cpu().numpy() - S1).max() <= 1e-5 * np.abs(S1).max() + 1e-7
    with torch.no_grad():
        again = relax_structures(model, structs + [short], torch.cat([feats, f_short]), fmax=0.0, steps=3,
                                 optimize_lattice=True, optimizer=optimizer)
    if optimizer == "LBFGS":
        for a, b in zip(got, again):
            assert torch.equal(a, b)
    else:
        assert torch.allclose(got.positions, again.positions, rtol=0, atol=1e-9)


def test_lbfgs_relax_is_batch_invariant():
    model = _model()
    structs, feats = _structures()
    got = relax_structures(model, structs, feats, fmax=0.0, steps=5, optimize_lattice=True, optimizer="LBFGS")
    off = got.atom_offsets.cpu().tolist()
    for b in (0, len(structs) - 1):
        one = relax_structures(model, [structs[b]], feats[off[b]:off[b + 1]], fmax=0.0, steps=5, optimize_lattice=True,
                               optimizer="LBFGS")
        assert torch.equal(one.positions, got.positions[off[b]:off[b + 1]])
        assert torch.equal(one.cells[0], got.cells[b])


def test_optimizer_rejections():
    model = _model()
    structs, feats = _structures(count=2)
    for bad in (None, 1, "fire", "Nope", b"FIRE"):
        with pytest.raises(ValueError, match="FIRE, LBFGS, BFGS"):
            relax_structures(model, structs, feats, optimizer=bad)
    for name in ("MDMin", "GPMin", "LBFGSLineSearch", "BFGSLineSearch", "SciPyFminCG", "SciPyFminBFGS"):
        with pytest.raises(NotImplementedError, match=name):
            relax_structures(model, structs, feats, optimizer=name)
    fire = relax_structures(model, structs, feats, fmax=0.0, steps=2)
    same = relax_structures(model, structs, feats, fmax=0.0, steps=2, optimizer="FIRE")
    for a, b in zip(fire, same):
        assert torch.equal(a, b)
