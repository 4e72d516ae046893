"""GPU (-m gpu): batched FIRE on ASE's ExpCellFilter, atoms and cells relaxed together.  The step kernel
(`ops.fire_cell_step`, csrc/fire_cell_device.cu) against `oracle/cell_filter_oracle.py` on scripted forces and
stresses, and `relax_structures(optimize_lattice=True)` against a host loop that relaxes each crystal alone the
reference's way (host graph build on the current cell, the same model on a one-crystal batch, the oracle's filtered
FIRE)."""
import os

import numpy as np
import pytest
import torch
from scipy.linalg import expm

from alignn_b200 import neighbors, ops, relax_structures
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from oracle import cell_filter_oracle as CF
from oracle import fire_oracle as FO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- 1. the step kernel on scripted forces and stresses ---------------------------------------------------------------
SIZES = [1, 2, 30, 1000]
MULT, WT, FMAX, STEPS = 1.5, 0.8, 0.05, 40
SHEAR = np.array([[0.0, 2.5, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]])   # preloaded on crystal 3: the fallback branch


def _script(b, s, n, rng_cache={}):
    """(grad, model stress) of crystal b at its evaluation s: a constant push (step limit), a push that flips every 7
    evaluations (uphill resets) and a decaying field (both converging, at different evaluations), and for the large
    sheared crystal a field that stays above fmax."""
    key = (b, n)
    if key not in rng_cache:
        rng = np.random.default_rng(100 + b)
        S = rng.normal(size=(3, 3))
        rng_cache[key] = (rng.normal(size=(n, 3)), S + S.T)
    base, S = rng_cache[key]
    if b == 0:
        g, st = 0.3 * base / np.linalg.norm(base), 0.05 * S
    elif b == 1:
        sign = 1.0 if (s // 7) % 2 == 0 else -1.0
        g, st = sign * base * 0.8 ** (s / 2), sign * S * 0.8 ** (s / 2)
    elif b == 2:
        g, st = base * 0.8 ** s, 0.2 * S * 0.8 ** s
    else:
        g, st = base * (1.0 + 0.1 * np.sin(s)), np.diag([0.32, -0.16, 0.24]) + 0.01 * np.sin(s) * S
    return g.astype(np.float32), st.astype(np.float32)


def _scripted_run(freeze_probe=False):
    sizes = SIZES
    aoff = neighbors.ragged_offsets(sizes)
    N, B = int(aoff[-1]), len(sizes)
    rng = np.random.default_rng(0)
    C0 = np.stack([np.diag([4.0, 4.5, 5.0]) + 0.3 * rng.normal(size=(3, 3)) for _ in range(3)] + [np.diag([20., 21., 22.])])
    x0 = np.concatenate([rng.random((n, 3)) @ C0[b] for b, n in enumerate(sizes)])
    L0 = np.zeros((B, 3, 3))
    L0[3] = SHEAR
    F0 = np.stack([expm(L) for L in L0])
    cells_start = np.einsum("bij,bkj->bik", C0, F0)                          # C0 @ F.T
    pos = torch.from_numpy(x0.copy()).to(DEV)
    vel = torch.zeros_like(pos)
    forces = torch.zeros(N, 3, device=DEV, dtype=torch.float32)
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)        # noqa: E731
    cells0, logdef, defgrad, cells = t64(C0), t64(L0), t64(F0), t64(cells_start)
    cvel, cforces = torch.zeros_like(cells0), torch.zeros_like(cells0)
    stress_out = torch.zeros(B, 6, device=DEV, dtype=torch.float32)
    fstate = torch.tensor([[ops.FIRE_DT0, ops.FIRE_A0]] * B, device=DEV, dtype=torch.float64)
    istate = torch.tensor([[0, 1, 0, 0]] * B, device=DEV, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(DEV)
    filts = []
    for b in range(B):
        f = CF.ExpCellFilter(C0[b], x0[aoff[b]:aoff[b + 1]])
        f.C = cells_start[b].copy()
        filts.append(f)
    opts = [FO.Fire(f.get_positions()) for f in filts]
    o_state = [dict(status=0, nsteps=0) for _ in range(B)]
    frozen_at = {}
    active, s = list(range(B)), 0
    seen = dict(reset=False, fallback=False, exact=False, capped=False)
    worst = dict(cell_forces=0.0, L=0.0, cells=0.0, positions=0.0, velocities=0.0)   # largest relative differences

    def rel(key, a, w, scale=None):
        d = float(np.abs(a - w).max()) / max(float(np.abs(w).max()) if scale is None else scale, 1e-300)
        worst[key] = max(worst[key], d)
        return d <= 1e-12
    while active:
        scripted = [_script(b, s, sizes[b]) for b in active]
        boff = torch.tensor(neighbors.ragged_offsets([sizes[b] for b in active]), dtype=torch.int32).to(DEV)
        grad = torch.from_numpy(np.concatenate([g for g, _ in scripted])).to(DEV)
        stress = torch.from_numpy(np.stack([st for _, st in scripted])).to(DEV)
        ops.fire_cell_step(grad, stress, torch.tensor(active, dtype=torch.int32).to(DEV), boff, aoff_d, pos, vel, forces,
                           cells0, logdef, defgrad, cells, cvel, cforces, stress_out, fstate, istate, fmax=FMAX, steps=STEPS,
                           force_multiplier=MULT, stress_wt=WT)
        for b, (g, stv) in zip(active, scripted):                            # the oracle's decision per crystal
            st, opt, filt = o_state[b], opts[b], filts[b]
            st["forces"] = FO.scaled_forces(g, MULT)
            st["stress"] = CF.calculator_stress(stv, WT)
            rows = filt.get_forces(st["forces"], st["stress"])
            st["cell_rows"] = rows[-3:]
            seen["fallback" if not filt.exact else "exact"] = True
            if FO.converged(rows, FMAX):
                st["status"] = FO.CONVERGED
            elif st["nsteps"] >= STEPS:
                st["status"] = FO.STEP_LIMIT
            else:
                n_before = opt.Nsteps
                opt.x = filt.get_positions()
                x_before = opt.x.copy()
                opt.step(rows)
                filt.set_positions(opt.x)
                st["nsteps"] += 1
                seen["reset"] |= (n_before > 0 and opt.Nsteps == 0)
                seen["capped"] |= bool(np.sqrt(((opt.x - x_before) ** 2).sum()) > 0.2 - 1e-12)
        P, V, Fo = pos.cpu().numpy(), vel.cpu().numpy(), forces.cpu().numpy()
        FS, IS = fstate.cpu().numpy(), istate.cpu().numpy()
        CL, CC, CV, CFo, SO = (t.cpu().numpy() for t in (logdef, cells, cvel, cforces, stress_out))
        for b in active:
            st, opt, filt, sl = o_state[b], opts[b], filts[b], slice(aoff[b], aoff[b + 1])
            n = sizes[b]
            first = 1 if opt.v is None else 0
            assert IS[b].tolist() == [opt.Nsteps, first, st["nsteps"], st["status"]], (b, s, IS[b])
            assert np.array_equal(Fo[sl], st["forces"]), (b, s)
            assert np.array_equal(SO[b], st["stress"]), (b, s)
            assert rel("cell_forces", CFo[b], st["cell_rows"]), (b, s, CFo[b], st["cell_rows"])
            np.testing.assert_allclose(FS[b], [opt.dt, opt.a], rtol=1e-12, atol=0)
            assert rel("positions", P[sl], filt.X), (b, s)
            assert rel("cells", CC[b], filt.C), (b, s)
            if np.abs(opt.x[n:]).max() > 0:
                assert rel("L", CL[b], opt.x[n:]), (b, s)
            if opt.v is not None:
                vmax = float(np.abs(opt.v).max())
                assert rel("velocities", V[sl], opt.v[:n], vmax), (b, s)
                assert rel("velocities", CV[b], opt.v[n:], vmax), (b, s)
            if st["status"] != 0:
                frozen_at[b] = (P[sl].copy(), V[sl].copy(), Fo[sl].copy(), FS[b].copy(), IS[b].copy(), CL[b].copy(),
                                CC[b].copy(), CV[b].copy(), CFo[b].copy(), SO[b].copy())
        for b, saved in frozen_at.items():                                    # frozen crystals stay bitwise as they were
            sl = slice(aoff[b], aoff[b + 1])
            now = (P[sl], V[sl], Fo[sl], FS[b], IS[b], CL[b], CC[b], CV[b], CFo[b], SO[b])
            assert all(np.array_equal(a, w) for a, w in zip(now, saved)), b
        active = [b for b in active if IS[b][3] == 0]
        s += 1
    tensors = (pos, vel, forces, fstate, istate, logdef, defgrad, cells, cvel, cforces, stress_out)
    if freeze_probe:                                                          # a frozen id in the list is not touched
        before = [t.clone() for t in tensors]
        ops.fire_cell_step(torch.full((SIZES[2], 3), 7.0, device=DEV), torch.ones(1, 3, 3, device=DEV),
                           torch.tensor([2], dtype=torch.int32, device=DEV),
                           torch.tensor([0, SIZES[2]], dtype=torch.int32, device=DEV), aoff_d, pos, vel, forces, cells0,
                           logdef, defgrad, cells, cvel, cforces, stress_out, fstate, istate, fmax=FMAX, steps=STEPS,
                           force_multiplier=MULT, stress_wt=WT)
        for a, b in zip(before, tensors):
            assert torch.equal(a, b)
    return dict(o_state=o_state, seen=seen, tensors=tensors, worst=worst)


def test_fire_cell_step_matches_oracle_on_scripted_forces():
    r = _scripted_run(freeze_probe=True)
    st = [o["status"] for o in r["o_state"]]
    steps = [o["nsteps"] for o in r["o_state"]]
    print(f"[fire cell scripted] status {st} nsteps {steps} seen {r['seen']}")
    print("[fire cell scripted] largest relative differences " + " ".join(f"{k} {v:.2g}" for k, v in r["worst"].items()))
    assert r["seen"] == dict(reset=True, fallback=True, exact=True, capped=True)
    assert FO.CONVERGED in st and FO.STEP_LIMIT in st
    again = _scripted_run()
    for a, b in zip(r["tensors"], again["tensors"]):
        assert torch.equal(a, b)                                               # bitwise repeatable


def _one_crystal_state(cell, n, L=None):
    t = dict(pos=torch.zeros(n, 3, dtype=torch.float64, device=DEV), vel=torch.zeros(n, 3, dtype=torch.float64, device=DEV),
             forces=torch.zeros(n, 3, device=DEV), cells0=torch.tensor(cell, dtype=torch.float64, device=DEV).view(1, 3, 3))
    t["logdef"] = torch.zeros_like(t["cells0"])
    t["defgrad"] = torch.eye(3, dtype=torch.float64, device=DEV).view(1, 3, 3).clone()
    t["cells"] = t["cells0"].clone()
    t["cvel"], t["cforces"] = torch.zeros_like(t["cells0"]), torch.zeros_like(t["cells0"])
    t["stress_out"] = torch.zeros(1, 6, device=DEV)
    t["fstate"] = torch.tensor([[0.1, 0.1]], dtype=torch.float64, device=DEV)
    t["istate"] = torch.tensor([[0, 1, 0, 0]], dtype=torch.int32, device=DEV)
    return t


def _step_one(t, grad, stress, steps=5):
    n = t["pos"].shape[0]
    ops.fire_cell_step(grad, stress, torch.tensor([0], dtype=torch.int32, device=DEV),
                       torch.tensor([0, n], dtype=torch.int32, device=DEV),
                       torch.tensor([0, n], dtype=torch.int64, device=DEV), t["pos"], t["vel"], t["forces"], t["cells0"],
                       t["logdef"], t["defgrad"], t["cells"], t["cvel"], t["cforces"], t["stress_out"], t["fstate"],
                       t["istate"], fmax=0.0, steps=steps)


def test_degenerate_cell_gives_status_4():
    # a cell without volume: nothing but the status is written
    t = _one_crystal_state(np.zeros((3, 3)), 2)
    before = {k: v.clone() for k, v in t.items()}
    _step_one(t, torch.ones(2, 3, device=DEV), torch.ones(1, 3, 3, device=DEV))
    assert t["istate"].tolist() == [[0, 1, 0, ops.FIRE_CELL_DEGENERATE]]
    for k in before:
        if k != "istate":
            assert torch.equal(before[k], t[k]), k
    # a NaN stress: expm of the new L is not finite; positions and the cell state are not written
    t = _one_crystal_state(np.eye(3) * 4.0, 2)
    before = {k: v.clone() for k, v in t.items()}
    _step_one(t, torch.ones(2, 3, device=DEV), torch.full((1, 3, 3), float("nan"), device=DEV))
    assert t["istate"][0, 3].item() == ops.FIRE_CELL_DEGENERATE
    for k in ("pos", "logdef", "defgrad", "cells"):
        assert torch.equal(before[k], t[k]), k
    # the operand checks
    t = _one_crystal_state(np.eye(3) * 4.0, 2)
    with pytest.raises(ValueError, match="shapes"):
        _step_one(t, torch.ones(2, 3, device=DEV), torch.ones(2, 3, 3, device=DEV))
    with pytest.raises(ValueError, match="steps"):
        _step_one(t, torch.ones(2, 3, device=DEV), torch.ones(1, 3, 3, device=DEV), steps=0)


# ---- 2-5. relax_structures(optimize_lattice=True) -------------------------------------------------------------------
def _model(seed=11, **kw):
    torch.manual_seed(seed)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64,
                               embedding_features=64, atom_input_features=92, stresswise_weight=1.0, **kw)
    return ALIGNNAtomWise(cfg).to(DEV).eval()


def _structures(count=8, seed=3):
    """Jittered sample structures with strained and sheared cells (atoms moved with their cell), none with a tie at the
    12th neighbour (`neighbors.knn_cut_is_tied`): there the two arms' rounding would pick different images."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    sizes = off[1:] - off[:-1]
    idx = [i for i in range(len(sizes)) if sizes[i] <= 12]
    rng = np.random.default_rng(seed)
    out = []
    for i in rng.permutation(idx):
        D = np.eye(3) + np.diag(rng.uniform(-0.04, 0.04, 3)) + rng.uniform(-0.03, 0.03, (3, 3))
        lat, X = z["lattices"][i] @ D.T, z["cart_coords"][off[i]:off[i + 1]] @ D.T
        X = X + rng.normal(scale=0.05, size=X.shape)
        if not neighbors.knn_cut_is_tied(lat, X):
            out.append((lat, X))
        if len(out) == count:
            break
    feats = torch.from_numpy(rng.normal(size=(sum(x.shape[0] for _, x in out), 92)).astype(np.float32)).to(DEV)
    return out, feats


def _host_evaluator(model, feats, strategy, cutoff):
    def evaluate(cell, x):
        g, lg = neighbors.crystal_graph(cell, x, feats.cpu(), cutoff=cutoff, neighbor_strategy=strategy, max_neighbors=12)
        vol = abs(float(np.dot(np.cross(cell[0], cell[1]), cell[2])))
        g.ndata["V"] = torch.full((x.shape[0],), vol, dtype=torch.float32)
        lat_t = torch.tensor(cell, dtype=torch.float32).view(1, 3, 3).to(DEV)
        res = model((g.to(DEV), lg.to(DEV), lat_t))
        e = (res["out"].detach().reshape(-1) * float(x.shape[0])).cpu().numpy()[0]
        return e, res["grad"].detach().reshape(-1, 3).cpu().numpy(), res["stresses"].detach().reshape(3, 3).cpu().numpy()
    return evaluate


@pytest.mark.parametrize("strategy,cutoff", [("k-nearest", 8.0), ("radius_graph", 6.0)])
def test_relax_cells_matches_host_loop(strategy, cutoff):
    model = _model()
    structs, feats = _structures()
    steps, mult = 12, 1.5
    evs, o = [], 0
    for lat, X in structs:
        evs.append(_host_evaluator(model, feats[o:o + X.shape[0]], strategy, cutoff))
        o += X.shape[0]
    # fmax from the oracle's own trajectories, as in the fixed-cell test
    srt = sorted(m for m in _min_rows(structs, evs, steps, mult) if m > 0)
    assert srt[0] < srt[-1]
    fmax = float(np.sqrt(np.sqrt(srt[0] * srt[len(srt) // 2])))             # between the lowest and the median
    ref = [CF.relax(ev, lat, X, fmax=fmax, steps=steps, force_multiplier=mult) for (lat, X), ev in zip(structs, evs)]
    got = relax_structures(model, structs, feats, fmax=fmax, steps=steps, neighbor_strategy=strategy, cutoff=cutoff,
                           force_multiplier=mult, optimize_lattice=True)
    nst, conv = got.nsteps.cpu().tolist(), got.converged.cpu().tolist()
    moved = [float(np.abs(r["cell"] - lat).max()) for r, (lat, _) in zip(ref, structs)]
    print(f"[relax cell {strategy}] fmax {fmax:.4g} nsteps {nst} converged {conv} cell moved {np.round(moved, 3)}")
    assert nst == [r["nsteps"] for r in ref] and conv == [r["converged"] for r in ref]
    assert any(conv) and not all(conv) and min(nst) < steps
    assert max(moved) > 1e-2
    off = got.atom_offsets.cpu().tolist()
    P, F, E = got.positions.cpu().numpy(), got.forces.cpu().numpy(), got.energy.cpu().numpy()
    Cg, Sg = got.cells.cpu().numpy(), got.stress.cpu().numpy()
    dpos = dcell = 0.0
    for b, r in enumerate(ref):
        sl = slice(off[b], off[b + 1])
        dpos, dcell = max(dpos, np.abs(P[sl] - r["positions"]).max()), max(dcell, np.abs(Cg[b] - r["cell"]).max())
        assert np.abs(P[sl] - r["positions"]).max() <= 1e-6, b
        assert np.abs(Cg[b] - r["cell"]).max() <= 1e-6, b
        assert np.abs(F[sl] - r["forces"]).max() <= 1e-5 * max(np.abs(r["forces"]).max(), 1e-30), b
        assert np.abs(Sg[b] - r["stress"]).max() <= 1e-5 * max(np.abs(r["stress"]).max(), 1e-30), b
        assert abs(E[b] - r["energy"]) <= 1e-5 * max(abs(r["energy"]), 1e-30), b
    print(f"[relax cell {strategy}] largest difference: positions {dpos:.3g} A, cells {dcell:.3g} A")


def _min_rows(structs, evs, steps, mult):
    """Per crystal, the smallest max |row|^2 of the filter's forces over the evaluations before the step limit of an
    fmax = 0 run (every crystal runs to the limit)."""
    out = []
    for (lat, X), ev in zip(structs, evs):
        m2 = []
        filt = CF.ExpCellFilter(lat, X)
        opt = FO.Fire(filt.get_positions())
        for s in range(steps + 1):
            _, g, st = ev(filt.C.copy(), filt.X.copy())
            rows = filt.get_forces(FO.scaled_forces(g, mult), CF.calculator_stress(st))
            m2.append((rows ** 2).sum(1).max())
            if s == steps:
                break
            opt.x = filt.get_positions()
            opt.step(rows)
            filt.set_positions(opt.x)
        out.append(min(m2[:-1]))
    return out


def test_relax_cells_is_batch_invariant():
    model = _model()
    structs, feats = _structures()
    got = relax_structures(model, structs, feats, fmax=0.0, steps=6, optimize_lattice=True, stress_wt=0.8)
    off = got.atom_offsets.cpu().tolist()
    for b in (0, 3, len(structs) - 1):
        one = relax_structures(model, [structs[b]], feats[off[b]:off[b + 1]], fmax=0.0, steps=6, optimize_lattice=True,
                               stress_wt=0.8)
        sl = slice(off[b], off[b + 1])
        assert torch.equal(one.positions, got.positions[sl]), b
        assert torch.equal(one.cells[0], got.cells[b]), b
        assert torch.equal(one.forces, got.forces[sl]), b
        assert torch.equal(one.stress[0], got.stress[b]), b
        assert torch.allclose(one.energy, got.energy[b:b + 1], rtol=1e-5, atol=0), b


def _with_short_bond(structs, feats):
    lat, X = structs[1]
    short = (lat, np.concatenate([X, X[:1] + np.array([0.8, 0.0, 0.0])]))
    return short, feats[:1].repeat(X.shape[0] + 1, 1)


def test_bond_penalty_counted_once_per_crystal_in_the_stress():
    model = _model()
    structs, feats = _structures(count=4)
    short, f_short = _with_short_bond(structs, feats)
    got = relax_structures(model, structs + [short], torch.cat([feats, f_short]), fmax=0.0, steps=3, optimize_lattice=True)
    one = relax_structures(model, [short], f_short, fmax=0.0, steps=3, optimize_lattice=True)
    off = got.atom_offsets.cpu().tolist()
    sl = slice(off[-2], off[-1])
    F1, S1 = one.forces.cpu().numpy(), one.stress.cpu().numpy()[0]
    assert np.abs(got.forces[sl].cpu().numpy() - F1).max() <= 1e-5 * np.abs(F1).max()
    assert np.abs(got.stress[-1].cpu().numpy() - S1).max() <= 1e-5 * np.abs(S1).max()
    assert np.abs(got.positions[sl].cpu().numpy() - one.positions.cpu().numpy()).max() <= 1e-6
    assert np.abs(got.cells[-1].cpu().numpy() - one.cells[0].cpu().numpy()).max() <= 1e-6


def test_relax_cells_under_no_grad():
    model = _model()
    structs, feats = _structures(count=3)
    short, f_short = _with_short_bond(structs, feats)
    structs, feats = structs + [short], torch.cat([feats, f_short])
    ref = relax_structures(model, structs, feats, fmax=0.0, steps=3, optimize_lattice=True)
    with torch.no_grad():
        got = relax_structures(model, structs, feats, fmax=0.0, steps=3, optimize_lattice=True)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)


def test_relax_cells_rejections():
    structs, feats = _structures(count=2)
    torch.manual_seed(0)
    no_stress = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=1, gcn_layers=1,
                                                    hidden_features=64, atom_input_features=92)).to(DEV).eval()
    with pytest.raises(ValueError, match="stress"):
        relax_structures(no_stress, structs, feats, optimize_lattice=True)
    model = _model()
    for wt in (float("nan"), float("inf"), "1.0", True, None):
        with pytest.raises(ValueError, match="stress_wt"):
            relax_structures(model, structs, feats, optimize_lattice=True, stress_wt=wt)
    for flag in ("False", 1, None):                                           # a truthy string must not pick the cells
        with pytest.raises(ValueError, match="optimize_lattice"):
            relax_structures(model, structs, feats, optimize_lattice=flag)
    with pytest.raises(ValueError, match="fmax"):                            # the existing rejections still apply
        relax_structures(model, structs, feats, fmax=-1.0, optimize_lattice=True)
    with pytest.raises(ValueError, match="eval"):
        relax_structures(model.train(), structs, feats, optimize_lattice=True)
    model.eval()
    # optimize_lattice=False is the fixed-cell path: a RelaxResult, cells untouched
    got = relax_structures(model, structs, feats, fmax=0.0, steps=2)
    assert type(got).__name__ == "RelaxResult"
    got = relax_structures(model, structs, feats, fmax=1e6, steps=2, optimize_lattice=np.bool_(True))
    assert type(got).__name__ == "CellRelaxResult" and got.converged.tolist() == [True, True]
    assert np.array_equal(got.cells.cpu().numpy(), np.stack([lat for lat, _ in structs]))
