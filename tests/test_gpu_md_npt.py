"""GPU (-m gpu): batched NPT Berendsen molecular dynamics.  The step kernel (`ops.md_npt_step`, csrc/md_device.cu)
against the numpy restatement `oracle/md_npt_oracle.py` on scripted forces and stresses, and
`run_md(ensemble="npt_berendsen")` against a host loop that runs each crystal alone the reference's way (host graph
build on the current cell, the same model on a one-crystal batch, the oracle's integrator)."""
import numpy as np
import pytest
import torch

from alignn_b200 import maxwell_boltzmann_momenta, neighbors, ops, run_md
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from oracle import md_npt_oracle as NO
from oracle import md_oracle as MO
from tests.test_gpu_relax_cell import _host_evaluator, _model, _structures

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max()) / max(float(np.abs(b).max()), 1e-300)


# ---- 1. the step kernel on scripted forces and stresses ----------------------------------------------------------------
SIZES = [1, 2, 30, 1000]
MULT, WT, STEPS, DT = 1.5, 0.8, 10, 1.0 * MO.fs
T0 = [300.0, 500.0, 200.0, 800.0]
P0 = [0.0, 0.01, -0.02, 0.005]                  # eV/A^3
COMP = 0.3                                      # A^3/eV: with taup = 10 dt and |P - P0| ~ 0.01-0.1, |1 - mu| ~ 1e-4-1e-3


def _script(b, k, n, cache={}):
    """(grad, model stress) of crystal b at its k-th evaluation (2e logged, 2e + 1 evaluation A of step e + 1)."""
    if (b, n) not in cache:
        rng = np.random.default_rng(100 + b)
        S = rng.normal(size=(3, 3))
        cache[(b, n)] = (rng.normal(size=(n, 3)), 20.0 * (S + S.T))
    g, S = cache[(b, n)]
    w = 1.0 + 0.3 * np.sin(k + b)
    return (g * w).astype(np.float32), (S * w + np.diag([5.0, 5.0, 5.0]) * b).astype(np.float32)


def _scripted_run(taut):
    aoff = neighbors.ragged_offsets(SIZES)
    N, B = int(aoff[-1]), len(SIZES)
    rng = np.random.default_rng(0)
    C0 = np.stack([np.diag([4.0, 4.5, 5.0]) + 0.3 * rng.normal(size=(3, 3)) for _ in range(3)] + [np.diag([20., 21., 22.])])
    x0 = np.concatenate([rng.random((n, 3)) @ C0[b] for b, n in enumerate(SIZES)])
    m = rng.choice([1.008, 12.011, 63.546, 196.97], N) * rng.uniform(0.9, 1.1, N)
    p0 = np.concatenate([MO.maxwell_boltzmann_momenta(m[aoff[b]:aoff[b + 1]], T, rng) for b, T in enumerate(T0)])
    p0[aoff[1]:aoff[2]] = 0.0                                          # crystal 1 starts at rest
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)   # noqa: E731
    pos, mom, m_d, cells = t64(x0), t64(p0), t64(m), t64(C0)
    t0, p0_d, comp = t64(T0), t64(P0), t64([COMP] * B)
    forces = torch.zeros(N, 3, device=DEV, dtype=torch.float32)
    stress_out = torch.zeros(B, 6, device=DEV, dtype=torch.float32)
    ekin, temp, press = (torch.zeros(B, dtype=torch.float64, device=DEV) for _ in range(3))
    status = torch.zeros(B, device=DEV, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(DEV)
    orc = [NO.NPT(C0[b], x0[aoff[b]:aoff[b + 1]], m[aoff[b]:aoff[b + 1]], dt=DT, temperature_K=T0[b], pressure_au_=P0[b],
                  compressibility_au_=COMP, taut=taut, taup=10 * DT, momenta=p0[aoff[b]:aoff[b + 1]]) for b in range(B)]
    kw = dict(steps=STEPS, dt=DT, kB=MO.kB, taut=taut, taup=10 * DT, force_multiplier=MULT, stress_wt=WT)
    worst, mus = 0.0, []

    def launch(k, e, phase):
        sc = [_script(b, k, SIZES[b]) for b in range(B)]
        grad = torch.from_numpy(np.concatenate([g for g, _ in sc])).to(DEV)
        stress = torch.from_numpy(np.stack([s for _, s in sc])).to(DEV)
        ops.md_npt_step(grad, stress, aoff_d, m_d, t0, p0_d, comp, cells, pos, mom, forces, stress_out, ekin, temp, press,
                        status, evaluation=e, phase=phase, **kw)
        return sc

    def compare(b, e):
        nonlocal worst
        sl = slice(aoff[b], aoff[b + 1])
        o = orc[b]
        for got, want in ((pos.cpu().numpy()[sl], o.x), (mom.cpu().numpy()[sl], o.p), (cells.cpu().numpy()[b], o.C)):
            d = _rel(got, want)
            worst = max(worst, d)
            assert d <= 1e-12, (b, e, d)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for e in range(STEPS + 1):
            sc = launch(2 * e, e, 0)
            assert status.tolist() == [0] * B
            F, SO = forces.cpu().numpy(), stress_out.cpu().numpy()
            EK, TT, PP = ekin.cpu().numpy(), temp.cpu().numpy(), press.cpu().numpy()
            for b, o in enumerate(orc):
                f = MO.scaled_forces(sc[b][0], MULT)
                sv = NO.calculator_stress(sc[b][1], WT)
                if e >= 1:
                    o.second_half(f.astype(np.float64))
                assert np.array_equal(F[aoff[b]:aoff[b + 1]], f) and np.array_equal(SO[b], sv), (b, e)
                assert _rel(EK[b], MO.kinetic_energy(o.p, o.m)) <= 1e-12 and _rel(TT[b], MO.temperature(o.p, o.m)) <= 1e-12
                assert _rel(PP[b], NO.pressure(NO.ideal_gas_stress(sv, o.p, o.m, o.C))) <= 1e-12, (b, e)
                if e < STEPS:
                    o.first_half(sv)
                    mus.append(o.mu)
                compare(b, e)
            if e == STEPS:
                break
            sc = launch(2 * e + 1, e, 1)
            for b, o in enumerate(orc):
                o.middle(MO.scaled_forces(sc[b][0], MULT).astype(np.float64))
                compare(b, e)
    return worst, mus, [t.clone() for t in (pos, mom, cells, forces, stress_out, ekin, temp, press, status)]


@pytest.mark.parametrize("taut", [DT, 10 * DT])
def test_md_npt_step_matches_oracle_on_scripted_forces(taut):
    worst, mus, first = _scripted_run(taut)
    dev = np.abs(np.array(mus) - 1.0)
    print(f"[npt scripted taut={taut / DT:g} dt] |1 - mu| {dev.min():.2g}..{dev.max():.2g}, largest relative "
          f"difference {worst:.2g}")
    assert 1e-4 < dev.max() < 1e-2
    _, _, again = _scripted_run(taut)
    for a, b in zip(first, again):
        assert torch.equal(a, b)                                          # bitwise repeatable


def _same(a, b):
    """Bitwise equality, NaN included."""
    if a.is_floating_point():
        a, b = (t.view(torch.int64 if t.dtype == torch.float64 else torch.int32) for t in (a, b))
    return torch.equal(a, b)


def _one(n, cell, stress):
    t = dict(grad=torch.ones(n, 3, device=DEV), stress=torch.tensor(stress, dtype=torch.float32, device=DEV).view(1, 3, 3),
             aoff=torch.tensor([0, n], dtype=torch.int64, device=DEV),
             m=torch.full((n,), 12.0, dtype=torch.float64, device=DEV),
             t0=torch.tensor([300.0], dtype=torch.float64, device=DEV),
             p0=torch.tensor([0.0], dtype=torch.float64, device=DEV),
             comp=torch.tensor([1.0], dtype=torch.float64, device=DEV),
             cells=torch.tensor(cell, dtype=torch.float64, device=DEV).view(1, 3, 3),
             pos=torch.randn(n, 3, dtype=torch.float64, device=DEV), mom=torch.randn(n, 3, dtype=torch.float64, device=DEV),
             forces=torch.zeros(n, 3, device=DEV), so=torch.zeros(1, 6, device=DEV),
             ek=torch.full((1,), -1.0, dtype=torch.float64, device=DEV),
             tt=torch.full((1,), -1.0, dtype=torch.float64, device=DEV),
             pp=torch.full((1,), -1.0, dtype=torch.float64, device=DEV), st=torch.zeros(1, dtype=torch.int32, device=DEV))
    return t


def _launch(t, **kw):
    base = dict(evaluation=0, steps=3, phase=0, dt=DT, kB=MO.kB, taut=10 * DT, taup=100 * DT, force_multiplier=1.0,
                stress_wt=1.0)
    ops.md_npt_step(t["grad"], t["stress"], t["aoff"], t["m"], t["t0"], t["p0"], t["comp"], t["cells"], t["pos"], t["mom"],
                    t["forces"], t["so"], t["ek"], t["tt"], t["pp"], t["st"], **dict(base, **kw))


def test_bad_slice_and_degenerate_cells_touch_nothing_but_their_status():
    cases = [(_one(2, np.zeros((3, 3)), np.eye(3)), ops.MD_CELL_DEGENERATE, 0),           # no volume
             (_one(2, np.eye(3) * 4.0, np.full((3, 3), np.nan)), ops.MD_CELL_DEGENERATE, 0),   # NaN stress: mu is NaN
             (_one(2, np.eye(3) * 4.0, np.eye(3)), ops.MD_BAD_INPUT, 0)]                     # slice outside grad
    cases[2][0]["grad"] = torch.ones(1, 3, device=DEV)
    for t, want, e in cases:
        before = {k: v.clone() for k, v in t.items()}
        _launch(t, evaluation=e)
        assert t["st"].item() == want
        for k in before:
            if k != "st":
                assert _same(before[k], t[k]), (want, k)
        for phase in (0, 1):                                              # a reported crystal is not touched again
            _launch(t, evaluation=1, phase=phase)
            for k in before:
                if k != "st":
                    assert _same(before[k], t[k]), (want, k)
    t = _one(2, np.eye(3) * 4.0, np.full((3, 3), np.nan))                 # NaN stress at the last evaluation: logged
    _launch(t, evaluation=3)
    assert t["st"].item() == 0 and np.isnan(t["pp"].item())


def test_md_npt_step_rejects_bad_parameters():
    t = _one(2, np.eye(3) * 4.0, np.eye(3))
    for bad in (dict(dt=0.0), dict(dt=float("nan")), dict(dt=float("inf")), dict(kB=0.0), dict(taut=0.5 * DT),
                dict(taut=float("inf")), dict(taup=0.0), dict(taup=-1.0), dict(taup=float("nan")),
                dict(force_multiplier=float("nan")), dict(stress_wt=float("inf")), dict(stress_wt=float("nan")),
                dict(phase=2), dict(phase=-1), dict(phase=1, evaluation=3)):
        with pytest.raises(RuntimeError, match="alignn_b200_md_npt_step failed"):
            _launch(t, **bad)
    for bad in (dict(evaluation=4), dict(evaluation=-1), dict(steps=0)):
        with pytest.raises(ValueError):
            _launch(t, **bad)
    t["cells"] = torch.zeros(2, 3, 3, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="shapes"):
        _launch(t)
    assert t["st"].item() == 0


# ---- 2-7. run_md(ensemble="npt_berendsen") -------------------------------------------------------------------------------
def _inputs(count=8, seed=3):
    structs, feats = _structures(count=count, seed=seed)
    n = sum(x.shape[0] for _, x in structs)
    rng = np.random.default_rng(seed + 1)
    masses = rng.uniform(1.0, 200.0, n)
    return structs, feats, masses, maxwell_boltzmann_momenta(masses, 300.0, rng)


NPT_KW = dict(compressibility=2e-6, taup=100.0, taut=50.0)


@pytest.mark.parametrize("strategy,cutoff", [("k-nearest", 8.0), ("radius_graph", 6.0)])
def test_run_md_npt_matches_host_loop(strategy, cutoff):
    model = _model()
    structs, feats, masses, p0 = _inputs()
    B = len(structs)
    steps, mult, dt_fs = 20, 1.5, 1.0
    pressure = [1e4 * (b - 3) for b in range(B)]
    got = run_md(model, structs, feats, masses, ensemble="npt_berendsen", steps=steps, timestep=dt_fs,
                 temperature_K=300.0, pressure=pressure, momenta=p0, neighbor_strategy=strategy, cutoff=cutoff,
                 force_multiplier=mult, **NPT_KW)
    assert type(got).__name__ == "NPTResult"
    off = got.atom_offsets.cpu().tolist()
    P, Q, F = got.positions.cpu().numpy(), got.momenta.cpu().numpy(), got.forces.cpu().numpy()
    E, EK, T, PR = (t.cpu().numpy() for t in (got.energy, got.kinetic_energy, got.temperature, got.pressure))
    CL, SL = got.cells.cpu().numpy(), got.stress.cpu().numpy()
    assert CL.shape == (steps + 1, B, 3, 3) and SL.shape == (steps + 1, B, 6) and PR.shape == (steps + 1, B)
    moved, dpos, dcell = 0.0, 0.0, 0.0
    for b, (lat, X) in enumerate(structs):
        sl = slice(off[b], off[b + 1])
        r = NO.run(_host_evaluator(model, feats[sl], strategy, cutoff), lat, X, masses[sl], steps=steps,
                   dt=dt_fs * MO.fs, temperature_K=300.0, pressure=pressure[b], compressibility=NPT_KW["compressibility"],
                   taut=NPT_KW["taut"] * MO.fs, taup=NPT_KW["taup"] * MO.fs, momenta=p0[sl], force_multiplier=mult)
        dpos, dcell = max(dpos, np.abs(P[sl] - r["positions"]).max()), max(dcell, np.abs(CL[:, b] - r["cells"]).max())
        assert np.abs(P[sl] - r["positions"]).max() <= 1e-9, b
        assert np.abs(CL[:, b] - np.stack(r["cells"])).max() <= 1e-9, b
        assert _rel(Q[sl], r["momenta"]) <= 1e-9, b
        for got_, want in ((EK[:, b], r["kinetic_energy"]), (T[:, b], r["temperature"]), (PR[:, b], r["pressure"])):
            assert _rel(got_, want) <= 1e-9, b
        assert _rel(F[sl], r["forces"]) <= 1e-5 and _rel(E[:, b], r["energy"]) <= 1e-5, b
        assert _rel(SL[:, b], np.stack(r["stress"])) <= 1e-5, b
        moved = max(moved, float(np.abs(CL[-1, b] - lat).max()))
    print(f"[npt {strategy}] cells moved by up to {moved:.3g} A; largest difference positions {dpos:.3g} A, "
          f"cells {dcell:.3g} A")
    assert moved > 1e-3, moved


def test_zero_compressibility_is_nvt_berendsen_bitwise():
    model = _model()
    structs, feats, masses, p0 = _inputs(count=4)
    kw = dict(steps=6, timestep=1.0, temperature_K=[250.0, 300.0, 350.0, 400.0], taut=20.0, momenta=p0)
    npt = run_md(model, structs, feats, masses, ensemble="npt_berendsen", pressure=1e4, compressibility=0.0, **kw)
    nvt = run_md(model, structs, feats, masses, ensemble="nvt_berendsen", **kw)
    for name in ("positions", "momenta", "forces", "kinetic_energy", "temperature"):
        assert torch.equal(getattr(npt, name), getattr(nvt, name)), name
    assert torch.equal(npt.cells, torch.from_numpy(np.stack([lat for lat, _ in structs])).to(DEV).expand_as(npt.cells))


def test_run_md_npt_is_batch_invariant():
    model = _model()
    structs, feats, masses, p0 = _inputs()
    B = len(structs)
    T0, P = [200.0 + 50.0 * b for b in range(B)], [-1e4 + 5e3 * b for b in range(B)]
    kw = dict(ensemble="npt_berendsen", steps=5, timestep=1.0, **NPT_KW)
    got = run_md(model, structs, feats, masses, temperature_K=T0, pressure=P, momenta=p0, **kw)
    off = got.atom_offsets.cpu().tolist()
    for b in (0, 3, B - 1):
        sl = slice(off[b], off[b + 1])
        one = run_md(model, [structs[b]], feats[sl], masses[sl], temperature_K=T0[b], pressure=P[b], momenta=p0[sl], **kw)
        for name in ("positions", "momenta", "forces"):
            assert torch.equal(getattr(one, name), getattr(got, name)[sl]), (b, name)
        for name in ("kinetic_energy", "temperature", "pressure", "cells", "stress"):
            assert torch.equal(getattr(one, name)[:, 0], getattr(got, name)[:, b]), (b, name)
        assert torch.allclose(one.energy[:, 0], got.energy[:, b], rtol=1e-5, atol=0), b


def _with_short_bond(structs, feats, masses, p0):
    lat, X = structs[1]
    short = (lat, np.concatenate([X, X[:1] + np.array([0.8, 0.0, 0.0])]))
    f_short = feats[:1].repeat(X.shape[0] + 1, 1)
    m_short, p_short = np.full(X.shape[0] + 1, 30.0), np.zeros((X.shape[0] + 1, 3))
    return (structs + [short], torch.cat([feats, f_short]), np.concatenate([masses, m_short]),
            np.concatenate([p0, p_short]), (short, f_short, m_short, p_short))


def test_bond_penalty_counted_once_per_crystal_in_the_stress():
    model = _model()
    structs, feats, masses, p0, (short, f_s, m_s, p_s) = _with_short_bond(*_inputs(count=4))
    kw = dict(ensemble="npt_berendsen", steps=3, timestep=1.0, pressure=0.0, **NPT_KW)
    got = run_md(model, structs, feats, masses, momenta=p0, **kw)
    one = run_md(model, [short], f_s, m_s, momenta=p_s, **kw)
    S1 = one.stress[:, 0].cpu().numpy()
    assert _rel(got.stress[:, -1].cpu().numpy(), S1) <= 1e-5
    assert np.abs(got.cells[:, -1].cpu().numpy() - one.cells[:, 0].cpu().numpy()).max() <= 1e-6
    sl = slice(int(got.atom_offsets[-2]), int(got.atom_offsets[-1]))
    assert np.abs(got.positions[sl].cpu().numpy() - one.positions.cpu().numpy()).max() <= 1e-6


def test_run_md_npt_under_no_grad_and_trajectory():
    model = _model()
    structs, feats, masses, p0, _ = _with_short_bond(*_inputs(count=3))
    kw = dict(ensemble="npt_berendsen", timestep=1.0, pressure=5e3, momenta=p0, **NPT_KW)
    ref = run_md(model, structs, feats, masses, steps=7, trajectory_interval=3, **kw)
    with torch.no_grad():
        got = run_md(model, structs, feats, masses, steps=7, trajectory_interval=3, **kw)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    X = torch.from_numpy(np.concatenate([x for _, x in structs])).to(DEV)
    assert ref.trajectory.shape == (3, X.shape[0], 3) and torch.equal(ref.trajectory[0], X)
    for i, s in ((1, 3), (2, 6)):
        stop = run_md(model, structs, feats, masses, steps=s, **kw)
        assert torch.equal(ref.trajectory[i], stop.positions) and torch.equal(ref.cells[s], stop.cells[-1]), s


def test_run_md_npt_rejections():
    model = _model()
    structs, feats, masses, p0 = _inputs(count=2)
    ok = dict(ensemble="npt_berendsen", steps=2, pressure=1.0, compressibility=1e-6)
    torch.manual_seed(0)
    no_stress = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=1, gcn_layers=1,
                                                    hidden_features=64, atom_input_features=92)).to(DEV).eval()
    with pytest.raises(ValueError, match="stress"):
        run_md(no_stress, structs, feats, masses, **ok)
    bad = [dict(pressure=None), dict(pressure=float("nan")), dict(pressure=[1.0]), dict(pressure="1"),
           dict(compressibility=None), dict(compressibility=-1e-6), dict(compressibility=float("inf")),
           dict(compressibility=[1e-6, 1e-6, 1e-6]), dict(taup=0.0), dict(taup=float("nan")), dict(taup=None),
           dict(stress_wt=float("nan")), dict(stress_wt=True), dict(timestep=1.0, taut=0.5),
           dict(temperature_K=0.0), dict(temperature_K=[300.0])]
    for kw in bad:
        with pytest.raises(ValueError):
            run_md(model, structs, feats, masses, **dict(ok, **kw))
    # a barostat scale that turns negative on crystal 1 in the first step
    with pytest.raises(RuntimeError, match="cell of crystal 1 became degenerate in step 1"):
        run_md(model, structs, feats, masses, **dict(ok, pressure=[0.0, 1e9], compressibility=[0.0, 1e6]))
    # accepted: per-crystal values, negative pressure, numpy scalars; ignored by the other ensembles
    got = run_md(model, structs, feats, masses, **dict(ok, pressure=[-1e3, np.float64(2e3)], compressibility=np.float32(0)))
    assert got.cells.shape == (3, 2, 3, 3)
    run_md(model, structs, feats, masses, steps=1, pressure=float("nan"), compressibility=-1.0, taup=None)
