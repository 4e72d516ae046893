"""GPU (-m gpu): batched NPT Nose-Hoover / Parrinello-Rahman molecular dynamics (ASE's NPT).  The step kernel
(`ops.md_nose_hoover_step`, csrc/md_device.cu) against the numpy restatement `oracle/md_nose_hoover_oracle.py` on
scripted forces and stresses, and `run_md(ensemble="npt_nose_hoover")` against a host loop that runs each crystal alone
the reference's way (host graph build on the current cell, the same model on a one-crystal batch, the oracle's
integrator)."""
import numpy as np
import pytest
import torch

from alignn_b200 import maxwell_boltzmann_momenta, md, neighbors, ops, run_md, upper_triangular
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from oracle import md_nose_hoover_oracle as NH
from oracle import md_oracle as MO
from tests.test_gpu_relax_cell import _host_evaluator, _model, _structures

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max()) / max(float(np.abs(b).max()), 1e-300)


def _t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(DEV)


# ---- 1. the step kernel on scripted forces and stresses ----------------------------------------------------------------
SIZES = [1, 2, 30, 1000]
MULT, WT, STEPS, DT = 1.5, 0.8, 10, 1.0 * MO.fs
T0 = [300.0, 500.0, 200.0, 800.0]
SYM = np.array([[0.01, 0.002, -0.001], [0.002, -0.02, 0.003], [-0.001, 0.003, 0.005]])
EXT = [0.0, 0.01, SYM, -0.02]                    # eV/A^3: pressures, and one symmetric 3 x 3 stress


def _script(b, k, n, cache={}):
    """(grad, model stress) of crystal b at its k-th evaluation; crystal 1, which starts at rest, gets first forces
    gentle enough for ASE's initialisation to stop after its first pass."""
    if (b, n) not in cache:
        rng = np.random.default_rng(200 + b)
        S = rng.normal(size=(3, 3))
        cache[(b, n)] = (rng.normal(size=(n, 3)), 20.0 * (S + S.T))
    g, S = cache[(b, n)]
    w = 1.0 + 0.3 * np.sin(k + b)
    gentle = 1e-3 if (b, k) == (1, 0) else 1.0
    return (g * w * gentle).astype(np.float32), (S * w + np.diag([5.0, 5.0, 5.0]) * b).astype(np.float32)


# relative bounds for positions, momenta and cells.  The momenta are a central difference, (q_future - q_past) h m /
# (2 dt), of fractional coordinates of about 0.5 that move by 1e-4..1e-3 per step in the 20 A cell: an ulp of q is
# 1e-13..1e-12 of that difference, so numpy's and the kernel's rounding orders part by up to a few 1e-12 there, and the
# kinetic energy and temperature, quadratic in the momenta, by twice that.
TOL = (1e-12, 5e-12, 1e-12)


def _scripted_run(ttime, pfactor):
    aoff = neighbors.ragged_offsets(SIZES)
    N, B = int(aoff[-1]), len(SIZES)
    rng = np.random.default_rng(0)
    C0 = np.stack([np.triu(np.diag([4.0, 4.5, 5.0]) + 0.3 * rng.normal(size=(3, 3))) for _ in range(3)]
                  + [np.diag([20., 21., 22.])])
    x0 = np.concatenate([rng.random((n, 3)) @ C0[b] for b, n in enumerate(SIZES)])
    m = rng.choice([1.008, 12.011, 63.546, 196.97], N) * rng.uniform(0.9, 1.1, N)
    p0 = np.concatenate([MO.maxwell_boltzmann_momenta(m[aoff[b]:aoff[b + 1]], T, rng) for b, T in enumerate(T0)])
    p0[aoff[1]:aoff[2]] = 0.0                                          # crystal 1 starts at rest
    tf, pf, de = md._nose_hoover_constants(SIZES, T0, ttime, pfactor, C0)
    ext = np.concatenate([md._external_stress(s, 1) for s in EXT])
    pos, mom, m_d, cells = _t64(x0), _t64(p0), _t64(m), _t64(C0)
    tf_d, pf_d, de_d, ext_d = _t64(tf), _t64(pf), _t64(de), _t64(ext)
    state = torch.zeros(B, ops.MD_NH_STATE, dtype=torch.float64, device=DEV)
    q, qf = torch.zeros(N, 3, dtype=torch.float64, device=DEV), torch.zeros(N, 3, dtype=torch.float64, device=DEV)
    forces = torch.zeros(N, 3, device=DEV, dtype=torch.float32)
    stress_out = torch.zeros(B, 6, device=DEV, dtype=torch.float32)
    ekin, temp, press = (torch.zeros(B, dtype=torch.float64, device=DEV) for _ in range(3))
    status = torch.zeros(B, device=DEV, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(DEV)
    orc = [NH.NPT(C0[b], x0[aoff[b]:aoff[b + 1]], m[aoff[b]:aoff[b + 1]], dt=DT, temperature_K=T0[b],
                  externalstress=EXT[b], ttime=ttime, pfactor=pfactor, momenta=p0[aoff[b]:aoff[b + 1]])
           for b in range(B)]
    worst = [0.0, 0.0, 0.0]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for e in range(STEPS + 1):
            sc = [_script(b, e, SIZES[b]) for b in range(B)]
            grad = torch.from_numpy(np.concatenate([g for g, _ in sc])).to(DEV)
            stress = torch.from_numpy(np.stack([s for _, s in sc])).to(DEV)
            ops.md_nose_hoover_step(grad, stress, aoff_d, m_d, tf_d, pf_d, de_d, ext_d, cells, state, pos, mom, q, qf,
                                    forces, stress_out, ekin, temp, press, status, evaluation=e, steps=STEPS, dt=DT,
                                    kB=MO.kB, force_multiplier=MULT, stress_wt=WT)
            assert status.tolist() == [0] * B
            F, SO = forces.cpu().numpy(), stress_out.cpu().numpy()
            EK, TT, PP = ekin.cpu().numpy(), temp.cpu().numpy(), press.cpu().numpy()
            P, Q, CC = pos.cpu().numpy(), mom.cpu().numpy(), cells.cpu().numpy()
            for b, o in enumerate(orc):
                sl = slice(aoff[b], aoff[b + 1])
                f = MO.scaled_forces(sc[b][0], MULT)
                sv = NH.calculator_stress(sc[b][1], WT)
                if e == 0:
                    o.initialize(f.astype(np.float64), sv)
                else:
                    o.finish_step(f.astype(np.float64))
                assert np.array_equal(F[sl], f) and np.array_equal(SO[b], sv), (b, e)
                assert _rel(EK[b], MO.kinetic_energy(o.p, o.m)) <= 2 * TOL[1], (b, e)
                assert _rel(TT[b], MO.temperature(o.p, o.m)) <= 2 * TOL[1], (b, e)
                assert _rel(PP[b], NH.pressure(NH.ideal_gas_stress(sv, o.p, o.m, o.h))) <= 1e-12, (b, e)
                if e < STEPS:
                    o.begin_step(sv)
                for j, (got, want) in enumerate(((P[sl], o.x), (Q[sl], o.p), (CC[b], o.h))):
                    d = _rel(got, want)
                    worst[j] = max(worst[j], d)
                    assert d <= TOL[j], (b, e, j, d)
    assert [o.passes for o in orc] == [2, 1, 2, 2]                     # the crystal at rest stops after one pass
    moved = max(float(np.abs(o.h - C0[b]).max()) for b, o in enumerate(orc))
    return worst, moved, [t.clone() for t in (pos, mom, cells, state, q, qf, forces, stress_out, ekin, temp, press)]


@pytest.mark.parametrize("ttime,pfactor", [(None, None), (20 * DT, None), (20 * DT, 500.0)])
def test_md_nose_hoover_step_matches_oracle_on_scripted_forces(ttime, pfactor):
    worst, moved, first = _scripted_run(ttime, pfactor)
    print(f"[nose-hoover scripted ttime={ttime} pfactor={pfactor}] largest relative differences: positions "
          f"{worst[0]:.2g}, momenta {worst[1]:.2g}, cells {worst[2]:.2g}; cells moved by up to {moved:.2g} A")
    if pfactor is None:
        C0 = first[2].cpu().numpy()
        assert moved == 0.0 and np.all(np.triu(C0) == C0)
    else:
        assert moved > 1e-3
    _, _, again = _scripted_run(ttime, pfactor)
    for a, b in zip(first, again):
        assert torch.equal(a, b)                                          # bitwise repeatable


def _same(a, b):
    """Bitwise equality, NaN included."""
    if a.is_floating_point():
        a, b = (t.view(torch.int64 if t.dtype == torch.float64 else torch.int32) for t in (a, b))
    return torch.equal(a, b)


def _one(n, cell):
    f64 = dict(dtype=torch.float64, device=DEV)
    return dict(grad=torch.ones(n, 3, device=DEV), stress=torch.eye(3, device=DEV).view(1, 3, 3),
                aoff=torch.tensor([0, n], dtype=torch.int64, device=DEV), m=torch.full((n,), 12.0, **f64),
                tf=torch.full((1,), 0.1, **f64), pf=torch.full((1,), 0.01, **f64), de=torch.full((1,), 0.05, **f64),
                ext=torch.zeros(1, 6, **f64), cells=torch.tensor(cell, **f64).view(1, 3, 3),
                state=torch.zeros(1, ops.MD_NH_STATE, **f64), pos=torch.randn(n, 3, **f64),
                mom=torch.randn(n, 3, **f64), q=torch.randn(n, 3, **f64), qf=torch.randn(n, 3, **f64),
                forces=torch.zeros(n, 3, device=DEV), so=torch.zeros(1, 6, device=DEV),
                ek=torch.full((1,), -1.0, **f64), tt=torch.full((1,), -1.0, **f64), pp=torch.full((1,), -1.0, **f64),
                st=torch.zeros(1, dtype=torch.int32, device=DEV))


def _launch(t, **kw):
    base = dict(evaluation=0, steps=3, dt=DT, kB=MO.kB, force_multiplier=1.0, stress_wt=1.0)
    ops.md_nose_hoover_step(t["grad"], t["stress"], t["aoff"], t["m"], t["tf"], t["pf"], t["de"], t["ext"], t["cells"],
                            t["state"], t["pos"], t["mom"], t["q"], t["qf"], t["forces"], t["so"], t["ek"], t["tt"],
                            t["pp"], t["st"], **dict(base, **kw))


def test_bad_slice_and_degenerate_crystals_touch_nothing_but_their_status():
    sheared = np.eye(3) * 4.0
    sheared[2, 1] = 0.5
    cases = [(_one(2, sheared), ops.MD_BAD_INPUT, dict(evaluation=0)),                 # not upper triangular
             (_one(2, np.eye(3) * 4.0), ops.MD_BAD_INPUT, dict(evaluation=0)),          # slice outside grad
             (_one(2, np.zeros((3, 3))), ops.MD_CELL_DEGENERATE, dict(evaluation=0)),   # no volume
             (_one(2, np.eye(3) * 4.0), ops.MD_CELL_DEGENERATE, dict(evaluation=1)),    # h_past = eta = 0: h_future 0
             (_one(2, np.eye(3) * 4.0), ops.MD_CELL_DEGENERATE, dict(evaluation=1, dt=1.0)),   # beta + I = 0
             (_one(2, np.eye(3) * 4.0), ops.MD_CELL_DEGENERATE, dict(evaluation=1))]    # a NaN eta
    cases[1][0]["grad"] = torch.ones(1, 3, device=DEV)
    for t in (cases[4][0], cases[5][0]):
        t["state"][0, 0:9] = t["cells"].reshape(-1)                                  # h_past = h
        t["state"][0, 9:18] = -torch.eye(3, dtype=torch.float64, device=DEV).reshape(-1)   # eta = -I/dt for dt = 1
    cases[5][0]["state"][0, 10] = float("nan")
    for t, want, kw in cases:
        before = {k: v.clone() for k, v in t.items()}
        _launch(t, **kw)
        assert t["st"].item() == want, (want, kw)
        for k in before:
            if k != "st":
                assert _same(before[k], t[k]), (want, k)
        for ev in (1, 2, 3):                                              # a reported crystal is not touched again
            _launch(t, evaluation=ev)
            for k in before:
                if k != "st":
                    assert _same(before[k], t[k]), (want, k)
    t = _one(2, np.eye(3) * 4.0)                                          # the sheared-cell check is evaluation 0's
    t["state"][0, 0:9] = t["cells"].reshape(-1)
    t["cells"][0, 2, 1] = 0.5
    _launch(t, evaluation=1)
    assert t["st"].item() == 0


def test_md_nose_hoover_step_rejects_bad_parameters():
    t = _one(2, np.eye(3) * 4.0)
    for bad in (dict(dt=0.0), dict(dt=float("nan")), dict(dt=float("inf")), dict(dt=-1.0), dict(kB=0.0),
                dict(kB=float("nan")), dict(force_multiplier=float("nan")), dict(stress_wt=float("inf")),
                dict(stress_wt=float("nan"))):
        with pytest.raises(RuntimeError, match="alignn_b200_md_nose_hoover_step failed"):
            _launch(t, **bad)
    for bad in (dict(evaluation=4), dict(evaluation=-1), dict(steps=0), dict(evaluation=True)):
        with pytest.raises(ValueError):
            _launch(t, **bad)
    for k, v in (("state", torch.zeros(1, 28, dtype=torch.float64, device=DEV)),
                 ("ext", torch.zeros(1, 3, 3, dtype=torch.float64, device=DEV)),
                 ("qf", torch.zeros(3, 3, dtype=torch.float64, device=DEV))):
        u = dict(t, **{k: v})
        with pytest.raises(ValueError, match="shapes"):
            _launch(u)
    assert t["st"].item() == 0


# ---- 3-5. run_md(ensemble="npt_nose_hoover") ---------------------------------------------------------------------------
def _inputs(count=8, seed=3):
    structs, feats = _structures(count=count, seed=seed)
    structs, _ = upper_triangular(structs)
    n = sum(x.shape[0] for _, x in structs)
    rng = np.random.default_rng(seed + 1)
    masses = rng.uniform(1.0, 200.0, n)
    p0 = maxwell_boltzmann_momenta(masses, 300.0, rng)
    off = np.cumsum([0] + [x.shape[0] for _, x in structs])
    for b in range(len(structs)):                                        # centre-of-mass momentum removed
        p0[off[b]:off[b + 1]] -= p0[off[b]:off[b + 1]].sum(0) / (off[b + 1] - off[b])
    return structs, feats, masses, p0


NH_KW = dict(ttime=25.0, pfactor=100.0)


@pytest.mark.parametrize("strategy,cutoff", [("k-nearest", 8.0), ("radius_graph", 6.0)])
def test_run_md_nose_hoover_matches_host_loop(strategy, cutoff):
    model = _model()
    structs, feats, masses, p0 = _inputs()
    B = len(structs)
    steps, mult, dt_fs = 20, 1.5, 1.0
    ext = [0.01 * (b - 3) for b in range(B)]
    got = run_md(model, structs, feats, masses, ensemble="npt_nose_hoover", steps=steps, timestep=dt_fs,
                 temperature_K=300.0, externalstress=np.stack([NH.external_stress(s) for s in ext]), momenta=p0,
                 neighbor_strategy=strategy, cutoff=cutoff, force_multiplier=mult, **NH_KW)
    assert type(got).__name__ == "NPTResult"
    off = got.atom_offsets.cpu().tolist()
    P, Q, F = got.positions.cpu().numpy(), got.momenta.cpu().numpy(), got.forces.cpu().numpy()
    E, EK, T, PR = (t.cpu().numpy() for t in (got.energy, got.kinetic_energy, got.temperature, got.pressure))
    CL, SL = got.cells.cpu().numpy(), got.stress.cpu().numpy()
    assert CL.shape == (steps + 1, B, 3, 3) and SL.shape == (steps + 1, B, 6) and PR.shape == (steps + 1, B)
    moved, dpos, dcell = 0.0, 0.0, 0.0
    for b, (lat, X) in enumerate(structs):
        sl = slice(off[b], off[b + 1])
        r = NH.run(_host_evaluator(model, feats[sl], strategy, cutoff), lat, X, masses[sl], steps=steps,
                   dt=dt_fs * MO.fs, temperature_K=300.0, externalstress=ext[b], ttime=NH_KW["ttime"] * MO.fs,
                   pfactor=NH_KW["pfactor"], momenta=p0[sl], force_multiplier=mult)
        dpos = max(dpos, np.abs(P[sl] - r["positions"]).max())
        dcell = max(dcell, np.abs(CL[:, b] - np.stack(r["cells"])).max())
        assert np.abs(P[sl] - r["positions"]).max() <= 1e-9, b
        assert np.abs(CL[:, b] - np.stack(r["cells"])).max() <= 1e-9, b
        assert _rel(Q[sl], r["momenta"]) <= 1e-9, b
        for got_, want in ((EK[:, b], r["kinetic_energy"]), (T[:, b], r["temperature"]), (PR[:, b], r["pressure"])):
            assert _rel(got_, want) <= 1e-9, b
        assert _rel(F[sl], r["forces"]) <= 1e-5 and _rel(E[:, b], r["energy"]) <= 1e-5, b
        assert _rel(SL[:, b], np.stack(r["stress"])) <= 1e-5, b
        moved = max(moved, float(np.abs(CL[-1, b] - lat).max()))
        assert np.all(CL[:, b][:, [1, 2, 2], [0, 0, 1]] == 0.0), b
    print(f"[nose-hoover {strategy}] cells moved by up to {moved:.3g} A; largest difference positions {dpos:.3g} A, "
          f"cells {dcell:.3g} A")
    assert moved > 1e-3, moved


def test_thermostat_and_barostat_off_is_velocity_verlet():
    """The reference's call (ttime = pfactor = None) against run_md's NVE on the same centre-of-mass-free momenta.  In
    exact arithmetic the two trajectories are the same; here they part by rounding only: NPT goes through fractional
    coordinates and a central difference, so positions differ by a few ulps per step (measured on an H100 over 20
    steps: 2e-14 A) and the momenta, a difference of such positions over 2 dt, by about 1e-12 relative.  The bounds
    leave 50-100 times that; an fp32 force that rounds differently between the two would show as a much larger gap."""
    model = _model()
    structs, feats, masses, p0 = _inputs(count=6)
    kw = dict(steps=20, timestep=1.0, momenta=p0)
    nh = run_md(model, structs, feats, masses, ensemble="npt_nose_hoover", temperature_K=300.0, **kw)
    vv = run_md(model, structs, feats, masses, ensemble="nve_velocity_verlet", **kw)
    cells = torch.from_numpy(np.stack([lat for lat, _ in structs])).to(DEV)
    assert torch.equal(nh.cells, cells.expand_as(nh.cells))
    dpos = float((nh.positions - vv.positions).abs().max())
    dmom = float((nh.momenta - vv.momenta).abs().max() / vv.momenta.abs().max())
    dek = float(((nh.kinetic_energy - vv.kinetic_energy).abs() / vv.kinetic_energy.abs().max()).max())
    print(f"[nose-hoover off vs velocity Verlet] positions {dpos:.3g} A, momenta {dmom:.3g} relative, ekin {dek:.3g}")
    assert float((nh.positions - torch.from_numpy(np.concatenate([x for _, x in structs])).to(DEV)).abs().max()) > 1e-3
    assert dpos <= 1e-12 and dmom <= 1e-10 and dek <= 1e-10


def test_run_md_nose_hoover_is_batch_invariant():
    model = _model()
    structs, feats, masses, p0 = _inputs()
    B = len(structs)
    T0, ext = [200.0 + 50.0 * b for b in range(B)], [-0.01 + 0.005 * b for b in range(B)]
    kw = dict(ensemble="npt_nose_hoover", steps=5, timestep=1.0, **NH_KW)
    got = run_md(model, structs, feats, masses, temperature_K=T0, externalstress=np.stack(
        [NH.external_stress(s) for s in ext]), momenta=p0, **kw)
    off = got.atom_offsets.cpu().tolist()
    for b in (0, 3, B - 1):
        sl = slice(off[b], off[b + 1])
        one = run_md(model, [structs[b]], feats[sl], masses[sl], temperature_K=T0[b], externalstress=ext[b],
                     momenta=p0[sl], **kw)
        for name in ("positions", "momenta", "forces"):
            assert torch.equal(getattr(one, name), getattr(got, name)[sl]), (b, name)
        for name in ("kinetic_energy", "temperature", "pressure", "cells", "stress"):
            assert torch.equal(getattr(one, name)[:, 0], getattr(got, name)[:, b]), (b, name)
        assert torch.allclose(one.energy[:, 0], got.energy[:, b], rtol=1e-5, atol=0), b


def test_run_md_nose_hoover_no_grad_trajectory_and_one_forward_per_step():
    model = _model()
    structs, feats, masses, p0 = _inputs(count=3)
    kw = dict(ensemble="npt_nose_hoover", timestep=1.0, externalstress=0.005, momenta=p0, **NH_KW)
    calls = []
    hook = model.register_forward_hook(lambda *a: calls.append(1))
    try:
        ref = run_md(model, structs, feats, masses, steps=7, trajectory_interval=3, **kw)
    finally:
        hook.remove()
    assert len(calls) == 7 + 1                                            # one model call per step
    with torch.no_grad():
        got = run_md(model, structs, feats, masses, steps=7, trajectory_interval=3, **kw)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    X = torch.from_numpy(np.concatenate([x for _, x in structs])).to(DEV)
    assert ref.trajectory.shape == (3, X.shape[0], 3) and torch.equal(ref.trajectory[0], X)
    for i, s in ((1, 3), (2, 6)):
        stop = run_md(model, structs, feats, masses, steps=s, **kw)
        assert torch.equal(ref.trajectory[i], stop.positions) and torch.equal(ref.cells[s], stop.cells[-1]), s


def test_run_md_nose_hoover_rejections():
    model = _model()
    raw, feats = _structures(count=2)
    structs, _ = upper_triangular(raw)
    n = sum(x.shape[0] for _, x in structs)
    masses = np.full(n, 30.0)
    ok = dict(ensemble="npt_nose_hoover", steps=2)
    torch.manual_seed(0)
    no_stress = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=1, gcn_layers=1,
                                                    hidden_features=64, atom_input_features=92)).to(DEV).eval()
    with pytest.raises(ValueError, match="stress"):
        run_md(no_stress, structs, feats, masses, **ok)
    mixed = [structs[0], raw[1]]
    assert raw[1][0][1, 0] != 0.0
    with pytest.raises(ValueError, match="crystal 1 is not upper triangular.*upper_triangular"):
        run_md(model, mixed, feats, masses, **ok)
    S = np.array([[0.0, 1.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    bad = [dict(ttime=0.0), dict(ttime=-25.0), dict(ttime=float("nan")), dict(ttime="25"), dict(pfactor=0.0),
           dict(pfactor=float("inf")), dict(pfactor=True), dict(externalstress=[1.0, 2.0, 3.0]),
           dict(externalstress=np.zeros((2, 2))), dict(externalstress=float("nan")), dict(externalstress=S),
           dict(externalstress=np.zeros((3, 6))), dict(externalstress=None, pfactor=10.0),
           dict(stress_wt=float("nan")), dict(temperature_K=0.0), dict(temperature_K=[300.0])]
    for kw in bad:
        with pytest.raises(ValueError):
            run_md(model, structs, feats, masses, **dict(ok, **kw))
    # accepted: the forms of externalstress, numpy scalars, taut (ignored); the other ensembles ignore the new keywords
    for v in (np.float32(0.01), np.zeros(6), S + S.T, np.zeros((2, 6)), np.zeros((2, 3, 3)), None):
        got = run_md(model, structs, feats, masses, **dict(ok, externalstress=v, taut=1e-9))
        assert got.cells.shape == (3, 2, 3, 3)
    run_md(model, raw, feats, masses, steps=1, ttime=-1.0, pfactor="x", externalstress=None)


def test_upper_triangular_properties():
    model = _model()
    raw, feats = _structures(count=8)
    rot, R = upper_triangular(raw)
    assert R.shape == (8, 3, 3)
    off = np.cumsum([0] + [x.shape[0] for _, x in raw])
    for b, ((L0, X0), (L, X)) in enumerate(zip(raw, rot)):
        assert L[1, 0] == 0.0 and L[2, 0] == 0.0 and L[2, 1] == 0.0 and L[1, 1] > 0 and L[2, 2] > 0
        assert np.abs(R[b] @ R[b].T - np.eye(3)).max() <= 1e-15 and abs(np.linalg.det(R[b]) - 1.0) <= 1e-15
        assert np.abs(L @ L.T - L0 @ L0.T).max() <= 1e-12 * np.abs(L0).max() ** 2     # lengths and angles
        assert np.abs(np.linalg.norm(X[:, None] - X[None], axis=-1)
                      - np.linalg.norm(X0[:, None] - X0[None], axis=-1)).max() <= 1e-12
        assert np.abs((X @ np.linalg.inv(L)) - (X0 @ np.linalg.inv(L0))).max() <= 1e-12   # same fractional coordinates
        f = feats[off[b]:off[b + 1]]
        e0 = _host_evaluator(model, f, "k-nearest", 8.0)(L0, X0)[0]
        e1 = _host_evaluator(model, f, "k-nearest", 8.0)(L, X)[0]
        assert abs(e1 - e0) <= 1e-5 * max(abs(e0), 1.0), (b, e0, e1)
    again, R2 = upper_triangular(rot)                                     # already in form: unchanged
    assert np.array_equal(R2, np.broadcast_to(np.eye(3), R2.shape))
    assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(again, rot))
