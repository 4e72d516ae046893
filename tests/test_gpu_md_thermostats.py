"""GPU (-m gpu): batched NVT Langevin and Andersen.  The noise stream (`ops.md_noise`, csrc/md_noise.cuh) against its
numpy restatement, the thermostat kernel (`ops.md_thermostat_step`, csrc/md_device.cu) against
`oracle/md_thermostat_oracle.py` on scripted forces, and `run_md` against a host loop that runs each crystal alone
the reference's way with the same per-crystal stream."""
import os

import numpy as np
import pytest
import torch

from alignn_b200 import maxwell_boltzmann_momenta, neighbors, ops, run_md
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from oracle import md_oracle as MO
from oracle import md_thermostat_oracle as TO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIND = {TO.LANGEVIN: ops.MD_NVT_LANGEVIN, TO.ANDERSEN: ops.MD_NVT_ANDERSEN}


def _close(a, b, rtol):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() <= rtol * max(np.abs(b).max(), 1e-300)


# ---- 1. the noise stream -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,step,tag,atom0,count,blocks", [(0, 0, 2, 0, 1000, 3), (2 ** 64 - 1, 2 ** 31 - 1, 3, 0, 7, 5),
                                                               (123456789012345, 17, 3, 0xFFFFFFFD, 5, 5)])
def test_md_noise_matches_the_restatement(seed, step, tag, atom0, count, blocks):
    words, u, z = ops.md_noise(seed, step, count, tag=tag, atom0=atom0, blocks=blocks, device=DEV)
    atoms = (atom0 + np.arange(count)) % 2 ** 32                                 # the last case wraps past kComAtom
    w_ref, u_ref, z_ref = TO.noise_blocks(seed, atoms, step, blocks, tag)
    assert np.array_equal(words.cpu().numpy(), w_ref.astype(np.int64))
    assert np.array_equal(u.cpu().numpy(), u_ref)
    assert np.abs(z.cpu().numpy() - z_ref).max() <= 1e-13


def test_md_noise_rejects_bad_arguments():
    for kw in (dict(step=-1), dict(blocks=0), dict(blocks=65)):
        with pytest.raises(RuntimeError, match="alignn_b200_md_noise failed"):
            ops.md_noise(1, **dict(dict(step=0, count=4), **kw), device=DEV)
    with pytest.raises(ValueError):
        ops.md_noise(-1, 0, 4, device=DEV)


# ---- 2. the thermostat kernel on scripted forces ---------------------------------------------------------------------
SIZES = [2, 30, 1000]
MULT, STEPS, DT = 1.5, 12, 1.0 * MO.fs
T0 = [300.0, 500.0, 200.0]
SEEDS = [7, 2 ** 64 - 5, 2 ** 40 + 3]
FRICTION, PROB = 0.05 / MO.fs, 0.3


def _script(b, e, n, cache={}):
    if (b, n) not in cache:
        cache[(b, n)] = np.random.default_rng(100 + b).normal(size=(n, 3))
    return (cache[(b, n)] * (1.0 + 0.3 * np.sin(e + b))).astype(np.float32)


def _buffers(N, B):
    z = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.float64)  # noqa: E731
    return dict(vel=z(N, 3), rnd=z(N, 3), forces=torch.zeros(N, 3, device=DEV), ekin=z(STEPS + 1, B),
                temp=z(STEPS + 1, B), status=torch.zeros(B, device=DEV, dtype=torch.int32))


def _seeds_tensor(seeds):
    return torch.from_numpy(np.array(seeds, dtype=np.uint64).view(np.int64)).to(DEV)


def _scripted_run(ensemble):
    aoff = neighbors.ragged_offsets(SIZES)
    N, B = int(aoff[-1]), len(SIZES)
    rng = np.random.default_rng(0)
    x0 = rng.normal(size=(N, 3))
    m = rng.choice([1.008, 12.011, 63.546, 196.97], N) * rng.uniform(0.9, 1.1, N)
    p0 = np.concatenate([MO.maxwell_boltzmann_momenta(m[aoff[b]:aoff[b + 1]], T, rng) for b, T in enumerate(T0)])
    p0[aoff[1]:aoff[2]] *= 4.0
    pos, mom = torch.from_numpy(x0.copy()).to(DEV), torch.from_numpy(p0.copy()).to(DEV)
    m_d, t0 = torch.from_numpy(m).to(DEV), torch.tensor(T0, dtype=torch.float64, device=DEV)
    buf = _buffers(N, B)
    aoff_d, seeds = torch.from_numpy(aoff).to(DEV), _seeds_tensor(SEEDS)
    orc = [TO.Thermostat(x0[aoff[b]:aoff[b + 1]], m[aoff[b]:aoff[b + 1]], ensemble=ensemble, dt=DT, temperature_K=T0[b],
                         noise=TO.PhiloxNoise(SEEDS[b]), friction=FRICTION, andersen_prob=PROB,
                         momenta=p0[aoff[b]:aoff[b + 1]]) for b in range(B)]
    for e in range(STEPS + 1):
        grads = [_script(b, e, SIZES[b]) for b in range(B)]
        ops.md_thermostat_step(torch.from_numpy(np.concatenate(grads)).to(DEV), aoff_d, m_d, t0, seeds, pos, mom,
                               buf["vel"], buf["rnd"], buf["forces"], buf["ekin"][e], buf["temp"][e], buf["status"],
                               evaluation=e, steps=STEPS, dt=DT, kB=MO.kB, ensemble=KIND[ensemble], friction=FRICTION,
                               andersen_prob=PROB, force_multiplier=MULT)
        P, Q, F = pos.cpu().numpy(), mom.cpu().numpy(), buf["forces"].cpu().numpy()
        EK, TT = buf["ekin"][e].cpu().numpy(), buf["temp"][e].cpu().numpy()
        assert buf["status"].tolist() == [0] * B
        for b, o in enumerate(orc):
            sl = slice(aoff[b], aoff[b + 1])
            f = MO.scaled_forces(grads[b], MULT)
            if e >= 1:
                o.second_half(f.astype(np.float64))
            assert _close(EK[b], MO.kinetic_energy(o.p, o.m.ravel()), 1e-12), (b, e)
            assert _close(TT[b], MO.temperature(o.p, o.m.ravel()), 1e-12), (b, e)
            if e < STEPS:
                o.first_half(f.astype(np.float64))
            assert np.array_equal(F[sl], f), (b, e)
            assert _close(P[sl], o.x, 1e-12) and _close(Q[sl], o.p, 1e-12), (b, e)
    if ensemble == TO.ANDERSEN:
        assert all(o.reassigned > 0 for o in orc)
    return [t.clone() for t in (pos, mom, buf["vel"], buf["rnd"], buf["forces"], buf["ekin"], buf["temp"])]


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_md_thermostat_step_matches_oracle_on_scripted_forces(ensemble):
    first = _scripted_run(ensemble)
    again = _scripted_run(ensemble)
    for a, b in zip(first, again):
        assert torch.equal(a, b)                                                 # bitwise repeatable


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_bad_slice_and_one_atom_langevin_touch_nothing_but_their_status(ensemble):
    aoff = torch.tensor([0, 1, 3, 6], dtype=torch.int64, device=DEV)             # crystal 0 has one atom
    pos = torch.randn(6, 3, dtype=torch.float64, device=DEV)
    mom = torch.randn(6, 3, dtype=torch.float64, device=DEV)
    m = torch.full((6,), 12.0, dtype=torch.float64, device=DEV)
    vel, rnd = torch.full((6, 3), 7.0, dtype=torch.float64, device=DEV), torch.full((6, 3), 8.0, dtype=torch.float64, device=DEV)
    forces = torch.full((6, 3), 9.0, device=DEV)
    ekin, temp = torch.full((3,), -1.0, dtype=torch.float64, device=DEV), torch.full((3,), -1.0, dtype=torch.float64, device=DEV)
    status = torch.zeros(3, dtype=torch.int32, device=DEV)
    t0, seeds = torch.full((3,), 300.0, dtype=torch.float64, device=DEV), _seeds_tensor([1, 2, 3])

    def crystal(sl, c):
        return [t[sl].clone() for t in (pos, mom, vel, rnd, forces)] + [ekin[c].clone(), temp[c].clone()]
    skipped = [(slice(3, 6), 2)] + ([(slice(0, 1), 0)] if ensemble == TO.LANGEVIN else [])
    before = [crystal(*s) for s in skipped]
    kw = dict(steps=3, dt=DT, kB=MO.kB, ensemble=KIND[ensemble], friction=FRICTION, andersen_prob=PROB)
    ops.md_thermostat_step(torch.ones(5, 3, device=DEV), aoff, m, t0, seeds, pos, mom, vel, rnd, forces, ekin, temp,
                           status, evaluation=0, **kw)                         # crystal 2 needs rows 3..6, grad has 5
    want = [ops.MD_ONE_ATOM if ensemble == TO.LANGEVIN else 0, 0, ops.MD_BAD_INPUT]
    assert status.tolist() == want
    assert ekin[1].item() > 0 and torch.equal(forces[1:3], torch.ones(2, 3, device=DEV))
    for s, b in zip(skipped, before):
        assert all(torch.equal(x, y) for x, y in zip(b, crystal(*s)))
    ops.md_thermostat_step(torch.ones(6, 3, device=DEV), aoff, m, t0, seeds, pos, mom, vel, rnd, forces, ekin, temp,
                           status, evaluation=1, **kw)
    assert status.tolist() == want
    for s, b in zip(skipped, before):                                            # a reported crystal stays untouched
        assert all(torch.equal(x, y) for x, y in zip(b, crystal(*s)))


def test_md_thermostat_step_rejects_bad_parameters():
    aoff = torch.tensor([0, 2], dtype=torch.int64, device=DEV)
    z3 = lambda: torch.zeros(2, 3, dtype=torch.float64, device=DEV)  # noqa: E731
    pos, mom, vel, rnd = z3(), z3(), z3(), z3()
    m = torch.ones(2, dtype=torch.float64, device=DEV)
    f, g = torch.zeros(2, 3, device=DEV), torch.zeros(2, 3, device=DEV)
    ek, tt = torch.zeros(1, dtype=torch.float64, device=DEV), torch.zeros(1, dtype=torch.float64, device=DEV)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    t0, seeds = torch.tensor([300.0], dtype=torch.float64, device=DEV), _seeds_tensor([5])
    args = (g, aoff, m, t0, seeds, pos, mom, vel, rnd, f, ek, tt, st)
    base = dict(evaluation=0, steps=2, dt=DT, kB=MO.kB, ensemble=ops.MD_NVT_LANGEVIN, friction=0.1, andersen_prob=0.5,
                force_multiplier=1.0)
    nan, inf = float("nan"), float("inf")
    for bad in (dict(dt=0.0), dict(dt=-DT), dict(dt=nan), dict(dt=inf), dict(kB=0.0), dict(kB=nan), dict(friction=-0.1),
                dict(friction=nan), dict(friction=inf), dict(andersen_prob=-0.01), dict(andersen_prob=1.01),
                dict(andersen_prob=nan), dict(force_multiplier=nan), dict(ensemble=0), dict(ensemble=1),
                dict(ensemble=4)):
        with pytest.raises(RuntimeError, match="alignn_b200_md_thermostat_step failed"):
            ops.md_thermostat_step(*args, **dict(base, **bad))
    for bad in (dict(evaluation=3), dict(evaluation=-1), dict(steps=0), dict(steps=True)):
        with pytest.raises(ValueError):
            ops.md_thermostat_step(*args, **dict(base, **bad))
    with pytest.raises(ValueError, match="shapes"):
        ops.md_thermostat_step(g, aoff, m, t0, seeds, pos, mom, vel, rnd[:1], f, ek, tt, st, **base)
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.md_thermostat_step(g, aoff, m, t0, seeds.to(torch.int32), pos, mom, vel, rnd, f, ek, tt, st, **base)
    with pytest.raises(RuntimeError, match="device"):
        ops.md_thermostat_step(g, aoff, m, t0, seeds.cpu(), pos, mom, vel, rnd, f, ek, tt, st, **base)
    for ens in (ops.MD_NVT_LANGEVIN, ops.MD_NVT_ANDERSEN):                       # the edges are accepted
        for kw in (dict(friction=0.0, andersen_prob=0.0), dict(andersen_prob=1.0)):
            ops.md_thermostat_step(*args, **dict(base, ensemble=ens, **kw))
    ops.md_thermostat_step(g, aoff, m, t0, seeds.view(torch.uint64), pos, mom, vel, rnd, f, ek, tt, st, **base)
    assert st.item() == 0


# ---- 3. run_md --------------------------------------------------------------------------------------------------------
def _model(seed=11):
    torch.manual_seed(seed)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64,
                               embedding_features=64, atom_input_features=92)
    return ALIGNNAtomWise(cfg).to(DEV).eval()


def _structures(count=8, seed=3):
    """test_gpu_md's samples: jittered, <= 12 atoms, no distance tie at the 12th-neighbour cut at the start."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    sizes = off[1:] - off[:-1]
    rng = np.random.default_rng(seed)
    out = []
    for i in rng.permutation([i for i in range(len(sizes)) if 2 <= sizes[i] <= 12]):
        s = (z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]] + rng.normal(scale=0.05, size=(sizes[i], 3)))
        if not neighbors.knn_cut_is_tied(*s):
            out.append(s)
        if len(out) == count:
            break
    n = sum(x.shape[0] for _, x in out)
    feats = torch.from_numpy(rng.normal(size=(n, 92)).astype(np.float32)).to(DEV)
    masses = rng.uniform(1.0, 200.0, n)
    return out, feats, masses, maxwell_boltzmann_momenta(masses, 300.0, rng)


def _host_evaluator(model, lat, feats, strategy, cutoff):
    lat_t = torch.tensor(lat, dtype=torch.float32).view(1, 3, 3).to(DEV)

    def evaluate(x):
        g, lg = neighbors.crystal_graph(lat, x, feats.cpu(), cutoff=cutoff, neighbor_strategy=strategy, max_neighbors=12)
        res = model((g.to(DEV), lg.to(DEV), lat_t))
        e = (res["out"].detach().reshape(-1) * float(x.shape[0])).cpu().numpy()[0]
        return e, res["grad"].detach().reshape(-1, 3).cpu().numpy()
    return evaluate


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
@pytest.mark.parametrize("strategy,cutoff", [("k-nearest", 8.0), ("radius_graph", 6.0)])
def test_run_md_matches_host_loop(strategy, cutoff, ensemble):
    model = _model()
    structs, feats, masses, p0 = _structures()
    steps, mult, dt_fs, seed = 20, 1.5, 1.0, 2 ** 62 + 11
    fr = 0.02                                                                    # 1/fs: the noise is not negligible
    got = run_md(model, structs, feats, masses, ensemble=ensemble, steps=steps, timestep=dt_fs, temperature_K=300.0,
                 momenta=p0, neighbor_strategy=strategy, cutoff=cutoff, force_multiplier=mult, friction=fr,
                 andersen_prob=0.1, seed=seed)
    off = got.atom_offsets.cpu().tolist()
    P, Q, F = got.positions.cpu().numpy(), got.momenta.cpu().numpy(), got.forces.cpu().numpy()
    E, EK, T = got.energy.cpu().numpy(), got.kinetic_energy.cpu().numpy(), got.temperature.cpu().numpy()
    assert E.shape == EK.shape == T.shape == (steps + 1, len(structs)) and got.trajectory is None
    moved = 0.0
    for b, (lat, X) in enumerate(structs):
        sl = slice(off[b], off[b + 1])
        r = TO.run(_host_evaluator(model, lat, feats[sl], strategy, cutoff), X, masses[sl], ensemble=ensemble,
                   steps=steps, dt=dt_fs * MO.fs, temperature_K=300.0, noise=TO.PhiloxNoise(seed + b),
                   friction=fr / MO.fs, andersen_prob=0.1, momenta=p0[sl], force_multiplier=mult)
        assert np.abs(P[sl] - r["positions"]).max() <= 1e-9, b
        assert _close(Q[sl], r["momenta"], 1e-9), b
        assert _close(EK[:, b], r["kinetic_energy"], 1e-9) and _close(T[:, b], r["temperature"], 1e-9), b
        assert _close(F[sl], r["forces"], 1e-5) and _close(E[:, b], r["energy"], 1e-5), b
        moved = max(moved, float(np.abs(P[sl] - X).max()))
    assert moved > 1e-3, moved


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_run_md_is_batch_invariant_with_per_crystal_seeds(ensemble):
    model = _model()
    structs, feats, masses, p0 = _structures()
    T0 = [200.0 + 50.0 * b for b in range(len(structs))]
    seeds = [2 ** 64 - 1 - 1000 * b for b in range(len(structs))]
    kw = dict(ensemble=ensemble, steps=6, timestep=1.0, friction=0.05, andersen_prob=0.3)
    got = run_md(model, structs, feats, masses, temperature_K=T0, momenta=p0, seed=seeds, **kw)
    off = got.atom_offsets.cpu().tolist()
    for b in (0, 3, len(structs) - 1):
        sl = slice(off[b], off[b + 1])
        one = run_md(model, [structs[b]], feats[sl], masses[sl], temperature_K=T0[b], momenta=p0[sl], seed=[seeds[b]],
                     **kw)
        assert torch.equal(one.positions, got.positions[sl]) and torch.equal(one.momenta, got.momenta[sl]), b
        assert torch.equal(one.forces, got.forces[sl]), b
        assert torch.equal(one.kinetic_energy[:, 0], got.kinetic_energy[:, b]), b
        assert torch.equal(one.temperature[:, 0], got.temperature[:, b]), b
        assert torch.allclose(one.energy[:, 0], got.energy[:, b], rtol=1e-5, atol=0), b
    # one int seed s gives crystal b the stream s + b
    a = run_md(model, structs[:3], feats[:off[3]], masses[:off[3]], momenta=p0[:off[3]], seed=40, **kw)
    b = run_md(model, structs[:3], feats[:off[3]], masses[:off[3]], momenta=p0[:off[3]], seed=[40, 41, 42], **kw)
    assert torch.equal(a.positions, b.positions) and torch.equal(a.momenta, b.momenta)
    c = run_md(model, structs[:3], feats[:off[3]], masses[:off[3]], momenta=p0[:off[3]], seed=41, **kw)
    assert not torch.equal(a.positions, c.positions)


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_run_md_under_no_grad(ensemble):
    model = _model()
    structs, feats, masses, p0 = _structures(count=3)
    kw = dict(ensemble=ensemble, steps=3, timestep=1.0, momenta=p0, trajectory_interval=1, seed=9)
    ref = run_md(model, structs, feats, masses, **kw)
    with torch.no_grad():
        got = run_md(model, structs, feats, masses, **kw)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)


def test_default_friction_is_the_references_ase_value():
    """friction=None is 1e-4 in ASE units exactly; friction=f in 1/fs is f / fs in ASE units."""
    model = _model()
    structs, feats, masses, p0 = _structures(count=2)
    kw = dict(ensemble="nvt_langevin", steps=2, timestep=1.0, momenta=p0, seed=3)
    a = run_md(model, structs, feats, masses, **kw)
    b = run_md(model, structs, feats, masses, friction=1e-4 * MO.fs, **kw)
    assert torch.allclose(a.positions, b.positions, rtol=0, atol=1e-14)


def test_run_md_thermostat_rejections():
    model = _model()
    structs, feats, masses, p0 = _structures(count=2)
    for ens in ("nvt_langevin", "nvt_andersen"):
        bad = [dict(), dict(seed=None), dict(seed=-1), dict(seed=2 ** 63), dict(seed=1.0), dict(seed=True),
               dict(seed=[1]), dict(seed=[1, 2, 3]), dict(seed=[1, 2 ** 64]), dict(seed=[1, -1]), dict(seed=[1, 2.0]),
               dict(seed=0, friction=-0.1), dict(seed=0, friction=float("nan")), dict(seed=0, friction=float("inf")),
               dict(seed=0, friction="0.1"), dict(seed=0, andersen_prob=-0.1), dict(seed=0, andersen_prob=1.5),
               dict(seed=0, andersen_prob=float("nan")), dict(seed=0, temperature_K=0.0),
               dict(seed=0, temperature_K=[300.0]), dict(seed=0, temperature_K=float("nan"))]
        for kw in bad:
            with pytest.raises(ValueError):
                run_md(model, structs, feats, masses, **dict(dict(ensemble=ens, steps=2), **kw))
    lat, X = structs[0]
    one = [(lat, X[:1])] + structs[1:]
    n0 = X.shape[0] - 1
    with pytest.raises(ValueError, match="at least 2 atoms"):
        run_md(model, one, feats[n0:], masses[n0:], ensemble="nvt_langevin", steps=2, seed=0)
    got = run_md(model, one, feats[n0:], masses[n0:], ensemble="nvt_andersen", steps=2, seed=0)   # Andersen: fine
    assert got.energy.shape == (3, 2)
    # accepted: the edges, numpy integers and a uint64 seed array
    run_md(model, structs, feats, masses, ensemble="nvt_langevin", steps=1, friction=0.0, seed=np.int64(2 ** 63 - 2))
    run_md(model, structs, feats, masses, ensemble="nvt_andersen", steps=1, andersen_prob=1.0,
           seed=np.array([2 ** 64 - 1, 0], dtype=np.uint64))
