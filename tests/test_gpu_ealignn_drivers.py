"""GPU (-m gpu): the batched drivers (`relax_structures`, `run_md`, `phonons`, `single_point`, `ev_curve`) with an
`eALIGNNAtomWise`, against a host loop that is the reference calculator alone: per crystal and per evaluation, the
device graph of that one crystal, the model's unchanged forward on it, and the oracle's optimizer or integrator."""
import os

import numpy as np
import pytest
import torch

from alignn_b200 import (ev_curve, maxwell_boltzmann_momenta, neighbors, phonons, relax_structures, run_md, single_point,
                         upper_triangular)
from alignn_b200.eos import strained
from alignn_b200.ealignn_atomwise import eALIGNNAtomWise, eALIGNNAtomWiseConfig
from alignn_b200.phonons import displaced_supercells
from oracle import cell_filter_oracle as CF
from oracle import fire_oracle as FO
from oracle import md_nose_hoover_oracle as NH
from oracle import md_npt_oracle as NO
from oracle import md_oracle as MO
from oracle import md_thermostat_oracle as TO
from oracle import phonon_oracle as PO
from oracle import qn_oracle as QN

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# radius_graph at 5 A, so that eALIGNN's 4 A inner cutoff drops bonds
GRAPH = dict(neighbor_strategy="radius_graph", cutoff=5.0)
MULT = 1.5


def _model(seed=11, **kw):
    torch.manual_seed(seed)
    cfg = dict(name="ealignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64, embedding_features=64,
               atom_input_features=92, stresswise_weight=1.0)
    cfg.update(kw)
    return eALIGNNAtomWise(eALIGNNAtomWiseConfig(**cfg)).to(DEV).eval()


def _structures(count=8, seed=3):
    """Jittered sample structures of at most 12 atoms with strained and sheared cells; the first is a 3-atom crystal."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    sizes = off[1:] - off[:-1]
    three = [i for i in range(len(sizes)) if sizes[i] == 3]
    rest = [i for i in range(len(sizes)) if sizes[i] <= 12 and sizes[i] != 3]
    rng = np.random.default_rng(seed)
    out = []
    for i in [three[0]] + list(rng.permutation(rest)[:count - 1]):
        D = np.eye(3) + np.diag(rng.uniform(-0.04, 0.04, 3)) + rng.uniform(-0.03, 0.03, (3, 3))
        lat, X = z["lattices"][i] @ D.T, z["cart_coords"][off[i]:off[i + 1]] @ D.T
        out.append((lat, X + rng.normal(scale=0.05, size=X.shape)))
    feats = torch.from_numpy(rng.normal(size=(sum(x.shape[0] for _, x in out), 92)).astype(np.float32)).to(DEV)
    return out, feats


def _with_short_bond(structs, feats):
    lat, X = structs[1]
    short = (lat, np.concatenate([X, X[:1] + np.array([0.8, 0.0, 0.0])]))
    return short, feats[:1].repeat(X.shape[0] + 1, 1)


def _alone(model, feats):
    """The calculator on one crystal: (energy out * n, grad, stress [3,3]) from the unchanged forward."""
    def evaluate(cell, x):
        g, lg, lat = neighbors.crystal_graphs_device([(cell, x)], feats, device=DEV, **GRAPH)
        res = model((g, lg, lat))
        e = (res["out"].detach().reshape(-1) * float(x.shape[0])).cpu().numpy()[0]
        return e, res["grad"].detach().reshape(-1, 3).cpu().numpy(), res["stresses"].detach().reshape(3, 3).cpu().numpy()
    return evaluate


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _slices(res):
    off = res.atom_offsets.cpu().tolist()
    return [slice(off[b], off[b + 1]) for b in range(len(off) - 1)]


# ---- relaxation ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["FIRE", "LBFGS", "BFGS"])
@pytest.mark.parametrize("cell", [False, True])
def test_relax_matches_host_loop(optimizer, cell):
    model = _model()
    structs, feats = _structures()
    steps, fmax = 8, 0.05
    sl = [slice(a, a + x.shape[0]) for a, x in zip(np.cumsum([0] + [x.shape[0] for _, x in structs]), (x for _, x in structs))]
    evs = [_alone(model, feats[s]) for s in sl]
    ref = []
    for (lat, X), ev in zip(structs, evs):
        if cell and optimizer == "FIRE":
            ref.append(CF.relax(ev, lat, X, fmax=fmax, steps=steps, force_multiplier=MULT))
        elif cell:
            ref.append(QN.relax_cell(optimizer, ev, lat, X, fmax=fmax, steps=steps, force_multiplier=MULT))
        elif optimizer == "FIRE":
            ref.append(FO.relax(lambda x, ev=ev, lat=lat: ev(lat, x)[:2], X, fmax=fmax, steps=steps, force_multiplier=MULT))
        else:
            ref.append(QN.relax(optimizer, lambda x, ev=ev, lat=lat: ev(lat, x)[:2], X, fmax=fmax, steps=steps,
                                force_multiplier=MULT))
    got = relax_structures(model, structs, feats, fmax=fmax, steps=steps, force_multiplier=MULT, optimize_lattice=cell,
                           optimizer=optimizer, **GRAPH)
    nst = got.nsteps.cpu().tolist()
    print(f"[ealignn relax {optimizer} cell={cell}] nsteps {nst} converged {got.converged.cpu().tolist()}")
    assert nst == [r["nsteps"] for r in ref]
    assert got.converged.cpu().tolist() == [r["converged"] for r in ref]
    P, F, E = got.positions.cpu().numpy(), got.forces.cpu().numpy(), got.energy.cpu().numpy()
    for b, (r, s) in enumerate(zip(ref, _slices(got))):
        assert np.abs(P[s] - r["positions"]).max() <= 1e-6, b
        assert np.abs(F[s] - r["forces"]).max() <= 1e-5 * max(np.abs(r["forces"]).max(), 1e-30) + 1e-6, b
        assert abs(E[b] - r["energy"]) <= 1e-5 * abs(r["energy"]), b
        if cell:
            assert np.abs(got.cells[b].cpu().numpy() - r["cell"]).max() <= 1e-6, b
            assert _rel(got.stress[b].cpu().numpy(), r["stress"]) <= 1e-5, b


@pytest.mark.parametrize("optimizer", ["FIRE", "LBFGS"])
def test_relax_is_batch_invariant(optimizer):
    model = _model()
    structs, feats = _structures()
    got = relax_structures(model, structs, feats, fmax=0.0, steps=5, optimize_lattice=True, optimizer=optimizer, **GRAPH)
    for b, s in enumerate(_slices(got)):
        one = relax_structures(model, [structs[b]], feats[s], fmax=0.0, steps=5, optimize_lattice=True,
                               optimizer=optimizer, **GRAPH)
        assert torch.equal(one.positions, got.positions[s]) and torch.equal(one.forces, got.forces[s]), b
        assert torch.equal(one.cells[0], got.cells[b]) and torch.equal(one.stress[0], got.stress[b]), b
        assert torch.allclose(one.energy, got.energy[b:b + 1], rtol=1e-5, atol=0), b


def test_bond_penalty_counted_once_and_no_grad():
    model = _model()
    structs, feats = _structures(count=4)
    short, f_short = _with_short_bond(structs, feats)
    allf = torch.cat([feats, f_short])
    got = relax_structures(model, structs + [short], allf, fmax=0.0, steps=3, optimize_lattice=True, **GRAPH)
    one = relax_structures(model, [short], f_short, fmax=0.0, steps=3, optimize_lattice=True, **GRAPH)
    s = _slices(got)[-1]
    assert torch.equal(got.forces[s], one.forces) and torch.equal(got.stress[-1], one.stress[0])
    assert torch.equal(got.positions[s], one.positions)
    ref = CF.relax(_alone(model, f_short), *short, fmax=0.0, steps=3)
    assert np.abs(one.positions.cpu().numpy() - ref["positions"]).max() <= 1e-6
    assert _rel(one.forces.cpu().numpy(), ref["forces"]) <= 1e-5
    with torch.no_grad():
        again = relax_structures(model, structs + [short], allf, fmax=0.0, steps=3, optimize_lattice=True, **GRAPH)
    for a, b in zip(got, again):
        assert torch.equal(a, b)
    # the default batched forward, which counts the penalty once per crystal of the batch and scales by the batch's
    # atoms, gives this crystal other forces
    g, lg, lat = neighbors.crystal_graphs_device(structs + [short], allf, device=DEV, **GRAPH)
    sp = single_point(model, structs + [short], allf, **GRAPH)
    assert not torch.allclose(model((g, lg, lat))["grad"][s], sp.forces[s])


# ---- molecular dynamics ---------------------------------------------------------------------------------------------------
def _md_inputs(count=8, seed=3, upper=False):
    structs, feats = _structures(count=count, seed=seed)
    if upper:
        structs, _ = upper_triangular(structs)
    n = sum(x.shape[0] for _, x in structs)
    rng = np.random.default_rng(seed + 1)
    masses = rng.uniform(1.0, 200.0, n)
    p0 = maxwell_boltzmann_momenta(masses, 300.0, rng)
    if upper:
        off = np.cumsum([0] + [x.shape[0] for _, x in structs])
        for b in range(len(structs)):
            p0[off[b]:off[b + 1]] -= p0[off[b]:off[b + 1]].sum(0) / (off[b + 1] - off[b])
    return structs, feats, masses, p0


ENSEMBLES = ["nve_velocity_verlet", "nvt_berendsen", "nvt_langevin", "nvt_andersen", "npt_berendsen", "npt_nose_hoover"]


@pytest.mark.parametrize("ensemble", ENSEMBLES)
def test_run_md_matches_host_loop(ensemble):
    model = _model()
    nh = ensemble == "npt_nose_hoover"
    structs, feats, masses, p0 = _md_inputs(upper=nh)
    B, steps, dt_fs, seed = len(structs), 10, 1.0, 2 ** 62 + 11
    kw = dict(ensemble=ensemble, steps=steps, timestep=dt_fs, temperature_K=300.0, momenta=p0, force_multiplier=MULT,
              **GRAPH)
    pressure = [1e4 * (b - 3) for b in range(B)]
    ext = [0.01 * (b - 3) for b in range(B)]
    if ensemble == "nvt_berendsen":
        kw.update(taut=100 * dt_fs)
    elif ensemble in ("nvt_langevin", "nvt_andersen"):
        kw.update(friction=0.02, andersen_prob=0.1, seed=seed)
    elif ensemble == "npt_berendsen":
        kw.update(pressure=pressure, compressibility=2e-6, taup=100.0, taut=50.0)
    elif nh:
        kw.update(externalstress=np.stack([NH.external_stress(s) for s in ext]), ttime=25.0, pfactor=100.0)
    got = run_md(model, structs, feats, masses, **kw)
    P, Q, F = got.positions.cpu().numpy(), got.momenta.cpu().numpy(), got.forces.cpu().numpy()
    E, EK = got.energy.cpu().numpy(), got.kinetic_energy.cpu().numpy()
    dt = dt_fs * MO.fs
    for b, ((lat, X), s) in enumerate(zip(structs, _slices(got))):
        ev = _alone(model, feats[s])
        evx = lambda x, ev=ev, lat=lat: ev(lat, x)[:2]                     # noqa: E731
        common = dict(steps=steps, dt=dt, temperature_K=300.0, momenta=p0[s], force_multiplier=MULT)
        if ensemble in (MO.NVE, MO.NVT_BERENDSEN):
            r = MO.run(evx, X, masses[s], ensemble=ensemble, taut=100 * dt, **common)
        elif ensemble in (TO.LANGEVIN, TO.ANDERSEN):
            r = TO.run(evx, X, masses[s], ensemble=ensemble, noise=TO.PhiloxNoise(seed + b), friction=0.02 / MO.fs,
                       andersen_prob=0.1, **common)
        elif ensemble == "npt_berendsen":
            r = NO.run(ev, lat, X, masses[s], pressure=pressure[b], compressibility=2e-6, taut=50.0 * MO.fs,
                       taup=100.0 * MO.fs, **common)
        else:
            r = NH.run(ev, lat, X, masses[s], externalstress=ext[b], ttime=25.0 * MO.fs, pfactor=100.0, **common)
        assert np.abs(P[s] - r["positions"]).max() <= 1e-9, b
        assert _rel(Q[s], r["momenta"]) <= 1e-9 and _rel(EK[:, b], r["kinetic_energy"]) <= 1e-9, b
        assert _rel(F[s], r["forces"]) <= 1e-5 and _rel(E[:, b], r["energy"]) <= 1e-5, b
        if ensemble.startswith("npt"):
            assert np.abs(got.cells[:, b].cpu().numpy() - np.stack(r["cells"])).max() <= 1e-9, b
            assert _rel(got.stress[:, b].cpu().numpy(), np.stack(r["stress"])) <= 1e-5, b


@pytest.mark.parametrize("ensemble", ["nvt_berendsen", "nvt_langevin", "npt_berendsen"])
def test_run_md_is_batch_invariant_and_the_same_under_no_grad(ensemble):
    model = _model()
    structs, feats, masses, p0 = _md_inputs()
    kw = dict(ensemble=ensemble, steps=5, timestep=1.0, trajectory_interval=1, **GRAPH)
    if ensemble == "nvt_langevin":
        kw.update(seed=[100 + b for b in range(len(structs))])
    if ensemble == "npt_berendsen":
        kw.update(pressure=1e4, compressibility=2e-6, taup=100.0, taut=50.0)
    got = run_md(model, structs, feats, masses, momenta=p0, **kw)
    with torch.no_grad():
        again = run_md(model, structs, feats, masses, momenta=p0, **kw)
    for a, b in zip(got, again):
        assert (a is None and b is None) or torch.equal(a, b)
    for b, s in enumerate(_slices(got)):
        one_kw = dict(kw, seed=[kw["seed"][b]]) if "seed" in kw else kw
        one = run_md(model, [structs[b]], feats[s], masses[s], momenta=p0[s], **one_kw)
        assert torch.equal(one.positions, got.positions[s]) and torch.equal(one.momenta, got.momenta[s]), b
        assert torch.equal(one.forces, got.forces[s]), b
        assert torch.allclose(one.energy[:, 0], got.energy[:, b], rtol=1e-5, atol=0), b


# ---- phonons, single points, E(V) ----------------------------------------------------------------------------------------
def test_phonons_match_host_loop():
    model = _model()
    structs, feats = _structures(count=3)
    rng = np.random.default_rng(5)
    masses = rng.uniform(1.0, 200.0, feats.shape[0])
    q = [np.concatenate([np.zeros((1, 3)), rng.uniform(-0.5, 0.5, size=(3, 3))]) for _ in structs]
    N, delta, kpts = (2, 2, 2), 0.01, (3, 3, 3)
    got = phonons(model, structs, feats, masses, supercell=N, delta=delta, qpoints=q, dos_kpts=kpts, dos_npts=30,
                  force_multiplier=MULT, **GRAPH)
    for b, ((lat, X), s) in enumerate(zip(structs, _slices(got))):
        ev = _alone(model, feats[s].repeat(8, 1))
        latN, disp = displaced_supercells(lat, X, N, delta)
        f = np.stack([FO.scaled_forces(ev(latN, x)[1], MULT) for x in disp]).astype(np.float64)
        r = PO.postprocess(f, masses[s], N, delta, qpoints=q[b], dos_kpts=kpts, dos_npts=30, dos_width=1e-3)
        # the force constants are differences of forces at +-delta: the 1e-5 of the forces over delta = 0.01
        assert _rel(got.force_constants[b].cpu().numpy(), r["C_N"]) <= 1e-3, b


def test_single_point_and_ev_curve_match_host_loop():
    model = _model()
    structs, feats = _structures()
    got = single_point(model, structs, feats, force_multiplier=MULT, **GRAPH)
    E, F = got.energy.cpu().numpy(), got.forces.cpu().numpy()
    for b, ((lat, X), s) in enumerate(zip(structs, _slices(got))):
        e, g, _ = _alone(model, feats[s])(lat, X)
        assert abs(E[b] - e) <= 1e-5 * abs(e), b
        assert np.abs(F[s] - FO.scaled_forces(g, MULT)).max() <= 1e-5 * max(np.abs(g).max(), 1e-30), b
    strains = np.linspace(-0.06, 0.06, 7)
    curve = ev_curve(model, structs[:4], feats[:_slices(got)[3].stop], strains=strains, **GRAPH)
    Eg = curve.energies.cpu().numpy()
    for b, ((lat, X), s) in enumerate(zip(structs[:4], _slices(got)[:4])):
        host = [_alone(model, feats[s])(*strained(lat, X, k)[:2])[0] for k in strains]
        assert np.abs(Eg[b] - host).max() <= 1e-5 * np.abs(host).max(), b


# ---- rejections and the graph builder ------------------------------------------------------------------------------------
def test_rejections_and_accepted_settings():
    structs, feats = _structures(count=2)
    with pytest.raises(ValueError, match="eval"):
        relax_structures(_model().train(), structs, feats, **GRAPH)
    with pytest.raises(ValueError, match="calculate_gradient"):
        relax_structures(_model(gradwise_weight=0.0), structs, feats, **GRAPH)
    with pytest.raises(ValueError, match="output_features"):
        run_md(_model(output_features=2), structs, feats, np.ones(feats.shape[0]), steps=1, **GRAPH)
    with pytest.raises(NotImplementedError, match="energy_mult_natoms"):
        single_point(_model(energy_mult_natoms=False), structs, feats, **GRAPH)
    with pytest.raises(ValueError, match="cart_coords"):
        relax_structures(_model(alignn_layers=0), structs, feats, **GRAPH)
    with pytest.raises(ValueError, match="stress"):
        relax_structures(_model(stresswise_weight=0.0), structs, feats, optimize_lattice=True, **GRAPH)
    with pytest.raises(ValueError, match="stress"):
        run_md(_model(stresswise_weight=0.0), structs, feats, np.ones(feats.shape[0]), steps=1,
               ensemble="npt_berendsen", pressure=0.0, compressibility=1e-6, taup=100.0, taut=50.0, **GRAPH)
    # accepted: force_mult_natoms (eALIGNN ignores it), no penalty with energies not multiplied, no ALIGNN layers
    # without torque removal
    for kw in (dict(force_mult_natoms=True), dict(energy_mult_natoms=False, use_penalty=False),
               dict(alignn_layers=0, remove_torque=False)):
        got = single_point(_model(**kw), structs, feats, **GRAPH)
        assert torch.isfinite(got.forces).all(), kw


def test_crystal_graphs_without_the_line_graph():
    structs, feats = _structures()
    g, lg, lat = neighbors.crystal_graphs_device(structs, feats, device=DEV, **GRAPH)
    g2, lg2, lat2 = neighbors.crystal_graphs_device(structs, feats, device=DEV, line_graph=False, **GRAPH)
    assert lg is not None and lg2 is None
    assert torch.equal(g.index.src, g2.index.src) and torch.equal(g.index.dst, g2.index.dst)
    assert torch.equal(g.batch_num_nodes(), g2.batch_num_nodes()) and torch.equal(g.batch_num_edges(), g2.batch_num_edges())
    for k in g.ndata:
        assert torch.equal(g.ndata[k], g2.ndata[k]), k
    for k in g.edata:
        assert torch.equal(g.edata[k], g2.edata[k]), k
    assert torch.equal(lat, lat2)
