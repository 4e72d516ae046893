"""GPU (-m gpu): batched FIRE relaxation.  The step kernel (`ops.fire_step`, csrc/fire_device.cu) against the numpy
restatement `oracle/fire_oracle.py` on scripted forces, and `relax_structures` against a host loop that relaxes each
crystal alone the reference's way (host graph build, the same model on a one-crystal batch, the oracle's FIRE)."""
import os

import numpy as np
import pytest
import torch

from alignn_b200 import neighbors, ops, relax_structures
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from oracle import fire_oracle as FO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- 1. the step kernel on scripted forces --------------------------------------------------------------------------
SIZES = [1, 2, 30, 1000]
MULT, FMAX, STEPS = 1.5, 0.05, 40


def _script(b, s, n, rng_cache={}):
    """grad of crystal b at its evaluation s: a constant push (dt grows to dtmax, steps get capped), a push that flips
    every 7 evaluations (uphill resets), and random fields decaying at different rates (converging at different
    evaluations; the 1000-atom one stays above fmax and hits the step limit)."""
    key = (b, n)
    if key not in rng_cache:
        rng_cache[key] = np.random.default_rng(100 + b).normal(size=(n, 3))
    base = rng_cache[key]
    if b == 0:
        g = 0.3 * base / np.linalg.norm(base)
    elif b == 1:
        g = (1.0 if (s // 7) % 2 == 0 else -1.0) * base * 0.8 ** (s / 2)
    elif b == 2:
        g = base * 0.8 ** s
    else:
        g = base * (1.0 + 0.1 * np.sin(s))
    return g.astype(np.float32)


def _scripted_run(freeze_probe=False):
    sizes = SIZES
    aoff = neighbors.ragged_offsets(sizes)
    N, B = int(aoff[-1]), len(sizes)
    rng = np.random.default_rng(0)
    x0 = rng.normal(size=(N, 3))
    pos = torch.from_numpy(x0.copy()).to(DEV)
    vel = torch.zeros_like(pos)
    forces = torch.zeros(N, 3, device=DEV, dtype=torch.float32)
    fstate = torch.tensor([[ops.FIRE_DT0, ops.FIRE_A0]] * B, device=DEV, dtype=torch.float64)
    istate = torch.tensor([[0, 1, 0, 0]] * B, device=DEV, dtype=torch.int32)
    aoff_d = torch.from_numpy(aoff).to(DEV)
    oracle = [FO.Fire(x0[aoff[b]:aoff[b + 1]]) for b in range(B)]
    o_state = [dict(status=0, nsteps=0, forces=None) for _ in range(B)]
    frozen_at = {}
    active, s = list(range(B)), 0
    seen = dict(reset=False, dtmax=False, capped=False)
    while active:
        grads = [_script(b, s, sizes[b]) for b in active]
        boff = torch.tensor(neighbors.ragged_offsets([sizes[b] for b in active]), dtype=torch.int32).to(DEV)
        grad = torch.from_numpy(np.concatenate(grads)).to(DEV)
        ops.fire_step(grad, torch.tensor(active, dtype=torch.int32).to(DEV), boff, aoff_d, pos, vel, forces, fstate, istate,
                      fmax=FMAX, steps=STEPS, force_multiplier=MULT)
        for b, g in zip(active, grads):                                    # the oracle's decision per crystal
            st, opt = o_state[b], oracle[b]
            st["forces"] = FO.scaled_forces(g, MULT)
            if FO.converged(st["forces"], FMAX):
                st["status"] = FO.CONVERGED
            elif st["nsteps"] >= STEPS:
                st["status"] = FO.STEP_LIMIT
            else:
                n_before, dt_before = opt.Nsteps, opt.dt
                x_before = opt.x.copy()
                opt.step(st["forces"])
                st["nsteps"] += 1
                seen["reset"] |= (n_before > 0 and opt.Nsteps == 0)
                seen["dtmax"] |= opt.dt == 1.0
                seen["capped"] |= bool(np.sqrt(((opt.x - x_before) ** 2).sum()) > 0.2 - 1e-12 and dt_before > 0)
        P, V, Fo = pos.cpu().numpy(), vel.cpu().numpy(), forces.cpu().numpy()
        FS, IS = fstate.cpu().numpy(), istate.cpu().numpy()
        for b in active:
            st, opt, sl = o_state[b], oracle[b], slice(aoff[b], aoff[b + 1])
            first = 1 if opt.v is None else 0
            assert IS[b].tolist() == [opt.Nsteps, first, st["nsteps"], st["status"]], (b, s, IS[b])
            assert np.array_equal(Fo[sl], st["forces"]), (b, s)
            np.testing.assert_allclose(FS[b], [opt.dt, opt.a], rtol=1e-12, atol=0)
            assert np.abs(P[sl] - opt.x).max() <= 1e-12 * np.abs(opt.x).max(), (b, s)
            if opt.v is not None:
                assert np.abs(V[sl] - opt.v).max() <= 1e-12 * max(np.abs(opt.v).max(), 1e-300), (b, s)
            if st["status"] != 0:
                frozen_at[b] = (P[sl].copy(), V[sl].copy(), Fo[sl].copy(), FS[b].copy(), IS[b].copy())
        for b, (p, v, f, fs, is_) in frozen_at.items():                   # frozen crystals stay bitwise as they were
            sl = slice(aoff[b], aoff[b + 1])
            assert np.array_equal(P[sl], p) and np.array_equal(V[sl], v) and np.array_equal(Fo[sl], f)
            assert np.array_equal(FS[b], fs) and np.array_equal(IS[b], is_)
        active = [b for b in active if IS[b][3] == 0]
        s += 1
    if freeze_probe:                                                      # a frozen id in the list is not touched
        before = [t.clone() for t in (pos, vel, forces, fstate, istate)]
        grad = torch.full((SIZES[2], 3), 7.0, device=DEV)
        ops.fire_step(grad, torch.tensor([2], dtype=torch.int32, device=DEV),
                      torch.tensor([0, SIZES[2]], dtype=torch.int32, device=DEV), aoff_d, pos, vel, forces, fstate, istate,
                      fmax=FMAX, steps=STEPS, force_multiplier=MULT)
        for a, b in zip(before, (pos, vel, forces, fstate, istate)):
            assert torch.equal(a, b)
    return dict(o_state=o_state, seen=seen, tensors=(pos, vel, forces, fstate, istate))


def test_fire_step_matches_oracle_on_scripted_forces():
    r = _scripted_run(freeze_probe=True)
    st = [o["status"] for o in r["o_state"]]
    steps = [o["nsteps"] for o in r["o_state"]]
    print(f"[fire scripted] status {st} nsteps {steps} seen {r['seen']}")
    assert r["seen"] == dict(reset=True, dtmax=True, capped=True)
    assert FO.CONVERGED in st and FO.STEP_LIMIT in st
    conv_steps = {steps[b] for b in range(len(st)) if st[b] == FO.CONVERGED}
    assert len(conv_steps) >= 2                                            # converging at different steps
    again = _scripted_run()
    for a, b in zip(r["tensors"], again["tensors"]):
        assert torch.equal(a, b)                                           # bitwise repeatable


# ---- 2-5. relax_structures ---------------------------------------------------------------------------------------------
def _model(seed=11):
    torch.manual_seed(seed)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64,
                               embedding_features=64, atom_input_features=92)
    return ALIGNNAtomWise(cfg).to(DEV).eval()


def _structures(count=8, seed=3):
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    sizes = off[1:] - off[:-1]
    idx = [i for i in range(len(sizes)) if sizes[i] <= 12]
    rng = np.random.default_rng(seed)
    pick = rng.choice(idx, count, replace=False)
    out = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]] + rng.normal(scale=0.05, size=(sizes[i], 3)))
           for i in pick]
    feats = torch.from_numpy(rng.normal(size=(sum(x.shape[0] for _, x in out), 92)).astype(np.float32)).to(DEV)
    return out, feats


def _host_evaluator(model, lat, feats, strategy, cutoff):
    lat_t = torch.tensor(lat, dtype=torch.float32).view(1, 3, 3).to(DEV)

    def evaluate(x):
        g, lg = neighbors.crystal_graph(lat, x, feats.cpu(), cutoff=cutoff, neighbor_strategy=strategy, max_neighbors=12)
        res = model((g.to(DEV), lg.to(DEV), lat_t))
        e = (res["out"].detach().reshape(-1) * float(x.shape[0])).cpu().numpy()[0]
        return e, res["grad"].detach().reshape(-1, 3).cpu().numpy()
    return evaluate


def _host_relax(model, structs, feats, strategy, cutoff, **kw):
    out, o = [], 0
    for lat, X in structs:
        n = X.shape[0]
        out.append(FO.relax(_host_evaluator(model, lat, feats[o:o + n], strategy, cutoff), X, **kw))
        o += n
    return out


@pytest.mark.parametrize("strategy,cutoff", [("k-nearest", 8.0), ("radius_graph", 6.0)])
def test_relax_structures_matches_host_loop(strategy, cutoff):
    model = _model()
    structs, feats = _structures()
    steps, mult = 12, 1.5
    # fmax from the oracle's own trajectories (fmax = 0: every crystal runs to the limit): the smallest max |F_i|^2 of
    # each crystal over the evaluations it reaches before the limit
    rec, o = [], 0
    for lat, X in structs:
        n = X.shape[0]
        base = _host_evaluator(model, lat, feats[o:o + n], strategy, cutoff)
        m2 = []

        def ev(x, base=base, m2=m2):
            e, g = base(x)
            f = FO.scaled_forces(g, mult).astype(np.float64)
            m2.append((f ** 2).sum(1).max())
            return e, g
        FO.relax(ev, X, fmax=0.0, steps=steps, force_multiplier=mult)
        rec.append(min(m2[:-1]))                                          # reachable before the step limit
        o += n
    srt = sorted(m for m in rec if m > 0)                                 # a 1-atom cell has no force at all
    assert srt[0] < srt[-1]
    fmax = float(np.sqrt(np.sqrt(srt[0] * srt[len(srt) // 2])))           # between the lowest and the median
    ref = _host_relax(model, structs, feats, strategy, cutoff, fmax=fmax, steps=steps, force_multiplier=mult)
    got = relax_structures(model, structs, feats, fmax=fmax, steps=steps, neighbor_strategy=strategy, cutoff=cutoff,
                           force_multiplier=mult)
    nst = got.nsteps.cpu().tolist()
    conv = got.converged.cpu().tolist()
    print(f"[relax {strategy}] fmax {fmax:.4g} nsteps {nst} converged {conv}")
    assert nst == [r["nsteps"] for r in ref] and conv == [r["converged"] for r in ref]
    assert any(conv) and not all(conv) and min(nst) < steps
    off = got.atom_offsets.cpu().tolist()
    P, F, E = got.positions.cpu().numpy(), got.forces.cpu().numpy(), got.energy.cpu().numpy()
    for b, r in enumerate(ref):
        sl = slice(off[b], off[b + 1])
        assert np.abs(P[sl] - r["positions"]).max() <= 1e-9, b
        assert np.abs(F[sl] - r["forces"]).max() <= 1e-5 * max(np.abs(r["forces"]).max(), 1e-30), b
        assert abs(E[b] - r["energy"]) <= 1e-5 * max(abs(r["energy"]), 1e-30), b


def test_relax_structures_is_batch_invariant():
    """Positions and forces bitwise; the energy within 1e-5 relative: the readout `fc` (torch's Linear on the pooled
    [B, d] rows) sums in an order that depends on the number of crystals in the batch (DESIGN section 10)."""
    model = _model()
    structs, feats = _structures()
    got = relax_structures(model, structs, feats, fmax=0.0, steps=6)
    off = got.atom_offsets.cpu().tolist()
    for b in (0, 3, len(structs) - 1):
        one = relax_structures(model, [structs[b]], feats[off[b]:off[b + 1]], fmax=0.0, steps=6)
        sl = slice(off[b], off[b + 1])
        assert torch.equal(one.positions, got.positions[sl]), b
        assert torch.equal(one.forces, got.forces[sl]), b
        assert torch.allclose(one.energy, got.energy[b:b + 1], rtol=1e-5, atol=0), b


def test_relax_structures_edge_cases():
    model = _model()
    structs, feats = _structures(count=4)
    got = relax_structures(model, structs, feats, fmax=1e6, steps=5, force_multiplier=2.0)
    assert got.nsteps.tolist() == [0] * 4 and got.converged.tolist() == [True] * 4
    X = np.concatenate([x for _, x in structs])
    assert np.array_equal(got.positions.cpu().numpy(), X)
    g, lg, lat = neighbors.crystal_graphs_device(structs, feats, device=DEV)
    res = model((g, lg, lat))
    assert torch.equal(got.energy, res["out"].detach() * g.batch_num_nodes_on_device().float())
    assert torch.equal(got.forces, res["grad"].detach() * torch.tensor(2.0, device=DEV))
    # steps=1: evaluate, step, evaluate -- two model calls for the batch
    calls = []
    hook = model.register_forward_hook(lambda *a: calls.append(1))
    try:
        got = relax_structures(model, structs[:1], feats[:structs[0][1].shape[0]], fmax=0.0, steps=1)
    finally:
        hook.remove()
    assert len(calls) == 2 and got.nsteps.tolist() == [1] and got.converged.tolist() == [False]


def test_relax_structures_rejections():
    model = _model()
    structs, feats = _structures(count=2)
    with pytest.raises(ValueError, match="eval"):
        relax_structures(model.train(), structs, feats)
    model.eval()
    with pytest.raises(ValueError, match="rows"):
        relax_structures(model, structs, feats[:-1])
    with pytest.raises(ValueError, match="fmax"):
        relax_structures(model, structs, feats, fmax=-0.1)
    with pytest.raises(ValueError, match="steps"):
        relax_structures(model, structs, feats, steps=0)
    with pytest.raises(ValueError, match="steps"):
        relax_structures(model, structs, feats, steps=2 ** 32 + 5)                # would wrap to 5 as an int32
    with pytest.raises(ValueError, match="fmax"):
        relax_structures(model, structs, feats, fmax=float("nan"))
    got = relax_structures(model, structs, feats, fmax=np.float32(1e6), steps=np.int64(2))   # numpy scalars are numbers
    assert got.converged.tolist() == [True, True]
    with pytest.raises(ValueError, match="device"):
        relax_structures(model, structs, feats.cpu())
    with pytest.raises(ValueError, match="CUDA"):
        relax_structures(_model().cpu(), structs, feats)
    for kw, err in ((dict(calculate_gradient=False), ValueError), (dict(output_features=2), ValueError),
                    (dict(energy_mult_natoms=False, use_penalty=True), NotImplementedError)):
        torch.manual_seed(0)
        m = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=1, gcn_layers=1, hidden_features=64,
                                                atom_input_features=92, **kw)).to(DEV).eval()
        with pytest.raises(err):
            relax_structures(m, structs, feats)


def test_bond_penalty_counted_once_per_crystal():
    """A crystal with bonds under the penalty threshold (1 A) relaxes in a batch as it does alone: the model adds the
    batch's penalty to every crystal's energy, and relax_structures takes the extra copies of its gradient back out
    (fp32 rounding on those bonds' pair forces only)."""
    model = _model()
    structs, feats = _structures(count=4)
    lat, X = structs[1]
    short = (lat, np.concatenate([X, X[:1] + np.array([0.8, 0.0, 0.0])]))
    f_short = feats[:1].repeat(X.shape[0] + 1, 1)
    batch_structs = structs + [short]
    batch_feats = torch.cat([feats, f_short])
    got = relax_structures(model, batch_structs, batch_feats, fmax=0.0, steps=3)
    one = relax_structures(model, [short], f_short, fmax=0.0, steps=3)
    off = got.atom_offsets.cpu().tolist()
    sl = slice(off[-2], off[-1])
    F1 = one.forces.cpu().numpy()
    assert np.abs(got.forces[sl].cpu().numpy() - F1).max() <= 1e-5 * np.abs(F1).max()
    assert np.abs(got.positions[sl].cpu().numpy() - one.positions.cpu().numpy()).max() <= 1e-6


def test_relax_structures_under_no_grad():
    """The usual inference context: forces come from autograd inside, so torch.no_grad() around the call changes
    nothing, also for a batch whose bond-penalty gradient is taken back out."""
    model = _model()
    structs, feats = _structures(count=3)
    lat, X = structs[1]
    structs = structs + [(lat, np.concatenate([X, X[:1] + np.array([0.8, 0.0, 0.0])]))]
    feats = torch.cat([feats, feats[:1].repeat(X.shape[0] + 1, 1)])
    ref = relax_structures(model, structs, feats, fmax=0.0, steps=3)
    with torch.no_grad():
        got = relax_structures(model, structs, feats, fmax=0.0, steps=3)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)


def test_fire_step_rejects_a_batch_slice_that_is_not_the_crystal():
    """A batch slice whose length differs from the crystal's atom count, or that runs past the end of grad, is not read:
    the crystal's status becomes FIRE_BAD_INPUT and nothing else changes; a consistent crystal in the same launch steps."""
    aoff = torch.tensor([0, 2, 5], dtype=torch.int64, device=DEV)
    pos = torch.randn(5, 3, dtype=torch.float64, device=DEV)
    vel, forces = torch.zeros_like(pos), torch.zeros(5, 3, device=DEV)
    fstate = torch.tensor([[0.1, 0.1]] * 2, dtype=torch.float64, device=DEV)
    istate = torch.tensor([[0, 1, 0, 0]] * 2, dtype=torch.int32, device=DEV)
    crystal1 = lambda: [pos[2:].clone(), vel[2:].clone(), forces[2:].clone(), fstate[1].clone()]  # noqa: E731
    before = crystal1()
    grad = torch.ones(4, 3, device=DEV)                                    # crystal 1 needs 3 rows, gets 2
    ops.fire_step(grad, torch.tensor([0, 1], dtype=torch.int32, device=DEV),
                  torch.tensor([0, 2, 4], dtype=torch.int32, device=DEV), aoff, pos, vel, forces, fstate, istate,
                  fmax=0.0, steps=5)
    assert istate[1].tolist() == [0, 1, 0, ops.FIRE_BAD_INPUT] and istate[0].tolist() == [0, 0, 1, 0]
    for a, b in zip(before, crystal1()):
        assert torch.equal(a, b)
    istate[1, 3] = 0
    ops.fire_step(grad[:3], torch.tensor([1], dtype=torch.int32, device=DEV),    # past the end of grad
                  torch.tensor([1, 4], dtype=torch.int32, device=DEV), aoff, pos, vel, forces, fstate, istate,
                  fmax=0.0, steps=5)
    assert istate[1, 3].item() == ops.FIRE_BAD_INPUT
    with pytest.raises(ValueError, match="steps"):
        ops.fire_step(grad, torch.tensor([0], dtype=torch.int32, device=DEV),
                      torch.tensor([0, 2], dtype=torch.int32, device=DEV), aoff, pos, vel, forces, fstate, istate,
                      fmax=0.0, steps=2 ** 32 + 5)
