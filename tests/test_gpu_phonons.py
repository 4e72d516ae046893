"""GPU (-m gpu): batched finite-displacement phonons.  The force-constant and dynamical-matrix kernels
(`ops.phonon_force_constants` / `ops.phonon_dynamical_matrix`, csrc/phonon_device.cu) against the numpy restatement
`oracle/phonon_oracle.py`, and `phonons` against a host loop that evaluates each displaced supercell alone the
reference's way (host graph build, the same model on a one-crystal batch) and post-processes with the oracle."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from alignn_b200 import _lib, neighbors, ops, phonons
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from alignn_b200.phonons import displaced_supercells
from oracle import phonon_oracle as PO
from oracle.fire_oracle import scaled_forces

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _close(a, b, rtol):
    a, b = np.asarray(a), np.asarray(b)
    return np.abs(a - b).max() <= rtol * max(np.abs(b).max(), 1e-300)


# ---- 1. the force-constant kernel on scripted forces -------------------------------------------------------------------
def _scripted(sizes, N, seed=0, mult=1.5, delta=0.013):
    rng = np.random.default_rng(seed)
    Nc = int(np.prod(N))
    grads = [rng.normal(size=(6 * n * Nc * n, 3)).astype(np.float32) for n in sizes]
    masses = [rng.uniform(1.0, 200.0, n) for n in sizes]
    aoff = neighbors.ragged_offsets(sizes)
    roff = neighbors.ragged_offsets([g.shape[0] for g in grads])
    foff = neighbors.ragged_offsets([Nc * 9 * n * n for n in sizes])
    t = dict(grad=torch.from_numpy(np.concatenate(grads)).to(DEV), aoff=torch.from_numpy(aoff).to(DEV),
             roff=torch.from_numpy(roff).to(DEV), foff=torch.from_numpy(foff).to(DEV),
             m=torch.from_numpy(np.concatenate(masses)).to(DEV))
    return grads, masses, foff, t, mult, delta


def _launch(t, fo, N, mult, delta, fill=0.0, **over):
    a = dict(t, **over)
    B = a["aoff"].numel() - 1
    Cn = torch.full((int(fo[-1]),), fill, dtype=torch.float64, device=DEV)
    Dn = torch.full_like(Cn, fill)
    st = torch.zeros(B, dtype=torch.int32, device=DEV)
    ops.phonon_force_constants(a["grad"], a["aoff"], a["roff"], a["foff"], a["m"], Cn, Dn, st, supercell=N, delta=delta,
                               force_multiplier=mult)
    return Cn, Dn, st


@pytest.mark.parametrize("N", [(2, 2, 2), (3, 3, 3), (1, 2, 3), (2, 3, 1)])
def test_force_constants_match_oracle_on_scripted_forces(N):
    sizes = [1, 2, 5, 8] + ([20] if N != (3, 3, 3) else [11])
    grads, masses, foff, t, mult, delta = _scripted(sizes, N)
    Cn, Dn, st = _launch(t, foff, N, mult, delta)
    assert st.tolist() == [0] * len(sizes)
    Nc = int(np.prod(N))
    Ch, Dh = Cn.cpu().numpy(), Dn.cpu().numpy()
    for b, n in enumerate(sizes):
        f = scaled_forces(grads[b], mult).astype(np.float64).reshape(6 * n, Nc * n, 3)
        C_N, D_N = PO.force_constants(f, masses[b], N, delta)
        got_C = Ch[foff[b]:foff[b + 1]].reshape(C_N.shape)
        got_D = Dh[foff[b]:foff[b + 1]].reshape(D_N.shape)
        assert _close(got_C, C_N, 1e-12) and _close(got_D, D_N, 1e-12), (N, n)
    again = _launch(t, foff, N, mult, delta)
    assert torch.equal(again[0], Cn) and torch.equal(again[1], Dn)        # bitwise repeatable
    # one crystal alone gives the same bits as in the batch
    b = 2
    sub = dict(grad=t["grad"][int(t["roff"][b]):int(t["roff"][b + 1])], aoff=torch.tensor([0, sizes[b]], device=DEV),
               roff=torch.tensor([0, int(t["roff"][b + 1] - t["roff"][b])], device=DEV),
               foff=torch.tensor([0, int(foff[b + 1] - foff[b])], device=DEV), m=torch.from_numpy(masses[b]).to(DEV))
    one = _launch(sub, np.array([0, foff[b + 1] - foff[b]]), N, mult, delta)
    assert torch.equal(one[0], Cn[foff[b]:foff[b + 1]]) and torch.equal(one[1], Dn[foff[b]:foff[b + 1]])


def test_bad_slices_and_non_finite_forces_touch_only_their_status():
    N, sizes = (2, 2, 2), [2, 3, 1, 2]
    grads, masses, foff, t, mult, delta = _scripted(sizes, N, seed=4)
    clean = _launch(t, foff, N, mult, delta)
    roff = t["roff"].clone()
    roff[2] = roff[1] + 1                                                    # crystal 1's row slice is short
    g = t["grad"].clone()
    g[int(t["roff"][3]) + 5, 1] = float("nan")                               # crystal 3 has a NaN force
    Cn, Dn, st = _launch(t, foff, N, mult, delta, fill=-7.0, roff=roff, grad=g)
    assert st.tolist() == [0, ops.PHONON_BAD_INPUT, ops.PHONON_BAD_INPUT, ops.PHONON_NON_FINITE]
    for b in range(4):
        sl = slice(int(foff[b]), int(foff[b + 1]))
        if b == 0:
            assert torch.equal(Cn[sl], clean[0][sl]) and torch.equal(Dn[sl], clean[1][sl])
        else:
            assert (Cn[sl] == -7.0).all() and (Dn[sl] == -7.0).all(), b
    big = torch.full_like(t["grad"], 3e38)                                   # finite, but 3e38 * 1.5 is not
    _, _, st = _launch(t, foff, N, 1.5, delta, grad=big)
    assert st.tolist() == [ops.PHONON_NON_FINITE] * 4
    short = t["foff"].clone()
    short[-1] -= 1                                                           # the last C_N slice is one short
    _, _, st = _launch(t, foff, N, mult, delta, foff=short)
    assert st.tolist() == [0, 0, 0, ops.PHONON_BAD_INPUT]


# ---- 2. the dynamical-matrix kernel --------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [(2, 2, 2), (3, 3, 3), (1, 2, 3)])
def test_dynamical_matrix_matches_oracle(N):
    rng = np.random.default_rng(7)
    Nc, sizes = int(np.prod(N)), [3, 1, 3, 8]
    D = [rng.normal(size=(Nc, 3 * n, 3 * n)) for n in sizes]
    foff = neighbors.ragged_offsets([d.size for d in D])
    D_all = torch.from_numpy(np.concatenate([d.ravel() for d in D])).to(DEV)
    foff_d = torch.from_numpy(foff).to(DEV)
    st = torch.zeros(len(sizes), dtype=torch.int32, device=DEV)
    for n in sorted(set(sizes)):
        M = 3 * n
        crystals = [b for b in range(len(sizes)) if sizes[b] == n for _ in range(7)]
        q = np.concatenate([rng.uniform(-1.5, 1.5, size=(6, 3)), np.zeros((1, 3))] * (len(crystals) // 7))
        out = torch.zeros(len(crystals), M, M, dtype=torch.complex128, device=DEV)
        ops.phonon_dynamical_matrix(D_all, foff_d, torch.tensor(crystals, dtype=torch.int32, device=DEV),
                                    torch.from_numpy(q).to(DEV), out, st, supercell=N, modes=M)
        got = out.cpu().numpy()
        iu = np.triu_indices(M, 1)
        for k, (b, qk) in enumerate(zip(crystals, q)):
            want = PO.dynamical_matrix(D[b], N, qk)
            assert _close(got[k][iu], want[iu], 1e-12), (n, k)
            assert _close(np.diag(got[k]).real, np.diag(want).real, 1e-12) and (np.diag(got[k]).imag == 0).all()
            assert np.array_equal(got[k], got[k].conj().T)
        again = torch.zeros_like(out)
        ops.phonon_dynamical_matrix(D_all, foff_d, torch.tensor(crystals, dtype=torch.int32, device=DEV),
                                    torch.from_numpy(q).to(DEV), again, st, supercell=N, modes=M)
        assert torch.equal(again, out)
    assert st.tolist() == [0] * len(sizes)
    # a crystal whose slice does not hold [Nc, M, M] gets status 3 and its pairs are not written
    out = torch.full((2, 9, 9), 5.0 + 5.0j, dtype=torch.complex128, device=DEV)
    ops.phonon_dynamical_matrix(D_all, foff_d, torch.tensor([0, 1], dtype=torch.int32, device=DEV),
                                torch.zeros(2, 3, dtype=torch.float64, device=DEV), out, st, supercell=N, modes=9)
    assert st.tolist() == [0, ops.PHONON_BAD_INPUT, 0, 0]
    assert (out[1] == 5.0 + 5.0j).all() and not (out[0] == 5.0 + 5.0j).any()


def test_kernels_reject_bad_arguments():
    N, sizes = (2, 2, 2), [1, 2]
    grads, masses, foff, t, mult, delta = _scripted(sizes, N)
    for kw in (dict(supercell=(0, 2, 2)), dict(supercell=(2, -1, 2)), dict(supercell=(16, 16, 16)),
               dict(supercell=None), dict(delta=0.0), dict(delta=-0.01), dict(delta=float("nan")),
               dict(delta=float("inf")), dict(force_multiplier=float("nan")), dict(force_multiplier=float("inf"))):
        a = dict(dict(supercell=N, delta=delta, force_multiplier=mult), **kw)
        Cn = torch.zeros(int(foff[-1]), dtype=torch.float64, device=DEV)
        with pytest.raises(RuntimeError, match="alignn_b200_phonon_force_constants failed"):
            ops.phonon_force_constants(t["grad"], t["aoff"], t["roff"], t["foff"], t["m"], Cn, Cn.clone(),
                                       torch.zeros(2, dtype=torch.int32, device=DEV), **a)
    lib = _lib.load()
    sc = C.cast((C.c_int32 * 3)(2, 2, 2), C.c_void_p)
    p = [x.data_ptr() for x in (t["aoff"], t["roff"], t["grad"], t["m"], t["foff"])]
    buf = torch.zeros(int(foff[-1]) * 2 + 2, dtype=torch.float64, device=DEV)
    st = torch.zeros(2, dtype=torch.int32, device=DEV)
    args = [sc, delta, mult, p[0], 2, p[1], p[2], t["grad"].shape[0], p[3], p[4], int(foff[-1]), buf.data_ptr(),
            buf.data_ptr() + 8 * int(foff[-1]), st.data_ptr(), None]
    assert lib.alignn_b200_phonon_force_constants(*args) == 0
    for i in (0, 3, 5, 6, 8, 9, 11, 12, 13):                                 # every pointer NULL in turn
        bad = list(args)
        bad[i] = None
        assert lib.alignn_b200_phonon_force_constants(*bad) != 0, i
    bad = list(args)
    bad[4] = 0                                                               # no crystals
    assert lib.alignn_b200_phonon_force_constants(*bad) != 0
    torch.cuda.synchronize()
    D_all = torch.zeros(8 * 9, dtype=torch.float64, device=DEV)
    fo = torch.tensor([0, 72], device=DEV)
    cr = torch.zeros(1, dtype=torch.int32, device=DEV)
    q = torch.zeros(1, 3, dtype=torch.float64, device=DEV)
    out = torch.zeros(1, 3, 3, dtype=torch.complex128, device=DEV)
    st1 = torch.zeros(1, dtype=torch.int32, device=DEV)
    for kw in (dict(supercell=(0, 2, 2)), dict(supercell=None), dict(supercell=(1, 1, 3073)), dict(modes=4)):
        a = dict(dict(supercell=N, modes=3), **kw)
        with pytest.raises((RuntimeError, ValueError)):
            ops.phonon_dynamical_matrix(D_all, fo, cr, q, out if a["modes"] == 3 else out.new_zeros(1, 4, 4), st1, **a)
    dargs = [sc, 3, D_all.data_ptr(), fo.data_ptr(), 1, 72, cr.data_ptr(), q.data_ptr(), 1, out.data_ptr(),
             st1.data_ptr(), None]
    assert lib.alignn_b200_phonon_dynamical_matrix(*dargs) == 0
    for i in (0, 2, 3, 6, 7, 9, 10):
        bad = list(dargs)
        bad[i] = None
        assert lib.alignn_b200_phonon_dynamical_matrix(*bad) != 0, i
    for i, v in ((1, 0), (1, 5), (4, 0), (5, -1), (8, -1)):
        bad = list(dargs)
        bad[i] = v
        assert lib.alignn_b200_phonon_dynamical_matrix(*bad) != 0, (i, v)
    torch.cuda.synchronize()
    assert st1.item() == 0


# ---- 3. phonons() -------------------------------------------------------------------------------------------------------
def _model(seed=11):
    torch.manual_seed(seed)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64,
                               embedding_features=64, atom_input_features=92)
    return ALIGNNAtomWise(cfg).to(DEV).eval()


def _structures(count=3, seed=3, max_atoms=3):
    """The smallest sample structures, random features and masses, and a few q-points each."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    sizes = off[1:] - off[:-1]
    pick = [i for i in np.argsort(sizes, kind="stable") if sizes[i] <= max_atoms][:count]
    out = [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]]) for i in pick]
    rng = np.random.default_rng(seed)
    n = sum(x.shape[0] for _, x in out)
    feats = torch.from_numpy(rng.normal(size=(n, 92)).astype(np.float32)).to(DEV)
    masses = rng.uniform(1.0, 200.0, n)
    q = [np.concatenate([np.zeros((1, 3)), rng.uniform(-0.5, 0.5, size=(4 + b, 3))]) for b in range(len(out))]
    return out, feats, masses, q


def _host_forces(model, latN, x, feats_tiled, mult):
    g, lg = neighbors.crystal_graph(latN, x, feats_tiled, cutoff=8.0, neighbor_strategy="k-nearest", max_neighbors=12)
    lat_t = torch.tensor(latN, dtype=torch.float32).view(1, 3, 3).to(DEV)
    res = model((g.to(DEV), lg.to(DEV), lat_t))
    return scaled_forces(res["grad"].detach().reshape(-1, 3).cpu().numpy(), mult)


def test_phonons_match_host_loop():
    model = _model()
    structs, feats, masses, q = _structures()
    N, delta, mult, kpts = (2, 2, 2), 0.01, 1.5, (4, 4, 4)
    got = phonons(model, structs, feats, masses, supercell=N, delta=delta, qpoints=q, dos_kpts=kpts, dos_npts=50,
                  dos_width=1e-3, force_multiplier=mult)
    off = got.atom_offsets.cpu().tolist()
    for b, (lat, X) in enumerate(structs):
        sl = slice(off[b], off[b + 1])
        tiled = feats[sl].cpu().repeat(8, 1)
        latN, disp = displaced_supercells(lat, X, N, delta)
        f = np.stack([_host_forces(model, latN, x, tiled, mult) for x in disp]).astype(np.float64)
        r = PO.postprocess(f, masses[sl], N, delta, qpoints=q[b], dos_kpts=kpts, dos_npts=50, dos_width=1e-3)
        assert _close(got.force_constants[b].cpu().numpy(), r["C_N"], 1e-12), b
        assert _close(got.dynamical_matrix[b].cpu().numpy(), r["D_N"], 1e-12), b
        e = got.band_energies[b].cpu().numpy()
        w2 = np.sign(e) * (e / PO.EV_PER_SQRT_EV_A2_AMU) ** 2
        assert e.shape == r["omega2"].shape and np.abs(w2 - r["omega2"]).max() <= 1e-10 * np.abs(r["omega2"]).max(), b
        assert _close(got.dos_energies[b].cpu().numpy(), r["dos_energies"], 1e-9), b
        assert _close(got.dos_weights[b].cpu().numpy(), r["dos_weights"], 1e-6), b


def _equal(a, b):
    for x, y in zip(a, b):
        if isinstance(x, list):
            assert all(torch.equal(u, v) for u, v in zip(x, y))
        elif x is None:
            assert y is None
        else:
            assert torch.equal(x, y)


def test_phonons_are_batch_invariant_and_chunk_invariant():
    model = _model()
    structs, feats, masses, q = _structures(count=4, max_atoms=4)
    kw = dict(supercell=(2, 2, 2), dos_kpts=(3, 3, 3), dos_npts=30)
    got = phonons(model, structs, feats, masses, qpoints=q, **kw)
    off = got.atom_offsets.cpu().tolist()
    for b in range(len(structs)):
        sl = slice(off[b], off[b + 1])
        one = phonons(model, [structs[b]], feats[sl], masses[sl], qpoints=[q[b]], **kw)
        assert torch.equal(one.force_constants[0], got.force_constants[b]), b
        assert torch.equal(one.dynamical_matrix[0], got.dynamical_matrix[b]), b
        assert torch.equal(one.band_energies[0], got.band_energies[b]), b
        assert torch.equal(one.dos_energies[0], got.dos_energies[b]) and torch.equal(one.dos_weights[0], got.dos_weights[b])
    smallest = 8 * max(x.shape[0] for _, x in structs)
    tight = phonons(model, structs, feats, masses, qpoints=q, max_batch_atoms=smallest, **kw)
    _equal(tight, got)


def test_phonons_with_a_penalised_short_bond():
    model = _model()
    structs, feats, masses, q = _structures(count=2)
    lat, X = structs[1]
    short = (lat, np.concatenate([X, X[:1] + np.array([0.8, 0.0, 0.0])]))
    fs = feats[:1].repeat(X.shape[0] + 1, 1)
    ms = np.full(X.shape[0] + 1, 30.0)
    kw = dict(supercell=(2, 2, 2), dos_kpts=None)
    got = phonons(model, structs + [short], torch.cat([feats, fs]), np.concatenate([masses, ms]), **kw)
    one = phonons(model, [short], fs, ms, **kw)
    C1 = one.force_constants[0].cpu().numpy()
    assert np.abs(got.force_constants[-1].cpu().numpy() - C1).max() <= 1e-3 * np.abs(C1).max()
    assert got.band_energies is None and got.dos_energies is None and got.dos_weights is None


def test_phonons_under_no_grad():
    model = _model()
    structs, feats, masses, q = _structures(count=2)
    kw = dict(qpoints=q, dos_kpts=(2, 2, 2), dos_npts=20)
    ref = phonons(model, structs, feats, masses, **kw)
    with torch.no_grad():
        got = phonons(model, structs, feats, masses, **kw)
    _equal(ref, got)


def test_phonons_rejections():
    model = _model()
    structs, feats, masses, q = _structures(count=2)
    n = masses.shape[0]
    with pytest.raises(ValueError, match="phonons needs the model in eval mode"):
        phonons(model.train(), structs, feats, masses)
    model.eval()
    bad = [dict(supercell=(2, 2)), dict(supercell=(0, 2, 2)), dict(supercell=(2.0, 2, 2)), dict(supercell=(True, 2, 2)),
           dict(supercell=(16, 16, 16)), dict(delta=0.0), dict(delta=-0.01), dict(delta=float("nan")),
           dict(delta=float("inf")), dict(qpoints=q[:1]), dict(qpoints=[q[0], q[1][:, :2]]),
           dict(qpoints=[q[0], np.full((2, 3), np.nan)]), dict(qpoints=[q[0], np.zeros((0, 3))]),
           dict(qpoints=np.zeros((2, 3))), dict(dos_kpts=(0, 2, 2)), dict(dos_kpts=(2, 2)), dict(dos_npts=1),
           dict(dos_npts=2.0), dict(dos_width=0.0), dict(dos_width=float("nan")), dict(force_multiplier=float("nan")),
           dict(max_batch_atoms=8 * max(x.shape[0] for _, x in structs) - 1), dict(max_batch_atoms=1e6)]
    for kw in bad:
        with pytest.raises(ValueError):
            phonons(model, structs, feats, masses, **kw)
    for m in (masses[:-1], np.where(np.arange(n) == 0, 0.0, masses), -masses, np.full(n, np.inf)):
        with pytest.raises(ValueError, match="masses"):
            phonons(model, structs, feats, m)
    with pytest.raises(ValueError, match="rows"):
        phonons(model, structs, feats[:-1], masses)
    with pytest.raises(ValueError, match="device"):
        phonons(model, structs, feats.cpu(), masses)
    with pytest.raises(ValueError, match="phonons needs the model on a CUDA device"):
        phonons(_model().cpu(), structs, feats, masses)
    for kw, err in ((dict(calculate_gradient=False), ValueError), (dict(output_features=2), ValueError),
                    (dict(force_mult_natoms=True), NotImplementedError)):
        torch.manual_seed(0)
        m = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=1, gcn_layers=1, hidden_features=64,
                                                atom_input_features=92, **kw)).to(DEV).eval()
        with pytest.raises(err, match="phonons"):
            phonons(m, structs, feats, masses)


def test_non_finite_forces_raise_naming_the_crystal():
    model = _model()
    structs, feats, masses, q = _structures(count=3)
    bad = feats.clone()
    bad[0] = float("nan")                                                    # crystal 0's model forces become NaN
    with pytest.raises(RuntimeError, match="crystal 0 are not finite"):
        phonons(model, structs, bad, masses, dos_kpts=None)
