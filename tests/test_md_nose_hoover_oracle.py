"""CPU: the ASE NPT restatement `oracle/md_nose_hoover_oracle.py` -- velocity Verlet with thermostat and barostat off,
the first-pass exit of a crystal at rest, the thermostat's exact leapfrog identity and its pull towards desiredEkin,
the barostat's direction with the cell kept upper triangular bitwise, ASE's rejections, run_md's host constants
against the oracle's, and the C layout of the step's parameter struct."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from alignn_b200 import _lib, md, ops
from oracle import md_nose_hoover_oracle as NH
from oracle import md_oracle as MO
from tests.test_cell_filter_oracle import _fcc_springs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FCC = np.array([[0.0, 0.0, 0.0], [0.0, 0.5, 0.5], [0.5, 0.0, 0.5], [0.5, 0.5, 0.0]])


def _spring_crystal(cells=(1, 1, 1), shear=0.0, seed=0, T=300.0):
    """A conventional FCC cell (a = 2.5 sqrt(2) * 1.01 A) repeated `cells` times, its cell upper triangular with an
    optional xy / xz shear, atoms jittered, mixed masses and Maxwell-Boltzmann momenta at T with zero sum."""
    a = 2.5 * np.sqrt(2.0) * 1.01
    rep = np.array([[i, j, k] for i in range(cells[0]) for j in range(cells[1]) for k in range(cells[2])], dtype=float)
    frac = ((FCC[None, :, :] + rep[:, None, :]) / np.array(cells, dtype=float)).reshape(-1, 3)
    h = np.diag(np.array(cells, dtype=float) * a)
    h[0, 1], h[0, 2] = shear * a, 0.5 * shear * a
    rng = np.random.default_rng(seed)
    X = frac @ h + rng.normal(scale=0.03, size=frac.shape)
    m = rng.choice([12.011, 28.085, 63.546], len(X))
    p = MO.maxwell_boltzmann_momenta(m, T, rng)
    return h, X, m, p - p.sum(0) / len(p)


def _coarse(ev):
    """ev with its forces rounded to multiples of 2^-12 eV/A: the two integrators' positions part by rounding (about
    1e-15 A), and an fp32 force would turn that into a full fp32 ulp whenever it straddles a rounding boundary, which
    then grows; on the coarse grid the forces of both stay identical."""
    def evaluate(cell, x):
        e, f, s = ev(cell, x)
        return e, (np.round(f.astype(np.float64) * 4096.0) / 4096.0).astype(np.float32), s
    return evaluate


@pytest.mark.parametrize("shear", [0.0, 0.2])
def test_thermostat_and_barostat_off_is_velocity_verlet(shear):
    ev = _coarse(_fcc_springs(r0=2.5, k=1.0))
    h, X, m, p0 = _spring_crystal(shear=shear)
    kw = dict(steps=300, dt=2.0 * MO.fs, momenta=p0, force_multiplier=1.5)
    r = NH.run(ev, h, X, m, temperature_K=300.0, **kw)
    q = MO.run(lambda x: ev(h, x)[:2], X, m, **kw)
    assert r["md"].passes == 2
    for key in ("positions", "momenta"):
        assert np.abs(r[key] - q[key]).max() <= 1e-10 * np.abs(q[key]).max(), key
    for key in ("kinetic_energy", "energy"):
        assert np.abs(np.subtract(r[key], q[key])).max() <= 1e-10 * np.abs(q[key]).max(), key
    assert np.abs(r["positions"] - X).max() > 0.05                    # it moved
    assert all(np.array_equal(c, h) for c in r["cells"]) and np.array_equal(r["cell"], h)
    npt = r["md"]
    assert not npt.eta.any() and not npt.eta_past.any() and npt.zeta == 0.0 and npt.zeta_past == 0.0


def test_crystal_at_rest_leaves_after_the_first_pass():
    ev = _fcc_springs(r0=2.5, k=1.0)
    h, X, m, _ = _spring_crystal()
    dt = 1.0 * MO.fs
    r = NH.run(ev, h, X, m, steps=1, dt=dt, temperature_K=300.0)
    assert r["md"].passes == 1
    f0 = ev(h, X)[1].astype(np.float64)
    assert np.abs(r["positions"] - (X + dt * dt * f0 / m[:, None])).max() <= 1e-13
    assert r["kinetic_energy"][0] == 0.0


def test_thermostat_leapfrog_identity_and_its_target():
    """ttime = 20 fs on a 32-atom spring crystal started at 600 K towards 300 K: summing the leapfrog zeta update over K
    steps gives mean_k (Ekin_k - desiredEkin) = (zeta_K + zeta_{K-1} - zeta_0 - zeta_past) / (2 tfact K dt), and the
    kinetic energy averaged over the run is within 10 % of desiredEkin."""
    ev = _fcc_springs(r0=2.5, k=1.0)
    h, X, m, p0 = _spring_crystal(cells=(2, 2, 2), T=600.0, seed=1)
    dt, ttime, K = 2.0 * MO.fs, 20.0 * MO.fs, 400
    r = NH.run(ev, h, X, m, steps=K, dt=dt, temperature_K=300.0, ttime=ttime, momenta=p0)
    npt = r["md"]
    E = np.array(r["kinetic_energy"])
    zeta_past0 = 0.0 - dt * npt.tfact * (E[0] - npt.desiredEkin)
    lhs = np.mean(E[:K] - npt.desiredEkin)
    rhs = (npt.zeta + npt.zeta_past - 0.0 - zeta_past0) / (2 * npt.tfact * K * dt)
    assert abs(lhs - rhs) <= 1e-9 * np.abs(E - npt.desiredEkin).max(), (lhs, rhs)
    assert npt.desiredEkin == 1.5 * (len(m) - 1) * (MO.kB * 300.0)
    assert E[0] > 1.6 * npt.desiredEkin and abs(E.mean() - npt.desiredEkin) <= 0.1 * npt.desiredEkin, E.mean()
    assert all(np.array_equal(c, h) for c in r["cells"])


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_barostat_moves_the_cell_towards_the_target(sign):
    ev = _fcc_springs(r0=2.5, k=1.0)
    h, X, m, p0 = _spring_crystal(shear=0.1, seed=2)
    _, _, S = ev(h, X)
    P = NH.pressure(NH.ideal_gas_stress(NH.calculator_stress(S), p0, m, h))
    target = P + sign * 0.02                                              # eV/A^3 above or below the crystal's
    B = 0.37                                                              # eV/A^3, about the springs' bulk modulus
    r = NH.run(ev, h, X, m, steps=40, dt=2.0 * MO.fs, temperature_K=300.0, externalstress=target, ttime=25 * MO.fs,
               pfactor=(50 * MO.fs) ** 2 * B, momenta=p0)
    V = [abs(np.linalg.det(c)) for c in r["cells"]]
    assert (V[-1] < V[0]) if sign > 0 else (V[-1] > V[0]), (P, V[0], V[-1])
    assert abs(V[-1] / V[0] - 1.0) > 1e-3
    for c in r["cells"]:
        assert c[1, 0] == 0.0 and c[2, 0] == 0.0 and c[2, 1] == 0.0       # U() keeps h upper triangular exactly
    assert r["md"].pfact == 1.0 / ((50 * MO.fs) ** 2 * B * np.linalg.det(h))


def test_rejections_mirror_ase():
    ev = _fcc_springs(r0=2.5, k=1.0)
    h, X, m, _ = _spring_crystal()
    kw = dict(steps=2, dt=1.0 * MO.fs)
    sheared = h.copy()
    sheared[2, 1] = 0.1
    with pytest.raises(NotImplementedError, match="upper triangular"):
        NH.run(ev, sheared, X, m, temperature_K=300.0, **kw)
    with pytest.raises(TypeError, match="temperature"):
        NH.run(ev, h, X, m, **kw)
    with pytest.raises(TypeError, match="externalstress"):
        NH.run(ev, h, X, m, temperature_K=300.0, externalstress=None, pfactor=1.0, **kw)
    with pytest.raises(ValueError, match="wrong shape"):
        NH.run(ev, h, X, m, temperature_K=300.0, externalstress=np.zeros(4), **kw)
    with pytest.raises(ValueError, match="symmetric"):
        NH.run(ev, h, X, m, temperature_K=300.0, externalstress=np.arange(9.0).reshape(3, 3), **kw)
    NH.run(ev, h, X, m, temperature_K=300.0, externalstress=None, **kw)   # unused without a barostat


def test_external_stress_forms_and_host_constants():
    assert np.array_equal(NH.external_stress(0.25), [-0.25, -0.25, -0.25, 0.0, 0.0, 0.0])
    S = np.array([[1.0, 6.0, 5.0], [6.0, 2.0, 4.0], [5.0, 4.0, 3.0]])
    assert np.array_equal(NH.external_stress(S), [1.0, 2.0, 3.0, 4.0, 5.0, 6.0])
    assert np.array_equal(NH.external_stress([1.0, 2.0, 3.0, 4.0, 5.0, 6.0]), [1.0, 2.0, 3.0, 4.0, 5.0, 6.0])
    assert md.ENSEMBLES["npt_nose_hoover"] == ops.MD_NPT_NOSE_HOOVER
    # run_md's numpy constants are the oracle's, bitwise
    rng = np.random.default_rng(4)
    cells = [np.triu(np.diag([4.0, 5.0, 6.0]) + rng.uniform(-0.5, 0.5, (3, 3))) for _ in range(3)]
    sizes, T0 = [1, 4, 9], [300.0, 10.0, 1234.5]
    for ttime, pfactor in ((None, None), (25 * MO.fs, None), (25 * MO.fs, 17.0)):
        tf, pf, de = md._nose_hoover_constants(sizes, T0, ttime, pfactor, cells)
        for b in range(3):
            want = NH.constants(sizes[b], MO.kB * T0[b], ttime, pfactor, cells[b])
            assert (tf[b], pf[b], de[b]) == want, (ttime, pfactor, b)
    ext = md._external_stress(S, 3)
    assert ext.shape == (3, 6) and all(np.array_equal(e, NH.external_stress(S)) for e in ext)
    per = md._external_stress(np.stack([S, 2 * S]), 2)
    assert np.array_equal(per[1], NH.external_stress(2 * S))
    assert np.array_equal(md._external_stress(0.1, 2), np.stack([NH.external_stress(0.1)] * 2))


def test_md_nose_hoover_params_struct_matches_c_layout(tmp_path):
    S = _lib.MdNoseHooverParams
    fields = [f for f, _ in S._fields_]
    src = tmp_path / "nh.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\nint main(){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(alignn_b200_md_nose_hoover_params)'
                   + "".join(f", offsetof(alignn_b200_md_nose_hoover_params, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "nh"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in fields]
