"""CPU: the NPTBerendsen restatement `oracle/md_npt_oracle.py` -- its units against ase.units' formulas and
ForceField's literals, the sign of the ideal-gas term, the barostat switched off (NVT Berendsen), the direction of the
cell's response, an FCC spring crystal held at two pressures, ASE's construction rejections, the batched driver against
one-by-one runs, and the C layout of the NPT step's parameter struct."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from alignn_b200 import _lib, md, ops
from oracle import md_npt_oracle as NO
from oracle import md_oracle as MO
from tests.test_cell_filter_oracle import _fcc_springs, _morse, _morse_crystal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FCC = np.array([[0.0, 0.0, 0.0], [0.0, 0.5, 0.5], [0.5, 0.0, 0.5], [0.5, 0.5, 0.0]])


def test_units_and_forcefield_literals():
    _e = 1.6021766208e-19                                  # ase.units, CODATA 2014
    pascal = (1 / _e) / 1e30
    assert NO.Pascal == pascal and md.BAR == 1e5 * pascal
    for v in (1.0, -250.0, 1.01325, 3e4):
        assert NO.pressure_au(v) == v * (1e5 * pascal)     # NPTBerendsen._process_pressure
        assert NO.compressibility_au(v) == v / (1e5 * pascal)
    assert NO.TAUT == 49.11347394232032 == 500 * MO.fs and NO.TAUP == 98.22694788464064 == 1000 * MO.fs
    assert md.NPT_TAUT == NO.TAUT and 1000.0 * md.FS == NO.TAUP    # run_md's defaults, bitwise
    assert md.ENSEMBLES["npt_berendsen"] == ops.MD_NPT_BERENDSEN


def test_ideal_gas_pressure_is_n_kb_t_over_v():
    """No forces, no model stress: the barostat's pressure is the ideal gas's N kB T / V of the (scaled) momenta."""
    rng = np.random.default_rng(1)
    cell = np.diag([5.0, 6.0, 7.0]) + rng.normal(scale=0.3, size=(3, 3))
    m = rng.uniform(1.0, 100.0, 20)
    p = MO.maxwell_boltzmann_momenta(m, 500.0, rng)
    s = NO.ideal_gas_stress(np.zeros(6, dtype=np.float32), p, m, cell)
    assert s.dtype == np.float32
    want = len(m) * MO.kB * MO.temperature(p, m) / abs(np.linalg.det(cell))
    assert want > 0 and abs(NO.pressure(s) - want) <= 2e-7 * want

    def free(cell, x):
        return 0.0, np.zeros_like(x, dtype=np.float32), np.zeros((3, 3), dtype=np.float32)
    # after step 1's velocity scaling: mu from the scaled momenta; an ideal gas above its target pressure expands
    dt, comp = 1.0 * MO.fs, 1e-4
    r = NO.run(free, cell, rng.random((20, 3)) @ cell, m, steps=1, dt=dt, temperature_K=300.0, pressure=0.0,
               compressibility=comp, momenta=p)
    npt = r["md"]
    s_T = MO.berendsen_scale(MO.temperature(p, m), 300.0, dt, NO.TAUT)
    P = len(m) * MO.kB * MO.temperature(s_T * p, m) / abs(np.linalg.det(cell))
    grow = dt / NO.TAUP * NO.compressibility_au(comp) / 3.0 * P             # mu - 1, to the fp32 stress's precision
    assert abs((npt.mu - 1.0) - grow) <= 2e-7 * grow
    assert npt.mu > 1.0 and abs(np.linalg.det(r["cell"])) > abs(np.linalg.det(cell))


def test_zero_compressibility_is_nvt_berendsen():
    ev = _morse()
    cell, X = _morse_crystal(seed=3, n=4)
    m = np.array([12.0, 30.0, 63.5, 1.008])
    p0 = MO.maxwell_boltzmann_momenta(m, 400.0, np.random.default_rng(2))
    kw = dict(steps=25, dt=1.0 * MO.fs, temperature_K=300.0, taut=10 * MO.fs, momenta=p0, force_multiplier=1.5)
    r = NO.run(ev, cell, X, m, pressure=1e4, compressibility=0.0, **kw)
    q = MO.run(lambda x: ev(cell, x)[:2], X, m, ensemble=MO.NVT_BERENDSEN, **kw)
    assert all(np.array_equal(c, cell) for c in r["cells"]) and np.array_equal(r["cell"], cell)
    for key in ("positions", "momenta"):
        assert np.abs(r[key] - q[key]).max() <= 1e-12 * np.abs(q[key]).max(), key
    for key in ("kinetic_energy", "temperature"):
        assert np.abs(np.subtract(r[key], q[key])).max() <= 1e-12 * np.abs(q[key]).max(), key
    assert np.abs(r["positions"] - X).max() > 1e-3
    assert r["evaluations"] == 2 * 25 + 1 and len(r["pressure"]) == len(r["stress"]) == 26


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_cell_shrinks_below_and_grows_above_the_target(sign):
    ev = _morse()
    cell, X = _morse_crystal(seed=4, n=3)
    m = np.full(3, 40.0)
    _, _, S = ev(cell, X)
    P = NO.pressure(NO.ideal_gas_stress(NO.calculator_stress(S), np.zeros((3, 3)), m, cell))
    target = (P + sign * 0.01) / NO.pressure_au(1.0)                     # bar, 0.01 eV/A^3 above or below
    r = NO.run(ev, cell, X, m, steps=1, dt=1.0 * MO.fs, temperature_K=300.0, pressure=target, compressibility=1e-5)
    V0, V1 = abs(np.linalg.det(cell)), abs(np.linalg.det(r["cell"]))
    assert (V1 < V0) if sign > 0 else (V1 > V0), (P, V0, V1)
    assert abs(r["md"].mu - 1.0) > 1e-9


def test_fcc_spring_crystal_holds_its_target_pressure():
    """A 4-atom FCC cell of nearest-neighbour springs (r0 = 2.5 A, k = 1 eV/A^2, bulk modulus about 60 GPa) at 300 K,
    compressibility 1.6e-6 / bar (about 1 / B), taup = 250 fs, 400 steps of 5 fs: over the last half the mean pressure
    is within 0.0015 eV/A^3 (0.24 GPa, below one standard deviation of the instantaneous pressure) of each target, and
    the higher target gives the smaller mean volume."""
    ev = _fcc_springs(r0=2.5, k=1.0)
    cell = np.eye(3) * 2.5 * np.sqrt(2.0) * 1.01
    rng = np.random.default_rng(0)
    X = FCC @ cell + rng.normal(scale=0.02, size=(4, 3))
    m = np.full(4, 63.546)
    p0 = MO.maxwell_boltzmann_momenta(m, 300.0, rng)
    volumes = []
    for bar in (0.0, 2e4):
        r = NO.run(ev, cell, X, m, steps=400, dt=5 * MO.fs, temperature_K=300.0, pressure=bar, compressibility=1.6e-6,
                   taut=100 * MO.fs, taup=250 * MO.fs, momenta=p0)
        P = np.array(r["pressure"][200:])
        assert abs(P.mean() - NO.pressure_au(bar)) <= 0.0015, (bar, P.mean(), P.std())
        assert abs(np.mean(r["temperature"][200:]) - 300.0) <= 60.0
        volumes.append(np.mean([abs(np.linalg.det(c)) for c in r["cells"][200:]]))
    assert volumes[1] < volumes[0], volumes


def test_construction_rejections_mirror_ase():
    ev = _morse()
    cell, X = _morse_crystal()
    kw = dict(steps=2, dt=1.0 * MO.fs, temperature_K=300.0)
    with pytest.raises(TypeError, match="pressure"):
        NO.run(ev, cell, X, np.ones(3), compressibility=1e-5, **kw)
    with pytest.raises(TypeError, match="None"):
        NO.run(ev, cell, X, np.ones(3), pressure=1.0, **kw)
    with pytest.raises(TypeError):                                      # the reference's own default call
        NO.run(ev, cell, X, np.ones(3), **kw)


def test_batched_oracle_equals_one_by_one_bitwise():
    ev = _morse()
    crystals = [_morse_crystal(seed=s, n=n) for s, n in ((5, 2), (6, 3), (7, 1), (8, 4))]
    masses = [np.linspace(10.0, 60.0, x.shape[0]) for _, x in crystals]
    rng = np.random.default_rng(9)
    mom = [MO.maxwell_boltzmann_momenta(mb, 300.0, rng) if b != 2 else None for b, mb in enumerate(masses)]
    T0, P0, comp = [100.0, 300.0, 500.0, 1000.0], [0.0, 1e4, -5e3, 2e3], [1e-5, 0.0, 3e-5, 1e-5]
    kw = dict(steps=12, dt=1.0 * MO.fs, taut=5 * MO.fs, taup=50 * MO.fs, force_multiplier=1.5, stress_wt=0.8,
              trajectory_interval=4)
    alone = [NO.run(ev, c, x, masses[b], temperature_K=T0[b], pressure=P0[b], compressibility=comp[b], momenta=mom[b],
                    **kw) for b, (c, x) in enumerate(crystals)]
    bat = NO.run_batch(lambda cx: [ev(c, x) for c, x in cx], [c for c, _ in crystals], [x for _, x in crystals], masses,
                       temperature_K=T0, pressure=P0, compressibility=comp, momenta=mom, **kw)
    for r, q in zip(alone, bat):
        for key in ("positions", "momenta", "forces", "cell"):
            assert np.array_equal(r[key], q[key]), key
        for key in ("energy", "kinetic_energy", "temperature", "pressure"):
            assert r[key] == q[key], key
        assert all(np.array_equal(a, b) for a, b in zip(r["cells"], q["cells"]))
        assert all(np.array_equal(a, b) for a, b in zip(r["stress"], q["stress"]))
        assert len(r["trajectory"]) == 4 and all(np.array_equal(a, b) for a, b in zip(r["trajectory"], q["trajectory"]))
    assert np.array_equal(alone[1]["cell"], crystals[1][0])                 # compressibility 0
    assert all(np.abs(alone[b]["cell"] - crystals[b][0]).max() > 1e-6 for b in (0, 2, 3))


def test_md_npt_params_struct_matches_c_layout(tmp_path):
    S = _lib.MdNptParams
    fields = [f for f, _ in S._fields_]
    src = tmp_path / "np.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\nint main(){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(alignn_b200_md_npt_params)'
                   + "".join(f", offsetof(alignn_b200_md_npt_params, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "np"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in fields]
