"""CPU: oracle/eos_oracle.py, the restatement of ASE 3.22.1's `EquationOfState.fit` that `alignn_b200.fit_eos` and
`ev_curve` are tested against: exact curves are recovered, the tight least-squares fit and the ASE restatement agree,
the parabola seed, ASE's warning as status 1, curve_fit's rejection of too few points, the GPa constant, and the
package's strain and volume arithmetic against jarvis' restated."""
import numpy as np
import pytest

from alignn_b200 import eos as E
from oracle import eos_oracle as EO


@pytest.mark.parametrize("form", EO.FORMS)
def test_exact_curves_are_recovered(form):
    V = 40.0 * (1 + np.arange(-0.05, 0.05, 0.01)) ** 3
    true = np.array([-7.3, 0.6, 4.7, 40.5])
    e = EO.FUNCS[form](V, *true)
    for fit in (EO.ase_fit, EO.tight_fit):
        p, st = fit(V, e, form)
        assert st == EO.OK
        assert np.allclose(p, true, rtol=1e-6 if fit is EO.ase_fit else 1e-9, atol=0), (fit, p)


@pytest.mark.parametrize("form", EO.FORMS)
def test_tight_fit_and_ase_restatement_agree_on_fp32_energies(form):
    V, En, _ = EO.random_rows(form, 60, 10, seed=5)
    worst = np.zeros(4)
    for r in range(V.shape[0]):
        a, sa = EO.ase_fit(V[r], En[r], form)
        t, st = EO.tight_fit(V[r], En[r], form)
        assert sa == st == EO.OK
        worst = np.maximum(worst, np.abs(a - t) / np.abs(t))
    # ASE's default curve_fit tolerance (1.49e-8) against the converged optimum: E0, B0, BP, V0
    assert (worst <= [1e-10, 1e-7, 3e-7, 1e-8]).all(), worst


def test_seed_of_an_exact_parabola():
    V = np.linspace(900.0, 1200.0, 10)
    a, b, c = 12.0, -0.3, 1.5e-4
    e = EO.parabola(V, a, b, c)
    vmin = -b / 2 / c
    want = [EO.parabola(vmin, a, b, c), 2 * c * vmin, 4.0, vmin]
    assert np.allclose(EO.lsq_seed(V, e), want, rtol=1e-9, atol=0)
    assert np.allclose(EO.ase_seed(V, e), want, rtol=1e-5, atol=0)


def test_minimum_outside_the_volumes_is_status_1():
    V = 40.0 * (1 + np.arange(-0.05, 0.05, 0.01)) ** 3
    e = EO.murnaghan(V, -7.3, 0.6, 4.7, 52.0)                  # V0 beyond every volume: a monotonic curve
    p, st = EO.ase_fit(V, e, "murnaghan")
    assert st == EO.OUTSIDE and p[3] > V.max()
    params, status = EO.fit_rows(V[None], e[None], "murnaghan", fit=EO.tight_fit)
    assert status.tolist() == [EO.OUTSIDE] and np.isfinite(params).all()


def test_curve_fit_rejects_fewer_points_than_parameters():
    V = np.array([38.0, 40.0, 42.0])
    with pytest.raises(TypeError):
        EO.ase_fit(V, EO.murnaghan(V, -7.3, 0.6, 4.7, 40.0), "murnaghan")
    V4 = np.array([38.0, 39.0, 41.0, 42.0])                   # four points: an exact fit
    p, st = EO.ase_fit(V4, EO.murnaghan(V4, -7.3, 0.6, 4.7, 40.0), "murnaghan")
    assert st == EO.OK and np.allclose(p, [-7.3, 0.6, 4.7, 40.0], rtol=1e-5)


def test_bad_rows_get_status_3():
    V, En, _ = EO.random_rows("vinet", 3, 10, seed=1)
    En[0, 4] = np.nan
    V[2, 0] = 0.0
    _, status = EO.fit_rows(V, En, "vinet")
    assert status.tolist() == [EO.BAD_INPUT, EO.OK, EO.BAD_INPUT]


def test_gpa_constant():
    assert E.kJ == EO.kJ and EO.kJ == 1000 / 1.6021766208e-19
    # 1 eV/A^3 = 160.21766208 GPa
    assert abs(EO.gpa(1.0) - 160.21766208) <= 1e-10
    assert EO.gpa(0.5) == 0.5 / EO.kJ * 1.0e24


def test_package_strain_matches_jarvis_restatement():
    rng = np.random.default_rng(3)
    lat = np.array([[3.1, 0.2, -0.1], [0.4, 4.2, 0.3], [-0.2, 0.1, 5.3]])
    x = rng.uniform(0, 3, (5, 3))
    for s in np.arange(-0.05, 0.05, 0.01):
        lat_p, x_p, vol_p = E.strained(lat, x, s)
        lat_o, x_o = EO.strain_atoms(lat, x, s)
        assert np.array_equal(lat_p, lat_o)                    # s I @ L is (1 + s) L, bit for bit
        assert vol_p == EO.volume(lat_o)
        assert np.abs(x_p - x_o).max() <= 1e-14                # via fractional coordinates: equal up to rounding
