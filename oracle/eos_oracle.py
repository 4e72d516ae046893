"""numpy/scipy restatement of the reference's `ev_curve` (alignn/ff/ff.py:762-805) fit with ASE 3.22.1's
`EquationOfState` (the version alignn's environment.yml pins): the specification `alignn_b200.fit_eos` /
`alignn_b200_eos_fit` and `alignn_b200.ev_curve` are tested against.

ASE sources restated (ase 3.22.1):
  ase/eos.py    murnaghan, birchmurnaghan, vinet and parabola, as written there (eta = (V0/V)**(1/3) for
                Birch-Murnaghan, (V/V0)**(1/3) for Vinet).
                EquationOfState.fit: p0 = [min(e), 1, 1]; curve_fit(parabola, v, e, p0); c, b, a = popt[2], popt[1],
                popt[0]; parabola_vmin = -b / 2 / c; E0 = parabola(parabola_vmin, a, b, c); B0 = 2 * c * parabola_vmin;
                BP = 4 (all three forms here); popt = curve_fit(func, v, e, [E0, B0, BP, parabola_vmin]); v0, e0, B =
                popt[3], popt[0], popt[1]; `warnings.warn` unless min(v) < v0 < max(v).
  ase/units.py  CODATA 2014: _e = 1.6021766208e-19, J = 1 / _e, kJ = 1000 * J; the reference's kv = B / kJ * 1.0e24.
jarvis (jarvis-tools, not in the reference tree; its documented behaviour):
  Atoms.strain_atoms(e): lattice s @ L with s = I + e I, fractional coordinates kept; Lattice.volume =
  |(a x b) . c|.

Statuses, as the kernel's: 0 ok; 1 V0 not strictly inside (min V, max V) (ASE's warning, parameters kept); 2 no fit
(a curve_fit raises, or the seed is not finite); 3 bad input (a volume not finite and > 0 or an energy not finite).
"""
from __future__ import annotations

import warnings

import numpy as np
from scipy.optimize import curve_fit, least_squares

_e = 1.6021766208e-19
J = 1 / _e
kJ = 1000 * J

OK, OUTSIDE, NO_FIT, BAD_INPUT = 0, 1, 2, 3
FORMS = ("murnaghan", "birchmurnaghan", "vinet")


def parabola(x, a, b, c):
    return a + b * x + c * x**2


def murnaghan(V, E0, B0, BP, V0):
    return E0 + B0 * V / BP * (((V0 / V)**BP) / (BP - 1) + 1) - V0 * B0 / (BP - 1.)


def birchmurnaghan(V, E0, B0, BP, V0):
    eta = (V0 / V)**(1 / 3)
    return E0 + 9 * B0 * V0 / 16 * (eta**2 - 1)**2 * (6 + BP * (eta**2 - 1.) - 4 * eta**2)


def vinet(V, E0, B0, BP, V0):
    eta = (V / V0)**(1 / 3)
    return (E0 + 2 * B0 * V0 / (BP - 1)**2 * (2 - (5 + 3 * BP * (eta - 1) - 3 * eta) *
                                              np.exp(-3 * (BP - 1) * (eta - 1) / 2)))


FUNCS = {"murnaghan": murnaghan, "birchmurnaghan": birchmurnaghan, "vinet": vinet}


def gpa(B):
    """The reference's kv = B / kJ * 1.0e24, B in eV/A^3."""
    return B / kJ * 1.0e24


def _seed_from(a, b, c):
    vmin = -b / 2 / c
    return np.array([parabola(vmin, a, b, c), 2 * c * vmin, 4.0, vmin])


def ase_seed(v, e):
    """EquationOfState.fit's initial guess, from curve_fit(parabola, v, e, [min(e), 1, 1])."""
    v, e = np.asarray(v, dtype=np.float64), np.asarray(e, dtype=np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                      # OptimizeWarning: covariance not estimated
        popt, _ = curve_fit(parabola, v, e, [min(e), 1, 1])
    return _seed_from(popt[0], popt[1], popt[2])


def lsq_seed(v, e):
    """The same seed from the exact least-squares parabola, solved in t = (V - mean) / (half range) (the raw
    Vandermonde is badly conditioned) and mapped back to a + b V + c V^2."""
    v, e = np.asarray(v, dtype=np.float64), np.asarray(e, dtype=np.float64)
    vm, h = v.mean(), 0.5 * (v.max() - v.min())
    t = (v - vm) / h
    al, be, ga = np.linalg.lstsq(np.stack([np.ones_like(t), t, t * t], 1), e, rcond=None)[0]
    c = ga / h**2
    b = be / h - 2 * c * vm
    a = al - be * vm / h + c * vm * vm
    return _seed_from(a, b, c)


def ase_fit(v, e, eos="murnaghan"):
    """ASE 3.22.1's EquationOfState(v, e, eos).fit() restated: (params [E0, B0, BP, V0], status 0 or 1).  Raises
    what curve_fit raises (TypeError for fewer points than parameters, RuntimeError without convergence)."""
    v, e = np.asarray(v, dtype=np.float64), np.asarray(e, dtype=np.float64)
    p0 = ase_seed(v, e)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                      # OptimizeWarning: covariance not estimated
        popt, _ = curve_fit(FUNCS[eos], v, e, p0)
    return popt, (OK if min(v) < popt[3] < max(v) else OUTSIDE)


def tight_fit(v, e, eos="murnaghan", seed=None):
    """The fully converged least-squares optimum from the seed: least_squares(method="lm", xtol=ftol=gtol=1e-15).
    (params, status 0 or 1)."""
    v, e = np.asarray(v, dtype=np.float64), np.asarray(e, dtype=np.float64)
    p0 = lsq_seed(v, e) if seed is None else seed
    f = FUNCS[eos]
    with np.errstate(all="ignore"):
        res = least_squares(lambda p: f(v, *p) - e, p0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    if not res.success:
        raise RuntimeError(f"least_squares: {res.message}")
    return res.x, (OK if v.min() < res.x[3] < v.max() else OUTSIDE)


def fit_rows(volumes, energies, eos="murnaghan", fit=ase_fit):
    """`fit` on every row of [R, S] arrays with the kernel's statuses: (params [R, 4] NaN for statuses 2 and 3,
    status [R])."""
    V, E = np.asarray(volumes, dtype=np.float64), np.asarray(energies, dtype=np.float64)
    params = np.full((V.shape[0], 4), np.nan)
    status = np.zeros(V.shape[0], dtype=np.int32)
    for r in range(V.shape[0]):
        if not (np.isfinite(V[r]).all() and (V[r] > 0).all() and np.isfinite(E[r]).all()):
            status[r] = BAD_INPUT
            continue
        try:
            with np.errstate(all="ignore"):
                seed = lsq_seed(V[r], E[r])
                if not np.isfinite(seed).all():
                    raise RuntimeError("no finite seed")
                p, status[r] = fit(V[r], E[r], eos)
            if not np.isfinite(p).all():
                raise RuntimeError("no finite fit")
            params[r] = p
        except (RuntimeError, ValueError, np.linalg.LinAlgError):
            status[r] = NO_FIT
    return params, status


def strain_atoms(lattice, cart, strain):
    """jarvis' strain_atoms(strain): (I + strain I) @ lattice, the fractional coordinates kept -> (lattice, cart)."""
    lat0 = np.asarray(lattice, dtype=np.float64)
    s = np.eye(3) + np.array(strain) * np.eye(3)
    lat = np.dot(s, lat0)
    frac = np.dot(np.asarray(cart, dtype=np.float64), np.linalg.inv(lat0))
    return lat, np.dot(frac, lat)


def volume(lattice):
    """jarvis' Lattice.volume: |(a x b) . c|."""
    m = np.asarray(lattice, dtype=np.float64)
    return float(abs(np.dot(np.cross(m[0], m[1]), m[2])))


def random_rows(eos, R, S, seed=0):
    """R test curves of S points in the regime ev_curve produces: V0 log-uniform in [10, 2000] A^3, B0 in
    [0.05, 2] eV/A^3, BP in [3, 6], E0 in [-5, 0] eV per 15 A^3, volumes (1 + strain)^3 V0 for S strains evenly over
    [-0.05, 0.04] times a per-row factor in [0.97, 1.03], energies of the exact curve rounded to fp32 (as the model's
    energies are).  Returns (volumes [R, S], energies [R, S], true params [R, 4])."""
    rng = np.random.default_rng(seed)
    V0 = np.exp(rng.uniform(np.log(10), np.log(2000), R))
    p = np.stack([rng.uniform(-5, 0, R) * V0 / 15, rng.uniform(0.05, 2, R), rng.uniform(3, 6, R), V0], 1)
    V = V0[:, None] * (1 + np.linspace(-0.05, 0.04, S))[None, :] ** 3 * rng.uniform(0.97, 1.03, R)[:, None]
    E = FUNCS[eos](V, *[p[:, k:k + 1] for k in range(4)]).astype(np.float32).astype(np.float64)
    return V, E, p
