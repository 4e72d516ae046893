"""CPU: the stochastic-thermostat restatement `oracle/md_thermostat_oracle.py` (ASE 3.22.1 `Langevin` and `Andersen`,
fixcm=True, on the counter-based stream of csrc/md_noise.cuh): Philox4x32-10 against Random123's known answers, the
uniforms' range, both thermostats against velocity Verlet with their coupling off, conserved zero momentum, an FCC
spring crystal thermalised from 50 K, Andersen's reassignment rate, the batched driver against one-by-one runs, and
the C layout and register report of the kernel."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from alignn_b200 import _lib, md, ops
from oracle import md_oracle as MO
from oracle import md_thermostat_oracle as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "alignn_b200", "csrc")


def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10."""
    cases = [([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
             ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
             ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
              [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for ctr, key, want in cases:
        assert TO.philox4x32_10(ctr, key).tolist() == want
    batch = TO.philox4x32_10([c for c, _, _ in cases], [k for _, k, _ in cases])     # vectorised: row by row
    assert batch.tolist() == [w for _, _, w in cases]


def test_uniforms_lie_strictly_inside_the_unit_interval():
    lo, hi = TO.unit_uniform(0, 0), TO.unit_uniform(0xffffffff, 0xffffffff)
    assert lo == 2.0 ** -53 and hi == 1.0 - 2.0 ** -53 and 0.0 < lo and hi < 1.0 and 1.0 - hi == 2.0 ** -53
    assert TO.unit_uniform(0, 0xfff) == lo                                     # the low 12 bits of lo are dropped
    w, u, z = TO.noise_blocks(2 ** 64 - 1, np.arange(4096), 7, 5, TO.TAG[TO.ANDERSEN])
    assert w.dtype == np.uint32 and u.shape == (4096, 5, 2) and z.shape == (4096, 5, 2)
    assert (u > 0).all() and (u < 1).all() and np.isfinite(np.log(1 - u)).all()
    assert abs(u.mean() - 0.5) < 0.01 and abs(z.mean()) < 0.02 and abs(z.std() - 1.0) < 0.02
    k = u * 2.0 ** 52 - 0.5                                                     # integers below 2^52
    assert np.array_equal(k, np.floor(k)) and k.max() < 2 ** 52


def test_streams_depend_on_every_counter_word_and_the_key():
    base = TO.noise_blocks(5, [0, 1], 3, 2, 2)[0]
    for other in (TO.noise_blocks(6, [0, 1], 3, 2, 2), TO.noise_blocks(5 + 2 ** 32, [0, 1], 3, 2, 2),
                  TO.noise_blocks(5, [2, 3], 3, 2, 2), TO.noise_blocks(5, [0, 1], 4, 2, 2),
                  TO.noise_blocks(5, [0, 1], 3, 2, 3)):
        assert not (other[0] == base).any()
    xi, eta = TO.PhiloxNoise(5).langevin(3, 4)
    assert not np.array_equal(xi, eta)
    cx, cy, x, y, c = TO.PhiloxNoise(5).andersen(3, 4)
    assert cx.shape == cy.shape == (3,) and x.shape == y.shape == c.shape == (4, 3)
    assert not np.isin(cx, x).any()                                           # the centre-of-mass atom word differs


def _pairs(n_pairs=6, k=1.5, seed=0):
    """Dimers on springs of rest length 1 around the origin; each pair's fp32 forces are exact negatives, so every
    crystal's forces sum to zero."""
    rng = np.random.default_rng(seed)
    a = rng.normal(size=(n_pairs, 3))
    d = rng.normal(size=(n_pairs, 3))
    X = np.concatenate([a - 0.5 * d, a + 0.5 * d])

    def evaluate(x):
        x = np.asarray(x)
        dd = x[n_pairs:] - x[:n_pairs]
        r = np.linalg.norm(dd, axis=1, keepdims=True)
        f = (k * (r - 1.0) / r * dd).astype(np.float32)                   # force on the first atom of each pair
        return 0.5 * k * float(((r - 1.0) ** 2).sum()), np.concatenate([f, -f])
    return X, evaluate


def _zero_momentum(m, T, seed):
    p = MO.maxwell_boltzmann_momenta(m, T, np.random.default_rng(seed))
    return p - p.sum(axis=0) / len(m)


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_uncoupled_thermostats_are_velocity_verlet(ensemble):
    """friction 0 (Langevin) or prob 0 (Andersen): the noise terms vanish and what remains is Verlet up to the
    rounding of v = (x_new - x) / dt and of the centre-of-mass corrections."""
    X, evaluate = _pairs()
    m = np.random.default_rng(1).uniform(1.0, 60.0, len(X))
    p0 = _zero_momentum(m, 300.0, 2)
    dt, steps = 2.0 * MO.fs, 40
    ref = MO.run(evaluate, X, m, steps=steps, dt=dt, momenta=p0)
    got = TO.run(evaluate, X, m, ensemble=ensemble, steps=steps, dt=dt, temperature_K=300.0, noise=TO.PhiloxNoise(9),
                 friction=0.0, andersen_prob=0.0, momenta=p0)
    assert _rel(got["positions"], ref["positions"]) <= 1e-12
    assert _rel(got["momenta"], ref["momenta"]) <= 1e-12
    assert _rel(got["kinetic_energy"], ref["kinetic_energy"]) <= 1e-12
    assert np.array_equal(got["forces"], ref["forces"]) or _rel(got["forces"], ref["forces"]) <= 1e-6
    assert got["md"].reassigned == 0


@pytest.mark.parametrize("ensemble,noise", [(TO.LANGEVIN, "philox"), (TO.ANDERSEN, "philox"), (TO.LANGEVIN, "numpy"),
                                            (TO.ANDERSEN, "numpy")])
def test_zero_total_momentum_stays_zero(ensemble, noise):
    X, evaluate = _pairs()
    m = np.random.default_rng(3).uniform(1.0, 60.0, len(X))
    src = TO.PhiloxNoise(11) if noise == "philox" else TO.NumpyNoise(np.random.default_rng(11))
    md_ = TO.Thermostat(X, m, ensemble=ensemble, dt=2.0 * MO.fs, temperature_K=500.0, noise=src,
                        friction=0.05 / MO.fs, andersen_prob=0.2, momenta=_zero_momentum(m, 300.0, 4))
    f = evaluate(md_.x)[1].astype(np.float64)
    for _ in range(100):
        md_.first_half(f)
        f = evaluate(md_.x)[1].astype(np.float64)
        md_.second_half(f)
        assert np.abs(md_.p.sum(axis=0)).max() <= 1e-10 * np.abs(md_.p).sum()


def _fcc_springs_crystal(reps=2, r0=2.55, k=1.0):
    """test_md_oracle's FCC nearest-neighbour spring crystal (32 atoms, minimum image in the fixed supercell)."""
    a = r0 * np.sqrt(2.0)
    basis = np.array([[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]])
    cells = np.stack(np.meshgrid(*[np.arange(reps)] * 3, indexing="ij"), -1).reshape(-1, 3)
    X = ((cells[:, None, :] + basis[None]) * a).reshape(-1, 3)
    L = reps * a
    d = X[None, :, :] - X[:, None, :]
    d -= L * np.round(d / L)
    r = np.linalg.norm(d, axis=2)
    i, j = np.nonzero(np.abs(r - r0) < 1e-6)

    def evaluate(x):
        dd = x[j] - x[i]
        dd -= L * np.round(dd / L)
        rr = np.linalg.norm(dd, axis=1)
        F = np.zeros_like(x)
        np.add.at(F, i, (k * (rr - r0) / rr)[:, None] * dd)
        return 0.25 * k * float(((rr - r0) ** 2).sum()), F.astype(np.float32)
    return X, evaluate


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_thermostat_brings_an_fcc_spring_crystal_to_its_target_temperature(ensemble):
    """From 50 K towards T0 = 300 K, with a friction of 0.01/fs (Langevin) or a reassignment probability of 2 % per
    component and step (Andersen): the late temperature averages within 10 % of T0."""
    X, evaluate = _fcc_springs_crystal()
    m = np.full(len(X), 63.546)
    p0 = MO.maxwell_boltzmann_momenta(m, 50.0, np.random.default_rng(0))
    res = TO.run(evaluate, X, m, ensemble=ensemble, steps=1500, dt=2.0 * MO.fs, temperature_K=300.0,
                 noise=TO.PhiloxNoise(2024), friction=0.01 / MO.fs, andersen_prob=0.02, momenta=p0)
    T = np.array(res["temperature"])
    assert T[0] < 100.0
    late = T[-700:].mean()
    assert abs(late - 300.0) <= 30.0, late


def test_andersen_reassigns_at_its_probability():
    X, evaluate = _pairs(n_pairs=16)
    m = np.full(len(X), 12.0)
    prob, steps = 0.1, 400
    res = TO.run(evaluate, X, m, ensemble=TO.ANDERSEN, steps=steps, dt=1.0 * MO.fs, temperature_K=300.0,
                 noise=TO.PhiloxNoise(77), andersen_prob=prob)
    trials = steps * len(X) * 3
    mean, sd = prob * trials, np.sqrt(trials * prob * (1 - prob))
    assert abs(res["md"].reassigned - mean) <= 5 * sd, (res["md"].reassigned, mean, sd)
    one = TO.run(evaluate, X, m, ensemble=TO.ANDERSEN, steps=20, dt=1.0 * MO.fs, temperature_K=300.0,
                 noise=TO.PhiloxNoise(77), andersen_prob=1.0)
    assert one["md"].reassigned == 20 * len(X) * 3                              # chance <= 1 always


def test_numpy_noise_makes_ases_draws_in_order():
    rng = np.random.default_rng(5)
    xi, eta = TO.NumpyNoise(np.random.default_rng(5)).langevin(0, 4)
    assert np.array_equal(xi, rng.standard_normal((4, 3))) and np.array_equal(eta, rng.standard_normal((4, 3)))
    np.random.seed(3)
    got = TO.NumpyNoise().andersen(0, 2)
    np.random.seed(3)
    want = [np.random.uniform(size=3), np.random.uniform(size=3), np.random.uniform(size=(2, 3)),
            np.random.uniform(size=(2, 3)), np.random.random((2, 3))]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_one_atom_langevin_is_rejected():
    with pytest.raises(ValueError, match="two atoms"):
        TO.Thermostat(np.zeros((1, 3)), [12.0], ensemble=TO.LANGEVIN, dt=0.1, temperature_K=300.0,
                      noise=TO.PhiloxNoise(0), friction=0.01)
    TO.Thermostat(np.zeros((1, 3)), [12.0], ensemble=TO.ANDERSEN, dt=0.1, temperature_K=300.0,
                  noise=TO.PhiloxNoise(0), andersen_prob=0.1)


def _analytic_crystals():
    rng = np.random.default_rng(5)
    out = []
    for n in [2, 3, 7, 5]:
        centre = rng.normal(size=(n, 3))
        k = 0.5 + 3.0 * rng.random((n, 3))
        x0 = centre + rng.normal(scale=0.4, size=(n, 3))
        m = rng.uniform(1.0, 200.0, n)

        def evaluate(x, centre=centre, k=k):
            d = np.asarray(x) - centre
            return float((0.5 * k * d ** 2 + 0.25 * d ** 4).sum()), (-(k * d + d ** 3)).astype(np.float32)
        out.append((x0, m, evaluate, MO.maxwell_boltzmann_momenta(m, 400.0, rng)))
    return out


@pytest.mark.parametrize("ensemble", [TO.LANGEVIN, TO.ANDERSEN])
def test_batched_oracle_equals_one_by_one_bitwise(ensemble):
    crystals = _analytic_crystals()
    T0 = [100.0, 300.0, 500.0, 1000.0]
    mom = [p if b != 2 else None for b, (_, _, _, p) in enumerate(crystals)]
    kw = dict(ensemble=ensemble, steps=30, dt=0.05, friction=0.3, andersen_prob=0.3, force_multiplier=1.5,
              trajectory_interval=4)
    alone = [TO.run(ev, x0, m, temperature_K=T0[b], momenta=mom[b], noise=TO.PhiloxNoise(40 + b), **kw)
             for b, (x0, m, ev, _) in enumerate(crystals)]
    bat = TO.run_batch(lambda xs: [crystals[b][2](x) for b, x in enumerate(xs)], [c[0] for c in crystals],
                       [c[1] for c in crystals], temperature_K=T0, momenta=mom,
                       noises=[TO.PhiloxNoise(40 + b) for b in range(len(crystals))], **kw)
    for r, q in zip(alone, bat):
        for key in ("positions", "momenta", "forces"):
            assert np.array_equal(r[key], q[key]), key
        for key in ("energy", "kinetic_energy", "temperature"):
            assert r[key] == q[key], key
        assert len(r["trajectory"]) == 8 and all(np.array_equal(a, b) for a, b in zip(r["trajectory"], q["trajectory"]))


def test_run_md_constants():
    assert md.LANGEVIN_FRICTION == 1e-4                                        # ff.py:450, in ASE units
    assert md.ENSEMBLES["nvt_langevin"] == ops.MD_NVT_LANGEVIN == TO.TAG[TO.LANGEVIN]
    assert md.ENSEMBLES["nvt_andersen"] == ops.MD_NVT_ANDERSEN == TO.TAG[TO.ANDERSEN]


def test_md_thermostat_params_struct_matches_c_layout(tmp_path):
    S = _lib.MdThermostatParams
    fields = [f for f, _ in S._fields_]
    src = tmp_path / "tp.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\nint main(){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(alignn_b200_md_thermostat_params)'
                   + "".join(f", offsetof(alignn_b200_md_thermostat_params, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "tp"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in fields]


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_md_thermostat_kernel_does_not_spill(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "md_device.cubin"),
           os.path.join(CSRC, "md_device.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    report, current = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current is not None:
            report[current] = tuple(int(v) for v in m.groups())
            current = None
    for name in ("md_thermostat_kernel", "md_noise_kernel"):
        hit = [v for n, v in report.items() if name in n]
        assert hit == [(0, 0, 0)], (name, report)
