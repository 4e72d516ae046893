"""CPU: the FIRE restatement `oracle/fire_oracle.py` (ASE 3.22.1 `FIRE.step` and `Dynamics.irun`) against steps worked
by hand on a 1-atom harmonic well, the batched oracle loop against the same crystals relaxed one by one, and the C
layout of the kernel's parameter struct."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from alignn_b200 import _lib
from oracle import fire_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _well(k=1.0, centre=(0.0, 0.0, 0.0)):
    """E = k/2 |x - c|^2 per atom; the 'grad' a model returns is the force -k (x - c), in fp32."""
    c = np.asarray(centre, dtype=np.float64)

    def evaluate(x):
        d = np.asarray(x, dtype=np.float64) - c
        return 0.5 * k * float((d ** 2).sum()), (-k * d).astype(np.float32)
    return evaluate


def test_first_step_only_zeroes_v():
    opt = FO.Fire([[1.0, 0.0, 0.0]])
    f = np.array([[-1.0, 0.0, 0.0]])
    opt.step(f)
    # v = 0 (no mix, no reset: dt and a unchanged), v += dt f, dr = dt v
    assert opt.dt == 0.1 and opt.a == 0.1 and opt.Nsteps == 0
    v = 0.1 * -1.0
    assert opt.v.tolist() == [[v, 0.0, 0.0]]
    assert opt.x.tolist() == [[1.0 + 0.1 * v, 0.0, 0.0]]
    # the same step through the run loop on the well E = |x|^2 / 2: two evaluations, the second at the moved atom
    res = FO.relax(_well(), [[1.0, 0.0, 0.0]], fmax=0.0, steps=1)
    assert res["nsteps"] == 1 and res["evaluations"] == 2 and not res["converged"]
    assert res["positions"].tolist() == [[1.0 + 0.1 * v, 0.0, 0.0]]
    assert res["forces"].tolist() == [[float(np.float32(-(1.0 + 0.1 * v))), 0.0, 0.0]]
    assert res["energy"] == 0.5 * (1.0 + 0.1 * v) ** 2


def test_downhill_mix_and_dt_growth_after_nmin_clipped_at_dtmax():
    opt = FO.Fire([[0.0, 0.0, 0.0]], maxstep=1e9)
    f = np.array([[1.0, 0.0, 0.0]])
    dts, as_, ns = [], [], []
    for _ in range(40):
        opt.step(f)
        dts.append(opt.dt)
        as_.append(opt.a)
        ns.append(opt.Nsteps)
    # step 1 sets v = 0; from step 2 on vf > 0 and Nsteps counts 1, 2, ...; dt and a change only once Nsteps > Nmin = 5
    # before the step, i.e. from step 8 on
    assert ns[:9] == [0, 1, 2, 3, 4, 5, 6, 7, 8]
    assert dts[:7] == [0.1] * 7 and as_[:7] == [0.1] * 7
    dt, a = 0.1, 0.1
    want_dt, want_a = [0.1] * 7, [0.1] * 7
    for _ in range(7, 40):
        dt, a = min(dt * 1.1, 1.0), a * 0.99
        want_dt.append(dt)
        want_a.append(a)
    assert dts == want_dt and as_ == want_a
    assert dts[-1] == 1.0 and dts[30] < 1.0 and dts[31] == 1.0          # 0.1 * 1.1^24 < 1 < 0.1 * 1.1^25
    # a force parallel to v leaves the mix at |v|: v_n = v_{n-1} + dt f exactly as without mixing, in 1-D
    v = opt.v[0, 0]
    assert v > 0 and opt.v[0, 1:].tolist() == [0.0, 0.0]


def test_uphill_reset():
    opt = FO.Fire([[0.0, 0.0, 0.0]])
    for _ in range(9):
        opt.step(np.array([[1.0, 0.0, 0.0]]))
    dt_before = opt.dt
    assert opt.Nsteps == 8 and dt_before > 0.1
    opt.step(np.array([[-2.0, 0.0, 0.0]]))                              # vf < 0
    assert opt.a == 0.1 and opt.Nsteps == 0 and opt.dt == dt_before * 0.5
    assert opt.v.tolist() == [[(dt_before * 0.5) * -2.0, 0.0, 0.0]]     # v = 0, then v += dt f


def test_maxstep_caps_the_whole_crystal():
    opt = FO.Fire([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]])
    opt.step(np.array([[30.0, 0.0, 0.0], [0.0, 40.0, 0.0]]))
    # v = dt f = (3, 4); dr = dt v = (0.3, 0.4), |dr| = 0.5 over the crystal > 0.2: both atoms scaled by 0.2 / 0.5
    dr = np.array([[0.1 * (0.1 * 30.0), 0, 0], [0, 0.1 * (0.1 * 40.0), 0]])
    norm = np.sqrt(np.vdot(dr, dr))
    assert norm > 0.2
    np.testing.assert_array_equal(opt.x, np.array([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]]) + 0.2 * dr / norm)
    step = opt.x - np.array([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]])
    assert np.linalg.norm(step[0]) < 0.2 and np.linalg.norm(step[1]) < 0.2   # a per-atom cap would not have moved them


def test_convergence_is_strict():
    assert not FO.converged(np.array([[0.5, 0.0, 0.0]]), 0.5)
    assert FO.converged(np.array([[np.nextafter(0.5, 0.0), 0.0, 0.0]]), 0.5)
    assert not FO.converged(np.array([[0.0, 0.0, 0.0], [0.3, 0.4, 0.0]]), 0.5)
    assert not FO.converged(np.array([[np.nan, 0.0, 0.0]]), 0.5)


def test_steps_plus_one_evaluations_when_not_converged():
    calls = []

    def constant(x):
        calls.append(np.array(x))
        return 0.0, np.array([[0.5, 0.0, 0.0]], dtype=np.float32)
    res = FO.relax(constant, [[0.0, 0.0, 0.0]], fmax=0.5, steps=3)       # |F| == fmax never converges
    assert res["nsteps"] == 3 and res["evaluations"] == 4 and len(calls) == 4 and not res["converged"]
    res = FO.relax(constant, [[0.0, 0.0, 0.0]], fmax=0.6, steps=3)
    assert res["nsteps"] == 0 and res["evaluations"] == 1 and res["converged"]
    with pytest.raises(ValueError):
        FO.relax(constant, [[0.0, 0.0, 0.0]], steps=0)


def test_force_multiplier_is_one_fp32_product():
    g = np.array([[0.1, -0.2, 0.3]], dtype=np.float32)
    f = FO.scaled_forces(g, 64 * 1.5)
    assert f.dtype == np.float32
    np.testing.assert_array_equal(f, g * np.float32(96.0))


def _analytic_crystals():
    """Crystals of 1..7 atoms in anisotropic quartic wells: different convergence times, some never within the limit."""
    rng = np.random.default_rng(5)
    out = []
    for b, n in enumerate([1, 3, 2, 7, 1, 5]):
        centre = rng.normal(size=(n, 3))
        k = 0.5 + 3.0 * rng.random((n, 3))
        x0 = centre + rng.normal(scale=0.6, size=(n, 3))

        def evaluate(x, centre=centre, k=k):
            d = np.asarray(x) - centre
            return float((0.5 * k * d ** 2 + 0.25 * d ** 4).sum()), (-(k * d + d ** 3)).astype(np.float32)
        out.append((x0, evaluate))
    return out


def test_batched_oracle_equals_one_by_one_bitwise():
    crystals = _analytic_crystals()
    fmax, steps, mult = 0.05, 38, 1.5
    alone = [FO.relax(ev, x0, fmax=fmax, steps=steps, force_multiplier=mult) for x0, ev in crystals]
    assert any(r["converged"] for r in alone) and not all(r["converged"] for r in alone)
    assert len({r["nsteps"] for r in alone}) > 2

    def evaluate_batch(ids, xs):
        return [crystals[b][1](x) for b, x in zip(ids, xs)]
    bat = FO.relax_batch(evaluate_batch, [x0 for x0, _ in crystals], fmax=fmax, steps=steps, force_multiplier=mult)
    for b, r in enumerate(alone):
        assert bat["nsteps"][b] == r["nsteps"] and bat["converged"][b] == r["converged"]
        assert bat["evaluations"][b] == r["evaluations"]
        assert np.array_equal(bat["positions"][b], r["positions"])
        assert np.array_equal(bat["forces"][b], r["forces"]) and bat["energy"][b] == r["energy"]
        assert bat["fire"][b].dt == r["fire"].dt and bat["fire"][b].a == r["fire"].a
        assert np.array_equal(bat["fire"][b].v, r["fire"].v)


def test_fire_params_struct_matches_c_layout(tmp_path):
    fields = [f for f, _ in _lib.FireParams._fields_]
    src = tmp_path / "fp.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\nint main(){printf("%zu'
                   + " %zu" * len(fields) + '\\n", sizeof(alignn_b200_fire_params)'
                   + "".join(f", offsetof(alignn_b200_fire_params, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "fp"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(_lib.FireParams)] + [getattr(_lib.FireParams, f).offset for f in fields]
