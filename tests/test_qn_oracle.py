"""CPU: the quasi-Newton restatement `oracle/qn_oracle.py` -- the two-loop recursion against an explicit inverse-BFGS
matrix, LBFGS against BFGS on strictly convex problems (the direct and inverse updates are dual, and |H|^-1 = H^-1
while H stays positive definite), BFGS's skipped update and its |omega| on an indefinite H, the strained FCC spring
cell relaxed to its ideal geometry under the filter, the batched driver against one-by-one runs, and the C layouts of
the parameter structs."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from alignn_b200 import _lib
from oracle import qn_oracle as QN
from tests.test_cell_filter_oracle import _fcc_cell, _fcc_springs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pairs(rng, n, count):
    """Rows r_k with forces f_k = -A r_k for a random SPD A: every pair has y.s = s^T A s > 0."""
    M = rng.normal(size=(3 * n, 3 * n))
    A = M @ M.T + 3 * n * np.eye(3 * n)
    rs = [rng.normal(size=(n, 3)) for _ in range(count)]
    return A, rs, [-(A @ r.ravel()).reshape(n, 3) for r in rs]


def _inverse_bfgs(pairs, alpha):
    n = len(pairs[0][0])
    Hi = np.eye(n) / alpha
    for s, y in pairs:
        rho = 1.0 / np.dot(y, s)
        V = np.eye(n) - rho * np.outer(y, s)
        Hi = V.T @ Hi @ V + rho * np.outer(s, s)
    return Hi


@pytest.mark.parametrize("memory", [100, 3])
def test_two_loop_equals_dense_inverse_bfgs(memory):
    rng = np.random.default_rng(0)
    n, count = 4, 7
    A, rs, fs = _pairs(rng, n, count)
    opt = QN.LBFGS(memory=memory, maxstep=1e9)
    for r, f in zip(rs[:-1], fs[:-1]):
        opt.step(r, f)
    r, f = rs[-1], fs[-1]
    got = opt.step(r, f) - r
    pairs = [((rs[k + 1] - rs[k]).ravel(), (fs[k] - fs[k + 1]).ravel()) for k in range(count - 1)]
    assert len(opt.s) == min(memory, count - 1)
    want = (_inverse_bfgs(pairs[-memory:], 70.0) @ f.ravel()).reshape(n, 3)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def _quadratic(n=3, seed=1):
    rng = np.random.default_rng(seed)
    M = rng.normal(size=(3 * n, 3 * n))
    A = 0.05 * (M @ M.T) + 0.5 * np.eye(3 * n)
    xs = rng.normal(size=(n, 3))

    def evaluate(x):
        d = (x - xs).ravel()
        return 0.5 * d @ A @ d, (-(A @ d)).reshape(n, 3).astype(np.float32)
    return evaluate, xs + rng.normal(scale=0.3, size=(n, 3))


def test_lbfgs_and_bfgs_follow_one_trajectory_on_an_spd_quadratic():
    evaluate, x0 = _quadratic()
    a = QN.relax("LBFGS", evaluate, x0, fmax=1e-4, steps=15)
    b = QN.relax("BFGS", evaluate, x0, fmax=1e-4, steps=15)
    assert a["nsteps"] == b["nsteps"] and a["nsteps"] > 3
    assert np.abs(a["positions"] - b["positions"]).max() <= 1e-9


@pytest.mark.parametrize("optimize_lattice", [False, True])
def test_lbfgs_and_bfgs_agree_on_the_fcc_springs_crystal(optimize_lattice):
    evaluate = _fcc_springs(2.5)
    cell = _fcc_cell(2.5, [[1.03, 0.02, 0.0], [0.0, 1.02, -0.01], [0.01, 0.0, 1.03]])
    X = np.array([[0.0, 0.0, 0.0], [0.1, 1.2, 1.3]]) @ np.eye(3)
    X = np.concatenate([X, X[:1] + cell[0] * 0.5 + 0.05])
    if optimize_lattice:
        a = QN.relax_cell("LBFGS", evaluate, cell, X, fmax=0.0, steps=6)
        b = QN.relax_cell("BFGS", evaluate, cell, X, fmax=0.0, steps=6)
        assert np.abs(a["cell"] - b["cell"]).max() <= 1e-9
    else:
        ev = lambda x: evaluate(cell, x)[:2]                               # noqa: E731
        a = QN.relax("LBFGS", ev, X, fmax=0.0, steps=6)
        b = QN.relax("BFGS", ev, X, fmax=0.0, steps=6)
    assert np.abs(a["positions"] - b["positions"]).max() <= 1e-9


def test_bfgs_skips_a_repeated_configuration_and_steps_along_abs_omega():
    opt = QN.BFGS(1)
    r, f = np.zeros((1, 3)), np.array([[0.1, -0.2, 0.05]])
    opt.step(r, f)
    H = opt.H.copy()
    opt.step(opt.r0.reshape(1, 3) + 5e-8, f * 0.5)                 # |dr| < 1e-7: no update
    assert np.array_equal(opt.H, H)
    opt.H = np.diag([-2.0, 70.0, 4.0])                              # indefinite: the step uses |omega|
    opt.r0 = None
    opt.update = lambda r, f: None
    x = opt.step(np.zeros((1, 3)), f)
    assert np.allclose(x, f / np.array([2.0, 70.0, 4.0]), rtol=1e-14, atol=0)


@pytest.mark.parametrize("optimizer", ["LBFGS", "BFGS"])
def test_fcc_springs_relax_to_the_ideal_cell(optimizer):
    r0 = 2.5
    evaluate = _fcc_springs(r0)
    cell = _fcc_cell(r0, [[1.04, 0.03, 0.0], [0.0, 1.04, -0.02], [0.01, 0.0, 1.04]])
    res = QN.relax_cell(optimizer, evaluate, cell, np.zeros((1, 3)), fmax=1e-6, steps=500)
    assert res["converged"], res["nsteps"]
    C = res["cell"]
    d = np.array([np.linalg.norm(v) for v in (C[0], C[1], C[2], C[0] - C[1], C[0] - C[2], C[1] - C[2])])
    assert np.abs(d - r0).max() <= 1e-5, d
    assert abs(abs(np.linalg.det(C)) - r0 ** 3 / np.sqrt(2.0)) <= 1e-5 * r0 ** 3


@pytest.mark.parametrize("optimizer", ["LBFGS", "BFGS"])
@pytest.mark.parametrize("optimize_lattice", [False, True])
def test_batched_oracle_equals_one_by_one(optimizer, optimize_lattice):
    springs = _fcc_springs()
    crystals = [(_fcc_cell(2.5, np.diag([1.04, 1.0, 0.98]) + 0.02), np.zeros((1, 3))),
                (_fcc_cell(2.5, np.eye(3) * 1.06), np.zeros((1, 3))),
                (_fcc_cell(2.5, np.eye(3) * 1.01 + 0.01), np.zeros((1, 3)))]
    if not optimize_lattice:
        crystals = [(c, np.array([[0.0, 0.0, 0.0], [0.3, 0.2, 0.1]]) @ c + 0.7 * c[0]) for c, _ in crystals]
    kw = dict(fmax=1e-3, steps=30, force_multiplier=1.5, memory=5) if optimizer == "LBFGS" else \
        dict(fmax=1e-3, steps=30, force_multiplier=1.5)
    if optimize_lattice:
        alone = [QN.relax_cell(optimizer, springs, c, x, stress_wt=0.9, **kw) for c, x in crystals]

        def evaluate_batch(ids, cx):
            return [springs(c, x) for c, x in cx]
        bat = QN.relax_batch(optimizer, evaluate_batch, crystals, optimize_lattice=True, stress_wt=0.9, **kw)
    else:
        alone = [QN.relax(optimizer, lambda x, c=c: springs(c, x)[:2], x, **kw) for c, x in crystals]

        def evaluate_batch(ids, xs):
            return [springs(crystals[b][0], x)[:2] for b, x in zip(ids, xs)]
        bat = QN.relax_batch(optimizer, evaluate_batch, [x for _, x in crystals], **kw)
    assert len({r["nsteps"] for r in alone}) > 1
    for b, r in enumerate(alone):
        assert bat["nsteps"][b] == r["nsteps"] and bat["converged"][b] == r["converged"]
        assert np.array_equal(bat["positions"][b], r["positions"]) and np.array_equal(bat["forces"][b], r["forces"])
        if optimize_lattice:
            assert np.array_equal(bat["cell"][b], r["cell"])


def _layout(tmp_path, ctype, cls):
    fields = [f for f, _ in cls._fields_]
    src = tmp_path / "qn.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\nint main(){printf("%zu'
                   + " %zu" * len(fields) + f'\\n", sizeof({ctype})'
                   + "".join(f", offsetof({ctype}, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "qn"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f in fields]


def test_lbfgs_params_struct_matches_c_layout(tmp_path):
    _layout(tmp_path, "alignn_b200_lbfgs_params", _lib.LbfgsParams)


def test_bfgs_params_struct_matches_c_layout(tmp_path):
    _layout(tmp_path, "alignn_b200_bfgs_params", _lib.BfgsParams)
