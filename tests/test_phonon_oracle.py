"""CPU: oracle/phonon_oracle.py, the numpy restatement of ASE 3.22.1's finite-displacement `Phonons` that
`alignn_b200.phonons` is tested against: supercell order, lattice vectors, harmonic spring crystals against their
analytic dispersions, the acoustic sum rule, Hermitian symmetry, negative frequencies, the DOS grid, the batched oracle,
and the package's displaced-supercell builder against the oracle's."""
import itertools
import math

import numpy as np
import pytest

from alignn_b200.phonons import displaced_supercells as pkg_displaced_supercells
from alignn_b200.phonons import EV_PER_SQRT_EV_A2_AMU
from alignn_b200.phonons import monkhorst_pack as pkg_monkhorst_pack
from oracle import phonon_oracle as PO


# ---- supercell order and lattice vectors ------------------------------------------------------------------------------
CELLS_222 = [(0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]
R_222 = [(0, 0, 0), (0, 0, -1), (0, -1, 0), (0, -1, -1), (-1, 0, 0), (-1, 0, -1), (-1, -1, 0), (-1, -1, -1)]
CELLS_123 = [(0, 0, 0), (0, 0, 1), (0, 0, 2), (0, 1, 0), (0, 1, 1), (0, 1, 2)]
R_123 = [(0, 0, 0), (0, 0, 1), (0, 0, -1), (0, -1, 0), (0, -1, 1), (0, -1, -1)]
AXIS3 = {0: 0, 1: 1, 2: -1}                                   # (m + 1) % 3 - 1


@pytest.mark.parametrize("N,cells,R", [((2, 2, 2), CELLS_222, R_222), ((1, 2, 3), CELLS_123, R_123),
                                       ((3, 3, 3), list(itertools.product(range(3), repeat=3)),
                                        [tuple(AXIS3[v] for v in c) for c in itertools.product(range(3), repeat=3)])])
def test_supercell_order_and_lattice_vectors(N, cells, R):
    lat = np.array([[3.0, 0.1, 0.0], [0.2, 4.0, 0.0], [0.0, 0.3, 5.0]])
    x = np.array([[0.1, 0.2, 0.3], [1.0, 1.5, 2.0]])
    latN, pos = PO.supercell(lat, x, N)
    assert np.allclose(latN, lat * np.array(N)[:, None], rtol=0, atol=0)
    assert pos.shape == (len(cells) * 2, 3)
    for c, m in enumerate(cells):
        assert np.allclose(pos[2 * c:2 * c + 2], x + np.array(m, dtype=float) @ lat, rtol=0, atol=1e-13)
    assert PO.lattice_vectors(N).T.tolist() == [list(r) for r in R]


def test_displacement_order_and_the_package_builder():
    lat = np.array([[3.0, 0.1, 0.0], [0.2, 4.0, 0.0], [0.0, 0.3, 5.0]])
    x = np.array([[0.1, 0.2, 0.3], [1.0, 1.5, 2.0], [2.0, 0.5, 4.0]])
    for N in ((2, 2, 2), (1, 2, 3), (3, 1, 1)):
        latN, disp = PO.displaced_supercells(lat, x, N, 0.01)
        _, base = PO.supercell(lat, x, N)
        assert disp.shape == (18,) + base.shape
        for k, (a, i, s) in enumerate(PO.displacements(3)):
            assert k == 6 * a + 2 * i + (s > 0)
            d = disp[k] - base
            d[a, i] -= s * 0.01
            assert np.abs(d).max() <= 1e-15
        latP, dispP = pkg_displaced_supercells(lat, x, N, 0.01)
        assert np.array_equal(latP, latN) and np.array_equal(dispP, disp)     # bit for bit
    assert np.array_equal(pkg_monkhorst_pack((3, 4, 5)), PO.monkhorst_pack((3, 4, 5)))
    mp = PO.monkhorst_pack((2, 1, 3))
    assert np.allclose(mp, [[-0.25, 0, -1 / 3], [-0.25, 0, 0], [-0.25, 0, 1 / 3], [0.25, 0, -1 / 3], [0.25, 0, 0],
                            [0.25, 0, 1 / 3]], rtol=0, atol=1e-15)


# ---- harmonic spring crystals -----------------------------------------------------------------------------------------
def _springs(lattice, x, N, bonds, k, onsite=None):
    """F_i = -sum_j K (u_i - u_j) over `bonds` (a, b, shift): atom a of cell m bonds atom b of cell m + shift (periodic
    in the supercell) with the 3x3 tensor K (k times the identity for a scalar k), minus onsite[a] u_i if given (a
    term that breaks the acoustic sum rule).  u is the displacement from the undisplaced supercell."""
    n = len(x)
    cells = list(itertools.product(*(range(v) for v in N)))
    index = {c: i for i, c in enumerate(cells)}
    L = np.zeros((len(cells) * n, 3, len(cells) * n, 3))
    for c in cells:
        for bi, (a, b, sh) in enumerate(bonds):
            K = k[bi] if np.ndim(k) == 3 else k * np.eye(3)
            i = index[c] * n + a
            j = index[tuple((c[d] + sh[d]) % N[d] for d in range(3))] * n + b
            L[i, :, i] += K
            L[j, :, j] += K
            L[i, :, j] -= K
            L[j, :, i] -= K
            if onsite is not None and bi == 0:
                for a_ in range(n):
                    L[index[c] * n + a_, :, index[c] * n + a_] += onsite[a_]
    L = L.reshape(len(cells) * n * 3, -1)
    _, x0 = PO.supercell(lattice, x, N)

    def forces(latN, pos):
        return -(L @ (pos - x0).ravel()).reshape(-1, 3)
    return forces


CUBIC = [(0, 0, (1, 0, 0)), (0, 0, (0, 1, 0)), (0, 0, (0, 0, 1))]
CHAIN = [(0, 1, (0, 0, 0)), (1, 0, (1, 0, 0))]


def test_simple_cubic_springs_match_the_analytic_dispersion():
    k, m, a = 2.5, 7.0, 3.0
    lat, x = a * np.eye(3), np.zeros((1, 3))
    N = (3, 3, 3)
    q = np.random.default_rng(0).uniform(-0.7, 0.7, size=(25, 3))
    r = PO.run(_springs(lat, x, N, CUBIC, k), lat, x, [m], N=N, delta=0.01, qpoints=q)
    want = (4 * k / m) * (np.sin(np.pi * q) ** 2).sum(1)
    assert np.abs(r["omega2"] - want[:, None]).max() <= 1e-10 * want.max()
    s = PO.EV_PER_SQRT_EV_A2_AMU
    assert np.abs(r["band_energies"] - s * np.sqrt(want)[:, None]).max() <= 1e-9 * s * np.sqrt(want.max())
    assert s == EV_PER_SQRT_EV_A2_AMU and math.isclose(s, 0.0646541510518066, rel_tol=1e-14)   # CODATA 2014


def test_two_mass_chain_has_the_analytic_acoustic_and_optical_branches():
    k, m1, m2 = 1.7, 2.0, 11.0
    lat = np.diag([4.0, 10.0, 10.0])
    x = np.array([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0]])
    N = (3, 1, 1)
    q = np.column_stack([np.linspace(-0.5, 0.5, 21), np.random.default_rng(1).uniform(-0.5, 0.5, (21, 2))])
    r = PO.run(_springs(lat, x, N, CHAIN, k), lat, x, [m1, m2], N=N, delta=0.02, qpoints=q)
    s_ = 1 / m1 + 1 / m2
    root = np.sqrt(s_ ** 2 - 4 * np.sin(np.pi * q[:, 0]) ** 2 / (m1 * m2))
    acoustic, optical = k * (s_ - root), k * (s_ + root)
    want = np.column_stack([acoustic] * 3 + [optical] * 3)
    assert np.abs(r["omega2"] - want).max() <= 1e-10 * optical.max()


def test_negative_omega2_is_reported_as_a_negative_energy():
    lat, x = 3.0 * np.eye(3), np.zeros((1, 3))
    N = (3, 3, 3)
    q = np.array([[0.1, 0.2, 0.3], [0.5, 0.0, 0.25]])
    r = PO.run(_springs(lat, x, N, CUBIC, -1.0), lat, x, [4.0], N=N, qpoints=q)
    want = -(4 / 4.0) * (np.sin(np.pi * q) ** 2).sum(1)
    assert (r["omega2"] < 0).all() and np.allclose(r["omega2"], want[:, None], rtol=1e-10, atol=0)
    assert np.allclose(r["band_energies"], -PO.EV_PER_SQRT_EV_A2_AMU * np.sqrt(-want)[:, None], rtol=1e-10, atol=0)
    e = PO.energies_from_omega2(np.array([-4.0, 0.0, 9.0]))
    assert e.tolist() == [-2 * PO.EV_PER_SQRT_EV_A2_AMU, 0.0, 3 * PO.EV_PER_SQRT_EV_A2_AMU]


def _sym(rng, count):
    a = rng.normal(size=(count, 3, 3))
    return a + a.transpose(0, 2, 1)


@pytest.mark.parametrize("N", [(3, 3, 3), (2, 2, 2), (1, 2, 3)])
def test_acoustic_gives_three_zero_modes_at_gamma_from_random_forces(N):
    """Random forces obey neither the sum rule nor any symmetry.  After the last `acoustic` round D(Gamma) annihilates
    the three mass-weighted rigid translations; one more `symmetrize` without `acoustic` breaks that again."""
    n, m = 2, np.array([3.0, 5.0])
    f = np.random.default_rng(5).normal(size=(6 * n, int(np.prod(N)) * n, 3))
    C_N, D_N = PO.force_constants(f, m, N, 0.01)
    rows = C_N.sum(0).reshape(3 * n, n, 3).sum(1)               # sum over cells and a' of each row block
    assert np.abs(rows).max() <= 1e-12 * np.abs(C_N).max()
    t = np.kron(np.sqrt(m)[:, None], np.eye(3))                 # [3n, 3]: sqrt(m_a) e_j
    D0 = PO.dynamical_matrix(D_N, N, [0.0, 0.0, 0.0])
    assert np.abs(D0 @ t).max() <= 1e-12 * np.abs(D0).max()
    w = np.sort(np.abs(np.linalg.eigvals(D0)))
    assert w[:3].max() <= 1e-12 * w[-1] and w[3] > 1e-6 * w[-1], w
    S = PO.symmetrize(C_N, N)
    assert np.abs(S.sum(0).reshape(3 * n, n, 3).sum(1)).max() > 1e-3 * np.abs(C_N).max()


@pytest.mark.parametrize("N", [(3, 3, 3), (1, 3, 5)])
def test_dynamical_matrix_is_hermitian_after_symmetrize(N):
    M = 6
    C = np.random.default_rng(2).normal(size=(int(np.prod(N)), M, M))
    S = PO.symmetrize(C, N)
    for q in np.random.default_rng(3).uniform(-1, 1, size=(5, 3)):
        Dq = PO.dynamical_matrix(S, N, q)
        assert np.abs(Dq - Dq.conj().T).max() <= 1e-12 * np.abs(Dq).max()
    # for an even N the cells at N/2 are left out: (2,2,2) symmetrizes only cell 0
    S2 = PO.symmetrize(C[:8], (2, 2, 2))
    assert np.array_equal(S2[0], 0.5 * C[0] + 0.5 * C[0].T) and np.array_equal(S2[1:], C[1:8])


def test_dos_sample_grid_on_two_peaks():
    e, w = np.array([0.010, 0.014]), 1e-3
    grid, dos = PO.sample_grid(e, 11, w)
    assert grid[0] == 0.010 - 3 * w and grid[-1] == 0.014 + 3 * w and len(grid) == 11
    want = sum(np.exp(-0.5 * ((grid - x) / w) ** 2) / (np.sqrt(2 * np.pi) * w) for x in e)
    assert np.allclose(dos, want, rtol=1e-14, atol=0)
    grid, dos = PO.sample_grid(e, 4001, w)
    inside = sum(0.5 * (math.erf((grid[-1] - x) / (w * 2 ** 0.5)) - math.erf((grid[0] - x) / (w * 2 ** 0.5))) for x in e)
    assert math.isclose(np.trapezoid(dos, grid) if hasattr(np, "trapezoid") else np.trapz(dos, grid), inside,
                        rel_tol=1e-6)
    assert 1.99 < inside < 2.0                                   # every energy has weight 1


def test_batched_oracle_equals_one_crystal_at_a_time():
    N = (3, 3, 3)
    crystals = [(3.0 * np.eye(3), np.zeros((1, 3)), CUBIC, [5.0]),
                (np.diag([4.0, 9.0, 9.0]), np.array([[0.0, 0.0, 0.0], [2.0, 0.1, 0.0]]), CHAIN, [2.0, 11.0])]
    q = [np.array([[0.1, 0.2, 0.3]]), np.array([[0.0, 0.0, 0.0], [0.25, 0.0, 0.0]])]
    fns = {id(lat): _springs(lat, x, N, bonds, 1.3) for lat, x, bonds, _ in crystals}
    lat_of = {}
    for lat, x, bonds, _ in crystals:
        lat_of[tuple((lat * np.array(N)[:, None]).ravel())] = fns[id(lat)]

    def batch(items):
        return [lat_of[tuple(latN.ravel())](latN, x) for latN, x in items]
    got = PO.run_batch(batch, [c[0] for c in crystals], [c[1] for c in crystals], [c[3] for c in crystals], N=N,
                       qpoints=q, dos_kpts=(3, 3, 3), dos_npts=20)
    for b, (lat, x, _, m) in enumerate(crystals):
        one = PO.run(fns[id(lat)], lat, x, m, N=N, qpoints=q[b], dos_kpts=(3, 3, 3), dos_npts=20)
        for key in ("C_N", "D_N", "omega2", "band_energies", "dos_energies", "dos_weights"):
            assert np.array_equal(got[b][key], one[key]), (b, key)
