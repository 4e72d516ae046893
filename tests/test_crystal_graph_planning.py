"""CPU: the host-side planning of the batched device crystal-graph builder (`neighbors._neighbors_device`,
csrc/crystal_graph_device.cu) -- image tables, growth rules, ragged offsets -- the sample-structure fixture, and a numpy
restatement of the device k-NN pipeline's integer logic (rank by (dist, v, image), shell cut, canonicalisation with
c -> I-1-c, stable sort by pair, order by (first rank, image)) against `neighbors.knn_graph`."""
import os

import numpy as np
import pytest

from alignn_b200 import neighbors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "sample_structures.npz")


def _random_cell(seed, n, skew=0.2):
    rng = np.random.default_rng(seed)
    lat = np.eye(3) * (4.0 + 2.0 * rng.random(3)) + skew * rng.normal(size=(3, 3))
    frac = rng.random((n, 3))
    return lat, frac @ lat


def load_samples():
    z = np.load(FIXTURE)
    off = z["atom_offsets"]
    return [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]]) for i in range(len(z["ids"]))]


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("cutoff", [4.0, 8.0, 13.7])
def test_knn_image_table_is_symmetric(seed, cutoff):
    lat, _ = _random_cell(seed, 3)
    cells = neighbors.knn_image_cells(lat, cutoff)
    assert np.array_equal(cells[::-1], -cells)                         # negating an image is c -> I-1-c
    order = np.lexsort((cells[:, 2], cells[:, 1], cells[:, 0]))
    assert np.array_equal(order, np.arange(cells.shape[0]))           # index order == lexicographic image order
    # and the shifts are the same doubles row by row as cells[c] @ lat (what knn_graph recomputes)
    sh = cells @ lat
    assert np.array_equal(np.stack([c @ lat for c in cells]), sh)


def test_radius_image_table_covers_the_coordinates():
    lat, X = _random_cell(4, 5)
    frac = X @ np.linalg.inv(lat)
    cells = neighbors.radius_image_cells(lat, frac, 4.0)
    lo, hi = cells.min(0), cells.max(0)
    assert (lo <= np.floor(frac.min(0)) - 1).all() and (hi >= np.ceil(frac.max(0))).all()
    order = np.lexsort((cells[:, 2], cells[:, 1], cells[:, 0]))
    assert np.array_equal(order, np.arange(cells.shape[0]))


def test_growth_rules():
    lat = np.diag([3.0, 5.0, 7.0])
    assert neighbors.grow_knn_cutoff(4.0, lat) == 7.0                  # below max(|a|, |b|, |c|): jump to it
    assert neighbors.grow_knn_cutoff(7.0, lat) == 14.0                 # at or above: double
    assert neighbors.grow_knn_cutoff(9.0, lat) == 18.0
    assert neighbors.grow_radius_cutoff(8.0, 3.5) == 11.5


def test_ragged_offsets():
    off = neighbors.ragged_offsets([3, 1, 64, 2])
    assert off.dtype == np.int64 and off.tolist() == [0, 3, 4, 68, 70]
    assert neighbors.ragged_offsets([]).tolist() == [0]


def test_structure_checks_reject_bad_input():
    lat, X = _random_cell(1, 2)
    with pytest.raises(ValueError):
        neighbors._checked_structures([(lat, X)], "k-nearest", 0)
    with pytest.raises(ValueError):
        neighbors._checked_structures([(lat, np.zeros((0, 3)))], "k-nearest", 12)
    with pytest.raises(ValueError):
        neighbors._checked_structures([(np.array([[1., 2., 3.], [4., 5., 6.], [7., 8., 9.]]), X)], "k-nearest", 12)
    with pytest.raises(ValueError):
        neighbors._checked_structures([(lat, X)], "voronoi", 12)
    with pytest.raises(ValueError):
        neighbors._checked_structures([], "radius_graph", 12)


def test_sample_fixture_and_knn_degree():
    samples = load_samples()
    sizes = [x.shape[0] for _, x in samples]
    assert len(samples) == 70 and min(sizes) == 1 and max(sizes) == 64
    for lat, X in samples:
        u, v, r, im = neighbors.knn_graph(lat, X, max_neighbors=12, cutoff=8.0)
        assert np.bincount(v, minlength=X.shape[0]).min() >= 12
        assert np.array_equal(u[0::2], v[1::2]) and np.array_equal(v[0::2], u[1::2])     # reverse bond adjacent
        assert np.array_equal(r[0::2], -r[1::2]) and np.array_equal(im[0::2], im[1::2])


def _knn_pipeline(lat, X, k, cutoff):
    """The device pipeline's integer logic in numpy, on the native host scan's candidates."""
    n = X.shape[0]
    while True:
        cells = neighbors.knn_image_cells(lat, cutoff)
        u, v, img, dist = neighbors._all_neighbors(lat, X, cutoff)
        if np.bincount(u, minlength=n).min() >= k:
            break
        cutoff = neighbors.grow_knn_cutoff(cutoff, lat)
    I = cells.shape[0]
    c = np.array([np.flatnonzero((cells == row).all(1))[0] for row in img])     # image -> table index
    kept = []
    for a in range(n):                                   # knn_shell_kernel: counting rank, then the shell cut
        m = np.flatnonzero(u == a)
        d, key = dist[m], v[m] * I + c[m]
        rank = np.array([np.sum((d < d[i]) | ((d == d[i]) & (key < key[i]))) for i in range(m.size)])
        srt = np.empty(m.size, dtype=np.int64)
        srt[rank] = m
        kth = dist[srt[k - 1]]
        kept += [e for e in srt if dist[e] <= kth]
    kept = np.asarray(kept)
    ku, kv, kc = u[kept], v[kept], c[kept]
    swap = kv < ku                                       # knn_canon_kernel
    a, b, cc = np.where(swap, kv, ku), np.where(swap, ku, kv), np.where(swap, I - 1 - kc, kc)
    g = np.arange(kept.size)
    o1 = np.argsort(a * n + b, kind="stable")            # sort 1: pair key, stable
    pk = (a * n + b)[o1]
    head = np.where(np.r_[True, pk[1:] != pk[:-1]], np.arange(pk.size), 0)
    first = g[o1][np.maximum.accumulate(head)]          # smallest rank of the pair
    key2 = first * I + cc[o1]
    o2 = np.argsort(key2, kind="stable")                 # sort 2: (first rank, image)
    k2 = key2[o2]
    uniq = np.r_[True, k2[1:] != k2[:-1]]
    rec = o1[o2][uniq]
    fr = X @ np.linalg.inv(lat)
    d = ((fr[b[rec]] + cells[cc[rec]]) - fr[a[rec]]) @ lat
    uu = np.stack([a[rec], b[rec]], 1).ravel()
    vv = np.stack([b[rec], a[rec]], 1).ravel()
    rr = np.stack([d, -d], 1).reshape(-1, 3).astype(np.float32)
    ii = np.repeat(cells[cc[rec]], 2, axis=0).astype(np.int64)
    return uu, vv, rr, ii


@pytest.mark.parametrize("case", ["n1", "n2", "n5", "diamond", "samples"])
def test_device_knn_pipeline_restatement_matches_knn_graph(case):
    if case == "samples":
        structs = load_samples()[::7]
    elif case == "diamond":
        structs = [neighbors.diamond_supercell(reps=1)]
    else:
        structs = [_random_cell(int(case[1:]), int(case[1:]))]
    for lat, X in structs:
        ref = neighbors.knn_graph(lat, X, max_neighbors=12, cutoff=8.0)
        got = _knn_pipeline(lat, X, 12, 8.0)
        for x, y in zip(got[:2] + got[3:], ref[:2] + ref[3:]):
            assert np.array_equal(x, y)
        assert np.abs(got[2].view(np.int32).astype(np.int64) - ref[2].view(np.int32)).max() <= 1
