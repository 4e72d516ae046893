"""GPU (-m gpu): the batched device crystal-graph builder (csrc/crystal_graph_device.cu, `neighbors.knn_graph_device`,
`neighbors.crystal_graphs_device`) against the host builders `neighbors.knn_graph` / `neighbors.radius_graph`: identical
bonds, order and images, fp32 displacements within one ulp (expected bitwise), graphs and line graphs laid out like
`dgl.batch` of `atom_dgl_multigraph` outputs, and bitwise-equal model outputs on the two batches."""
import os

import numpy as np
import pytest
import torch

from alignn_b200 import _lib, neighbors
from alignn_b200.graph import Graph, batch, bond_cosines
from oracle import golden_inputs as GI

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_cell(seed, n, skew=0.2):
    rng = np.random.default_rng(seed)
    lat = np.eye(3) * (4.0 + 2.0 * rng.random(3)) + skew * rng.normal(size=(3, 3))
    frac = rng.random((n, 3))
    return lat, frac @ lat


def _samples():
    z = np.load(os.path.join(ROOT, "tests", "golden", "sample_structures.npz"))
    off = z["atom_offsets"]
    return [(z["lattices"][i], z["cart_coords"][off[i]:off[i + 1]]) for i in range(len(z["ids"]))]


def _ulp_rows(a, b):
    """(max distance in fp32 ulps of the larger magnitude, rows not bitwise equal) of two [E,3] float32 arrays."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    d = np.abs(a.astype(np.float64) - b) / np.spacing(np.maximum(np.abs(a), np.abs(b))).astype(np.float64)
    return (float(d.max()) if d.size else 0.0), int((a.view(np.int32) != b.view(np.int32)).any(1).sum())


def _same_bonds(got, ref, what):
    u, v, r, im = (np.asarray(x.cpu()) if isinstance(x, torch.Tensor) else np.asarray(x) for x in got)
    ru, rv, rr, rim = ref
    assert np.array_equal(u, ru) and np.array_equal(v, rv), what
    assert np.array_equal(im.astype(np.int64), np.asarray(rim).astype(np.int64)), what
    ulp, rows = _ulp_rows(np.ascontiguousarray(r, dtype=np.float32), np.ascontiguousarray(rr, dtype=np.float32))
    print(f"[{what}] {u.size} bonds, {rows} rows not bitwise equal, max {ulp} ulp")
    assert ulp <= 1, what
    return rows


def _single_cases():
    cases = [(f"random seed {s} n {n}", *_random_cell(s, n), k, 4.0) for s, n, k in [(1, 1, 12), (2, 2, 12), (3, 5, 8), (4, 9, 12)]]
    cases.append(("diamond", *neighbors.diamond_supercell(reps=2), 12, 8.0))
    cases.append(("diamond jittered", *neighbors.diamond_supercell(reps=2, jitter=0.02, seed=1), 12, 8.0))
    cases.append(("1-atom 1.2 A cell", np.eye(3) * 1.2, np.zeros((1, 3)), 12, 8.0))      # > 1000 candidates: untiled rank
    return cases


def test_knn_graph_device_matches_host_builder():
    rows = 0
    for name, lat, X, k, cutoff in _single_cases():
        ref = neighbors.knn_graph(lat, X, max_neighbors=k, cutoff=cutoff)
        got = neighbors.knn_graph_device(lat, X, max_neighbors=k, cutoff=cutoff, device=DEV)
        assert got[0].is_cuda and got[0].dtype == torch.int64 and got[3].dtype == torch.int64
        rows += _same_bonds(got, ref, name)
    for i, (lat, X) in enumerate(_samples()):
        ref = neighbors.knn_graph(lat, X, max_neighbors=12, cutoff=8.0)
        rows += _same_bonds(neighbors.knn_graph_device(lat, X, device=DEV), ref, f"sample {i}")
    print(f"[knn single] rows not bitwise equal in all: {rows}")


def _mixed_batch():
    s = _samples()
    return [s[0], _random_cell(1, 1), s[17], _random_cell(2, 2), s[33], neighbors.diamond_supercell(reps=1), s[61]]


def _host_batch(structs, feats, strategy, cutoff, cutoff_extra):
    graphs, o = [], 0
    for lat, X in structs:
        n = X.shape[0]
        if strategy == "k-nearest":
            u, v, r, im = neighbors.knn_graph(lat, X, max_neighbors=12, cutoff=cutoff)
        else:
            u, v, r, im = neighbors.radius_graph(lat, X, cutoff=cutoff, cutoff_extra=cutoff_extra)
        g = Graph(u, v, n)
        g.ndata["atom_features"] = feats[o:o + n]
        lat = np.asarray(lat, dtype=np.float64)
        g.ndata["V"] = torch.full((n,), abs(float(np.dot(np.cross(lat[0], lat[1]), lat[2]))), dtype=torch.float32)
        g.ndata["frac_coords"] = torch.from_numpy((X @ np.linalg.inv(lat)).astype(np.float32))
        g.edata["r"] = torch.from_numpy(r)
        g.edata["images"] = torch.from_numpy(np.asarray(im, dtype=np.float32))
        graphs.append(g)
        o += n
    g = batch(graphs).to(DEV)
    lg = g.line_graph(shared=True)
    lg.edata["h"] = bond_cosines(g.edata["r"], lg)
    lat = torch.from_numpy(np.stack([np.asarray(l, dtype=np.float64) for l, _ in structs]).astype(np.float32)).to(DEV)
    return g, lg, lat


def _assert_same_batch(got, ref, what):
    (g, lg, lat), (rg, rlg, rlat) = got, ref
    assert torch.equal(g.batch_num_nodes(), rg.batch_num_nodes()) and torch.equal(g.batch_num_edges(), rg.batch_num_edges())
    s, t = g.edges()
    rs, rt = rg.edges()
    assert torch.equal(s, rs) and torch.equal(t, rt), what
    assert torch.equal(g.edata["images"], rg.edata["images"]), what
    ulp, rows = _ulp_rows(g.edata["r"].cpu().numpy(), rg.edata["r"].cpu().numpy())
    print(f"[{what}] {s.numel()} bonds, {rows} r rows not bitwise equal, max {ulp} ulp")
    assert ulp <= 1
    for k in ("V", "frac_coords", "atom_features"):
        assert torch.equal(g.ndata[k], rg.ndata[k]), k
    assert torch.equal(lat, rlat)
    ls, lt = lg.edges()
    rls, rlt = rlg.edges()
    assert torch.equal(ls, rls) and torch.equal(lt, rlt) and torch.equal(lg.batch_num_edges(), rlg.batch_num_edges())
    if rows == 0:
        assert torch.equal(lg.edata["h"], rlg.edata["h"])


@pytest.mark.parametrize("strategy", ["k-nearest", "radius_graph"])
def test_batch_matches_concatenated_single_builds(strategy):
    structs = _mixed_batch()
    n = sum(x.shape[0] for _, x in structs)
    feats = GI.features(5, n, 92)
    got = neighbors.crystal_graphs_device(structs, feats, neighbor_strategy=strategy, cutoff=4.0, device=DEV)
    ref = _host_batch(structs, feats, strategy, 4.0, 3.5)
    _assert_same_batch(got, ref, strategy)
    # repeatability: a second build is bitwise the same
    again = neighbors.crystal_graphs_device(structs, feats, neighbor_strategy=strategy, cutoff=4.0, device=DEV)
    for a, b in ((got[0], again[0]), (got[1], again[1])):
        assert all(torch.equal(x, y) for x, y in zip(a.edges(), b.edges()))
        assert all(torch.equal(a.edata[k], b.edata[k]) for k in a.edata)
    with pytest.raises(ValueError):
        neighbors.crystal_graphs_device(structs, feats, neighbor_strategy="voronoi", device=DEV)


def test_alignn_on_device_built_knn_batch_is_bitwise_the_host_batch():
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig
    structs = _samples()[:64]
    n = sum(x.shape[0] for _, x in structs)
    feats = GI.features(7, n, 92)
    got = neighbors.crystal_graphs_device(structs, feats, device=DEV)
    ref = _host_batch(structs, feats, "k-nearest", 8.0, 3.5)
    _assert_same_batch(got, ref, "k-NN 64 samples")
    model = ALIGNN(ALIGNNConfig(name="alignn"))
    GI.fill_state_dict(model, 91)
    model.to(DEV).eval()
    with torch.no_grad():
        assert torch.equal(model(got), model(ref))


def test_alignn_atomwise_forces_and_stress_on_device_built_radius_batch():
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    structs = _samples()[::4]
    n = sum(x.shape[0] for _, x in structs)
    feats = GI.features(8, n, 92)
    got = neighbors.crystal_graphs_device(structs, feats, neighbor_strategy="radius_graph", cutoff=5.0, device=DEV)
    ref = _host_batch(structs, feats, "radius_graph", 5.0, 3.5)
    _assert_same_batch(got, ref, "radius samples")
    m = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64,
                                            embedding_features=32, atom_input_features=92, stresswise_weight=0.1))
    GI.fill_state_dict(m, 401)
    m.to(DEV).eval()
    a, b = m(got), m(ref)
    for k in ("out", "grad", "stresses"):
        assert torch.equal(a[k], b[k]), k


def test_rejected_input_raises_before_any_launch():
    lat, X = _random_cell(3, 4)
    with pytest.raises(ValueError):
        neighbors.knn_graph_device(lat, X, max_neighbors=0, device=DEV)
    with pytest.raises(ValueError):
        neighbors.knn_graph_device(lat, np.zeros((0, 3)), device=DEV)
    with pytest.raises(ValueError):
        neighbors.knn_graph_device(np.array([[1., 2., 3.], [2., 4., 6.], [0., 0., 1.]]), X, device=DEV)
    # the library itself returns an error code for the same inputs (nothing is enqueued)
    lib = _lib.load()
    i64 = torch.tensor([0, 4], dtype=torch.int64, device=DEV)
    dbl = torch.zeros(64, dtype=torch.float64, device=DEV)
    i32 = torch.zeros(8, dtype=torch.int32, device=DEV)
    ws = torch.empty(1 << 16, dtype=torch.uint8, device=DEV)
    singular = np.array([[1., 2., 3.], [2., 4., 6.], [0., 0., 1.]])

    def bt(lat_host, n):
        return _lib.CrystalBatch(dbl.data_ptr(), dbl.data_ptr(), dbl.data_ptr(), lat_host.ctypes.data, i64.data_ptr(),
                                 i64.data_ptr(), i32.data_ptr(), dbl.data_ptr(), 1, n, 1, 1, 1e-8)
    st = _lib.stream_ptr()
    good = np.ascontiguousarray(lat)
    assert lib.alignn_b200_crystal_scan_count(bt(singular, 4), 1, i32.data_ptr(), i32.data_ptr(), ws.data_ptr(), ws.numel(), st) == -1
    assert lib.alignn_b200_crystal_scan_count(bt(good, 0), 1, i32.data_ptr(), i32.data_ptr(), ws.data_ptr(), ws.numel(), st) == -1
    assert lib.alignn_b200_knn_graph_select(bt(good, 4), i32.data_ptr(), 4, 0, i32.data_ptr(), ws.data_ptr(), ws.numel(), st) == -1
    torch.cuda.synchronize()
