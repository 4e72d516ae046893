"""CPU: host logic (graph container, sorted-CSR index, line graph, collation), the C-ABI library
loads and exports every symbol the header declares, ctypes struct layouts match the C structs,
and the product path refuses to run without CUDA (no CPU fallback)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import alignn_b200
from alignn_b200 import _lib, synthetic
from alignn_b200.graph import EdgeIndex, Graph, batch, reverse, unbatch
from oracle import alignn_oracle as O
from tests.helpers import to_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()


@pytest.mark.parametrize("seed,regular", [(1, True), (2, False), (3, False)])
def test_edge_index_bit_exact(seed, regular):
    g, lg, _, _ = synthetic.make_batch(batch_size=3, atoms=7, k=6, seed=seed, regular=regular, vary_atoms=True)
    for gr in (g, lg):
        s, d = gr.edges()
        ip, ie = O.csr_by_key(d.numpy(), gr.num_nodes())
        op, oe = O.csr_by_key(s.numpy(), gr.num_nodes())
        ix = gr.index
        assert ix.in_ptr.dtype == torch.int32
        assert np.array_equal(ix.in_ptr.numpy(), ip) and np.array_equal(ix.in_eid.numpy(), ie)
        assert np.array_equal(ix.out_ptr.numpy(), op) and np.array_equal(ix.out_eid.numpy(), oe)
    assert lg.index.dst_sorted and np.array_equal(lg.index.in_eid.numpy(), np.arange(lg.num_edges()))


def test_line_graph_same_edge_set_as_reference_semantics():
    g, lg, _, _ = synthetic.make_batch(batch_size=2, atoms=5, k=6, seed=11, regular=False)
    og = to_oracle(g)
    olg = O.line_graph(og)           # DGL order (i, j)
    ours = set(zip(lg.edges()[0].tolist(), lg.edges()[1].tolist()))
    # multigraph: compare as multisets
    a = sorted(zip(lg.edges()[0].tolist(), lg.edges()[1].tolist()))
    b = sorted(zip(olg.src.tolist(), olg.dst.tolist()))
    assert a == b and len(ours) > 0
    assert lg.num_nodes() == g.num_edges()
    assert lg.batch_num_edges().tolist() == olg.bne.tolist()
    # within each destination, sources ascend (same summation order as the reference)
    s, d = lg.edges()
    for v in range(0, lg.num_nodes(), 7):
        seg = s[d == v].tolist()
        assert seg == sorted(seg)
    # cosines: same values edge-for-edge after aligning the two orders
    h_ours = alignn_b200.bond_cosines(g.edata["r"], lg)
    h_ref = O.bond_cosines(og.edata["r"], olg.src, olg.dst)
    key = lambda s_, d_: np.lexsort((s_, d_))  # noqa: E731
    np.testing.assert_array_equal(h_ours.numpy()[key(s.numpy(), d.numpy())],
                                  h_ref.numpy()[key(olg.src.numpy(), olg.dst.numpy())])


def test_line_graph_self_loops_and_multi_edges():
    # node 0 has a self loop (edge 0) and a double bond to node 1 (edges 1, 2), reverse edges 3, 4
    g = Graph([0, 0, 0, 1, 1], [0, 1, 1, 0, 0], 2)
    lg = g.line_graph(shared=True)
    pairs = sorted(zip(lg.edges()[0].tolist(), lg.edges()[1].tolist()))
    expect = sorted((i, j) for i in range(5) for j in range(5)
                    if i != j and [0, 1, 1, 0, 0][i] == [0, 0, 0, 1, 1][j])
    assert pairs == expect
    assert (0, 0) not in pairs        # a bond never pairs with itself, even when it is a self loop


def test_headline_shapes():
    g, lg, lat, y = synthetic.make_batch(batch_size=64, atoms=30, k=12, seed=123)
    assert (g.num_nodes(), g.num_edges(), lg.num_edges()) == (1920, 23040, 276480)
    assert lat.shape == (64, 3, 3) and y.shape == (64,)
    s, d = g.edges()
    assert torch.equal(s[0::2], d[1::2]) and torch.equal(d[0::2], s[1::2])          # reverse bonds adjacent
    assert torch.equal(g.edata["r"][0::2], -g.edata["r"][1::2])
    assert float(torch.norm(g.edata["r"], dim=1).min()) >= 1.5


def test_batch_unbatch_reverse_roundtrip():
    rng = np.random.default_rng(0)
    gs = [synthetic.make_crystal(rng, n, 6, False)[0] for n in (3, 5, 4)]
    bg = batch(gs)
    assert bg.batch_size == 3 and bg.batch_num_nodes().tolist() == [3, 5, 4]
    back = unbatch(bg)
    for a, b in zip(gs, back):
        assert torch.equal(a.edges()[0], b.edges()[0]) and torch.equal(a.edges()[1], b.edges()[1])
        assert torch.equal(a.edata["r"], b.edata["r"])
    rg = reverse(bg, copy_edata=True)
    assert torch.equal(rg.edges()[0], bg.edges()[1]) and torch.equal(rg.index.in_ptr, bg.index.out_ptr)
    assert bg.local_var().ndata is not bg.ndata
    assert bg.node_graph_offsets().tolist() == [0, 3, 8, 12]


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "alignn_b200.h")).read()
    declared = set(re.findall(r"\b(alignn_b200_[a-z_0-9]+)\s*\(", header))
    declared -= {"alignn_b200_status", "alignn_b200_norm"}
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name)
    # and the reverse: the shared object exports no alignn_b200_* symbol the header does not declare
    nm = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {ln.split()[-1] for ln in nm.splitlines() if ln.split() and ln.split()[-1].startswith("alignn_b200_")}
    assert exported == declared, exported ^ declared
    assert lib.alignn_b200_version() == 101
    assert lib.alignn_b200_strerror(-2).decode().startswith("unsupported feature width")
    assert lib.alignn_b200_egc_partial_rows(1920, 256) == 240
    assert lib.alignn_b200_egc_partial_rows(10 ** 7, 256) == 132 * 4


def test_ctypes_structs_match_c_layout(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(alignn_b200_egc_fwd_args),'
                   'offsetof(alignn_b200_egc_fwd_args, x), offsetof(alignn_b200_egc_fwd_args, stream),'
                   'sizeof(alignn_b200_egc_bwd_args), offsetof(alignn_b200_egc_bwd_args, P),'
                   'offsetof(alignn_b200_egc_bwd_args, stream));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    F, B = _lib.EgcFwdArgs, _lib.EgcBwdArgs
    assert got == [ctypes.sizeof(F), F.x.offset, F.stream.offset, ctypes.sizeof(B), B.P.offset, B.stream.offset]


def test_bad_arguments_are_rejected_without_touching_the_gpu():
    lib = _lib.load()
    a = _lib.EgcFwdArgs(struct_size=1)
    assert lib.alignn_b200_egc_forward(ctypes.byref(a)) == -3
    a = _lib.EgcFwdArgs(struct_size=ctypes.sizeof(_lib.EgcFwdArgs), d=48, Nn=4, Ne=4)
    assert lib.alignn_b200_egc_forward(ctypes.byref(a)) == -2
    a = _lib.EgcFwdArgs(struct_size=ctypes.sizeof(_lib.EgcFwdArgs), d=64, Nn=4, Ne=4)
    assert lib.alignn_b200_egc_forward(ctypes.byref(a)) == -1          # NULL pointers
    assert lib.alignn_b200_colsum(None, 1, 1, 1, 1.0, None, None) == -1


def test_no_cpu_fallback():
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig, EdgeGatedGraphConv
    g, lg, lat, _ = synthetic.make_batch(batch_size=1, atoms=4, k=4, seed=1)
    conv = EdgeGatedGraphConv(64, 64)
    with pytest.raises(RuntimeError, match="no CPU path"):
        conv(g, torch.zeros(g.num_nodes(), 64), torch.zeros(g.num_edges(), 64))
    with pytest.raises(RuntimeError, match="fp32-only"):
        conv(g, torch.zeros(g.num_nodes(), 64, dtype=torch.float64), torch.zeros(g.num_edges(), 64, dtype=torch.float64))
    with pytest.raises(NotImplementedError):
        EdgeGatedGraphConv(32, 64)
    m = ALIGNN(ALIGNNConfig(name="alignn", alignn_layers=1, gcn_layers=1, hidden_features=32, embedding_features=32))
    with pytest.raises(RuntimeError):
        m((g, lg, lat))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "alignn_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            txt = open(os.path.join(pkg, fn)).read()
            assert "import oracle" not in txt and "from oracle" not in txt, fn


def test_state_dict_names_match_reference_layout():
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig
    m = ALIGNN(ALIGNNConfig(name="alignn"))
    o = O.ALIGNN()
    assert list(m.state_dict().keys()) == list(o.state_dict().keys())
    assert sum(p.numel() for p in m.parameters()) == 4026753            # SURVEY.md App. A
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(o.state_dict()[k].shape), k
    cfg = ALIGNNConfig(name="alignn")
    assert (cfg.alignn_layers, cfg.gcn_layers, cfg.hidden_features, cfg.atom_input_features) == (4, 4, 256, 92)
    with pytest.raises(Exception):
        ALIGNNConfig(name="not_alignn")


def test_as_graph_adapts_dglgraph_like_objects():
    """A DGLGraph-like object (here: the pure-torch DGL stand-in used for golden generation) is accepted at the
    boundary: structure is read once through the DGL API subset and the sorted-CSR index is cached on it."""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "dgl_stub"))
    try:
        import dgl
    finally:
        sys.path.pop(0)
    from alignn_b200.graph import as_graph
    g, _, _, _ = synthetic.make_batch(batch_size=2, atoms=5, k=4, seed=4)
    s, d = g.edges()
    dg = dgl.DGLGraph(s.long(), d.long(), g.num_nodes(), g.batch_num_nodes().clone(), g.batch_num_edges().clone())
    dg.ndata["atom_features"] = g.ndata["atom_features"]
    dg.edata["r"] = g.edata["r"]
    ours = as_graph(dg)
    assert torch.equal(ours.index.in_ptr, g.index.in_ptr) and torch.equal(ours.index.out_eid, g.index.out_eid)
    assert ours.batch_size == 2 and "r" in ours.edata and "atom_features" in ours.ndata
    again = as_graph(dg)
    assert again.index is ours.index                  # the STRUCTURE is cached on the DGL object ...
    dg.edata["r"] = g.edata["r"] * 2.0                # ... features are read from the live object on every call
    assert torch.equal(as_graph(dg).edata["r"], g.edata["r"] * 2.0) and torch.equal(ours.edata["r"], g.edata["r"])
    assert as_graph(g) is g
    with pytest.raises(TypeError):
        as_graph(object())


def test_native_structure_builders_edge_cases():
    """alignn_b200_csr_build_host / line_graph_*_host on degenerate inputs."""
    g = Graph(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 5)
    assert g.num_edges() == 0 and g.index.in_ptr.tolist() == [0] * 6 and g.index.max_in_deg == 0
    lg = g.line_graph(shared=True)
    assert lg.num_nodes() == 0 and lg.num_edges() == 0
    with pytest.raises(ValueError):
        Graph([0, 7], [1, 2], 3)
    # a batch whose second crystal has no bonds: per-graph line-graph counts still add up
    a = Graph([0, 1], [1, 0], 2)
    b = Graph(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 3)
    c = Graph([0, 1, 1, 2], [1, 0, 2, 1], 3)
    bg = batch([a, b, c])
    lg = bg.line_graph()
    assert lg.batch_num_edges().tolist() == [2, 0, 6] and lg.num_nodes() == 6
    olg = O.line_graph(to_oracle(bg))
    assert sorted(zip(lg.edges()[0].tolist(), lg.edges()[1].tolist())) == sorted(zip(olg.src.tolist(), olg.dst.tolist()))


# ---- property tests on arbitrary small multigraphs (self-loops, parallel edges, isolated nodes, empty) ---------------
from hypothesis import given, settings, strategies as st  # noqa: E402


@st.composite
def _multigraphs(draw):
    n = draw(st.integers(min_value=1, max_value=9))
    e = draw(st.integers(min_value=0, max_value=40))
    src = draw(st.lists(st.integers(0, n - 1), min_size=e, max_size=e))
    dst = draw(st.lists(st.integers(0, n - 1), min_size=e, max_size=e))
    return n, np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64)


@settings(max_examples=60, deadline=None)
@given(_multigraphs())
def test_native_csr_is_a_stable_sort_on_any_multigraph(gr):
    n, src, dst = gr
    ix = Graph(src, dst, n).index
    for key, ptr, eid in ((dst, ix.in_ptr.numpy(), ix.in_eid.numpy()), (src, ix.out_ptr.numpy(), ix.out_eid.numpy())):
        assert np.array_equal(eid, np.argsort(key, kind="stable"))
        assert np.array_equal(ptr, np.concatenate([[0], np.cumsum(np.bincount(key, minlength=n))]))
    assert ix.dst_sorted == bool(np.all(np.diff(dst) >= 0))
    assert ix.max_in_deg == (int(np.bincount(dst, minlength=n).max()) if dst.size else 0)


@settings(max_examples=60, deadline=None)
@given(_multigraphs())
def test_native_line_graph_is_the_definition_on_any_multigraph(gr):
    """L(g) has an edge i -> j exactly when dst(i) == src(j) and i != j (DGL line_graph with backtracking; graphs.py:588);
    emitted destination-major with ascending sources."""
    n, src, dst = gr
    lg = Graph(src, dst, n).line_graph()
    want = [(i, j) for j in range(src.size) for i in range(src.size) if dst[i] == src[j] and i != j]
    ls, lt = (a.numpy() for a in lg.edges())
    assert list(zip(ls.tolist(), lt.tolist())) == want
    assert lg.num_nodes() == src.size


def test_flat_adamw_equals_per_parameter_adamw():
    """dp.FlatAdamW (one flat parameter, one fused launch on the GPU) performs the same update as torch.optim.AdamW
    on the individual tensors; parameters that never receive a gradient stay untouched; versions are bumped."""
    from alignn_b200 import dp
    torch.manual_seed(0)

    def make():
        torch.manual_seed(1)
        return torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.SiLU(), torch.nn.Linear(5, 3), torch.nn.Linear(3, 3))
    a, b = make(), make()
    x, y = torch.randn(16, 6), torch.randn(16, 3)

    def loss(m):
        return (m[2](m[1](m[0](x))) - y).abs().mean()          # m[3] never used: no gradient, like the dead norm layers
    ref_opt = torch.optim.AdamW(a.parameters(), lr=1e-2)
    red = dp.FlatGradAllReducer(b.parameters())
    red.zero_grad()
    loss(b).backward()
    red.gather()
    opt = dp.FlatAdamW(red, lr=1e-2)
    dead_before = b[3].weight.detach().clone()
    for _ in range(4):
        ref_opt.zero_grad(set_to_none=True)
        loss(a).backward()
        ref_opt.step()
        red.zero_grad()
        loss(b).backward()
        v0 = b[0].weight._version
        red.all_reduce()
        opt.step()
        assert b[0].weight._version > v0
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.allclose(pa, pb, rtol=1e-6, atol=1e-7)
    assert torch.equal(b[3].weight, dead_before)


def test_wgrad_batch_workspace_plan_on_the_host():
    """The slab planner behind alignn_b200_wgrad_batch runs on the host (no GPU needed): the workspace is one D x D fp32
    tile per slab, at least one slab per non-empty problem, never more than problems + 2 x 132 slabs, 0 for bad input."""
    import ctypes as C
    from alignn_b200 import _lib
    lib = _lib.load()

    def ws(Ks, d=256):
        arr = (_lib.WgradProblem * len(Ks))()
        for q, k in zip(arr, Ks):
            q.K = k
        return int(lib.alignn_b200_wgrad_batch_workspace_bytes(arr, len(Ks), d))
    tile = 256 * 256 * 4
    step = [276480] * 4 + [23040] * 24 + [1920] * 32               # one training step of the 4+4 stack at batch 64
    n = ws(step) // tile
    assert ws(step) % tile == 0 and len(step) <= n <= len(step) + 2 * 132
    assert ws([0]) == tile and ws([0, 0, 5]) == tile                 # empty problems need no slab (one tile minimum)
    # one huge problem is spread over the whole device: at d = 256 each slab runs on 4 CTAs (one per 128 x 128 block)
    assert ws([10 ** 7]) // tile >= 132 // 4
    small = ws([1920] * 8)
    assert 8 <= small // tile <= 8 + 2 * 132
    assert ws([1, 2, 3], d=48) == 0 and ws([-1]) == 0               # unsupported width / negative K
    assert ws([5] * 65) == 0                                         # more problems than one launch holds
    assert ws([100] * 64, d=32) % (32 * 32 * 4) == 0


def test_deferring_is_a_no_op_on_cpu_tensors():
    """FlatGradAllReducer.deferring() only defers CUDA weight gradients; on CPU tensors backward + gather behave as usual."""
    from alignn_b200 import dp
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(8, 8), torch.nn.SiLU(), torch.nn.Linear(8, 8))
    x = torch.randn(5, 8)
    red = dp.FlatGradAllReducer(m.parameters())
    flats = []
    for deferred in (False, True, True):
        red.zero_grad()
        if deferred:
            with red.deferring():
                m(x).square().mean().backward()
        else:
            m(x).square().mean().backward()
        red.gather()
        flats.append(red.flat.clone())
    assert torch.equal(flats[0], flats[1]) and torch.equal(flats[1], flats[2])
    from alignn_b200 import ops
    assert ops.WgradQueue.current is None


def test_deferring_drops_the_queue_when_backward_raises():
    from alignn_b200 import dp, ops
    m = torch.nn.Linear(4, 4)
    red = dp.FlatGradAllReducer(m.parameters())
    m(torch.randn(2, 4)).sum().backward()
    red.gather()
    with pytest.raises(RuntimeError):
        with red.deferring():
            red.queue.items.append(("stale", "stale", "stale"))
            red.queue.deferred_ptrs().add(123)
            raise RuntimeError("backward failed")
    assert red.queue.items == [] and red.queue.vec_items == [] and not red.queue.deferred_ptrs()
    assert ops.WgradQueue.current is None


def test_public_header_is_plain_c():
    """include/alignn_b200.h is the drop-in boundary: it has to compile as C99 (cgo / ctypes / JNI style bindings), not only
    as C++."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    hdr = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "alignn_b200.h")
    r = subprocess.run([gcc, "-x", "c", "-std=c99", "-fsyntax-only", "-Wall", "-Werror", hdr], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
