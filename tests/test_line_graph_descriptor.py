"""The line-graph descriptor (`EdgeIndex.parent`, set by `Graph.line_graph`): the edge-id arithmetic of the one-pass
line-graph backward, restated in numpy, reproduces L(g)'s edge list from the parent's CSR, and the descriptor moves
with the graph.  CPU except where marked."""
import copy

import numpy as np
import pytest
import torch

from alignn_b200.graph import Graph, batch, reverse, unbatch
from alignn_b200.runtime import BucketedForward


def random_multigraph(seed, n=23, E=90, hub=True):
    """Self-loops, multi-bonds, atoms without bonds (the last three), one atom with in- and out-degree > 32."""
    rng = np.random.default_rng(seed)
    m = n - 3
    src, dst = rng.integers(0, m, E), rng.integers(0, m, E)
    src[:4], dst[:4] = 5, 5                      # self-loop bonds (a multi-bond among them)
    src[4:7], dst[4:7] = 1, 2                    # multi-bond
    if hub:
        src = np.concatenate([src, np.zeros(40, np.int64), rng.integers(0, m, 37)])
        dst = np.concatenate([dst, rng.integers(0, m, 40), np.zeros(37, np.int64)])
    return Graph(src, dst, n)


def lg_edges_from_parent(in_ptr, in_eid, out_ptr, out_eid, lg_in_ptr):
    """The kernel's enumeration: atom a, destination j = out(a)[c], round t -> source in(a)[t], edge
    lg_in_ptr[j] + t - (t > position of j in in(a))."""
    in_ptr, in_eid, out_ptr, out_eid, lg_in_ptr = (np.asarray(t, dtype=np.int64) for t in
                                                   (in_ptr, in_eid, out_ptr, out_eid, lg_in_ptr))
    T = int(lg_in_ptr[-1])
    src, dst, seen = np.full(T, -1), np.full(T, -1), np.zeros(T, dtype=np.int64)
    for a in range(in_ptr.shape[0] - 1):
        ins = in_eid[in_ptr[a]:in_ptr[a + 1]]
        for j in out_eid[out_ptr[a]:out_ptr[a + 1]]:
            base = lg_in_ptr[j]
            selfpos = -1
            if lg_in_ptr[j + 1] - base != ins.shape[0]:
                selfpos = int(np.flatnonzero(ins == j)[0])
            for t, i in enumerate(ins):
                if t == selfpos:
                    continue
                e = base + t - (1 if 0 <= selfpos < t else 0)
                src[e], dst[e] = i, j
                seen[e] += 1
    return src, dst, seen


def _check_descriptor(g, lg):
    assert lg.index.parent is not None and lg.index.dst_sorted
    pin, peid, pout, poeid = (t.cpu().numpy() for t in lg.index.parent)
    ix = g.index
    for a, b in zip((pin, peid, pout, poeid), (ix.in_ptr, ix.in_eid, ix.out_ptr, ix.out_eid)):
        assert np.array_equal(a, b.cpu().numpy())
    s, d, seen = lg_edges_from_parent(pin, peid, pout, poeid, lg.index.in_ptr.cpu().numpy())
    assert (seen == 1).all()                       # every L(g) edge is enumerated exactly once
    assert np.array_equal(s, lg.index.src.cpu().numpy()) and np.array_equal(d, lg.index.dst.cpu().numpy())
    # the source-side order: for each source i its destinations come in ascending id == L(g)'s out-CSR order
    oe = lg.index.out_eid.cpu().numpy()
    op = lg.index.out_ptr.cpu().numpy()
    lg_dst = lg.index.dst.cpu().numpy()
    for i in range(lg.num_nodes()):
        assert (np.diff(lg_dst[oe[op[i]:op[i + 1]]]) >= 0).all()


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_edge_ids_from_parent_host_builder(seed):
    g = random_multigraph(seed)
    _check_descriptor(g, g.line_graph())


def test_edge_ids_from_parent_batched_synthetic():
    from alignn_b200 import synthetic
    g, lg, _, _ = synthetic.make_batch(batch_size=3, atoms=9, k=12, seed=5, vary_atoms=True)
    _check_descriptor(g, lg)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_edge_ids_from_parent_device_builder(seed):
    g = random_multigraph(seed).to("cuda:0")
    lg = g.line_graph()
    assert lg.index.parent[0].is_cuda
    _check_descriptor(g, lg)


def test_only_line_graph_sets_the_descriptor():
    g = random_multigraph(7)
    lg = g.line_graph()
    assert g.index.parent is None
    assert reverse(lg).index.parent is None
    assert batch([lg, lg]).index.parent is None
    assert all(h.index.parent is None for h in unbatch(lg))
    loc = lg.local_var()
    assert loc.index.parent is lg.index.parent


def test_descriptor_moves_with_the_graph():
    g = random_multigraph(8)
    lg = g.line_graph()
    n0 = lg.index.nbytes()
    assert n0 == sum(t.numel() * 4 for t in (lg.index.src, lg.index.dst, lg.index.in_ptr, lg.index.in_eid,
                                              lg.index.out_ptr, lg.index.out_eid, *lg.index.parent))
    moved = lg.index.to("cpu")
    assert all(torch.equal(a, b) for a, b in zip(moved.parent, lg.index.parent))
    # BucketedForward's static line graph takes the descriptor of each new batch with the same shapes
    dst = copy.copy(lg)
    dst.index = copy.copy(lg.index)
    dst.index.parent = tuple(torch.zeros_like(t) for t in lg.index.parent)
    dst._seg = lg._seg.clone()
    dst.ndata, dst.edata = {}, {}
    BucketedForward._copy_graph(dst, lg)
    assert all(torch.equal(a, b) for a, b in zip(dst.index.parent, lg.index.parent))


@pytest.mark.gpu
def test_descriptor_survives_pin_memory_and_to_device():
    lg = random_multigraph(9).line_graph()
    pinned = lg.pin_memory()
    assert all(t.is_pinned() for t in pinned.index.parent)
    dev = pinned.to("cuda:0", non_blocking=True)
    assert all(t.is_cuda and torch.equal(t.cpu(), u) for t, u in zip(dev.index.parent, lg.index.parent))
