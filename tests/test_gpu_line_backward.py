"""GPU (-m gpu): the one-pass line-graph backward (`egc_backward_line_kernel`) against the destination- and
source-keyed kernels on the same inputs -- the same `ops.egc_backward` call with and without the line-graph descriptor.

GM, GSh and all of GP must be bitwise equal.  The per-block partial rows are grouped differently (one CTA per parent atom
instead of one warp per node), so their column sums agree to 1e-6 of their scale, and a second fused run must repeat
them bit for bit."""
import copy

import numpy as np
import pytest
import torch

from alignn_b200 import ops, synthetic
from alignn_b200._lib import NORM_AFFINE, NORM_LAYER, NORM_STATS
from alignn_b200.graph import Graph

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NORMS = (NORM_LAYER, NORM_AFFINE, NORM_STATS)


def ragged_multigraph(seed, n=23, E=90):
    """Self-loops, multi-bonds, atoms without bonds, one atom with in- and out-degree > 32 (several warp chunks)."""
    rng = np.random.default_rng(seed)
    m = n - 3
    src, dst = rng.integers(0, m, E), rng.integers(0, m, E)
    src[:4], dst[:4] = 5, 5
    src[4:7], dst[4:7] = 1, 2
    src[7:9], dst[7:9] = 9, 11                   # atom 9: out-bonds only unless the random ones reach it
    src = np.concatenate([src, np.zeros(40, np.int64), rng.integers(0, m, 37)])
    dst = np.concatenate([dst, rng.integers(0, m, 40), np.zeros(37, np.int64)])
    return Graph(src, dst, n)


def _inputs(ix, Nn, Ne, d, norm, gy, seed):
    gen = torch.Generator(device="cpu").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=gen).to(DEV)  # noqa: E731
    pos = lambda *s: (torch.rand(*s, generator=gen) * 3 + 0.1).to(DEV)  # noqa: E731
    P, M, XP, S, H, gx = rnd(Nn, 4 * d), rnd(Ne, d), rnd(Nn, d), pos(Nn, d), rnd(Nn, d), rnd(Nn, d)
    gy_out = rnd(Ne, d) if gy else None

    def vecs():
        v = dict(w=pos(d), b=rnd(d))
        if norm != NORM_LAYER:
            v.update(mean=rnd(d), rstd=pos(d))
        if norm == NORM_STATS:
            v.update(c1=rnd(d) * 0.1, c2=rnd(d) * 0.1)
        return v
    return P, M, XP, S, H, gx, gy_out, vecs(), vecs()


def _compare(lg, d, norm, gy, seed=0):
    ix = lg.index
    assert ix.parent is not None
    two = copy.copy(ix)
    two.parent = None
    Nn, Ne = lg.num_nodes(), lg.num_edges()
    P, M, XP, S, H, gx, gy_out, n, e = _inputs(ix, Nn, Ne, d, norm, gy, seed)
    run = lambda index: ops.egc_backward(index, P, M, XP, S, H, gx, gy_out, n, e, reduce=False,  # noqa: E731
                                         norm_nodes=norm, norm_edges=norm, keep_gsh=True)
    GM0, GP0, pd0, ps0, GSh0 = run(two)
    GM1, GP1, pd1, ps1, GSh1 = run(ix)
    assert torch.equal(GM0, GM1)
    assert torch.equal(GSh0, GSh1)
    assert torch.equal(GP0, GP1)
    for a, b in ((pd0, pd1), (ps0, ps1)):
        sa, sb = ops.colsum(a), ops.colsum(b)
        scale = max(sa.abs().max().item(), 1e-30)
        assert (sa - sb).abs().max().item() <= 1e-6 * scale
    _, _, pd2, ps2, _ = run(ix)
    assert torch.equal(pd1, pd2) and torch.equal(ps1, ps2)


@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("gy", [True, False])
def test_ragged_multigraph_host_builder(d, norm, gy):
    lg = ragged_multigraph(d + norm).line_graph().to(DEV)
    _compare(lg, d, norm, gy, seed=d * 7 + norm)


@pytest.mark.parametrize("norm", NORMS)
def test_ragged_multigraph_device_builder(norm):
    lg = ragged_multigraph(11).to(DEV).line_graph()
    _compare(lg, 64, norm, True, seed=3)


@pytest.mark.parametrize("norm", NORMS)
@pytest.mark.parametrize("gy", [True, False])
def test_headline_line_graph(norm, gy):
    _, lg, _, _ = synthetic.make_batch(64, 30, 12, seed=123)
    _compare(lg.to(DEV), 256, norm, gy, seed=norm)


def test_atoms_without_out_bonds_zero_their_sources():
    # atoms 3 and 4 receive bonds but emit none: their in-bonds have no L(g) out-edges, GP[i, 0:2d] must be 0
    src = np.array([0, 1, 2, 0, 1, 2, 1, 0])
    dst = np.array([1, 2, 0, 3, 4, 3, 0, 2])
    lg = Graph(src, dst, 5).line_graph().to(DEV)
    _compare(lg, 32, NORM_LAYER, True)
