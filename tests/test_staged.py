"""Staged work (alignn_b200/csrc/staged): the one-kernel gate-GEMM + edge forward.

CPU part (always runs): the segment-aligned tile packer, and a numpy emulation of the kernel's tile / row-phase /
column-phase data flow driven by the packer's descriptors, against the oracle's formulas -- this pins the tiling
semantics the CUDA kernel implements.
GPU part: the fully fused kernels (bit-identical to the two-kernel path; not the shipped path) against the shipped
gemm_nt + egc_forward pair.
"""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from alignn_b200 import synthetic  # noqa: E402
from alignn_b200.graph import Graph  # noqa: E402
from oracle import golden_inputs as GI  # noqa: E402


@pytest.fixture(scope="module")
def staged():
    import staged_binding
    try:
        return staged_binding.load()
    except Exception as exc:  # no nvcc on this box and no prebuilt library
        pytest.skip(f"staged library not built: {exc}")


def pack_tiles(lib, in_ptr):
    import staged_binding
    return staged_binding.pack_tiles(lib, in_ptr)


@pytest.mark.parametrize("degs", [[12] * 40, [0] * 300, [128, 1, 127, 0, 0, 128], [3, 0, 0, 125, 1, 1, 126] * 9,
                                  list(range(0, 60)), []])
def test_tile_packer_covers_every_segment_once(staged, degs):
    in_ptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int32)
    n, tiles = pack_tiles(staged, in_ptr)
    assert n >= 0
    v = 0
    for v0, nseg, p0, rows in tiles:
        assert v0 == v and 1 <= nseg <= 128 and 0 <= rows <= 128
        assert p0 == in_ptr[v0] and rows == in_ptr[v0 + nseg] - in_ptr[v0]
        v += nseg
        if v < len(degs):      # greedy: the next segment did not fit
            assert nseg == 128 or rows + degs[v] > 128
    assert v == len(degs)


def test_ctypes_struct_matches_staged_header(staged):
    """The library rejects a binding whose struct layout drifted (struct_size guard); Nn = 0 returns before any CUDA call."""
    import ctypes as C
    import staged_binding
    a = staged_binding.FusedArgs(struct_size=C.sizeof(staged_binding.FusedArgs), Nn=0, Ne=0, d=64, norm_edges=2, residual=1,
                                 epilogue_groups=1)
    assert staged.alignn_b200_egc_forward_fused(C.byref(a)) == 0
    a.struct_size += 8
    assert staged.alignn_b200_egc_forward_fused(C.byref(a)) != 0
    staged.alignn_b200_egc_backward_fused.restype = C.c_int
    b = staged_binding.BwdFusedArgs(struct_size=C.sizeof(staged_binding.BwdFusedArgs), Nn=0, Ne=0, d=64, residual=1)
    assert staged.alignn_b200_egc_backward_fused(C.byref(b)) == 0
    b.d = 32                                   # the fused backward keeps d = 32 on the two-kernel path
    assert staged.alignn_b200_egc_backward_fused(C.byref(b)) != 0
    b.d, b.struct_size = 64, b.struct_size + 8
    assert staged.alignn_b200_egc_backward_fused(C.byref(b)) != 0


def test_tile_packer_rejects_oversized_segment(staged):
    in_ptr = np.array([0, 5, 134, 140], dtype=np.int32)
    assert pack_tiles(staged, in_ptr)[0] == -2


def _emulate(tiles, ix_in_ptr, in_eid, src, dst, y, W, b, P, eps=1e-6):
    """numpy restatement of the kernel's data flow (fp64): per tile, rows = gathered y rows -> GEMM -> row phase ->
    per-segment column sums -> S, H, x'."""
    d = y.shape[1]
    Nn = ix_in_ptr.size - 1
    M = np.zeros_like(y)
    S, H, XP = (np.zeros((Nn, d)) for _ in range(3))
    stat = np.zeros((2, d))
    for v0, nseg, p0, rows in tiles:
        e = in_eid[p0:p0 + rows]
        acc = y[e] @ W.T
        m = (acc + b) + (P[src[e], 0:d] + P[dst[e], 2 * d:3 * d])
        M[e] = m
        sg = 1.0 / (1.0 + np.exp(-m))
        sgc = sg * P[src[e], d:2 * d]
        seg = ix_in_ptr[v0:v0 + nseg + 1] - p0
        for j in range(nseg):
            s1, s2 = sg[seg[j]:seg[j + 1]].sum(0), sgc[seg[j]:seg[j + 1]].sum(0)
            h = s2 / (s1 + eps)
            S[v0 + j], H[v0 + j], XP[v0 + j] = s1, h, P[v0 + j, 3 * d:] + h
        stat[0] += m.sum(0)
        stat[1] += (m * m).sum(0)
    return M, S, H, XP, stat


def test_tiled_dataflow_matches_oracle_formulas(staged):
    from oracle import alignn_oracle as O
    g, lg, _, _ = synthetic.make_batch(batch_size=3, atoms=7, k=12, seed=5, vary_atoms=True)
    rng = np.random.default_rng(0)
    for gr in (g, lg):
        # shuffle the edge order so that in_eid is a real permutation
        s, t = (a.numpy() for a in gr.edges())
        perm = rng.permutation(s.size)
        gr2 = Graph(s[perm], t[perm], gr.num_nodes())
        ix = gr2.index
        d = 32
        conv = O.EdgeGatedGraphConv(d, d, norm="batchnorm").double()
        GI.fill_state_dict(conv, 9)
        x, y = GI.features(2, gr2.num_nodes(), d).double(), GI.features(3, gr2.num_edges(), d).double()
        Wcat = torch.cat([conv.src_gate.weight, conv.dst_update.weight, conv.dst_gate.weight, conv.src_update.weight])
        bcat = torch.cat([conv.src_gate.bias, conv.dst_update.bias, conv.dst_gate.bias, conv.src_update.bias])
        P = (x @ Wcat.T + bcat).detach().numpy()
        n, tiles = pack_tiles(staged, ix.in_ptr.numpy())
        assert n > 0
        M, S, H, XP, stat = _emulate(tiles, ix.in_ptr.numpy(), ix.in_eid.numpy().astype(np.int64),
                                     ix.src.numpy().astype(np.int64), ix.dst.numpy().astype(np.int64), y.numpy(),
                                     conv.edge_gate.weight.detach().numpy(), conv.edge_gate.bias.detach().numpy(), P)
        # the reference's intermediate quantities (alignn.py:98-110) by plain index_add
        src, dst = (a.long() for a in gr2.edges())
        with torch.no_grad():
            e_src = x @ conv.src_gate.weight.T + conv.src_gate.bias
            Bh = x @ conv.dst_update.weight.T + conv.dst_update.bias
            e_dst = x @ conv.dst_gate.weight.T + conv.dst_gate.bias
            m = e_src[src] + e_dst[dst] + y @ conv.edge_gate.weight.T + conv.edge_gate.bias
            sig = torch.sigmoid(m)
            Sref = torch.zeros(gr2.num_nodes(), d, dtype=torch.float64).index_add_(0, dst, sig)
            Shref = torch.zeros(gr2.num_nodes(), d, dtype=torch.float64).index_add_(0, dst, sig * Bh[src])
            href = Shref / (Sref + 1e-6)
            xpref = x @ conv.src_update.weight.T + conv.src_update.bias + href
        np.testing.assert_allclose(M, m.numpy(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(S, Sref.numpy(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(H, href.numpy(), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(XP, xpref.numpy(), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(stat[0], m.sum(0).numpy(), rtol=1e-10, atol=1e-10)


# ------------------------------------------------------------------------------------------------ GPU (opt-in)
def needs_optin(f):
    """The staged kernels' tests run with the GPU suite (kept as a marker for them)."""
    return f


def _run_fused(lib, gr, x, y, conv_w, norm_edges, d, train, e_w=None, e_b=None, residual=True, groups=1):
    """Returns the fused kernel's outputs and the shipped two-kernel path's, on the same inputs."""
    import staged_binding
    from alignn_b200 import ops
    dev = x.device
    ix = gr.index
    Wcat, bcat, W_eg, b_eg = conv_w
    P = ops.gemm_nt(x, ops.WeightImage(Wcat), bcat)
    img = ops.WeightImage(W_eg)
    n, tiles = pack_tiles(lib, ix.in_ptr.cpu().numpy())
    assert n > 0
    tiles_d = torch.from_numpy(tiles).to(dev)
    out = staged_binding.fused_forward(lib, ix, tiles_d, n, y, img, b_eg, P, norm_edges, train, e_w, e_b, residual,
                                       groups=groups)
    torch.cuda.synchronize()
    G = ops.gemm_nt(y, img, b_eg)
    zeros = torch.zeros(d, device=dev)
    ref = ops.egc_forward(ix, x, y, G, P, zeros + 1, zeros, e_w if e_w is not None else zeros + 1,
                          e_b if e_b is not None else zeros, norm_nodes=ops.NORM_STATS if train else ops.NORM_AFFINE,
                          norm_edges=norm_edges, residual=residual, save=True, need_edge_out=True)
    torch.cuda.synchronize()
    return out, ref


def _few_ulp(a, b, ulps=16):
    """Equal up to a few units in the last place of the larger magnitude in the tensor (sigmoid via ex2/rcp.approx)."""
    return (a - b).abs().max().item() <= ulps * 1.2e-7 * max(b.abs().max().item(), 1.0)


@pytest.mark.gpu
@needs_optin
@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("d", [256, 64])
@pytest.mark.parametrize("shuffle", [False, True])
def test_fused_forward_bit_identical_to_shipped_path(staged, d, shuffle, groups):
    from alignn_b200 import ops
    dev = torch.device("cuda:0")
    g, lg, _, _ = synthetic.make_batch(batch_size=4, atoms=9, k=12, seed=17, vary_atoms=True)
    for gr in (g, lg):
        if shuffle:
            s, t = (a.numpy() for a in gr.edges())
            perm = np.random.default_rng(1).permutation(s.size)
            gr = Graph(s[perm], t[perm], gr.num_nodes())
        grd = gr.to(dev)
        x, y = GI.features(2, gr.num_nodes(), d).to(dev), GI.features(3, gr.num_edges(), d).to(dev)
        gen = torch.Generator().manual_seed(3)
        Wcat = (torch.randn(4 * d, d, generator=gen) / d ** 0.5).to(dev)
        W_eg = (torch.randn(d, d, generator=gen) / d ** 0.5).to(dev)
        bcat, b_eg = torch.randn(4 * d, generator=gen).to(dev), torch.randn(d, generator=gen).to(dev)
        e_w, e_b = (torch.rand(d, generator=gen) + 0.5).to(dev), torch.randn(d, generator=gen).to(dev)
        # training BatchNorm: M, S, H, x' bit-identical; column sums to fp32 round-off
        out, ref = _run_fused(staged, grd, x, y, (Wcat, bcat, W_eg, b_eg), ops.NORM_STATS, d, True, groups=groups)
        assert torch.equal(out["M"], ref["M"])
        for k in ("S", "H", "XP"):          # the two libraries compile the 4-instruction sigmoid into different FMA groupings
            assert _few_ulp(out[k], ref[k]), k
        sums = out["partials"].double().sum(0)
        refs = ref["partials"].double().sum(0)[:2]
        assert torch.allclose(sums, refs, rtol=1e-5, atol=1e-3)
        # eval BatchNorm: y_out bit-identical; LayerNorm: the row statistics are summed in a different order
        out, ref = _run_fused(staged, grd, x, y, (Wcat, bcat, W_eg, b_eg), ops.NORM_AFFINE, d, False, e_w, e_b, groups=groups)
        assert _few_ulp(out["y_out"], ref["y_out"])
        assert _few_ulp(out["XP"], ref["XP"])
        out, ref = _run_fused(staged, grd, x, y, (Wcat, bcat, W_eg, b_eg), ops.NORM_LAYER, d, True, e_w, e_b, groups=groups)
        assert torch.equal(out["M"], ref["M"])
        err = (out["y_out"] - ref["y_out"]).abs().max().item()
        assert err <= 1e-5 * max(ref["y_out"].abs().max().item(), 1.0), err


@pytest.mark.gpu
@needs_optin
@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("mode", ["layernorm", "bn_eval", "bn_train"])
def test_fused_conv_forward_matches_shipped_forward(staged, mode, groups):
    """Fused kernel + node tail against `ops.egc_forward` (+ the BatchNorm finalize/apply steps) end to end."""
    import staged_binding
    from alignn_b200 import ops
    dev = torch.device("cuda:0")
    d = 128
    g, lg, _, _ = synthetic.make_batch(batch_size=5, atoms=8, k=12, seed=23, vary_atoms=True)
    for gr in (g, lg):
        grd = gr.to(dev)
        ix = grd.index
        Nn, Ne = gr.num_nodes(), gr.num_edges()
        x, y = GI.features(2, Nn, d).to(dev), GI.features(3, Ne, d).to(dev)
        gen = torch.Generator().manual_seed(5)
        Wcat = (torch.randn(4 * d, d, generator=gen) / d ** 0.5).to(dev)
        W_eg = (torch.randn(d, d, generator=gen) / d ** 0.5).to(dev)
        bcat, b_eg = torch.randn(4 * d, generator=gen).to(dev), torch.randn(d, generator=gen).to(dev)
        n_w, n_b, e_w, e_b = ((torch.rand(d, generator=gen) + 0.5).to(dev) for _ in range(4))
        P = ops.gemm_nt(x, ops.WeightImage(Wcat), bcat)
        img = ops.WeightImage(W_eg)
        G = ops.gemm_nt(y, img, b_eg)
        n, tiles = pack_tiles(staged, ix.in_ptr.cpu().numpy())
        tiles_d = torch.from_numpy(tiles).to(dev)
        norm = {"layernorm": ops.NORM_LAYER, "bn_eval": ops.NORM_AFFINE, "bn_train": ops.NORM_STATS}[mode]
        kw = dict(norm_nodes=norm, norm_edges=norm, residual=True, save=True, need_edge_out=True)
        ref = ops.egc_forward(ix, x, y, G, P, n_w, n_b, e_w, e_b, **kw)
        out = staged_binding.conv_forward_like(staged, ix, tiles_d, n, x, y, img, b_eg, P, n_w, n_b, e_w, e_b, groups=groups, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out["M"], ref["M"]), mode
        for k in ("XP", "S", "H"):
            assert _few_ulp(out[k], ref[k]), (mode, k)
        if mode == "bn_train":
            for which, cnt, part, R, res in ((1, Nn, out["partials_n"], out["XP"], x), (0, Ne, out["partials_e"], out["M"], y)):
                a = ops.bn_finalize(ref["partials"], which, cnt, n_w, n_b, 1e-5, 0.1, None, None)
                b = ops.bn_finalize(part, 0, cnt, n_w, n_b, 1e-5, 0.1, None, None)
                for u, v in zip(a, b):
                    assert torch.allclose(u, v, rtol=1e-5, atol=1e-6)
        else:
            tol = 1e-6 if mode == "bn_eval" else 1e-5   # the node tail is a separate kernel: FMA contraction may differ
            for k in ("x_out", "y_out"):
                err = (out[k] - ref[k]).abs().max().item()
                assert err <= tol * max(ref[k].abs().max().item(), 1.0), (mode, k, err)


# ---- thread-level restatement of the fused kernel's epilogue index arithmetic -------------------------------------------
def _emulate_threads(tiles, in_ptr, in_eid, src, dst, y, W, b, P, D, EG, eps=1e-6):
    """Python transcription of the epilogue of egc_fused_tc.cu at thread granularity (same formulas for et / col / rg /
    chunk ownership / staging strides / stat slots), with the GEMM done by numpy.  Catches index-arithmetic mistakes
    that the tile-level emulation above cannot see."""
    BM, GT = 128, 128
    CC = 32 // EG
    NG = GT // CC
    STG = CC + 4
    Nn = in_ptr.size - 1
    M = np.full_like(y, np.nan)
    S, H, XP = (np.full((Nn, D), np.nan) for _ in range(3))
    stat = np.zeros((NG, 2, D))
    for v0, nseg, p0, rows in tiles:
        acc = np.zeros((BM, D))
        if rows:
            acc[:rows] = y[in_eid[p0:p0 + rows]] @ W.T
        for grp in range(EG):
            seg = np.zeros(BM + 1, dtype=np.int64)
            for et in range(GT):                                     # seg[] fill, one entry per thread (+1 by thread 0)
                if et <= nseg:
                    seg[et] = in_ptr[v0 + et] - p0
                if et == 0 and nseg == BM:
                    seg[BM] = in_ptr[v0 + BM] - p0
            for c0 in range(grp * CC, D, EG * CC):
                stg = np.full((3, BM * STG), np.nan)
                for et in range(GT):                                 # row phase: thread = tile row
                    if et < rows:
                        e = in_eid[p0 + et]
                        s_, t_ = src[e], dst[e]
                        v = (acc[et, c0:c0 + CC] + b[c0:c0 + CC]) + (P[s_, c0:c0 + CC] + P[t_, 2 * D + c0:2 * D + c0 + CC])
                        M[e, c0:c0 + CC] = v
                        stg[2, et * STG:et * STG + CC] = v
                        stg[0, et * STG:et * STG + CC] = 1.0 / (1.0 + np.exp(-v))
                        stg[1, et * STG:et * STG + CC] = P[s_, D + c0:D + c0 + CC]
                    else:
                        stg[2, et * STG:et * STG + CC] = 0.0
                for et in range(GT):                                 # column phase: thread = (column, row group)
                    col, rg = et % CC, et // CC
                    for j in range(rg, nseg, NG):
                        vtx = v0 + j
                        s1 = s2 = 0.0
                        for r in range(seg[j], seg[j + 1]):
                            g_ = stg[0, r * STG + col]
                            s1 += g_
                            s2 += stg[1, r * STG + col] * g_
                        h = s2 / (s1 + eps)
                        XP[vtx, c0 + col] = P[vtx, 3 * D + c0 + col] + h
                        S[vtx, c0 + col], H[vtx, c0 + col] = s1, h
                    x = stg[2, [r * STG + col for r in range(rg * (BM // NG), (rg + 1) * (BM // NG))]]
                    stat[rg, 0, c0 + col] += x.sum()
                    stat[rg, 1, c0 + col] += (x * x).sum()
    return M, S, H, XP, stat.sum(0)


@pytest.mark.parametrize("EG", [1, 2])
def test_thread_level_restatement_agrees_with_tile_level_data_flow(staged, EG):
    g, lg, _, _ = synthetic.make_batch(batch_size=2, atoms=5, k=12, seed=9, vary_atoms=True)
    rng = np.random.default_rng(3)
    D = 64
    for gr in (g, lg):
        s, t = (a.numpy() for a in gr.edges())
        perm = rng.permutation(s.size)
        gr2 = Graph(s[perm], t[perm], gr.num_nodes())
        ix = gr2.index
        Nn, Ne = gr2.num_nodes(), gr2.num_edges()
        y, W, b = rng.normal(size=(Ne, D)), rng.normal(size=(D, D)) / 8, rng.normal(size=D)
        P = rng.normal(size=(Nn, 4 * D))
        n, tiles = pack_tiles(staged, ix.in_ptr.numpy())
        args = (tiles, ix.in_ptr.numpy().astype(np.int64), ix.in_eid.numpy().astype(np.int64), ix.src.numpy().astype(np.int64),
                ix.dst.numpy().astype(np.int64), y, W, b, P)
        ref = _emulate(*args)
        out = _emulate_threads(*args, D, EG)
        for a_, b_, name in zip(out, ref, ("M", "S", "H", "XP")):
            assert not np.isnan(a_).any(), name                      # every element written exactly by some thread
            np.testing.assert_allclose(a_, b_, rtol=1e-12, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(out[4], ref[4], rtol=1e-10, atol=1e-9)


@pytest.mark.gpu
@needs_optin
@pytest.mark.parametrize("dead_edge_out", [False, True])
@pytest.mark.parametrize("d", [256, 64])
def test_fused_backward_matches_shipped_backward(staged, d, dead_edge_out):
    """Node kernel + fused edge kernel (gm, GM, segment sums, gy = GM W_eg + gy_out) against `ops.egc_backward` followed
    by the shipped data-gradient GEMM, train-mode BatchNorm, on g and L(g) with permuted edge order."""
    import staged_binding
    from alignn_b200 import ops
    dev = torch.device("cuda:0")
    g, lg, _, _ = synthetic.make_batch(batch_size=4, atoms=9, k=12, seed=19, vary_atoms=True)
    for gr in (g, lg):
        s_, t_ = (a.numpy() for a in gr.edges())
        perm = np.random.default_rng(6).permutation(s_.size)
        grd = Graph(s_[perm], t_[perm], gr.num_nodes()).to(dev)
        ix = grd.index
        Nn, Ne = gr.num_nodes(), gr.num_edges()
        gen = torch.Generator().manual_seed(11)
        rnd = lambda *s: torch.randn(*s, generator=gen).to(dev)  # noqa: E731
        x, y, gx_out, gy_out = rnd(Nn, d), rnd(Ne, d), rnd(Nn, d), rnd(Ne, d)
        Wcat, W_eg = rnd(4 * d, d) / d ** 0.5, rnd(d, d) / d ** 0.5
        bcat, b_eg = rnd(4 * d), rnd(d)
        P = ops.gemm_nt(x, ops.WeightImage(Wcat), bcat)
        G = ops.gemm_nt(y, ops.WeightImage(W_eg), b_eg)
        ones = torch.ones(d, device=dev)
        fwd = ops.egc_forward(ix, x, y, G, P, None, None, None, None, norm_nodes=ops.NORM_STATS, norm_edges=ops.NORM_STATS,
                              residual=True, save=True, need_edge_out=True)
        n_aux = ops.bn_finalize(fwd["partials"], 1, Nn, ones, 0 * ones, 1e-5, 0.1, None, None)
        e_aux = ops.bn_finalize(fwd["partials"], 0, Ne, ones, 0 * ones, 1e-5, 0.1, None, None)
        nd = dict(w=n_aux[0], b=n_aux[1], mean=n_aux[2], rstd=n_aux[3])
        ed = dict(w=e_aux[0], b=e_aux[1], mean=e_aux[2], rstd=e_aux[3])
        nd["c1"], nd["c2"] = ops.bn_backward_reduce(fwd["XP"], gx_out, *n_aux)
        go = None if dead_edge_out else gy_out
        if go is not None:
            ed["c1"], ed["c2"] = ops.bn_backward_reduce(fwd["M"], go, *e_aux)
        GM, GP, vd, _ = ops.egc_backward(ix, P, fwd["M"], fwd["XP"], fwd["S"], fwd["H"], gx_out, go, nd, ed if go is not None else {},
                                         norm_nodes=ops.NORM_STATS, norm_edges=ops.NORM_STATS)
        img_t = ops.WeightImage(W_eg, transpose=True)
        gy_ref = ops.gemm_nt(GM, img_t, None, go)
        n, tiles = pack_tiles(staged, ix.in_ptr.cpu().numpy())
        tiles_d = torch.from_numpy(tiles).to(dev)
        out = staged_binding.backward_fused(staged, ix, tiles_d, n, P, fwd["M"], fwd["XP"], fwd["S"], fwd["H"], gx_out, go, nd, ed,
                                            img_t)
        torch.cuda.synchronize()

        def close(a_, b_, what, tol=2e-5):
            err = (a_ - b_).abs().max().item()
            assert err <= tol * max(b_.abs().max().item(), 1e-6), (what, err, b_.abs().max().item())
        close(out["GM"], GM, "GM")
        close(out["GP"][:, 2 * d:3 * d], GP[:, 2 * d:3 * d], "GP e_dst")
        close(out["GP"][:, 3 * d:], GP[:, 3 * d:], "GP src_update")
        # column sums of dL/dx' are mathematically zero in train-mode BatchNorm: judge them against the summands' scale
        def close_sum(a_, b_, what, scale):
            err = (a_ - b_).abs().max().item()
            assert err <= 1e-4 * scale, (what, err, scale)
        close_sum(out["sum_gD"], vd[4], "sum dL/dx'", GP[:, 3 * d:].abs().sum(0).max().item())
        close_sum(out["sum_gm"], vd[5], "sum gm", GM.abs().sum(0).max().item())
        close(out["gy"], gy_ref, "gy", 1e-4)      # the fused GEMM consumes the same gm to within the rounding of gm itself


def test_folded_batchnorm_backward_constants_are_the_same_function():
    """egc_bwd_fused_tc.cu folds  w (c1 + xhat c2),  xhat = (m - mean) rstd,  into  A + B m  with  B = w c2 rstd,
    A = w c1 - B mean: same function of m as norm_backward_row of the shipped kernel."""
    rng = np.random.default_rng(0)
    m, go = rng.normal(size=(50, 16)), rng.normal(size=(50, 16))
    w, b, mean, c1, c2 = (rng.normal(size=16) for _ in range(5))
    rstd = rng.random(16) + 0.5
    sig = lambda x: 1 / (1 + np.exp(-x))  # noqa: E731
    u = m * w + b
    gu = go * (sig(u) * (1 + u * (1 - sig(u))))
    shipped = w * gu - w * (c1 + (m - mean) * rstd * c2)
    B = w * c2 * rstd
    A = w * c1 - B * mean
    np.testing.assert_allclose(w * gu - (A + B * m), shipped, rtol=1e-12, atol=1e-12)
