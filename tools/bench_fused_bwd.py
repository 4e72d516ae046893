"""A/B timing of the staged fused backward (node kernel + gm-producer/dgrad wgmma kernel) against the shipped
`ops.egc_backward` (destination- AND source-keyed kernels) + data-gradient GEMM, train-mode BatchNorm, headline shapes.

    python tools/bench_fused_bwd.py [--iters 20] [--d 256] [--batch 64] [--graphs g,lg]

The shipped figure contains egc_backward_src_kernel (152 µs on L(g) in round 1), which the fused path still needs on
top of its own time; the JSON line says so."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--d", type=int, default=256)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--graphs", default="g,lg")
    args = ap.parse_args()
    import staged_binding as SB
    from alignn_b200 import ops, synthetic
    lib = SB.load()
    dev = torch.device("cuda:0")
    g, lg, _, _ = synthetic.make_batch(batch_size=args.batch, atoms=30, k=12, seed=123)
    d = args.d
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {}
    for name, gr in (("g", g), ("lg", lg)):
        if name not in args.graphs.split(","):
            continue
        ix = gr.to(dev).index
        Nn, Ne = gr.num_nodes(), gr.num_edges()
        gen = torch.Generator().manual_seed(1)
        rnd = lambda *s: torch.randn(*s, generator=gen).to(dev)  # noqa: E731
        x, y, gx_out, gy_out = rnd(Nn, d), rnd(Ne, d), rnd(Nn, d), rnd(Ne, d)
        Wcat, W_eg, bcat, b_eg = rnd(4 * d, d) / d ** 0.5, rnd(d, d) / d ** 0.5, rnd(4 * d), rnd(d)
        P = ops.gemm_nt(x, ops.WeightImage(Wcat), bcat)
        G = ops.gemm_nt(y, ops.WeightImage(W_eg), b_eg)
        ones = torch.ones(d, device=dev)
        fwd = ops.egc_forward(ix, x, y, G, P, None, None, None, None, norm_nodes=ops.NORM_STATS, norm_edges=ops.NORM_STATS,
                              residual=True, save=True, need_edge_out=True)
        del G
        n_aux = ops.bn_finalize(fwd["partials"], 1, Nn, ones, 0 * ones, 1e-5, 0.1, None, None)
        e_aux = ops.bn_finalize(fwd["partials"], 0, Ne, ones, 0 * ones, 1e-5, 0.1, None, None)
        nd = dict(w=n_aux[0], b=n_aux[1], mean=n_aux[2], rstd=n_aux[3])
        ed = dict(w=e_aux[0], b=e_aux[1], mean=e_aux[2], rstd=e_aux[3])
        nd["c1"], nd["c2"] = ops.bn_backward_reduce(fwd["XP"], gx_out, *n_aux)
        ed["c1"], ed["c2"] = ops.bn_backward_reduce(fwd["M"], gy_out, *e_aux)
        img_t = ops.WeightImage(W_eg, transpose=True)
        n, tiles = SB.pack_tiles(lib, ix.in_ptr.cpu().numpy())
        tiles_d = torch.from_numpy(tiles).to(dev)

        def shipped():
            GM, GP, _, _ = ops.egc_backward(ix, P, fwd["M"], fwd["XP"], fwd["S"], fwd["H"], gx_out, gy_out, nd, ed,
                                            norm_nodes=ops.NORM_STATS, norm_edges=ops.NORM_STATS)
            return ops.gemm_nt(GM, img_t, None, gy_out)

        def fused():
            return SB.backward_fused(lib, ix, tiles_d, n, P, fwd["M"], fwd["XP"], fwd["S"], fwd["H"], gx_out, gy_out, nd, ed, img_t)

        def timeit(fn):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            ts = []
            for _ in range(args.iters):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b) * 1e3)
            ts.sort()
            return ts[len(ts) // 2]
        t_f, t_s = timeit(fused), timeit(shipped)
        res[name] = dict(Nn=Nn, Ne=Ne, tiles=n, fused_nodes_plus_edge_us=round(t_f, 1),
                         shipped_dst_src_dgrad_us=round(t_s, 1),
                         fused_algorithmic_GBps=round(4 * d * 4 * Ne / t_f / 1e3, 1))
    print(json.dumps(dict(bench="fused_backward", d=d, batch=args.batch,
                          note="the fused path still needs egc_backward_src_kernel (included in the shipped figure)", **res)))


if __name__ == "__main__":
    main()
