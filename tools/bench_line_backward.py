"""A/B: the line-graph backward as one pass per parent atom (`egc_backward_line_kernel`) against the destination- and
source-keyed kernels, at the L(g) shape of the headline batch (Nn = 23 040 bonds, Ne = 276 480 bond pairs, d = 256), on
identical inputs.  Prints one JSON line: microseconds per launch (CUDA events, 256 MB L2 flush between launches),
compulsory bytes and GB/s of each path, and whether GM, GP and GSh are bit-identical."""
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from alignn_b200 import ops, synthetic  # noqa: E402
from alignn_b200._lib import NORM_AFFINE, NORM_LAYER, NORM_STATS  # noqa: E402

dev = torch.device("cuda:0")
g, lg, lat, _ = synthetic.make_batch(64, 30, 12, seed=123)
lgd = lg.to(dev)
ix_line = lgd.index
ix_two = copy.copy(ix_line)
ix_two.parent = None
Nn, Ne, d = lgd.num_nodes(), lgd.num_edges(), 256
gen = torch.Generator(device="cpu").manual_seed(1)
rnd = lambda *s: torch.randn(*s, generator=gen).to(dev)  # noqa: E731
pos = lambda *s: (torch.rand(*s, generator=gen) * 3 + 0.1).to(dev)  # noqa: E731
P, M, XP, S, H, gx, gy = rnd(Nn, 4 * d), rnd(Ne, d), rnd(Nn, d), pos(Nn, d), rnd(Nn, d), rnd(Nn, d), rnd(Ne, d)
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)


def vecs(norm):
    v = dict(w=pos(d), b=rnd(d))
    if norm != NORM_LAYER:
        v.update(mean=rnd(d), rstd=pos(d))
    if norm == NORM_STATS:
        v.update(c1=rnd(d) * 0.1, c2=rnd(d) * 0.1)
    return v


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    tot = 0.0
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps * 1e3


# compulsory bytes (what ops.egc_backward records for each path): the two-pass path also reads GM and M back
rows = 2 + 1                                             # M, gy_out read; GM written
bytes_line = 4 * d * (Ne * rows + 10 * Nn)
bytes_two = 4 * d * (Ne * rows + 9 * Nn) + 4 * d * 2 * Ne
out = {"gpu": torch.cuda.get_device_name(dev), "shape": {"Nn": Nn, "Ne": Ne, "d": d}}
for tag, norm, gy_out in (("layernorm", NORM_LAYER, gy), ("layernorm_dead_edge_output", NORM_LAYER, None),
                          ("bn_train", NORM_STATS, gy), ("bn_eval", NORM_AFFINE, gy)):
    n, e = vecs(norm), vecs(norm)
    res = {}
    for name, ix in (("two_pass", ix_two), ("line", ix_line)):
        def fn(ix=ix):
            return ops.egc_backward(ix, P, M, XP, S, H, gx, gy_out, n, e, reduce=False, norm_nodes=norm,
                                    norm_edges=norm, keep_gsh=True)
        r = fn()
        res[name] = (timeit(fn), r)
    same = all(torch.equal(a, b) for k, (a, b) in enumerate(zip(res["two_pass"][1], res["line"][1])) if k in (0, 1, 4))
    extra = 0 if gy_out is not None else 4 * d * Ne
    row = {"bit_identical_GM_GP_GSh": bool(same)}
    for name, nb in (("two_pass", bytes_two - extra), ("line", bytes_line - extra)):
        us = res[name][0]
        row[name] = {"us": round(us, 1), "bytes": nb, "GB_per_s": round(nb / us / 1e3, 1)}
    row["saved_us"] = round(res["two_pass"][0] - res["line"][0], 1)
    out[tag] = row
print(json.dumps(out))
