"""A/B: edge kernels with their rows staged through a shared-memory ring (cp.async) against the register-staged
kernels, at the L(g) shape of the headline batch (Nn = 23 040 bonds, Ne = 276 480 bond pairs, d = 256).  Prints one JSON
line: microseconds per launch (CUDA events, 256 MB L2 flush between launches) and whether the outputs are bit-identical."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from alignn_b200 import _lib, ops, synthetic  # noqa: E402
from alignn_b200._lib import NORM_AFFINE, NORM_LAYER, NORM_STATS  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
g, lg, lat, _ = synthetic.make_batch(64, 30, 12, seed=123)
lgd = lg.to(dev)
ix = lgd.index
Nn, Ne, d = lgd.num_nodes(), lgd.num_edges(), 256
gen = torch.Generator(device="cpu").manual_seed(1)
rnd = lambda *s: torch.randn(*s, generator=gen).to(dev)  # noqa: E731
x, y, G, P = rnd(Nn, d), rnd(Ne, d), rnd(Ne, d), rnd(Nn, 4 * d)
vec = [torch.rand(d, generator=gen).to(dev) + 0.5 for _ in range(4)]
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)


def timeit(fn, reps=10):
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


out = {"shape": {"Nn": Nn, "Ne": Ne, "d": d}}
for name, nn_, ne_, save in (("bn_train", NORM_STATS, NORM_AFFINE, True), ("layernorm_train", NORM_LAYER, NORM_LAYER, True),
                             ("bn_eval_inference", NORM_AFFINE, NORM_AFFINE, False)):
    def fwd():
        return ops.egc_forward(ix, x, y, G, P, *vec, norm_nodes=nn_, norm_edges=ne_, residual=True, save=save,
                               need_edge_out=True, gate_is_m=True)
    res = {}
    for flag, tag in ((1, "registers"), (0, "ring")):
        lib.alignn_b200_debug_egc_flags(flag)
        r = fwd()
        res[tag] = (timeit(fwd), r)
    same = all((res["ring"][1][k] is None and res["registers"][1][k] is None) or torch.equal(res["ring"][1][k], res["registers"][1][k])
               for k in ("x_out", "y_out", "XP", "S", "H", "partials"))
    out["forward_" + name] = {"us_registers": res["registers"][0], "us_ring": res["ring"][0], "bit_identical": bool(same)}
lib.alignn_b200_debug_egc_flags(0)
print(json.dumps(out))
