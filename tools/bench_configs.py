"""Secondary BASELINE.json configs (not the headline bench line):
  config 2: full ALIGNN (4+4, d=256) inference, batch 64, eval-mode BatchNorm;
  config 5: gather/segment-sum primitive, 1e4..1e7 edges, d=256 (1288 algorithmic bytes per edge)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from alignn_b200 import ops, synthetic  # noqa: E402
from alignn_b200.alignn import ALIGNN, ALIGNNConfig  # noqa: E402

dev = torch.device("cuda:0")
peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"] \
    if os.path.exists("MEASURED_PEAKS.json") else 6650.0


def timeit(fn, reps=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


out = {}
torch.manual_seed(123)
model = ALIGNN(ALIGNNConfig(name="alignn")).to(dev).eval()
batches = [tuple(t.to(dev) for t in synthetic.make_batch(64, 30, 12, seed=123 + b)) for b in range(4)]
i = [0]


def infer():
    g, lg, lat, _ = batches[i[0] % 4]
    i[0] += 1
    with torch.no_grad():
        return model((g, lg, lat))


ms = timeit(infer)
# the same inference replayed as one CUDA graph per resident batch (what a serving loop with bucketed shapes does,
# alignn_b200.runtime.BucketedForward)
side = torch.cuda.Stream()
side.wait_stream(torch.cuda.current_stream())
graphs = []
with torch.cuda.stream(side):
    for b in range(4):
        i[0] = b
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=side):
            o = infer()
        graphs.append((gr, o))
torch.cuda.current_stream().wait_stream(side)
j = [0]


def replay():
    graphs[j[0] % 4][0].replay()
    j[0] += 1


ms_graph = timeit(replay)
out["config2_inference"] = {"ms_per_batch": ms, "graphs_per_s": 64 / ms * 1e3, "ms_per_batch_cuda_graph": ms_graph,
                            "graphs_per_s_cuda_graph": 64 / ms_graph * 1e3, "conv_stack_bytes": 2.873e9,
                            "conv_stack_GBps": 2.873e9 / (ms_graph * 1e-3) / 1e9,
                            "frac_of_measured_hbm": 2.873e9 / (ms_graph * 1e-3) / 1e9 / peak}
sw = {}
for ne in (10_000, 100_000, 1_000_000, 10_000_000):
    g, bh, sigma = synthetic.make_segment_sweep(ne, d=256)
    gd, bh, sigma = g.to(dev), bh.to(dev), sigma.to(dev)
    ms = timeit(lambda: ops.gather_segment_sum(gd.index, bh, sigma), reps=10, warm=3)
    nb = 1288.0 * g.num_edges()
    sw[str(ne)] = {"us": ms * 1e3, "GBps": nb / (ms * 1e-3) / 1e9, "frac_of_measured_hbm": nb / (ms * 1e-3) / 1e9 / peak}
    del g, gd, bh, sigma
out["config5_gather_segment_sum"] = sw
print(json.dumps(out))
