"""BASELINE config 4: ALIGNN-FF energy + per-atom forces on a ~1000-atom periodic supercell, 1 GPU.
(Secondary config, not the headline bench line.)
Measures (a) the structure build -- periodic radius graph, sorted-CSR index, line graph, bond cosines -- on the host
(native scan) and on the device (csrc/graph_device.cu), (b) one energy+forces evaluation launched eagerly and
(c) replayed as ONE CUDA graph (forward, the autograd pass for the forces and the force reduction captured together)."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from alignn_b200 import neighbors  # noqa: E402
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig  # noqa: E402

dev = torch.device("cuda:0")
lat, X = neighbors.diamond_supercell(reps=5, jitter=0.03)
feats = torch.rand(X.shape[0], 92)
t0 = time.perf_counter()
g, lg = neighbors.crystal_graph(lat, X, feats, cutoff=4.0)
t_host = time.perf_counter() - t0
for _ in range(2):
    neighbors.crystal_graph_device(lat, X, feats, cutoff=4.0, device=dev)
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(5):
    gd, lgd = neighbors.crystal_graph_device(lat, X, feats, cutoff=4.0, device=dev)
torch.cuda.synchronize()
t_dev = (time.perf_counter() - t0) / 5
torch.manual_seed(0)
m = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", atom_input_features=92, alignn_layers=4, gcn_layers=4,
                                        hidden_features=256)).to(dev).eval()
latd = torch.from_numpy(lat).float().unsqueeze(0).to(dev)


def run():
    return m((gd, lgd, latd))


def timeit(fn, n=10):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


side = torch.cuda.Stream()
side.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(side):
    for _ in range(3):
        res = run()
torch.cuda.current_stream().wait_stream(side)
ms_eager = timeit(run)
gr = torch.cuda.CUDAGraph()
with torch.cuda.graph(gr):
    res_g = run()
gr.replay()
ms_graph = timeit(gr.replay)
same = bool(torch.equal(res_g["grad"], res["grad"]))
print(json.dumps({"config4_alignn_ff": {"atoms": gd.num_nodes(), "bonds": gd.num_edges(), "triplets": lgd.num_edges(),
                                         "ms_per_energy_force_eval_eager": ms_eager, "ms_per_energy_force_eval_cuda_graph": ms_graph,
                                         "evals_per_s_cuda_graph": 1e3 / ms_graph, "graph_replay_forces_equal_eager": same,
                                         "structure_build_host_s": t_host, "structure_build_device_s": t_dev,
                                         "max_force": float(res["grad"].abs().max())}}))
