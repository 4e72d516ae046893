#!/usr/bin/env python
"""eALIGNN (eALIGNNAtomWise) on the H100, timed with CUDA events.

    python tools/bench_ealignn.py [--steps 10] [--warmup 3] [--json OUT]

Arm (a), MD step: forward, forces and stress of one 1000-atom jittered diamond supercell (the BASELINE config 4
shape; bonds from the periodic radius graph at 5 A, so the model's 4 A inner cutoff filters), for the default eALIGNN
(2 + 2 layers, d = 64) and a 4 + 4, d = 256 variant.  Besides the whole step it times, separately, the structure built
inside forward (Cartesian coordinates, cutoff filter, index, L(g)), the conv stack (embeddings, convs, pooling and the
force backward through them) and the net-torque removal kernel.
Arm (b): one force + stress training step (forward, forces with create_graph=True, L1 losses, backward, AdamW) on 64
random crystals of 30 atoms, with the convs on the library kernels against the same model with its convs run as the
torch-operator composition.
Every number is the median of three timed runs; the device name, power limit and SM clock limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_force_training import device_info, timed, use_torch_ops_convs  # noqa: E402


def crystal_graph(lat, X, feats, seed):
    """One periodic crystal as eALIGNN reads it: ndata frac_coords / V / atom_features, edata r / images."""
    from alignn_b200 import neighbors
    from alignn_b200.graph import Graph
    u, v, r, images = neighbors.radius_graph(lat, X, cutoff=5.0)
    g = Graph(u, v, X.shape[0])
    g.ndata["frac_coords"] = torch.from_numpy(X @ np.linalg.inv(lat)).float()
    g.ndata["V"] = torch.full((X.shape[0],), float(abs(np.linalg.det(lat))))
    g.ndata["atom_features"] = feats
    g.edata["r"] = torch.from_numpy(r)
    g.edata["images"] = torch.from_numpy(images).float()
    return g


def make_model(alignn_layers, gcn_layers, d, train, dev):
    from alignn_b200 import eALIGNNAtomWise, eALIGNNAtomWiseConfig
    torch.manual_seed(0)
    m = eALIGNNAtomWise(eALIGNNAtomWiseConfig(name="ealignn_atomwise", alignn_layers=alignn_layers, gcn_layers=gcn_layers,
                                              hidden_features=d, atom_input_features=92, stresswise_weight=0.1))
    return m.to(dev).train(train)


def median3(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    runs = [timed(fn, steps) for _ in range(3)]
    return round(statistics.median(runs), 3), [round(v, 3) for v in runs]


def arm_md(args, dev):
    from alignn_b200 import neighbors, ops
    from alignn_b200.ealignn_atomwise import cartesian_coordinates
    from alignn_b200.graph import bond_cosines, lightweight_graph
    lat, X = neighbors.diamond_supercell(reps=5, jitter=0.03, seed=1)
    feats = torch.from_numpy(np.random.default_rng(5).normal(size=(X.shape[0], 92))).float()
    g = crystal_graph(lat, X, feats, 1).to(dev)
    latd = torch.from_numpy(lat).float().unsqueeze(0).to(dev)
    out = {}
    for name, (nal, ngcn, d) in (("2+2_d64", (2, 2, 64)), ("4+4_d256", (4, 4, 256))):
        m = make_model(nal, ngcn, d, False, dev)

        def structure():
            pos = cartesian_coordinates(g, latd)
            gf, r = lightweight_graph(g, pos, m.config.inner_cutoff)
            return pos, gf, r, gf.line_graph(shared=True)

        pos, gf, r0, lg = structure()

        def convs():
            r = r0.detach().requires_grad_(True)
            x = m.atom_embedding(gf.ndata["atom_features"])
            z = m.angle_embedding(bond_cosines(r, lg))
            y = m.edge_embedding(torch.norm(r, dim=1))
            for i, layer in enumerate(m.alignn_layers):
                x, y, z = layer(gf, lg, x, y, z, _need_z_out=(i + 1 < nal))
            for i, layer in enumerate(m.gcn_layers):
                x, y = layer(gf, x, y, _need_edge_out=(i + 1 < ngcn))
            e = m.fc(ops.segment_mean(x, gf.node_graph_offsets())).sum()
            with ops.input_grads_only():
                torch.autograd.grad(e, r)

        res = m((g, latd))
        forces = res["grad"].contiguous()
        noff = gf.node_graph_offsets().long()
        step_ms, step_runs = median3(lambda: m((g, latd)), args.steps, args.warmup)
        struct_ms, _ = median3(structure, args.steps, args.warmup)
        conv_ms, _ = median3(convs, args.steps, args.warmup)
        torque_ms, _ = median3(lambda: ops.remove_net_torque(pos, forces, noff), args.steps, args.warmup)
        out[name] = dict(atoms=g.num_nodes(), bonds_5A=g.num_edges(), bonds_kept=gf.num_edges(), line_graph_edges=lg.num_edges(),
                         step_ms=step_ms, step_runs_ms=step_runs, structure_ms=struct_ms, convs_fwd_and_force_bwd_ms=conv_ms,
                         torque_ms=torque_ms)
        print(name, out[name], flush=True)
    return out


def arm_training(args, dev):
    from alignn_b200.graph import batch
    rng = np.random.default_rng(3)
    graphs, lats = [], []
    for b in range(64):
        lat = np.diag(rng.uniform(7.6, 8.4, 3)) + rng.uniform(-0.3, 0.3, (3, 3)) * (1 - np.eye(3))
        X = rng.uniform(0, 1, (30, 3)) @ lat
        graphs.append(crystal_graph(lat, X, torch.from_numpy(rng.normal(size=(30, 92))).float(), b))
        lats.append(lat)
    g = batch(graphs).to(dev)
    latd = torch.from_numpy(np.stack(lats)).float().to(dev)
    tgt_e = torch.zeros(64, device=dev)
    tgt_f = torch.zeros(g.num_nodes(), 3, device=dev)
    out = {"crystals": 64, "atoms": g.num_nodes(), "bonds_5A": g.num_edges()}
    arms = {"kernels": make_model(4, 4, 256, True, dev), "torch_ops": use_torch_ops_convs(make_model(4, 4, 256, True, dev))}
    for name, m in arms.items():
        opt = torch.optim.AdamW(m.parameters(), lr=1e-4)

        def step(m=m, opt=opt):
            opt.zero_grad(set_to_none=True)
            res = m((g, latd))
            loss = (res["out"] - tgt_e).abs().mean() + (res["grad"] - tgt_f).abs().mean() + res["stresses"].abs().mean()
            loss.backward()
            opt.step()

        ms, runs = median3(step, max(1, args.steps // 2), args.warmup)
        out[name] = dict(median_ms=ms, runs_ms=runs, peak_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
        torch.cuda.reset_peak_memory_stats()
        print(name, out[name], flush=True)
    out["speedup_median"] = round(out["torch_ops"]["median_ms"] / out["kernels"]["median_ms"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ealignn.py times the GPU path and needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"device": device_info(), "md_step": arm_md(args, dev), "training_step_64": arm_training(args, dev)}
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
