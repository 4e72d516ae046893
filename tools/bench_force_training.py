#!/usr/bin/env python
"""One ALIGNN-FF force-training step (ALIGNNAtomWise, 4+4 layers, d = 256: the mlearn Si / Ge / Mo configuration),
timed with CUDA events, with the convs on the library kernels (double backward: alignn_b200_egc_backward_vjp) against
the same model with its convs run as the torch-operator composition `conv._torch_ops_forward`.

    python tools/bench_force_training.py [--batches 16 64] [--steps 5] [--warmup 2] [--json OUT]

The step is forward, forces by autograd with create_graph=True, loss = L1(energy) + gradwise_weight * L1(forces),
backward, AdamW; batches are synthetic JARVIS-shaped crystals (30 atoms, 12 neighbours).  Each batch size runs three
alternations of the two arms in this one process and reports the median step time, the peak memory of each arm, the
gradient agreement of the two arms from identical weights, and the time per step of egc_backward_vjp with its
compulsory bytes over time as a fraction of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The device name,
power limit and SM clock limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001 -- the timings stand without it
        out = f"nvidia-smi unavailable ({e})"
    return {"torch_device": torch.cuda.get_device_name(), "nvidia_smi": out}


def use_torch_ops_convs(model):
    """Run every conv of `model` as the torch-operator composition instead of the library Function."""
    from alignn_b200 import conv as CV
    from alignn_b200.graph import as_graph
    for mod in model.modules():
        if isinstance(mod, CV.EdgeGatedGraphConvBase):
            mod.forward = (lambda m: lambda g, x, y, _need_edge_out=True:
                           CV._torch_ops_forward(m, as_graph(g).index, x, y, _need_edge_out))(mod)
    return model


def make_model(seed, dev):
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    torch.manual_seed(seed)
    cfg = ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=4, gcn_layers=4, hidden_features=256,
                               atom_input_features=92, gradwise_weight=1.0)
    return ALIGNNAtomWise(cfg).to(dev).train()


def step_fn(model, opt, batch, tgt_e, tgt_f, gradwise):
    def step():
        opt.zero_grad(set_to_none=True)
        res = model(batch)
        loss = (res["out"] - tgt_e).abs().mean() + gradwise * (res["grad"] - tgt_f).abs().mean()
        loss.backward()
        opt.step()
    return step


def timed(step, n):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        step()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def grads_of_one_step(model, batch, tgt_e, tgt_f, gradwise):
    for p in model.parameters():
        p.grad = None
    res = model(batch)
    ((res["out"] - tgt_e).abs().mean() + gradwise * (res["grad"] - tgt_f).abs().mean()).backward()
    return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}


def run_batch(B, args, dev):
    from alignn_b200 import ops, synthetic
    g, lg, lat, _ = synthetic.make_batch(batch_size=B, atoms=30, k=12, seed=123)
    batch = (g.to(dev), lg.to(dev), lat.to(dev))
    gen = torch.Generator().manual_seed(7)
    tgt_e = torch.randn(B, generator=gen).to(dev)
    tgt_f = torch.randn(g.num_nodes(), 3, generator=gen).to(dev)
    gradwise = 1.0
    kern = make_model(1, dev)
    aten = use_torch_ops_convs(make_model(1, dev))
    # gradients of the two arms from identical weights
    gk = grads_of_one_step(kern, batch, tgt_e, tgt_f, gradwise)
    ga = grads_of_one_step(aten, batch, tgt_e, tgt_f, gradwise)
    rel = max(float((gk[n] - ga[n]).abs().max() / ga[n].abs().max().clamp_min(1e-30)) for n in ga if ga[n].abs().max() > 0)
    arms = {}
    for name, model in (("kernels", kern), ("torch_ops", aten)):
        opt = torch.optim.AdamW(model.parameters(), lr=1e-5)
        arms[name] = dict(step=step_fn(model, opt, batch, tgt_e, tgt_f, gradwise), ms=[], peak_gib=0.0)
        for _ in range(args.warmup):
            arms[name]["step"]()
    torch.cuda.synchronize()
    for _ in range(3):                                     # alternations
        for name, a in arms.items():
            torch.cuda.reset_peak_memory_stats()
            a["ms"].append(timed(a["step"], args.steps))
            a["peak_gib"] = max(a["peak_gib"], torch.cuda.max_memory_allocated() / 2 ** 30)
    # the double-backward kernel alone, inside one more kernel-arm step
    ops.TIMER = ops.KernelTimer()
    try:
        arms["kernels"]["step"]()
        torch.cuda.synchronize()
        vjp = ops.TIMER.summary().get("egc_backward_vjp", dict(launches=0, total_ms=0.0, total_bytes=0))
    finally:
        ops.TIMER = None
    out = dict(batch=B, atoms=g.num_nodes(), bonds=g.num_edges(), triplets=lg.num_edges(), grad_rel_err_arms=rel)
    for name, a in arms.items():
        out[name] = dict(ms_per_step=[round(v, 3) for v in a["ms"]], median_ms=round(statistics.median(a["ms"]), 3),
                         peak_mem_gib=round(a["peak_gib"], 2))
    out["speedup_median"] = round(out["torch_ops"]["median_ms"] / out["kernels"]["median_ms"], 3)
    ms = vjp["total_ms"]
    out["egc_backward_vjp"] = dict(launches=vjp["launches"], ms_per_step=round(ms, 3),
                                   compulsory_gb=round(vjp["total_bytes"] / 1e9, 3),
                                   hbm_fraction=round(vjp["total_bytes"] / (ms * 1e-3) / HBM_BYTES_PER_S, 3) if ms else None)
    del arms, kern, aten
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_force_training.py needs a CUDA device")
    import __graft_entry__
    __graft_entry__.build()
    dev = torch.device("cuda:0")
    result = dict(device=device_info(), steps=args.steps, warmup=args.warmup, runs=[])
    for B in args.batches:
        r = run_batch(B, args, dev)
        print(json.dumps(r), flush=True)
        result["runs"].append(r)
    result["device_after"] = device_info()
    print(json.dumps(result["device"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
