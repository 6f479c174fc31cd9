"""Throughput of instance-batched plan execution: NetworkPlan.run_batch(0, B) against the sequential loop
[run_slices(i, B) for i in range(B)] over the same B staged networks, in one process with the order alternated.

Workloads (every one a plan of one structure whose leaf payloads vary per instance):
  amp16 / amp20   16- / 20-qubit, 10-round random-circuit amplitude networks, random bitstrings
  obs36           36-qubit random_circuit_with_set_observable network (6 rounds, observables on qubits 5, 17, 30),
                  random x / y / z Paulis at those locations
  bench3          bench.py's network (36 qubits, 10 rounds, seed 1) with 3 bitstrings, where no gain is expected
Per workload and batch size one JSON line: networks/s of both paths (median, min, max over the repeats), kernel launches
of one batched call and of the loop, and whether the batch and the loop agree bit for bit.  The first line holds the
card's name and power limit (nvidia-smi query).  `--trace DIR` additionally writes a torch.profiler trace of one
batched and one looped call of amp16 at B = 64 (a run of its own, after the timed runs).

usage: python tools/bench_batch.py [--sizes 1,8,64,512] [--repeats 7] [--workloads amp16,amp20,obs36,bench3]
                                   [--out FILE] [--trace DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def amplitude_nets(qubits, rounds, seed, n, first_zero=False):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 1000)
    bits = ["".join(rng.choice(["0", "1"], qubits)) for _ in range(n)]
    if first_zero:
        bits[0] = "0" * qubits
    return [c.into_amplitude_network(b)[0] for b in bits]


def observable_nets(n, seed=1):
    """One light-cone structure; the Pauli at each observable location is drawn per instance (the first tensors of the
    network are the observables, in location order)"""
    from tnc_b200.builders import random_circuit_with_set_observable
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    locations = [5, 17, 30]
    tn = random_circuit_with_set_observable(36, 6, 0.5, 0.5, locations, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 1000)
    nets = []
    for _ in range(n):
        ts = list(tn.tensors)
        for q in range(len(locations)):
            t = Tensor(ts[q].legs, ts[q].bond_dims)
            t.set_tensor_data(TensorData.Gate("xyz"[int(rng.integers(0, 3))]))
            ts[q] = t
        nets.append(Tensor.new_composite(ts))
    return nets


def workload(name, n):
    if name == "amp16":
        return amplitude_nets(16, 10, 16, n)
    if name == "amp20":
        return amplitude_nets(20, 10, 20, n)
    if name == "obs36":
        return observable_nets(n)
    if name == "bench3":
        import bench
        return amplitude_nets(bench.NET["qubits"], bench.NET["rounds"], bench.NET["seed"], n, first_zero=True)
    raise ValueError(name)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the record says so instead of guessing
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def run_loop(plan, b):
    outs = [plan.run_slices(i, b) for i in range(b)]
    return outs


def measure(ctx, plan, b, repeats):
    # warm-up of both paths (module loads, K1 offset tables, arena slabs), then the bit-for-bit check
    _, dt = plan.run_batch(0, b)
    batch = dt.to_numpy()
    loop = np.stack([t.to_numpy() for t in run_loop(plan, b)])
    identical = bool(np.array_equal(batch, loop.reshape(batch.shape)))
    ctx.synchronize()
    ctx.reset_stats()
    plan.run_batch(0, b)
    ctx.synchronize()
    l_batch = ctx.stats()["kernel_launches"]
    ctx.reset_stats()
    run_loop(plan, b)
    ctx.synchronize()
    l_loop = ctx.stats()["kernel_launches"]
    tb, tl = [], []
    for r in range(repeats):
        for which in ((0, 1) if r % 2 == 0 else (1, 0)):
            ctx.synchronize()
            t0 = time.perf_counter()
            if which == 0:
                res = plan.run_batch(0, b)
            else:
                res = run_loop(plan, b)
            ctx.synchronize()
            (tb if which == 0 else tl).append(time.perf_counter() - t0)
            del res
    rate = lambda ts: {"median": b / statistics.median(ts), "min": b / max(ts), "max": b / min(ts)}
    return {"batch_networks_per_s": rate(tb), "loop_networks_per_s": rate(tl),
            "speedup_median": statistics.median(tl) / statistics.median(tb),
            "launches_batch": l_batch, "launches_loop": l_loop, "bit_identical": identical}


def trace(ctx, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from tnc_b200.tensornetwork import NetworkPlan
    nets = workload("amp16", 64)
    plan = NetworkPlan(nets[0], greedy(nets[0]), ctx=ctx)
    plan.stage_slices(nets)
    plan.run_batch(0, 64)
    run_loop(plan, 64)
    ctx.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in (("batch", lambda: plan.run_batch(0, 64)), ("loop", lambda: run_loop(plan, 64))):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            ctx.synchronize()
        prof.export_chrome_trace(os.path.join(out_dir, f"amp16_b64_{name}.pt.trace.json"))
        with open(os.path.join(out_dir, f"amp16_b64_{name}.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,512")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--workloads", default="amp16,amp20,obs36,bench3")
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace", default=None)
    args = ap.parse_args()
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    ctx = tb.Context(0)
    lines = [{"record": "card", **card()}]
    print(json.dumps(lines[0]), flush=True)
    sizes = [int(s) for s in args.sizes.split(",")]
    for wl in args.workloads.split(","):
        wl_sizes = [3] if wl == "bench3" else sizes
        nets = workload(wl, max(wl_sizes))
        path = greedy(nets[0])
        for b in wl_sizes:
            plan = NetworkPlan(nets[0], path, ctx=ctx)
            plan.stage_slices(nets[:b])
            rec = {"record": "throughput", "workload": wl, "B": b, "pairs": plan.info()["pairs"],
                   "kernels_per_network": plan.info()["kernels"], "repeats": args.repeats,
                   **measure(ctx, plan, b, args.repeats if wl != "bench3" else 3)}
            del plan
            ctx.trim()
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    if args.trace:
        trace(ctx, args.trace)
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
