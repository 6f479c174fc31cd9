"""Throughput of instance-batched reverse mode: NetworkPlan.vjp_batch(0, B, seeds) with the gradient sum or the
per-instance gradient rows, against the loop [stage(net_i); run(); vjp(seed_i) for i in range(B)] on the same gradient
plan, in one process with the order of the three arms rotated per repeat.

Workloads (every one a gradient plan of one structure, every leaf requested, bitstrings varying per instance):
  amp16 / amp20   16- / 20-qubit, 10-round random-circuit amplitude networks, random bitstrings
  bench3          bench.py's network (36 qubits, 10 rounds, seed 1) with 3 bitstrings
Every arm downloads what it returns (the sum, the rows, or each instance's gradient block), so the three return the
same data up to the sum.  Per workload and batch size one JSON line: networks/s of each arm (median, min, max over the
repeats, host clock around synchronised work), the median time of stage_batch (reported separately: the loop stages per
instance inside its timed window), kernel launches of one call of each arm, and whether the rows equal the loop's
gradients and the sum the left fold of the rows, bit for bit.  The first line holds the card's name and power limit
(nvidia-smi query).

usage: python tools/bench_vjp_batch.py [--sizes 1,8,64,512] [--repeats 5] [--workloads amp16,amp20,bench3] [--out FILE]
"""
import argparse
import functools
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import amplitude_nets, card, greedy  # noqa: E402


def workload(name, n):
    if name == "amp16":
        return amplitude_nets(16, 10, 16, n)
    if name == "amp20":
        return amplitude_nets(20, 10, 20, n)
    if name == "bench3":
        import bench
        return amplitude_nets(bench.NET["qubits"], bench.NET["rounds"], bench.NET["seed"], n, first_zero=True)
    raise ValueError(name)


def path_for(name, tn):
    if name == "bench3":            # bench.py's own path: the 15.24 GB gradient workspace
        import bench
        return bench.greedy_path(tn)
    return greedy(tn)


def run_loop(plan, nets, seeds):
    out = []
    for net, s in zip(nets, seeds):
        plan.stage(net)
        plan.run()
        out.append(plan.vjp(s))
    return out


def launches(ctx, fn):
    ctx.synchronize()
    ctx.reset_stats()
    fn()
    ctx.synchronize()
    return ctx.stats()["kernel_launches"]


def measure(ctx, plan, nets, seeds, repeats):
    b = len(nets)
    t0 = time.perf_counter()
    plan.stage_batch(nets)
    t_stage = [time.perf_counter() - t0]
    for _ in range(2):
        t0 = time.perf_counter()
        plan.stage_batch(nets)
        t_stage.append(time.perf_counter() - t0)
    arms = {
        "sum": lambda: plan.vjp_batch(0, b, seeds, rows=False, sum=True, values=False),
        "rows": lambda: plan.vjp_batch(0, b, seeds, rows=True, sum=False, values=False),
        "loop": lambda: run_loop(plan, nets, seeds),
    }
    # warm-up of every arm (module loads, K1 offset tables, arena slabs), then the bit-for-bit checks
    _, _, _, total = arms["sum"]()
    _, _, rows, _ = arms["rows"]()
    loop = arms["loop"]()
    rows_identical = all(np.array_equal(rows[leaf][i], loop[i][leaf]) for i in range(b) for leaf in rows)
    sum_identical = all(np.array_equal(total[leaf], functools.reduce(np.add, [rows[leaf][i] for i in range(b)],
                                                                       np.zeros(rows[leaf].shape[1:], np.complex128)))
                        for leaf in rows)
    n_launch = {k: launches(ctx, fn) for k, fn in arms.items()}
    times = {k: [] for k in arms}
    order = list(arms)
    for r in range(repeats):
        for k in order[r % 3:] + order[:r % 3]:
            ctx.synchronize()
            t0 = time.perf_counter()
            res = arms[k]()
            ctx.synchronize()
            times[k].append(time.perf_counter() - t0)
            del res
    rate = lambda ts: {"median": b / statistics.median(ts), "min": b / max(ts), "max": b / min(ts)}
    rec = {f"{k}_networks_per_s": rate(ts) for k, ts in times.items()}
    rec.update({"speedup_sum_median": statistics.median(times["loop"]) / statistics.median(times["sum"]),
                "speedup_rows_median": statistics.median(times["loop"]) / statistics.median(times["rows"]),
                "stage_batch_ms_median": 1e3 * statistics.median(t_stage),
                **{f"launches_{k}": v for k, v in n_launch.items()},
                "bit_identical": bool(rows_identical and sum_identical)})
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,512")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workloads", default="amp16,amp20,bench3")
    ap.add_argument("--out", default=None)
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
        path = path_for(wl, nets[0])
        rng = np.random.default_rng(7)
        all_seeds = rng.standard_normal(max(wl_sizes)) + 1j * rng.standard_normal(max(wl_sizes))
        for b in wl_sizes:
            plan = NetworkPlan.for_gradients(nets[0], path, ctx=ctx)
            info = plan.info()
            rec = {"record": "throughput", "workload": wl, "B": b, "pairs": info["pairs"], "leaves": len(plan.leaf_shapes),
                   "gradient_workspace_bytes": info["peak_bytes"], "repeats": args.repeats if wl != "bench3" else 3,
                   **measure(ctx, plan, nets[:b], all_seeds[:b], args.repeats if wl != "bench3" else 3)}
            del plan
            ctx.trim()
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
