"""Reverse-mode cost: `run` against `run` + `vjp` of a gradient plan (every leaf requested).

Networks: bench.py's 36-qubit network (488 forward pairs, the int8 engine) and a 20-qubit, 10-round random-circuit
amplitude network (launch-bound).  Each is warmed up, then timed with CUDA events on the context stream over --reps
repetitions of (a) the forward levels alone and (b) forward + backward levels + gather; the ratio
backward / forward = (b - a) / a.  The card's name and power limit are read in the same call.

    python tools/bench_vjp.py [--reps 10] [--out profiles/h100_vjp.jsonl]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:           # the numbers are still the card's; say that the label is missing
        return {"gpu": f"unknown ({e})"}


def networks():
    import bench
    from tnc_b200.builders import random_circuit_builder
    tn = bench.build_network()
    yield "bench_36q_10r", tn, bench.greedy_path(tn)
    c = random_circuit_builder(20, 10, 0.5, 0.5, np.random.default_rng(21))
    tn = c.into_amplitude_network("0" * 20)[0]
    yield "amp_20q_10r", tn, bench.greedy_path(tn)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_vjp.jsonl"))
    args = ap.parse_args()
    import torch
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    ctx = tb.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    info = card()
    lines = []
    for name, tn, path in networks():
        plan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
        pi = plan.info()
        fwd_plan = NetworkPlan(tn, path, ctx=ctx)
        plan.stage(tn)

        def fwd():
            plan.run()

        def both():
            plan.run()
            plan.vjp()                                   # (includes the one device-to-host copy of the gradients)

        def timed(fn, reps):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ms = []
            for _ in range(reps):
                ctx.synchronize()
                t0.record(stream)
                fn()
                t1.record(stream)
                t1.synchronize()
                ms.append(t0.elapsed_time(t1))
            return ms

        for fn in (fwd, both):                           # warm-up: modules, K1 tables, int8 planes, arena slabs
            timed(fn, 2)
        f_ms, b_ms = [], []
        for _ in range(args.reps):                       # alternate the two so that drift hits both alike
            f_ms += timed(fwd, 1)
            b_ms += timed(both, 1)
        ctx.reset_stats()
        both()
        ctx.synchronize()
        ec = ctx.engine_counts()
        # device time per kernel name of one forward and one forward + backward (separate, untimed passes)
        by_kernel = {}
        for tag, fn in (("run", fwd), ("run_vjp", both)):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fn()
                ctx.synchronize()
            for ev in prof.key_averages():
                t = getattr(ev, "self_device_time_total", 0) or getattr(ev, "self_cuda_time_total", 0)
                if t > 0:
                    by_kernel.setdefault(ev.key.split("<")[0][:60], {}).setdefault(tag, 0.0)
                    by_kernel[ev.key.split("<")[0][:60]][tag] += t / 1e3
        by_kernel = dict(sorted(by_kernel.items(), key=lambda kv: -kv[1].get("run_vjp", 0.0))[:12])
        f, b = float(np.median(f_ms)), float(np.median(b_ms))
        line = {"network": name, **info, "reps": args.reps,
                "forward_pairs": fwd_plan.info()["pairs"], "gradient_pairs": pi["pairs"],
                "forward_flops": fwd_plan.info()["flops"], "gradient_flops": pi["flops"],
                "forward_peak_bytes": fwd_plan.info()["peak_bytes"], "gradient_ws_bytes": pi["peak_bytes"],
                "run_ms_median": f, "run_vjp_ms_median": b, "run_ms_min": min(f_ms), "run_vjp_ms_min": min(b_ms),
                "backward_over_forward": (b - f) / f, "engine_counts_run_vjp": ec,
                "kernel_ms_profiled": by_kernel}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del plan, fwd_plan
        ctx.trim()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "a") as fh:
        for line in lines:
            fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
