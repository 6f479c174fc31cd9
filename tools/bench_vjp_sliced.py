"""Sliced gradients: `run_slices` and `vjp_sliced` over all slices of a sliced gradient plan (every leaf requested),
against the unsliced gradient plan's `run` + `vjp`, on bench.py's network at 0, 1, 2 and 3 sliced legs (find_slices).

Method (as tools/bench_vjp.py): warm-up, then CUDA events on the context stream around each call, alternating the
calls over --reps repetitions, medians.  The device time of the extract and accumulate kernels per slice comes from a
separate torch.profiler pass.  The expected sliced cost is one slice's pass times the slice count: the `flops` of
tncb_plan_info (one slice, forward + backward pairs) x slices, plus two small launches per slice, plus one more forward
per slice inside vjp_sliced (no workspace holds every slice's forward state).  The card's name and power limit are read
in the same call.

--sycamore-d12 also runs the committed depth-12 Sycamore-53 tree sliced on the committed 6 legs + 3 from find_slices
(512 slices, every leaf requested): its time, the value against bench.py's config-5 amplitude and multilinearity
sum_e G_l[e] X_l[e] = R on 16 sampled leaves.

    python tools/bench_vjp_sliced.py [--reps 5] [--sycamore-d12] [--out profiles/h100_vjp_sliced.jsonl]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

D12_LEGS = [157, 1115, 231, 606, 1084, 986, 1088, 155, 515]
CONFIG5_AMPLITUDE = complex(-6.148484459425177e-09, -5.130555022162778e-09)    # bench.py's committed config-5 value


def timed(ctx, stream, fn, reps):
    import torch
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


def kernel_ms(ctx, fn, names):
    """device ms of the kernels whose names start with one of `names`, over one call of fn (torch.profiler)"""
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        ctx.synchronize()
    out = {n: 0.0 for n in names}
    count = {n: 0 for n in names}
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", 0) or getattr(ev, "self_cuda_time_total", 0)
        for n in names:
            if ev.key.startswith(n) or ev.key.split(" ")[-1].startswith(n) or (n + "(") in ev.key:
                out[n] += t / 1e3
                count[n] += ev.count
    return out, count


def leaf_value(t):
    from tnc_b200.contractionpath.slicing import _leaf_array
    return np.asarray(_leaf_array(t), dtype=np.complex128)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--legs", default="0,1,2,3")
    ap.add_argument("--sycamore-d12", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_vjp_sliced.jsonl"))
    args = ap.parse_args()
    import torch
    import bench
    import tnc_b200 as tb
    from bench_vjp import card
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    from tnc_b200.tensornetwork import NetworkPlan
    ctx = tb.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    info = card()
    lines = []

    def emit(line):
        print(json.dumps(line), flush=True)
        lines.append(line)

    tn = bench.build_network()
    path = bench.greedy_path(tn)
    # the unsliced gradient plan: run + vjp (bench_vjp's method)
    g = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    g.stage(tn)

    def unsliced():
        g.run()
        g.vjp()
    timed(ctx, stream, unsliced, 2)
    u_ms = timed(ctx, stream, unsliced, args.reps)
    unsliced_fwd = g.info()
    del g
    ctx.trim()
    emit({"network": "bench_36q_10r", **info, "mode": "unsliced run+vjp", "reps": args.reps,
          "gradient_ws_bytes": unsliced_fwd["peak_bytes"], "gradient_flops": unsliced_fwd["flops"],
          "run_vjp_ms_median": float(np.median(u_ms)), "run_vjp_ms_min": min(u_ms)})
    for n in [int(x) for x in args.legs.split(",")]:
        legs = find_slices(tn, path, min_slices=2 ** n) if n else []
        p = SlicedPlan.for_gradients(tn, path, legs, ctx=ctx)
        p.stage(tn)
        pi = p.info()

        def run():
            p.run()

        def vjp():
            p.vjp()
        for fn in (run, vjp):
            timed(ctx, stream, fn, 2)
        r_ms, v_ms = [], []
        for _ in range(args.reps):
            r_ms += timed(ctx, stream, run, 1)
            v_ms += timed(ctx, stream, vjp, 1)
        km, kc = kernel_ms(ctx, vjp, ["slice_extract_kernel", "grad_accumulate_kernel"])
        ctx.reset_stats()
        vjp()
        ctx.synchronize()
        ec = ctx.engine_counts()
        v = float(np.median(v_ms))
        emit({"network": "bench_36q_10r", **info, "mode": "sliced", "sliced_legs": legs, "slices": p.n_slices,
              "reps": args.reps, "ws_bytes_per_slice": pi["peak_bytes"], "flops_per_slice": pi["flops"],
              "kernels_per_slice": pi["kernels"],
              "run_slices_ms_median": float(np.median(r_ms)), "run_slices_ms_min": min(r_ms),
              "vjp_sliced_ms_median": v, "vjp_sliced_ms_min": min(v_ms),
              "vjp_sliced_over_unsliced_run_vjp": v / float(np.median(u_ms)),
              "flops_all_slices_over_unsliced": pi["flops"] * p.n_slices / unsliced_fwd["flops"],
              "extract_ms_per_slice": km["slice_extract_kernel"] / p.n_slices,
              "accumulate_ms_per_slice": km["grad_accumulate_kernel"] / p.n_slices,
              "extract_launches": kc["slice_extract_kernel"], "accumulate_launches": kc["grad_accumulate_kernel"],
              "engine_counts_vjp": ec})
        del p
        ctx.trim()
    if args.sycamore_d12:
        from tnc_b200.builders import sycamore_circuit
        from tnc_b200.contractionpath import ContractionPath
        from tnc_b200.tensornetwork import leaves
        with open(os.path.join(ROOT, "bench_inputs", "sycamore53_d12.json")) as f:
            d = json.load(f)
        net = sycamore_circuit(53, 12, np.random.default_rng(1)).into_amplitude_network("0" * 53)[0]
        tree = ContractionPath.simple([tuple(x) for x in d["toplevel"]])
        t0 = time.perf_counter()
        p = SlicedPlan.for_gradients(net, tree, D12_LEGS, ctx=ctx)
        p.stage(net)
        t_setup = time.perf_counter() - t0
        pi = p.info()
        ctx.synchronize()
        t0 = time.perf_counter()
        res, G = p.vjp()
        ctx.synchronize()
        t_vjp = time.perf_counter() - t0
        t0 = time.perf_counter()
        run_val = complex(p.run().to_numpy())
        t_run = time.perf_counter() - t0
        r = complex(res.to_numpy())
        lv = leaves(net)
        rng = np.random.default_rng(0)
        sample = sorted(rng.choice(len(lv), 16, replace=False).tolist())
        worst = 0.0
        for i in sample:
            x = leaf_value(lv[i])
            lhs = complex(np.sum(G[i] * x))
            worst = max(worst, abs(lhs - r) / float(np.sum(np.abs(G[i]) * np.abs(x))))
        emit({"network": "sycamore53_d12_committed_tree", **info, "sliced_legs": D12_LEGS, "slices": p.n_slices,
              "ws_bytes_per_slice": pi["peak_bytes"], "flops_per_slice": pi["flops"], "setup_s": t_setup,
              "vjp_sliced_s": t_vjp, "run_slices_s": t_run, "value": [r.real, r.imag],
              "value_vs_config5_abs": abs(r - CONFIG5_AMPLITUDE), "value_equals_run_slices": r == run_val,
              "multilinearity_leaves": sample, "multilinearity_worst_rel": worst, "leaves": len(lv)})
        del p, G
        ctx.trim()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as fh:
        for line in lines:
            fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
