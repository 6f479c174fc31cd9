"""Sliced tangents and Hessian-vector products: `jvp_sliced` and `hvp_sliced` over all slices (every leaf requested)
against the unsliced tangent and Hessian-vector plans' `jvp` / `hvp`, on bench.py's network at 1, 2 and 3 sliced legs
(find_slices).

Method (as tools/bench_vjp_sliced.py): warm-up, then CUDA events on the context stream around each call, alternating
the calls over --reps repetitions, medians.  The device time of the extract and accumulate kernels per slice comes from
a separate torch.profiler pass.  The card's name and power limit are read in the same call.

--sycamore-d12 also runs one full sliced `hvp` of the committed depth-12 Sycamore-53 tree on the 10 legs whose per-slice
Hessian-vector workspace fits (1024 slices, every leaf requested, Ẋ = X): its time, and sum_e G_l[e] X_l[e] = R on 16
sampled leaves.

    python tools/bench_hvp_sliced.py [--reps 5] [--sycamore-d12] [--out profiles/h100_hvp_sliced.jsonl]"""
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

D12_HVP_LEGS = [157, 1115, 231, 606, 1084, 986, 1088, 155, 515, 424]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--legs", default="1,2,3")
    ap.add_argument("--sycamore-d12", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_hvp_sliced.jsonl"))
    args = ap.parse_args()
    import torch
    import bench
    import tnc_b200 as tb
    from bench_vjp import card
    from bench_vjp_sliced import kernel_ms, leaf_value, timed
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    ctx = tb.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    info = card()
    lines = []

    def emit(line):
        print(json.dumps(line), flush=True)
        lines.append(line)

    tn = bench.build_network()
    path = bench.greedy_path(tn)
    lv = leaves(tn)
    rng = np.random.default_rng(0)
    tans = {i: rng.standard_normal(l.bond_dims) + 1j * rng.standard_normal(l.bond_dims) for i, l in enumerate(lv)}
    S, Sd = np.asarray(0.3 - 0.7j), np.asarray(1.1 + 0.2j)
    unsliced = {}
    for kind in ("jvp", "hvp"):
        p = (NetworkPlan.for_tangents if kind == "jvp" else NetworkPlan.for_hvp)(tn, path, ctx=ctx)
        p.stage(tn)
        fn = (lambda: p.jvp(tans)) if kind == "jvp" else (lambda: p.hvp(tans, S, Sd))
        timed(ctx, stream, fn, 2)
        ms = timed(ctx, stream, fn, args.reps)
        pi = p.info()
        unsliced[kind] = (float(np.median(ms)), pi)
        emit({"network": "bench_36q_10r", **info, "mode": f"unsliced {kind}", "reps": args.reps,
              "ws_bytes": pi["peak_bytes"], "flops": pi["flops"], "kernels": pi["kernels"],
              "ms_median": float(np.median(ms)), "ms_min": min(ms)})
        del p, fn
        ctx.trim()
    for n in [int(x) for x in args.legs.split(",") if x]:
        legs = find_slices(tn, path, min_slices=2 ** n)
        jp = SlicedPlan.for_tangents(tn, path, legs, ctx=ctx)
        hp = SlicedPlan.for_hvp(tn, path, legs, ctx=ctx)
        jp.stage(tn)
        hp.stage(tn)

        def jvp():
            jp.jvp(tans)

        def hvp():
            hp.hvp(tans, S, Sd)
        for fn in (jvp, hvp):
            timed(ctx, stream, fn, 2)
        j_ms, h_ms = [], []
        for _ in range(args.reps):
            j_ms += timed(ctx, stream, jvp, 1)
            h_ms += timed(ctx, stream, hvp, 1)
        for kind, p, fn, ms in (("jvp", jp, jvp, j_ms), ("hvp", hp, hvp, h_ms)):
            km, kc = kernel_ms(ctx, fn, ["slice_extract_kernel", "grad_accumulate_kernel"])
            ctx.reset_stats()
            fn()
            ctx.synchronize()
            ec = ctx.engine_counts()
            pi = p.info()
            med = float(np.median(ms))
            u_ms, u_info = unsliced[kind]
            emit({"network": "bench_36q_10r", **info, "mode": f"sliced {kind}", "sliced_legs": legs, "slices": p.n_slices,
                  "reps": args.reps, "ws_bytes_per_slice": pi["peak_bytes"], "flops_per_slice": pi["flops"],
                  "kernels_per_slice": pi["kernels"], "ms_median": med, "ms_min": min(ms),
                  "sliced_over_unsliced_time": med / u_ms,
                  "flops_all_slices_over_unsliced": pi["flops"] * p.n_slices / u_info["flops"],
                  "extract_accumulate_ms_per_slice": (km["slice_extract_kernel"] + km["grad_accumulate_kernel"]) / p.n_slices,
                  "extract_ms_per_slice": km["slice_extract_kernel"] / p.n_slices,
                  "accumulate_ms_per_slice": km["grad_accumulate_kernel"] / p.n_slices,
                  "extract_launches": kc["slice_extract_kernel"], "accumulate_launches": kc["grad_accumulate_kernel"],
                  "engine_counts": ec})
        del jp, hp
        ctx.trim()
    if args.sycamore_d12:
        from tnc_b200.builders import sycamore_circuit
        from tnc_b200.contractionpath import ContractionPath
        with open(os.path.join(ROOT, "bench_inputs", "sycamore53_d12.json")) as f:
            d = json.load(f)
        net = sycamore_circuit(53, 12, np.random.default_rng(1)).into_amplitude_network("0" * 53)[0]
        tree = ContractionPath.simple([tuple(x) for x in d["toplevel"]])
        nlv = leaves(net)
        xs = [leaf_value(l) for l in nlv]
        t0 = time.perf_counter()
        p = SlicedPlan.for_hvp(net, tree, D12_HVP_LEGS, ctx=ctx)
        p.stage(net)
        t_setup = time.perf_counter() - t0
        pi = p.info()
        ctx.synchronize()
        t0 = time.perf_counter()
        val, tan, G, Gd = p.hvp({i: x for i, x in enumerate(xs)})
        ctx.synchronize()
        t_hvp = time.perf_counter() - t0
        r = complex(val)
        sample = sorted(np.random.default_rng(0).choice(len(nlv), 16, replace=False).tolist())
        worst = 0.0
        for i in sample:
            lhs = complex(np.sum(G[i] * xs[i]))
            worst = max(worst, abs(lhs - r) / float(np.sum(np.abs(G[i]) * np.abs(xs[i]))))
        k = len(nlv)
        emit({"network": "sycamore53_d12_committed_tree", **info, "mode": "sliced hvp", "sliced_legs": D12_HVP_LEGS,
              "slices": p.n_slices, "ws_bytes_per_slice": pi["peak_bytes"], "flops_per_slice": pi["flops"],
              "setup_s": t_setup, "hvp_sliced_s": t_hvp, "value": [r.real, r.imag],
              "tangent_over_leaves_times_value": [(complex(tan) / (k * r)).real, (complex(tan) / (k * r)).imag],
              "multilinearity_leaves": sample, "multilinearity_worst_rel": worst, "leaves": k})
        del p, G, Gd
        ctx.trim()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "a") as fh:
        for line in lines:
            fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
