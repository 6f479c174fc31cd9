"""Cost of forward mode: NetworkPlan.for_tangents + jvp against the plain plan's run, and Jacobian columns from
jvp_batch against Jacobian rows from vjp_batch.

Workloads:
  bench   bench.py's network (36 qubits, 10 rounds, seed 1, bench.py's path), every leaf requested
  amp20   a 20-qubit, 10-round random-circuit amplitude network, every leaf requested
For each, the plain plan's run and the tangent plan's jvp (random complex tangents of every leaf, packed on the device
once) are timed with CUDA events on the context stream, alternating the two arms per repeat.  One JSON line per
workload: median / min / max milliseconds of each arm, the measured tangent-over-forward time ratio next to the MNK
volume ratio of the two plans (3 with every leaf requested: a count, not a measurement), both workspaces, and the device
time per kernel name of one jvp from a separate torch.profiler pass.

Jacobian workload (jac16): a 16-qubit, 10-round partial-amplitude network with 10 open qubits (2^10 outputs), P
directions over every leaf.  jvp_batch over P stride-0 instances of the network (one tangent row per direction) against
vjp_batch over 2^10 stride-0 instances with one-hot seeds (the Jacobian's rows) followed by rows x directions on the
device, so that both arms end with the same [P, 2^10] columns; host clock around synchronised work, arms alternating.
The line records the largest difference between the two arms' columns relative to their largest entry.

The first line holds the card's name and power limit (nvidia-smi query, in the same process).

usage: python tools/bench_jvp.py [--repeats 5] [--workloads bench,amp20,jac16] [--directions 8,64]
                                 [--out profiles/h100_jvp.jsonl]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import card, greedy  # noqa: E402


def crandn(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def network(name):
    if name == "bench":
        import bench
        tn = bench.build_network()
        return tn, bench.greedy_path(tn)
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(20, 10, 0.5, 0.5, np.random.default_rng(20))
    tn = c.into_amplitude_network("0" * 20)[0]
    return tn, greedy(tn)


def event_ms(ctx, fn, tb):
    """device milliseconds of fn() on the context stream (CUDA events recorded there)"""
    import torch
    _, ext = tb.torch_streams(ctx)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx.synchronize()
    e0.record(ext)
    res = fn()
    e1.record(ext)
    e1.synchronize()
    return e0.elapsed_time(e1), res


def kernel_times(ctx, fn):
    """{kernel name: [device ms, launches]} of one fn() from torch.profiler (CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    ctx.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        ctx.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        t = getattr(ev, "device_time", None)
        if t is None:
            t = ev.cuda_time
        name = ev.name if len(ev.name) <= 80 else ev.name[:77] + "..."
        rec = out.setdefault(name, [0.0, 0])
        rec[0] += t / 1e3
        rec[1] += 1
    return dict(sorted(out.items(), key=lambda kv: -kv[1][0]))


def forward_vs_tangent(ctx, name, repeats):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = network(name)
    plain = NetworkPlan(tn, path, ctx=ctx)
    plain.stage(tn)
    tplan = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    tplan.stage(tn)
    rng = np.random.default_rng(3)
    offs = tplan.grad_offsets()
    block = tplan._tangent_block({i: crandn(rng, s) for i, (o, s) in enumerate(zip(offs, tplan.leaf_shapes)) if o >= 0})

    def run():
        out = plain.run()
        out.tensordata.matrix.free()

    def jvp():
        v, t = C.c_void_p(), C.c_void_p()
        tb._lib.check(ctx._l.tncb_plan_jvp(ctx.handle, tplan.handle, block.handle, C.byref(v), C.byref(t)))
        for h in (v, t):
            ctx._l.tncb_tensor_free(ctx.handle, h)

    for fn in (run, jvp):                      # warm-up: modules, K1 tables, arena slabs
        event_ms(ctx, fn, tb)
    times = {"run": [], "jvp": []}
    for r in range(repeats):
        for k in (["run", "jvp"] if r % 2 == 0 else ["jvp", "run"]):
            times[k].append(event_ms(ctx, run if k == "run" else jvp, tb)[0])
    fi, ti = plain.info(), tplan.info()
    stats = lambda ts: {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}
    rec = {"record": "tangent_vs_forward", "workload": name, "leaves": len(tplan.leaf_shapes),
           "requested": sum(o >= 0 for o in offs), "repeats": repeats, "forward_pairs": fi["pairs"],
           "tangent_plan_pairs": ti["pairs"], "mnk_ratio": ti["flops"] / fi["flops"],
           "run_ms": stats(times["run"]), "jvp_ms": stats(times["jvp"]),
           "time_ratio_median": statistics.median(times["jvp"]) / statistics.median(times["run"]),
           "forward_peak_bytes": fi["peak_bytes"], "tangent_workspace_bytes": ti["peak_bytes"],
           "jvp_kernels": {k: {"ms": round(v[0], 4), "launches": v[1]} for k, v in list(kernel_times(ctx, jvp).items())[:12]}}
    block.free()
    del plain, tplan
    ctx.trim()
    return rec


def jacobian(ctx, directions, repeats):
    """[P, 2^10] Jacobian columns of a 16-qubit partial-amplitude network: jvp_batch vs vjp_batch + rows x directions"""
    import torch
    from tnc_b200 import DeviceTensor
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    c = random_circuit_builder(16, 10, 0.5, 0.5, np.random.default_rng(16))
    tn = c.into_amplitude_network("*" * 10 + "0" * 6)[0]
    path = greedy(tn)
    tplan = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    gplan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    dims = gplan.result_dims
    n_out = int(np.prod(dims))
    offs = tplan.grad_offsets()
    assert offs == gplan.grad_offsets()
    te = sum(int(np.prod(s)) for o, s in zip(offs, tplan.leaf_shapes) if o >= 0)
    gplan.stage_instances(tn, {}, n_out)
    seeds = DeviceTensor.from_numpy(ctx, np.eye(n_out, dtype=np.complex128).reshape((n_out,) + tuple(dims)))
    dev = torch.device("cuda", ctx.device)
    lines = []
    for P in directions:
        rng = np.random.default_rng(P)
        dirs = crandn(rng, (P, te))
        dirs_t = torch.from_numpy(dirs).to(dev)
        tangents = {i: dirs_t[:, o:o + int(np.prod(s))].reshape((P,) + tuple(s))
                    for i, (o, s) in enumerate(zip(offs, tplan.leaf_shapes)) if o >= 0}
        tplan.stage_instances(tn, {}, P)

        def fwd():
            _, rows = tplan.jvp_batch_blocks(0, P, tangents, values=False)
            out = rows.to_torch().reshape(P, n_out)
            rows.free()
            return out

        def rev():
            _, rows, _ = gplan.vjp_batch_blocks(0, n_out, seeds, rows=True, sum=False, values=False)
            J = rows.to_torch()                       # [n_out, te]: row r = dR[r]/dX
            rows.free()
            return (J @ dirs_t.T).T                   # [P, n_out]

        def timed(fn):
            ctx.synchronize()
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            res = fn()
            ctx.synchronize()
            torch.cuda.synchronize(dev)
            return time.perf_counter() - t0, res

        _, a = timed(fwd)
        _, b = timed(rev)
        diff = float((a - b).abs().max() / b.abs().max())
        times = {"jvp_batch": [], "vjp_batch": []}
        for r in range(repeats):
            for k in (["jvp_batch", "vjp_batch"] if r % 2 == 0 else ["vjp_batch", "jvp_batch"]):
                times[k].append(1e3 * timed(fwd if k == "jvp_batch" else rev)[0])
        stats = lambda ts: {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}
        lines.append({"record": "jacobian", "workload": "jac16", "outputs": n_out, "directions": P, "tangent_elems": te,
                      "repeats": repeats, "jvp_batch_ms": stats(times["jvp_batch"]), "vjp_batch_ms": stats(times["vjp_batch"]),
                      "vjp_over_jvp_median": statistics.median(times["vjp_batch"]) / statistics.median(times["jvp_batch"]),
                      "max_rel_diff": diff})
    seeds.free()
    del tplan, gplan
    ctx.trim()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workloads", default="bench,amp20,jac16")
    ap.add_argument("--directions", default="8,64")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_jvp.jsonl"))
    args = ap.parse_args()
    import tnc_b200 as tb
    ctx = tb.Context(0)
    lines = [{"record": "card", **card()}]
    print(json.dumps(lines[0]), flush=True)
    for wl in args.workloads.split(","):
        recs = jacobian(ctx, [int(p) for p in args.directions.split(",")], args.repeats) if wl == "jac16" \
            else [forward_vs_tangent(ctx, wl, args.repeats)]
        for rec in recs:
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
