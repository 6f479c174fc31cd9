"""Cost of Hessian-vector products: NetworkPlan.for_hvp + hvp against the plain run, a gradient (run + vjp), a tangent
pass (jvp) and the finite-difference alternative (two gradient passes).

Workloads:
  bench   bench.py's network (36 qubits, 10 rounds, seed 1, bench.py's path), every leaf requested
  amp20   a 20-qubit, 10-round random-circuit amplitude network, every leaf requested
Every arm is timed with CUDA events on the context stream, the arms alternating per repeat.  bench.py's network does not
hold all four plans on one 80 GB card, so the arms run in two phases, each with its own run arm: {run, jvp} with the
plain and tangent plans, then {run, run + vjp, hvp, fd} with the gradient and Hessian-vector plans, where run is the
gradient plan's forward pass (the plain plan's pairs on the same engines).  hvp is one tncb_plan_hvp
call with random complex leaf tangents and a random seed (all four outputs); fd is two run + vjp passes, the cost of
G(X + hV) - G(X - hV) without the leaf updates between them.  One JSON line per workload: median / min / max
milliseconds of each arm, the time ratios to the run of the same phase, the MNK volume ratios of the plans (counts, not
measurements), the workspaces, and the device time per kernel name of one hvp from a separate torch.profiler pass.

The first line holds the card's name and power limit (nvidia-smi query, in the same process).

usage: python tools/bench_hvp.py [--repeats 5] [--workloads bench,amp20] [--out profiles/h100_hvp.jsonl]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import card  # noqa: E402
from bench_jvp import crandn, event_ms, kernel_times, network  # noqa: E402


def alternate(ctx, tb, arms, repeats):
    """{arm: [ms]}: every arm once to warm up, then `repeats` rounds, the order reversed every other round"""
    for fn in arms.values():
        event_ms(ctx, fn, tb)
    names = list(arms)
    times = {k: [] for k in names}
    for r in range(repeats):
        for k in (names if r % 2 == 0 else names[::-1]):
            times[k].append(event_ms(ctx, arms[k], tb)[0])
    return times


def hvp_costs(ctx, name, repeats):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = network(name)
    stats = lambda ts: {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}
    free = lambda *hs: [ctx._l.tncb_tensor_free(ctx.handle, h) for h in hs if h.value]
    plain = NetworkPlan(tn, path, ctx=ctx)
    plain.stage(tn)

    def run():
        plain.run().tensordata.matrix.free()

    # ---- phase 1: run against jvp ----
    tplan = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    tplan.stage(tn)
    rng = np.random.default_rng(3)
    offs = tplan.grad_offsets()
    tans = {i: crandn(rng, s) for i, (o, s) in enumerate(zip(offs, tplan.leaf_shapes)) if o >= 0}
    block = tplan._tangent_block(tans)

    def jvp():
        v, t = C.c_void_p(), C.c_void_p()
        tb._lib.check(ctx._l.tncb_plan_jvp(ctx.handle, tplan.handle, block.handle, C.byref(v), C.byref(t)))
        free(v, t)

    t1 = alternate(ctx, tb, {"run": run, "jvp": jvp}, repeats)
    fi, ti = plain.info(), tplan.info()
    del plain, tplan
    ctx.trim()
    # ---- phase 2: run, run + vjp, hvp, fd ----
    gplan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    gplan.stage(tn)
    hplan = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    hplan.stage(tn)
    assert hplan.grad_offsets() == offs
    seed = DeviceTensor.from_numpy(ctx, crandn(rng, hplan.result_dims))

    def forward():
        gplan.run().tensordata.matrix.free()

    def grad():
        forward()
        g = C.c_void_p()
        tb._lib.check(ctx._l.tncb_plan_vjp(ctx.handle, gplan.handle, seed.handle, C.byref(g)))
        free(g)

    def hvp():
        o = [C.c_void_p() for _ in range(4)]
        tb._lib.check(ctx._l.tncb_plan_hvp(ctx.handle, hplan.handle, block.handle, seed.handle, None, *[C.byref(x) for x in o]))
        free(*o)

    def fd():
        grad()
        grad()

    t2 = alternate(ctx, tb, {"run": forward, "run_vjp": grad, "hvp": hvp, "fd": fd}, repeats)
    gi, hi = gplan.info(), hplan.info()
    med = lambda ts: statistics.median(ts)
    rec = {"record": "hvp_vs_forward", "workload": name, "leaves": len(hplan.leaf_shapes),
           "requested": sum(o >= 0 for o in offs), "repeats": repeats, "forward_pairs": fi["pairs"],
           "hvp_plan_pairs": hi["pairs"],
           "mnk_ratio": {"run_vjp": gi["flops"] / fi["flops"], "jvp": ti["flops"] / fi["flops"], "hvp": hi["flops"] / fi["flops"]},
           "phase1_ms": {k: stats(v) for k, v in t1.items()}, "phase2_ms": {k: stats(v) for k, v in t2.items()},
           "time_ratio_median": {"jvp": med(t1["jvp"]) / med(t1["run"]), "run_vjp": med(t2["run_vjp"]) / med(t2["run"]),
                                 "hvp": med(t2["hvp"]) / med(t2["run"]), "fd": med(t2["fd"]) / med(t2["run"])},
           "workspace_bytes": {"run": fi["peak_bytes"], "run_vjp": gi["peak_bytes"], "jvp": ti["peak_bytes"],
                               "hvp": hi["peak_bytes"]},
           "hvp_kernels": {k: {"ms": round(v[0], 4), "launches": v[1]} for k, v in list(kernel_times(ctx, hvp).items())[:12]}}
    block.free()
    seed.free()
    del gplan, hplan
    ctx.trim()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workloads", default="bench,amp20")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_hvp.jsonl"))
    args = ap.parse_args()
    import tnc_b200 as tb
    ctx = tb.Context(0)
    lines = [{"record": "card", **card()}]
    print(json.dumps(lines[0]), flush=True)
    for wl in args.workloads.split(","):
        rec = hvp_costs(ctx, wl, args.repeats)
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
