"""Throughput of instance-batched Hessian-vector products: NetworkPlan.hvp_batch_blocks against the loop of single
tncb_plan_hvp calls on the same staged Hessian-vector plan (every leaf requested), in one process, the two arms
alternating per repeat, host clock around synchronised calls.

Workloads:
  block     Hessian blocks: P directions of one network (amp16 / amp20: 16- / 20-qubit, 10-round random-circuit
            amplitude networks) at P = 8, 64, 512, plus the full Hessian of amp16 (P = tangent_elems) if it fits.  The
            batched call returns R, Ṙ, G and Ġ rows; the loop calls hvp once per direction with the tangent row already
            on the device and the same four outputs.
  sampled   amp16 with B = 8, 64, 512 random output bitstrings from one [B, q, 2] device tensor, per-instance seeds and
            seed tangents: hvp_batch with grad_tangent_sum only, against the loop set_leaves(bitstring b) + hvp(row b,
            seed b, seed tangent b) returning Ġ_b (the loop's summation is not timed).
Per line: calls/s of both arms (median, min, max over the repeats), the speed-up of the medians, kernel launches of one
call of each arm, and whether the batched outputs equal the loop's bit for bit (rows, and the sum against the left fold
of the loop's rows).  The first line holds the card's name and power limit (nvidia-smi query).

usage: python tools/bench_hvp_batch.py [--sizes 8,64,512] [--repeats 5] [--workloads block,sampled] [--out FILE]
"""
import argparse
import ctypes as C
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


def raw_hvp(ctx, plan, tangents, seed=None, seed_tangent=None, outs=(True,) * 4):
    """one tncb_plan_hvp on device inputs; DeviceTensors (None where not requested)"""
    from tnc_b200 import DeviceTensor
    from tnc_b200._lib import check
    o = [C.c_void_p() if w else None for w in outs]
    h = lambda t: t.handle if t is not None else None
    check(ctx._l.tncb_plan_hvp(ctx.handle, plan.handle, tangents.handle, h(seed), h(seed_tangent),
                               *[C.byref(x) if x is not None else None for x in o]))
    return [None if x is None else DeviceTensor.adopt(ctx, x) for x in o]


def free_all(ts):
    for t in ts:
        if t is not None:
            t.free()


def launches(ctx, fn):
    ctx.synchronize()
    ctx.reset_stats()
    free_all(fn())
    ctx.synchronize()
    return ctx.stats()["kernel_launches"]


def timed(ctx, arms, repeats):
    """{arm: [seconds]}: the arms alternate, each call synchronised, its outputs freed outside the window"""
    times = {k: [] for k in arms}
    order = list(arms)
    for r in range(repeats):
        for k in order[r % len(order):] + order[:r % len(order)]:
            ctx.synchronize()
            t0 = time.perf_counter()
            res = arms[k]()
            ctx.synchronize()
            times[k].append(time.perf_counter() - t0)
            free_all(res)
    return times


def summary(times, n, ctx, arms, identical):
    rate = lambda ts: {"median": n / statistics.median(ts), "min": n / max(ts), "max": n / min(ts)}
    rec = {f"{k}_per_s": rate(ts) for k, ts in times.items()}
    rec["speedup_median"] = statistics.median(times["loop"]) / statistics.median(times["batched"])
    rec.update({f"launches_{k}": launches(ctx, fn) for k, fn in arms.items()})
    rec["bit_identical"] = bool(identical)
    return rec


def hessian_block(ctx, plan, rows, repeats):
    """P directions of the staged network: hvp_batch rows against the loop of hvp"""
    from tnc_b200 import DeviceTensor
    p = rows.shape[0]
    block = DeviceTensor.from_numpy(ctx, rows)
    singles = [DeviceTensor.from_numpy(ctx, r) for r in rows]
    arms = {"batched": lambda: plan.hvp_batch_blocks(p, block, outputs=(True, True, True, False, True, False)),
            "loop": lambda: [x for t in singles for x in raw_hvp(ctx, plan, t)]}
    got = [None if x is None else x.to_numpy() for x in arms["batched"]()]
    loop = [x.to_numpy() for x in arms["loop"]()]
    identical = all(np.array_equal(got[k][i], loop[4 * i + j]) for i in range(p) for j, k in enumerate((0, 1, 2, 4)))
    rec = summary(timed(ctx, arms, repeats), p, ctx, arms, identical)
    free_all([block] + singles)
    return rec


def sampled(ctx, plan, bit_leaves, onehot, tangents, seeds, seed_tans, repeats):
    """B bitstrings from one [B, q, 2] device tensor: hvp_batch's Ġ sum against the loop set_leaves + hvp"""
    import torch
    from tnc_b200 import DeviceTensor
    b = onehot.shape[0]
    dev_bits = torch.tensor(onehot, device=torch.device("cuda", ctx.device))
    payloads = {leaf: dev_bits[:, j, :] for j, leaf in enumerate(bit_leaves)}
    t_rows = [DeviceTensor.from_numpy(ctx, r) for r in tangents]
    s_rows = [DeviceTensor.from_numpy(ctx, np.asarray(s)) for s in seeds]
    sd_rows = [DeviceTensor.from_numpy(ctx, np.asarray(s)) for s in seed_tans]
    d_t, d_s, d_sd = (DeviceTensor.from_numpy(ctx, x) for x in (tangents, seeds, seed_tans))
    only_gd = (False, False, False, True)

    def loop():
        out = []
        for i in range(b):
            plan.set_leaves({leaf: dev_bits[i, j, :] for j, leaf in enumerate(bit_leaves)})
            out += raw_hvp(ctx, plan, t_rows[i], s_rows[i], sd_rows[i], only_gd)
        return out
    arms = {"batched": lambda: plan.hvp_batch_blocks(b, d_t, d_s, d_sd, payloads, outputs=(False,) * 5 + (True,)),
            "loop": loop}
    total = arms["batched"]()[5].to_numpy()
    rows = [x.to_numpy() for x in loop() if x is not None]
    identical = np.array_equal(total, functools.reduce(np.add, rows, np.zeros_like(total)))
    rec = summary(timed(ctx, arms, repeats), b, ctx, arms, identical)
    free_all(t_rows + s_rows + sd_rows + [d_t, d_s, d_sd])
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8,64,512")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--workloads", default="block,sampled")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    ctx = tb.Context(0)
    lines = [{"record": "card", **card()}]
    print(json.dumps(lines[0]), flush=True)
    sizes = [int(s) for s in args.sizes.split(",")]

    def emit(rec):
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    for wl in args.workloads.split(","):
        nets = {"amp16": amplitude_nets(16, 10, 16, 1, first_zero=True)[0],
                "amp20": amplitude_nets(20, 10, 20, 1, first_zero=True)[0]}
        for name, tn in nets.items():
            if wl == "sampled" and name != "amp16":
                continue
            plan = NetworkPlan.for_hvp(tn, greedy(tn), ctx=ctx)
            plan.stage(tn)
            info = plan.info()
            offs = plan.grad_offsets()
            te = sum(int(np.prod(s)) for o, s in zip(offs, plan.leaf_shapes) if o >= 0)
            head = {"record": wl, "network": name, "leaves": len(plan.leaf_shapes), "tangent_elems": te,
                    "hvp_workspace_bytes": info["peak_bytes"], "repeats": args.repeats}
            rng = np.random.default_rng(7)
            if wl == "block":
                for p in sizes + ([te] if name == "amp16" else []):
                    rows = rng.standard_normal((p, te)) + 1j * rng.standard_normal((p, te)) if p != te else np.eye(te)
                    try:
                        emit({**head, "P": p, "full_hessian": p == te, **hessian_block(ctx, plan, rows, args.repeats)})
                    except tb.TncbError as e:
                        emit({**head, "P": p, "full_hessian": p == te, "error": str(e)})
            else:
                q = 16
                k = len(plan.leaf_shapes)
                for b in sizes:
                    bits = rng.integers(0, 2, (b, q))
                    onehot = np.zeros((b, q, 2), np.complex128)
                    onehot[np.arange(b)[:, None], np.arange(q)[None, :], bits] = 1.0
                    tangents = rng.standard_normal((b, te)) + 1j * rng.standard_normal((b, te))
                    seeds = rng.standard_normal(b) + 1j * rng.standard_normal(b)
                    seed_tans = rng.standard_normal(b) + 1j * rng.standard_normal(b)
                    emit({**head, "B": b, **sampled(ctx, plan, list(range(k - q, k)), onehot, tangents, seeds, seed_tans,
                                                    args.repeats)})
            del plan
            ctx.trim()
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
