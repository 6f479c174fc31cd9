"""Staging leaf payloads from device memory against staging through the host.

  staging   NetworkPlan.stage_batch of B host networks against NetworkPlan.stage_instances with the B bitstring
            projectors from ONE device tensor [B, qubits, 2] (the other leaves from the host template), on a gradient
            plan.  Workloads amp16 / amp20 (16- / 20-qubit, 10-round random-circuit amplitude networks) at B = 1, 8, 64,
            512.  Both arms then run vjp_batch; its values and gradient sum must be equal bit for bit.
  training  one network_function step (forward, backward() of a linear loss, SGD step) with CPU inputs against on_device=True with CUDA
            inputs: amp16 unbatched with every gate an input; amp16 batched (bras per instance, gates shared) at B = 64
            and 512; bench.py's network (36 qubits, 489 leaves) unbatched with every leaf an input.  The first step of
            both arms starts from the same inputs; its values and gradients must be equal bit for bit.

Times: host clock around synchronised calls, median (and min, max) of --repeats repeats, the two arms alternating.  The
first line holds the card's name and power limit (nvidia-smi query); every other line one workload and size.

usage: python tools/bench_device_stage.py [--sizes 1,8,64,512] [--repeats 5] [--sections staging,training] [--out FILE]
"""
import argparse
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


def stats(ts):
    return {"median": 1e3 * statistics.median(ts), "min": 1e3 * min(ts), "max": 1e3 * max(ts)}


def alternate(arms, repeats, sync):
    """{arm: [seconds]} with the arms' order rotated per repeat"""
    times = {k: [] for k in arms}
    order = list(arms)
    for r in range(repeats):
        for k in order[r % len(order):] + order[:r % len(order)]:
            sync()
            t0 = time.perf_counter()
            arms[k]()
            sync()
            times[k].append(time.perf_counter() - t0)
    return times


def matrixify(leaves):
    from tnc_b200.contractionpath.slicing import _leaf_array
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    out = []
    for t in leaves:
        m = Tensor(list(t.legs), list(t.bond_dims))
        m.set_tensor_data(TensorData.Matrix(np.ascontiguousarray(_leaf_array(t), dtype=np.complex128)))
        out.append(m)
    return out


def staging(ctx, name, qubits, sizes, repeats):
    import torch
    from tnc_b200.contractionpath.slicing import _leaf_array
    from tnc_b200.tensornetwork import NetworkPlan, PreparedNetwork
    nets = amplitude_nets(qubits, 10, qubits, max(sizes))
    path = greedy(nets[0])
    n = len(nets[0].tensors)
    bras = torch.from_numpy(np.stack([np.stack([_leaf_array(t) for t in net.tensors[-qubits:]]) for net in nets])).cuda()
    lines = []
    for b in sizes:
        plan = NetworkPlan.for_gradients(nets[0], path, ctx=ctx)
        tmpl = PreparedNetwork(nets[0])
        X = bras[:b].contiguous()
        pay = {n - qubits + j: X[:, j, :] for j in range(qubits)}
        seeds = np.ones(b, dtype=np.complex128)
        arms = {"host": lambda: plan.stage_batch(nets[:b]), "device": lambda: plan.stage_instances(tmpl, pay, b)}
        res = {}
        for k, fn in arms.items():                 # warm-up and the bit-for-bit check
            fn()
            _, v, _, s = plan.vjp_batch(0, b, seeds, rows=False, sum=True, values=True)
            res[k] = (v, s)
        same = np.array_equal(res["host"][0], res["device"][0]) and all(
            np.array_equal(res["host"][1][leaf], res["device"][1][leaf]) for leaf in res["host"][1])
        times = alternate(arms, repeats, lambda: (ctx.synchronize(), torch.cuda.synchronize()))
        rec = {"record": "staging", "workload": name, "B": b, "leaves": n, "repeats": repeats,
               "stage_batch_ms": stats(times["host"]), "stage_instances_ms": stats(times["device"]),
               "speedup_median": statistics.median(times["host"]) / statistics.median(times["device"]),
               "bit_identical": bool(same)}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
        del plan
        ctx.trim()
    return lines


def training_step(f, xs, opt):
    """loss sum Re(w f(xs)) for a fixed w: linear, so its gradient (the seed) has the same bits on the CPU and the GPU"""
    import torch
    opt.zero_grad()
    out = f(*xs)
    (out * torch.full(out.shape, complex(0.3, -0.7), dtype=out.dtype, device=out.device)).real.sum().backward()
    opt.step()
    return out


def training(ctx, name, tn, path, wrt, batched, inputs, repeats):
    """inputs: the starting tensors (CPU), one per network_function input"""
    import torch
    from tnc_b200.autograd import network_function
    arms = {}
    first = {}
    for k, on_device in (("host", False), ("device", True)):
        f = network_function(tn, path, wrt, ctx=ctx, batched=batched, on_device=on_device)
        xs = [x.clone().cuda().requires_grad_(True) if on_device else x.clone().requires_grad_(True) for x in inputs]
        opt = torch.optim.SGD(xs, lr=1e-3)
        out = training_step(f, xs, opt)             # warm-up, from the same inputs in both arms
        first[k] = (out.detach().cpu(), [None if x.grad is None else x.grad.cpu() for x in xs])
        arms[k] = (lambda f=f, xs=xs, opt=opt: training_step(f, xs, opt))
    same = torch.equal(first["host"][0], first["device"][0]) and all(
        (a is None and b is None) or torch.equal(a, b) for a, b in zip(first["host"][1], first["device"][1]))
    times = alternate(arms, repeats, lambda: (ctx.synchronize(), torch.cuda.synchronize()))
    rec = {"record": "training_step", "workload": name, "B": int(inputs[-1].shape[0]) if batched else None,
           "inputs": len(inputs), "leaves": len(tn.tensors), "repeats": repeats,
           "cpu_inputs_ms": stats(times["host"]), "on_device_ms": stats(times["device"]),
           "speedup_median": statistics.median(times["host"]) / statistics.median(times["device"]), "bit_identical": bool(same)}
    print(json.dumps(rec), flush=True)
    ctx.trim()
    return [rec]


def training_workloads(ctx, repeats):
    import torch
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import Tensor
    lines = []
    c = random_circuit_builder(16, 10, 0.5, 0.5, np.random.default_rng(16))
    rng = np.random.default_rng(3)
    tn = Tensor.new_composite(matrixify(c.into_amplitude_network("0" * 16)[0].tensors))
    path = greedy(tn)
    leaves = list(tn.tensors)
    payload = lambda t: torch.from_numpy(np.asarray(t.tensordata.matrix).reshape([int(d) for d in t.bond_dims]).copy())
    lines += training(ctx, "amp16", tn, path, list(range(len(leaves))), (), [payload(t) for t in leaves], repeats)
    n = len(leaves)
    gates = list(range(n - 16))
    for b in (64, 512):
        bras = np.zeros((b, 2), dtype=np.complex128)
        rows = []
        for j in range(16):
            bits = rng.integers(0, 2, b)
            col = bras.copy()
            col[np.arange(b), bits] = 1.0
            rows.append(torch.from_numpy(col))
        lines += training(ctx, "amp16_batched", tn, path, gates, list(range(n - 16, n)),
                          [payload(leaves[i]) for i in gates] + rows, repeats)
    import bench
    q = bench.NET["qubits"]
    c = random_circuit_builder(q, bench.NET["rounds"], bench.NET["p1"], bench.NET["p2"], np.random.default_rng(bench.NET["seed"]))
    tn = Tensor.new_composite(matrixify(c.into_amplitude_network("0" * q)[0].tensors))
    lines += training(ctx, "bench", tn, bench.greedy_path(tn), list(range(len(tn.tensors))), (),
                      [payload(t) for t in tn.tensors], max(3, repeats // 2))
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,512")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sections", default="staging,training")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import tnc_b200 as tb
    ctx = tb.Context(0)
    lines = [{"record": "card", **card()}]
    print(json.dumps(lines[0]), flush=True)
    sizes = [int(s) for s in args.sizes.split(",")]
    sections = args.sections.split(",")
    with torch.cuda.device(ctx.device):
        if "staging" in sections:
            for name, q in (("amp16", 16), ("amp20", 20)):
                lines += staging(ctx, name, q, sizes, args.repeats)
        if "training" in sections:
            lines += training_workloads(ctx, args.repeats)
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
