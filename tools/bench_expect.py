"""One value_and_grad of a Pauli-sum energy (tnc_b200.Expectation, tncb_plan_expect) against the host recipes it replaces.

Workloads:
  qaoa20:        QAOA p = 2 MaxCut on a random 3-regular 20-qubit graph (seed 1): K = 30 ZZ terms, cx rz(2γ) cx cost
                 layers and rx(2β) mixers, γ and β tied through AngleMap scales;
  qaoa20_split:  the same Hamiltonian as 30 single-edge Expectation objects, their energies and gradients summed
                 (built, timed and freed one at a time: together they do not fit on the card);
  tfim24:        a 24-qubit transverse-field Ising chain (K = 47) on an ry + cz ansatz of depth 4.
Per workload one JSON line:
  device_ms:     this call (CUDA events around it, median of the repeats, alternated with the recipes below);
  recipe_ms:     the host recipe: K host networks, stage_batch, vjp_batch(seeds = c), Angles.pullback;
  single_ms:     K single calls: stage, run, vjp(c_k) per term, the gradient blocks added by torch, then the pullback;
  split_us:      from a torch.profiler run of its own: the device time of the expect kernels against everything else,
                 and the host-to-device copies of one call.
The first line holds the card's name and power limit (nvidia-smi query, same process).

usage: python tools/bench_expect.py [--repeats 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the record says so instead of guessing
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def regular3(n, seed):
    rng = np.random.default_rng(seed)
    while True:
        stubs = rng.permutation(np.repeat(np.arange(n), 3))
        edges = {tuple(sorted((int(a), int(b)))) for a, b in stubs.reshape(-1, 2)}
        if len(edges) == 3 * n // 2 and all(a != b for a, b in edges):
            return sorted(edges)


def qaoa(n, p, seed):
    from tnc_b200 import PauliSum
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    edges = regular3(n, seed)
    theta = np.random.default_rng(seed + 1).uniform(-1, 1, 2 * p)
    c = Circuit()
    c.allocate_register(n)
    for q in range(n):
        c.append_gate("h", [], [q])
    refs = []
    for l in range(p):
        for a, b in edges:
            c.append_gate("cx", [], [a, b])
            refs.append((len(c.tensors), 0, 2 * l, 2.0))
            c.append_gate("rz", [2 * theta[2 * l]], [b])
            c.append_gate("cx", [], [a, b])
        for q in range(n):
            refs.append((len(c.tensors), 0, 2 * l + 1, 2.0))
            c.append_gate("rx", [2 * theta[2 * l + 1]], [q])
    return c, [(0.5, f"Z{a} Z{b}") for a, b in edges], AngleMap(refs, 2 * p, theta)


def tfim(n, depth, seed):
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    theta = np.random.default_rng(seed).uniform(-np.pi, np.pi, n * depth)
    c = Circuit()
    c.allocate_register(n)
    refs = []
    for d in range(depth):
        for q in range(n):
            refs.append((len(c.tensors), 0, d * n + q, 1.0))
            c.append_gate("ry", [theta[d * n + q]], [q])
        for q in range(d % 2, n - 1, 2):
            c.append_gate("cz", [], [q, q + 1])
    terms = [(-1.0, f"Z{q} Z{q + 1}") for q in range(n - 1)] + [(-0.7, f"X{q}") for q in range(n)]
    return c, terms, AngleMap(refs, n * depth, theta)


def term_networks(exp):
    from tnc_b200 import pauli_layer_matrix
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    pn = exp.network
    x, z, _ = exp.hamiltonian.masks()
    nets = []
    for xk, zk in zip(x.tolist(), z.tolist()):
        leaves = list(pn.tn.tensors)
        for leaf, q in zip(pn.layer_leaf, pn.layer_qubit):
            t = Tensor(list(leaves[leaf].legs), list(leaves[leaf].bond_dims))
            t.set_tensor_data(TensorData.Matrix(pauli_layer_matrix((xk >> q) & 1, (zk >> q) & 1)))
            leaves[leaf] = t
        nets.append(Tensor.new_composite(leaves))
    return nets


def event_ms(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    from tnc_b200 import Context
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--workload", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.workload:
        print(json.dumps(workload(Context(0), args.workload, args.repeats)), flush=True)
        return
    lines = [card()]
    for name in ("qaoa20", "qaoa20_split", "tfim24"):
        # a process per workload: the memory one leaves in the caches does not size the next one's batch
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--workload", name, "--repeats", str(args.repeats)],
                           capture_output=True, text=True, check=True)
        row = json.loads(r.stdout.strip().splitlines()[-1])
        lines.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")
    print(json.dumps(lines[0]))


def workload(ctx, name, repeats):
    import torch
    from tnc_b200 import Expectation, PauliSum
    from tnc_b200.tensornetwork import NetworkPlan
    c, terms, amap = qaoa(20, 2, 1) if name.startswith("qaoa") else tfim(24, 4, 2)
    n = c.num_qubits()
    theta = torch.tensor(amap.theta0, dtype=torch.float64, device="cuda")
    if name == "qaoa20_split":
        # the 30 single-edge plans, whose greedy light-cone paths reach 5.4 GiB of forward workspace, do not fit on the
        # card together: each group is built, timed and freed in turn, and device_ms is the sum of the groups' medians
        row = {"workload": name, "qubits": n, "terms": len(terms), "plans": len(terms), "device_ms": 0.0, "energy": 0.0,
               "flops_per_group": [], "note": "groups timed one at a time, each plan freed before the next is built"}
        for t in terms:
            e = Expectation(c, PauliSum([t], n_qubits=n), angle_map=amap, ctx=ctx)
            row["flops_per_group"].append(e.plan.info()["flops"])
            row["energy"] += e.value_and_grad(theta)[0]
            row["device_ms"] += statistics.median(event_ms(lambda: e.value_and_grad(theta)) for _ in range(repeats))
            del e
        return row
    exps = [Expectation(c, PauliSum(terms, n_qubits=n), angle_map=amap, ctx=ctx)]

    def device():
        out = [e.value_and_grad(theta) for e in exps]
        return sum(o[0] for o in out), sum(o[1] for o in out)
    row = {"workload": name, "qubits": n, "terms": len(terms), "plans": 1, "flops_per_term": exps[0].plan.info()["flops"],
           "peak_bytes": exps[0].plan.info()["peak_bytes"]}
    E, g = device()
    recipe = single = None
    if len(exps) == 1:
        exp = exps[0]
        wrt = exp.angle_map.leaves()
        ref = NetworkPlan.for_gradients(exp.network.tn, exp.path, wrt=wrt, ctx=ctx)
        one = NetworkPlan.for_gradients(exp.network.tn, exp.path, wrt=wrt, ctx=ctx)
        _, _, coeff = exp.hamiltonian.masks()
        seeds = coeff.astype(np.complex128)

        def recipe():
            ref.stage_batch(term_networks(exp))
            gs = ref.vjp_batch_blocks(0, len(coeff), seeds=seeds, rows=False, sum=True, values=True)
            gs[0].free()
            rows = exp.angles.pullback(theta, gs[2])[0]
            gs[2].free()
            rows.free()

        def single():
            total = None
            for net, ck in zip(term_networks(exp), coeff.tolist()):
                one.stage(net)
                one.run()
                blk = one.vjp_block(np.array(ck, dtype=np.complex128))
                t = blk.to_torch()
                blk.free()
                total = t if total is None else total + t
            from tnc_b200 import DeviceTensor
            d = DeviceTensor.from_torch(ctx, total)
            rows = exp.angles.pullback(theta, d)[0]
            d.free()
            rows.free()
        recipe()
        single()
    ts = {"device_ms": [], "recipe_ms": [], "single_ms": []}
    for _ in range(repeats):           # alternated, so that the three see the same card state
        ts["device_ms"].append(event_ms(device))
        if recipe:
            ts["recipe_ms"].append(event_ms(recipe))
            ts["single_ms"].append(event_ms(single))
    for k, v in ts.items():
        row[k] = statistics.median(v) if v else None
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device()
        torch.cuda.synchronize()
    mine = rest = 0.0
    h2d = 0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        if "Memcpy HtoD" in ev.name:
            h2d += 1
        elif "expect_" in ev.name:
            mine += us
        else:
            rest += us
    row["split_us"] = {"expect_kernels": round(mine, 2), "other": round(rest, 2), "h2d_copies": h2d,
                       "h2d_copies_per_plan": h2d / len(exps)}
    row["energy"] = E
    row["max_imag"] = max(e.max_imag for e in exps)
    return row


if __name__ == "__main__":
    main()
