"""Planning (outside every timer): partition vectors + nested paths of the bench network for 2 / 4 / 8 ranks.

    python tools/plan_partitions.py            # writes bench_inputs/c4_partitions.json

Pipeline (all seeded, metadata only): FM bisection -> 400-evaluation simulated annealing into 2 parts
(contractionpath/repartitioning.py, the step-budget restatement of the reference's SA balancer) -> the resulting
nested path flattened into one contraction tree -> tree_cut(N) (contractionpath/tree_partition.py): N subtrees +
the N-1 top nodes as the fan-in path -> 6 seeded SA chains of 1500 evaluations per N started from that cut, scored by
the predicted critical-path time on GPUs (two-roof pair model + NVLink transfer of the fan-in operands); the
candidate with the smallest predicted time is kept."""
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "bench_inputs", "c4_partitions.json")
NETWORK = {"qubits": 36, "rounds": 10, "p1": 0.5, "p2": 0.5, "seed": 1}


def build_network():
    from tnc_b200.builders import random_circuit
    return random_circuit(NETWORK["qubits"], NETWORK["rounds"], NETWORK["p1"], NETWORK["p2"], np.random.default_rng(NETWORK["seed"]))


def network_hash(tn) -> str:
    h = hashlib.sha256()
    for t in tn.tensors:
        h.update(repr((list(t.legs), list(t.bond_dims), t.tensordata.kind, t.tensordata.gate if t.tensordata.kind == "gate" else None)).encode())
    return h.hexdigest()[:16]


def _evaluate(tn, partitioning):
    """compute_solution under the device time model: (predicted critical-path seconds, critical-path flops, total flops, ptn, path)"""
    from tnc_b200.contractionpath.contraction_cost import (communication_path_cost, contract_path_cost, gpu_fanin_time_tensors,
                                                           gpu_time_tensors)
    from tnc_b200.contractionpath.repartitioning import compute_solution
    ptn, path, t_par, _ = compute_solution(tn, partitioning, None, gpu_time_tensors, gpu_fanin_time_tensors)
    locs = [contract_path_cost(ptn.tensors[i].tensors, path.nested[i], False)[0] for i in range(len(ptn.tensors))]
    exts = [c.external_tensor() for c in ptn.tensors]
    crit, _ = communication_path_cost(exts, path.toplevel, False, True, locs)
    total = sum(locs) + communication_path_cost(exts, path.toplevel, False, False, None)[0]
    return t_par, crit, total, ptn, path


def _split_to(tn, partitioning, n):
    """more parts from a good partitioning: repeatedly bisect the partition with the most local flops along its own
    (greedy) contraction tree (tree_cut of the local network into 2)"""
    from tnc_b200.contractionpath.contraction_cost import contract_path_cost
    from tnc_b200.contractionpath.paths import Cotengrust
    from tnc_b200.contractionpath.tree_partition import tree_cut
    from tnc_b200.tensornetwork.tensor import Tensor
    part = list(partitioning)
    dead = set()                                     # partitions whose tree cannot be bisected (caterpillar root)
    while len(set(part)) < n:
        best_p, best_cost, best_cut = None, -1.0, None
        for pid in sorted(set(part) - dead):
            ids = [i for i, q in enumerate(part) if q == pid]
            if len(ids) < 4:
                continue
            comp = Tensor.new_composite([tn.tensors[i] for i in ids])
            opt = Cotengrust(comp); opt.find_path()
            lp = opt.get_best_replace_path()
            cost = contract_path_cost(comp.tensors, lp, False)[0]
            if cost > best_cost:
                best_p, best_cost, best_cut = pid, cost, (ids, tree_cut(comp, lp, 2, min_leaves=1)[0])
        if best_p is None:
            break
        ids, cut = best_cut
        if len(set(cut)) < 2:
            dead.add(best_p)
            continue
        new_id = max(part) + 1
        for i, c in zip(ids, cut):
            if c == 1:
                part[i] = new_id
    order = sorted(set(part), key=part.index)
    return [order.index(b) for b in part]


def _sa_job(args):
    n, start, steps, seed = args
    from tnc_b200.contractionpath.contraction_cost import gpu_fanin_time_tensors, gpu_time_tensors
    from tnc_b200.contractionpath.repartitioning import balance_partitions
    tn = build_network()
    best, score = balance_partitions(tn, n, start, steps=steps, seed=seed, cost_fn=gpu_time_tensors, fanin_cost_fn=gpu_fanin_time_tensors)
    return n, seed, score, best


def plan(tn, parts_list=(2, 4, 8), sa_steps=400, seed=1, refine_steps=1500, refine_seeds=(1, 2, 3, 4, 5, 6), workers=0):
    """Per rank count N: start = tree-cut(N) of the 2-part SA tree (op-count objective, like the reference), refined by
    `refine_seeds` independent seeded SA chains of `refine_steps` evaluations whose objective is the predicted
    critical-path TIME on GPUs (contraction_cost.gpu_time_tensors: two-roof pair times + NVLink transfer of every
    fan-in operand); the reference anneals 48 chains for minutes on an op-count objective
    (simulated_annealing.rs:406-592).  The candidate with the smallest predicted time wins.  Deterministic."""
    import multiprocessing as mp
    from tnc_b200.contractionpath.contraction_cost import contract_path_cost
    from tnc_b200.contractionpath.repartitioning import balance_partitions, compute_solution
    from tnc_b200.contractionpath.tree_partition import flatten_nested, tree_cut
    from tnc_b200.tensornetwork.partitioning import find_partitioning
    t0 = time.time()
    init = find_partitioning(tn, 2, seed=seed)
    best, _ = balance_partitions(tn, 2, init, steps=sa_steps, seed=seed)
    ptn, ppath, _, _ = compute_solution(tn, best)
    order = sorted(set(best), key=best.index)
    flat = flatten_nested(ptn, ppath, [order.index(b) for b in best])
    out = {"network": NETWORK, "network_hash": network_hash(tn), "sa_steps": sa_steps, "seed": seed, "refine_steps": refine_steps,
           "refine_seeds": list(refine_seeds), "tree_flops": contract_path_cost(tn.tensors, flat, False)[0], "plans": {}}
    workers = workers or min(2 * len(refine_seeds) or 1, os.cpu_count() or 1)
    prev_best = None
    for n in sorted(parts_list):
        cands = [("tree_cut", tree_cut(tn, flat, n)[0])]
        if prev_best is not None:
            cands.append((f"split of the {len(set(prev_best))}-part plan", _split_to(tn, prev_best, n)))
        jobs = [(ci, cands[ci][1], refine_steps, sd) for ci in range(len(cands)) for sd in refine_seeds]
        if jobs:
            with mp.get_context("spawn").Pool(workers) as pool:
                res = pool.map(_sa_job, [(n, j[1], j[2], j[3]) for j in jobs])
            for j, (_, sd, _, part) in zip(jobs, res):
                cands.append((f"{cands[j[0]][0]} + SA seed {sd}", part))
        best_c = None
        for name, part in cands:
            t_par, crit, total, ptn_n, path_n = _evaluate(tn, part)
            if best_c is None or t_par < best_c[0]:
                best_c = (t_par, crit, total, ptn_n, path_n, name, part)
        t_par, crit, total, ptn_n, path_n, name, part = best_c
        order_n = sorted(set(part), key=part.index)
        pv = [order_n.index(b) for b in part]
        prev_best = pv
        out["plans"][str(n)] = {"partitioning": pv, "nested": {str(k): [list(p) for p in v.toplevel] for k, v in path_n.nested.items()},
                                "toplevel": [list(p) for p in path_n.toplevel], "critical_path_flops": crit, "total_flops": total,
                                "predicted_critical_path_ms": t_par * 1e3, "partition_sizes": [len(c.tensors) for c in ptn_n.tensors], "chosen": name,
                                "boundary_tensor_bytes": [16.0 * c.external_tensor().size() for c in ptn_n.tensors]}
    out["planning_seconds"] = time.time() - t0
    return out


def load(tn, n):
    """(partitioned network, nested path, facts) for n ranks from the committed plan file; None if absent or stale."""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork.partitioning import partition_tensor_network
    try:
        with open(OUT) as f:
            d = json.load(f)
    except Exception:
        return None
    if d.get("network_hash") != network_hash(tn) or str(n) not in d["plans"]:
        return None
    p = d["plans"][str(n)]
    path = ContractionPath({int(k): ContractionPath.simple([tuple(x) for x in v]) for k, v in p["nested"].items()},
                           [tuple(x) for x in p["toplevel"]])
    return partition_tensor_network(tn, p["partitioning"]), path, {k: p[k] for k in ("critical_path_flops", "total_flops", "partition_sizes", "predicted_critical_path_ms", "boundary_tensor_bytes", "chosen") if k in p}


if __name__ == "__main__":
    tn = build_network()
    d = plan(tn)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(d, f)
    for n, p in d["plans"].items():
        print(n, "parts: predicted %.2f ms, critical path %.3e flop, total %.3e, sizes %s, boundary MB %s (%s)" % (
            p["predicted_critical_path_ms"], p["critical_path_flops"], p["total_flops"], p["partition_sizes"], [round(b / 1e6, 1) for b in p["boundary_tensor_bytes"]], p["chosen"]))
    print("planning took %.1f s ->" % d["planning_seconds"], OUT)
