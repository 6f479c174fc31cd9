"""Analytic cost model: mirror of tnc/src/contractionpath/contraction_cost.rs.
These formulas define the FLOP / byte accounting of the benchmark (SURVEY 8d) and the objective of
the partition refiner; every function is pinned by the reference's own KATs (:366-460 and the
doc-tests :15-25, :37-47, :59-69, :84-94) in tests/test_contraction_cost.py."""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

from ..tensornetwork.tensor import Tensor
from . import ContractionPath

COMPLEX64_BYTES = 16.0  # std::mem::size_of::<Complex64>() (contraction_cost.rs:135)


def contract_cost_tensors(t1: Tensor, t2: Tensor) -> float:
    """:26-32  ((K-1)*2 + K*6) * |t1 ^ t2|."""
    k = (t1 & t2).size()
    return ((k - 1.0) * 2.0 + k * 6.0) * (t1 ^ t2).size()


def contract_op_cost_tensors(t1: Tensor, t2: Tensor) -> float:
    """:50-53  |t1 | t2|."""
    return (t1 | t2).size()


def contract_size_tensors(t1: Tensor, t2: Tensor) -> float:
    """:71-74  |out| + |t1| + |t2| (elements)."""
    return (t1 ^ t2).size() + t1.size() + t2.size()


def contract_size_tensors_exact(i: Tensor, j: Tensor) -> float:
    """:95-136  bytes, with the transpose doubling: i is GEMM-ready iff the shared legs are a suffix
    of i's legs, j iff they are a prefix of j's."""
    shared = (i & j).legs
    n = len(shared)
    i_t = not (n <= len(i.legs) and i.legs[len(i.legs) - n:] == shared)
    j_t = not (n <= len(j.legs) and j.legs[:n] == shared)
    si, sj, sij = i.size(), j.size(), (i ^ j).size()
    base = si + sj + sij
    if i_t and j_t:
        el = max(2.0 * si + sj, si + 2.0 * sj, base)
    elif i_t:
        el = max(2.0 * si + sj, base)
    elif j_t:
        el = max(si + 2.0 * sj, base)
    else:
        el = base
    return el * COMPLEX64_BYTES


def _path_custom_cost(inputs: Sequence[Tensor], path: ContractionPath, cost_fn: Callable, size_fn: Callable) -> Tuple[float, float]:
    """:166-193 (nested first, then the top level; max over memory, sum over ops)."""
    op, mem = 0.0, 0.0
    inputs = list(inputs)
    for i in sorted(path.nested):
        o, m = _path_custom_cost(inputs[i].tensors, path.nested[i], cost_fn, size_fn)
        op += o
        mem = max(mem, m)
        inputs[i] = inputs[i].external_tensor()
    for (i, j) in path.toplevel:
        op += cost_fn(inputs[i], inputs[j])
        mem = max(mem, size_fn(inputs[i], inputs[j]))
        inputs[i] = inputs[i] ^ inputs[j]
    return op, mem


def contract_path_cost(inputs: List[Tensor], path: ContractionPath, only_count_ops: bool = False) -> Tuple[float, float]:
    """:146-157."""
    return _path_custom_cost(inputs, path, contract_op_cost_tensors if only_count_ops else contract_cost_tensors,
                             contract_size_tensors)


def compute_memory_requirements(inputs: List[Tensor], path: ContractionPath,
                                memory_estimator: Callable = contract_size_tensors) -> float:
    """:306-316."""
    return _path_custom_cost(inputs, path, lambda a, b: 0.0, memory_estimator)[1]


def communication_path_cost(inputs: Sequence[Tensor], path, only_count_ops: bool, only_critical_path: bool,
                            tensor_cost: Optional[Sequence[float]] = None) -> Tuple[float, float]:
    """:219-248 + :259-289: fan-in cost; the latency of a pair is its own cost plus the max
    (critical path) or the sum of its operands' latencies."""
    cost_fn = contract_op_cost_tensors if only_count_ops else contract_cost_tensors
    cost = list(tensor_cost) if tensor_cost is not None else [0.0] * len(inputs)
    assert len(cost) == len(inputs)
    if len(inputs) == 1:
        return cost[0], cost[0]
    ts = list(inputs)
    op, mem = 0.0, 0.0
    for (i, j) in path:
        mem = max(mem, contract_size_tensors(ts[i], ts[j]))
        c = cost_fn(ts[i], ts[j])
        op = c + (max(cost[i], cost[j]) if only_critical_path else cost[i] + cost[j])
        cost[i] = op
        ts[i] = ts[i] ^ ts[j]
    return op, mem


def _communication_custom_cost(inputs: Sequence[Tensor], path, cost_fn: Callable, only_critical_path: bool, tensor_cost: Sequence[float]):
    """:259-289 with an arbitrary per-pair cost."""
    cost = list(tensor_cost)
    if len(inputs) == 1:
        return cost[0], cost[0]
    ts = list(inputs)
    op, mem = 0.0, 0.0
    for (i, j) in path:
        mem = max(mem, contract_size_tensors(ts[i], ts[j]))
        op = cost_fn(ts[i], ts[j]) + (max(cost[i], cost[j]) if only_critical_path else cost[i] + cost[j])
        cost[i] = op
        ts[i] = ts[i] ^ ts[j]
    return op, mem


def communication_path_op_costs(inputs: Sequence[Tensor], path, only_count_ops: bool,
                                tensor_cost: Optional[Sequence[float]] = None):
    """:196-208: ((critical-path cost, serial cost), memory)."""
    par, _ = communication_path_cost(inputs, path, only_count_ops, True, tensor_cost)
    ser, mem = communication_path_cost(inputs, path, only_count_ops, False, tensor_cost)
    return (par, ser), mem


# ---- planning-only device time model (NOT in the reference) -------------------------------------------------------
# The reference scores partitionings by operation counts (contract_op_cost_tensors); on a GPU the pairs that dominate a
# partitioned or sliced contraction are as often bandwidth-bound (tensors of 2^28..2^30 elements meeting tiny ones) as
# compute-bound, and the fan-in moves them over NVLink.  `gpu_time_tensors` is a two-roof estimate per pair.  Its rates were
# fitted on the GPU generation this project targeted before the H100 and have NOT been re-measured on the H100; they are
# planning parameters (the committed paths in bench_inputs/ were ranked with them), and only the ranking of candidate
# trees depends on them:
#   * FP64 kernels (K1 DMMA, K2, K0): 34 TFLOP/s x K/(K+24) (short K loses to the per-chunk overheads; gate-sized K stay
#     HBM-bound);
#   * K1' (int8 engine; M, N >= 128, 256 <= K <= 2^20, MNK >= 2^28): 160 K/(K+600) TFLOP/s-equivalent (the residue /
#     reconstruction passes do not shrink with K) plus the operand conversion, 40 bytes of residue planes per operand element;
#   * 5 TB/s of HBM traffic, 5 us per launch.
# Used by tools/plan_partitions.py (partitionings) and csrc/reconf.cpp via tools/search_path.py (trees + slices): the C++
# Objective::pair restates exactly this function and tests/test_tree_reconfiguration.py pins the two against each other.
GPU_RATES = {"crt_flops": 160e12, "crt_k_half": 600.0, "dmma_flops": 34e12, "hbm_bytes": 5e12, "launch_s": 5e-6,
             "dmma_k_half": 24.0, "crt_k_max": 1048576.0, "crt_conv_bytes": 40.0, "nvlink_bytes": 6e11, "hop_s": 30e-6}


def gpu_time_mnk(m: float, n: float, k: float) -> float:
    R = GPU_RATES
    mnk = m * n * k
    flops = 8.0 * mnk
    t_mem = 16.0 * (m * k + n * k + m * n) / R["hbm_bytes"]
    t = max(flops / (R["dmma_flops"] * k / (k + R["dmma_k_half"])), t_mem)
    if m >= 128 and n >= 128 and 256 <= k <= R["crt_k_max"] and mnk >= 2.0 ** 28:
        t_crt = flops / (R["crt_flops"] * k / (k + R["crt_k_half"])) + R["crt_conv_bytes"] * (m * k + n * k) / R["hbm_bytes"]
        t = min(t, max(t_crt, t_mem))
    return t + R["launch_s"]


def gpu_time_tensors(t1: Tensor, t2: Tensor) -> float:
    k = (t1 & t2).size()
    return gpu_time_mnk((t1 - t2).size(), (t2 - t1).size(), k)


def gpu_fanin_time_tensors(t1: Tensor, t2: Tensor) -> float:
    """a fan-in pair: t2 travels to t1's device first (ncclSend/Recv of the raw buffer), then the pair runs there"""
    return gpu_time_tensors(t1, t2) + 16.0 * t2.size() / GPU_RATES["nvlink_bytes"] + GPU_RATES["hop_s"]
