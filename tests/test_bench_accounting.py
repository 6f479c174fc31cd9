"""bench.py's accounting (no GPU): the pair count, the 8MNK flop total and the host->device bytes it reports for the headline
network are the values the committed bench line carries (tests/golden/bench_n1.json: one H100 80GB HBM3 at a 400 W power
limit), and the flop total agrees with two independent counters -- the mirror
of the reference's cost model (contraction_cost.rs:26-32: (2(K-1) + 6K) M N per pair = 8MNK - 2MN) and the oracle's per-pair
statistics on a network it can contract in seconds."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_headline_network_accounting(built_lib):
    import bench
    from tnc_b200.contractionpath.contraction_cost import contract_path_cost
    tn = bench.build_network()
    path = bench.greedy_path(tn)
    pairs, flops = bench.count_pairs(path), bench.path_flops(tn, path)
    line = json.load(open(os.path.join(ROOT, "tests", "golden", "bench_n1.json")))
    assert pairs == 488 == line["config"]["pairs"] and len(tn.tensors) == 489
    assert flops == line["config"]["flops_8mnk"] == line["roofline"]["algorithmic_flops_per_step"]
    assert bench.leaf_bytes(tn) == line["e2e"]["h2d_bytes_per_step"]
    assert line["e2e"]["d2h_bytes_per_step"] == 16                                   # one complex128 amplitude
    assert abs(line["value"] - pairs / (line["ms_per_step"] * 1e-3)) <= 1e-9 * line["value"]
    assert abs(line["zgemm_tflops"] - flops / (line["ms_per_step"] * 1e-3) * 1e-12) <= 1e-9 * line["zgemm_tflops"]
    # the reference's cost model counts 8MNK - 2MN per pair: add 2 per output element of every pair
    cost, _ = contract_path_cost(tn.tensors, path, False)
    out_elems, ts = 0.0, list(tn.tensors)
    for i, j in path.toplevel:
        ts[i] = ts[j] ^ ts[i]
        out_elems += ts[i].size()
    assert abs(cost + 2.0 * out_elems - flops) <= 1e-12 * flops


def test_partitioned_accounting_matches_the_oracle_counter(built_lib):
    """nested paths: bench.path_flops / count_pairs == the oracle's per-pair counter (it contracts a 12-qubit network)"""
    import bench
    from oracle import tnc_oracle as orc
    from tnc_b200.builders import random_circuit
    from tnc_b200.contractionpath.paths import Cotengrust
    from tnc_b200.tensornetwork import Tensor
    tn = random_circuit(12, 6, 0.5, 0.5, np.random.default_rng(6))
    n = len(tn.tensors)
    ptn = Tensor.new_composite([Tensor.new_composite(tn.tensors[:n // 3]), Tensor.new_composite(tn.tensors[n // 3:2 * n // 3]),
                                Tensor.new_composite(tn.tensors[2 * n // 3:])])
    for net in (tn, ptn):
        opt = Cotengrust(net); opt.find_path()
        path = opt.get_best_replace_path()
        stats = {}
        orc.contract_tensor_network(bench.to_oracle(net), bench.to_opath(path), stats=stats)
        assert stats["pairs"] == bench.count_pairs(path) == n - 1
        assert stats["flops"] == bench.path_flops(net, path)
