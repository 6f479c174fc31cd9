"""GPU tests for whole networks: random-circuit amplitude networks (the reference's benchmark
inputs) against the oracle at sizes the oracle finishes in seconds, and size-independent
properties at larger sizes: <0|U^dagger U|0> = 1, path independence, partitioned == flat
(tnc/tests/integration_tests.rs:22-83)."""
import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu


def to_oracle(t):
    if t.is_composite():
        return orc.OTensor(children=[to_oracle(c) for c in t.tensors])
    td = t.tensordata
    if td.kind == "gate":
        d = ("gate", td.gate[0], td.gate[1], td.gate[2])
    elif td.kind == "matrix":
        d = np.asarray(td.matrix)
    else:
        d = None
    return orc.OTensor(list(t.legs), list(t.bond_dims), d)


def to_opath(p):
    return orc.OPath(list(p.toplevel), {i: to_opath(q) for i, q in p.nested.items()})


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


@pytest.mark.parametrize("qubits,rounds,seed", [(8, 6, 1), (12, 8, 2), (16, 8, 3), (20, 8, 4)])
def test_random_circuit_amplitude_vs_oracle(ctx, qubits, rounds, seed):
    from tnc_b200.builders import random_circuit
    from tnc_b200.tensornetwork import contract_tensor_network
    tn = random_circuit(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    path = greedy(tn)
    res = contract_tensor_network(tn, path, ctx=ctx)
    ref = orc.contract_tensor_network(to_oracle(tn), to_opath(path))
    assert res.legs == ref.legs == []
    got, exp = complex(res.to_numpy()), complex(ref.data)
    assert abs(got - exp) <= 1e-9 * max(abs(exp), 1e-300) + 1e-18, (got, exp)  # rel 1e-9 on amplitudes (SURVEY 8d)


def test_statevector_vs_oracle(ctx):
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import contract_tensor_network
    c = random_circuit_builder(10, 6, 0.5, 0.5, np.random.default_rng(5))
    tn, perm = c.into_statevector_network()
    path = greedy(tn)
    res = perm.apply(contract_tensor_network(tn, path, ctx=ctx), ctx=ctx)
    ref = orc.permute_to(orc.contract_tensor_network(to_oracle(tn), to_opath(path)), perm.target_leg_order)
    sv = res.to_numpy()
    assert np.abs(sv - ref.data).max() <= 1e-12
    assert abs(np.vdot(sv, sv) - 1) < 1e-12  # unitary circuit


def echo_circuit(qubits, rounds, seed):
    """U followed by U^dagger (adjoint gates in reverse order)."""
    from tnc_b200.builders import Circuit, random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    gates = [(t.tensordata.gate, None) for t in c.tensors if t.tensordata.kind == "gate"]
    # recover qubit indices by replaying the leg bookkeeping
    c2 = Circuit(); q = c2.allocate_register(qubits)
    log = []
    edge_owner = {e: i for i, e in enumerate(c2.open_edges)}
    for t in c.tensors:
        if t.tensordata.kind != "gate":
            continue
        k = len(t.legs) // 2
        qs = [edge_owner[e] for e in t.legs[:k]]
        for qq, e in zip(qs, t.legs[k:]):
            edge_owner[e] = qq
        name, angles, adj = t.tensordata.gate
        c2.append_gate(name, angles, qs, adjoint=adj)
        log.append((name, angles, qs, adj))
    for name, angles, qs, adj in reversed(log):
        c2.append_gate(name, angles, qs, adjoint=not adj)
    return c2


@pytest.mark.parametrize("qubits,rounds", [(12, 6), (16, 6), (20, 5)])
def test_echo_amplitude_is_one(ctx, qubits, rounds):
    from tnc_b200.tensornetwork import contract_tensor_network
    tn, _ = echo_circuit(qubits, rounds, 11).into_amplitude_network("0" * qubits)
    res = contract_tensor_network(tn, greedy(tn), ctx=ctx)
    assert abs(complex(res.to_numpy()) - 1.0) <= 1e-10


def test_partitioned_equals_flat(ctx):
    from tnc_b200.builders import random_circuit
    from tnc_b200.tensornetwork import Tensor, contract_tensor_network
    tn = random_circuit(10, 6, 0.5, 0.5, np.random.default_rng(22))
    flat = complex(contract_tensor_network(tn, greedy(tn), ctx=ctx).to_numpy())
    for parts in (2, 4, 7):
        n = len(tn.tensors)
        groups = [tn.tensors[i * n // parts:(i + 1) * n // parts] for i in range(parts)]
        ptn = Tensor.new_composite([Tensor.new_composite(g) for g in groups])
        path = greedy(ptn)
        assert set(path.nested) == set(range(parts))
        got = complex(contract_tensor_network(ptn, path, ctx=ctx).to_numpy())
        assert abs(got - flat) <= 1e-9 * abs(flat) + 1e-14  # amplitudes can be exactly 0


def test_path_independence(ctx):
    from tnc_b200.builders import random_circuit
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import contract_tensor_network
    tn = random_circuit(10, 6, 0.5, 0.5, np.random.default_rng(31))
    a = complex(contract_tensor_network(tn, greedy(tn), ctx=ctx).to_numpy())
    # a second valid path: greedy on the reversed tensor list, mapped back
    n = len(tn.tensors)
    from tnc_b200.tensornetwork import Tensor
    rev = Tensor.new_composite(list(reversed(tn.tensors)))
    p = greedy(rev)
    mapped = ContractionPath.simple([(n - 1 - i, n - 1 - j) for i, j in p.toplevel])
    b = complex(contract_tensor_network(tn, mapped, ctx=ctx).to_numpy())
    assert abs(a - b) <= 1e-10 * abs(a) + 1e-18


def test_twelve_partitions_equal_flat(ctx):
    """tnc/tests/integration_tests.rs:22-83: 15 qubits, 10 rounds, partitioned into 12 == flat
    (KaHyPar replaced by the FM bisection restatement, StdRng by PCG64)."""
    from tnc_b200.builders import random_circuit
    from tnc_b200.tensornetwork import contract_tensor_network
    from tnc_b200.tensornetwork.partitioning import find_partitioning, partition_tensor_network
    tn = random_circuit(15, 10, 0.5, 0.5, np.random.default_rng(52), layout="line", layout_n=15)
    flat = complex(contract_tensor_network(tn, greedy(tn), ctx=ctx).to_numpy())
    part = find_partitioning(tn, 12, seed=3)
    assert sorted(set(part)) == list(range(12))
    ptn = partition_tensor_network(tn, part)
    got = complex(contract_tensor_network(ptn, greedy(ptn), ctx=ctx).to_numpy())
    assert abs(got - flat) <= 1e-9 * abs(flat) + 1e-14


def test_sycamore_small_vs_oracle(ctx):
    """builders/sycamore_circuit.rs:74-95 structure check + amplitude vs oracle."""
    from collections import Counter
    from tnc_b200.builders import sycamore_circuit
    from tnc_b200.tensornetwork import contract_tensor_network
    c = sycamore_circuit(3, 3, np.random.default_rng(42))
    tn, _ = c.into_amplitude_network("000")
    ranks = Counter(len(t.legs) for t in tn.tensors)
    assert ranks == {1: 6, 2: 12, 4: 1}          # small_sycamore KAT
    tn, _ = sycamore_circuit(12, 4, np.random.default_rng(7)).into_amplitude_network("0" * 12)
    p = greedy(tn)
    got = complex(contract_tensor_network(tn, p, ctx=ctx).to_numpy())
    ref = complex(orc.contract_tensor_network(to_oracle(tn), to_opath(p)).data)
    assert abs(got - ref) <= 1e-9 * abs(ref) + 1e-14


def test_plan_graph_replay_matches_eager(ctx, monkeypatch):
    """K0-only plans replay as one CUDA graph; results must equal the eager pair-by-pair executor bit for bit
    (same kernels, same order) for every payload.  The eager side is a plan created with TNCB_NO_STATIC=1, which never
    gets a static layout (the plan cache behind contract_tensor_network would serve later calls with a graph too)."""
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    c = random_circuit_builder(12, 6, 0.5, 0.5, np.random.default_rng(9))
    tn0, _ = c.into_amplitude_network("0" * 12)
    path = greedy(tn0)
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    eager = NetworkPlan(tn0, path, ctx=ctx)
    monkeypatch.delenv("TNCB_NO_STATIC")
    plan = NetworkPlan(tn0, path, ctx=ctx)
    for bits in ["0" * 12, "1" * 12, "010101010101", "000011110000"]:
        c2 = random_circuit_builder(12, 6, 0.5, 0.5, np.random.default_rng(9))
        tn, _ = c2.into_amplitude_network(bits)
        ctx.reset_stats(); a = complex(plan.execute(tn).to_numpy()); la = ctx.stats()["kernel_launches"]
        ctx.reset_stats(); b = complex(eager.execute(tn).to_numpy()); lb = ctx.stats()["kernel_launches"]
        assert a == b, (bits, a, b)
        assert lb >= len(path.toplevel) > la, (la, lb)                   # eager: one launch per pair; graph: batched levels


def test_sliced_equals_flat(ctx):
    """Slicing (book/src/future_work.md:9-11): the sum over slices equals the unsliced contraction,
    also for an open (statevector) result accumulated on the device."""
    from tnc_b200.builders import random_circuit, random_circuit_builder
    from tnc_b200.contractionpath.slicing import contract_sliced, find_slices, path_cost
    from tnc_b200.tensornetwork import contract_tensor_network
    tn = random_circuit(16, 8, 0.5, 0.5, np.random.default_rng(3))
    p = greedy(tn)
    flat = complex(contract_tensor_network(tn, p, ctx=ctx).to_numpy())
    for ms in (2, 8):
        legs = find_slices(tn, p, min_slices=ms)
        assert 2 ** len(legs) >= ms
        got = complex(contract_sliced(tn, p, legs, ctx=ctx).to_numpy())
        assert abs(got - flat) <= 1e-10 * abs(flat) + 1e-14
    meta = [(t.legs, t.bond_dims) for t in tn.tensors]
    legs = find_slices(tn, p, min_slices=1, max_peak_elements=path_cost(meta, p)[1] / 4)
    assert path_cost(meta, p, legs)[1] <= path_cost(meta, p)[1] / 4          # memory-bounded slicing
    c = random_circuit_builder(8, 5, 0.5, 0.5, np.random.default_rng(4))
    tn, perm = c.into_statevector_network()
    p = greedy(tn)
    ref = contract_tensor_network(tn, p, ctx=ctx)
    legs = find_slices(tn, p, min_slices=4)
    got = contract_sliced(tn, p, legs, ctx=ctx)
    assert got.legs == ref.legs
    assert np.abs(got.to_numpy() - ref.to_numpy()).max() <= 1e-12


def test_reconfigured_and_sliced_paths_give_the_same_amplitude(ctx):
    """The planning chain of BASELINE config 5 on a network the oracle can check: greedy path, TreeReconfigure path
    (csrc/reconf.cpp) and slice_and_reconfigure + contract_sliced all return the oracle's amplitude."""
    from tnc_b200.builders import random_circuit
    from tnc_b200.contractionpath import ContractionPath, ssa_replace_ordering
    from tnc_b200.contractionpath.paths import TreeReconfigure, slice_and_reconfigure
    from tnc_b200.contractionpath.paths.cotengrust import optimize_greedy
    from tnc_b200.contractionpath.slicing import contract_sliced
    from tnc_b200.tensornetwork import contract_tensor_network
    tn = random_circuit(20, 10, 0.5, 0.5, np.random.default_rng(11))
    p0 = greedy(tn)
    ref = complex(orc.contract_tensor_network(to_oracle(tn), to_opath(p0)).data)
    opt = TreeReconfigure(tn, 10)
    opt.find_path()
    got = complex(contract_tensor_network(tn, opt.get_best_replace_path(), ctx=ctx).to_numpy())
    assert abs(got - ref) <= 1e-10 * abs(ref) + 1e-14
    inputs = [list(t.legs) for t in tn.tensors]
    size = {l: float(d) for t in tn.tensors for l, d in t.edges()}
    ssa = optimize_greedy(inputs, [], size)
    for objective in ("flops", "time"):
        sliced, new, flops, peak, _ = slice_and_reconfigure(inputs, size, ssa, opt.get_best_size() / 64.0, 10, 4, 0.0, 3, 8, objective)
        assert 1 <= len(sliced) <= 8
        rp = ssa_replace_ordering(ContractionPath.simple(new))
        got = complex(contract_sliced(tn, rp, sliced, ctx=ctx).to_numpy())
        assert abs(got - ref) <= 1e-10 * abs(ref) + 1e-14


@pytest.mark.parametrize("name,qubits,rounds", [("C3", 24, 12), ("C4", 36, 10)])
def test_baseline_networks_vs_oracle(built_lib, name, qubits, rounds):
    """BASELINE.json configs 3 and 4 as networks (seed 1, greedy Cotengrust path): the amplitude through
    contract_tensor_network against the oracle port of the same network and path (CPU: ~5 s / ~8 s), rel 1e-9
    (SURVEY 8d).  These are the only networks whose dominant pairs hit K1' (tcgen05) and K1 split-K in anger, so the
    engine counters are part of the assertion (VERDICT r1 weak #2)."""
    import torch
    import tnc_b200 as tb
    from tnc_b200.builders import random_circuit
    from tnc_b200.tensornetwork import contract_tensor_network
    tn = random_circuit(qubits, rounds, 0.5, 0.5, np.random.default_rng(1))
    path = greedy(tn)
    c = tb.Context(0)
    try:
        c.reset_stats()
        res = contract_tensor_network(tn, path, ctx=c)
        got = complex(res.to_numpy())
        ec = c.engine_counts()
        c.set_tcgen05_slices(0)                       # the same network on the FP64 pipe only
        got_dmma = complex(contract_tensor_network(tn, path, ctx=c).to_numpy())
    finally:
        c.close()
    torch.set_num_threads(max(1, min(16, torch.get_num_threads())))
    ref = complex(orc.contract_tensor_network(to_oracle(tn), to_opath(path), backend="torch").data)
    assert res.legs == []
    assert abs(got - ref) <= 1e-9 * abs(ref), (name, got, ref)
    assert abs(got_dmma - ref) <= 1e-9 * abs(ref), (name, got_dmma, ref)
    assert ec["k1_tcgen05"] >= 1 and ec["k1_dmma"] + ec["k1_dmma_splitk"] >= 1 and ec["k0"] >= 100, ec
    if name == "C4":
        assert ec["k1_dmma_splitk"] >= 1, ec      # the M=256, N=64, K=2^20 pair
    print(f"{name}: |gpu-cpu|/|cpu| = {abs(got - ref) / abs(ref):.2e} (tcgen05 on), {abs(got_dmma - ref) / abs(ref):.2e} (DMMA only); engines {ec}")


def test_direct_calls_reuse_a_cached_plan(built_lib):
    """tncb_contract_tensor_network compiles a plan on the second sighting of a structure and replays it afterwards
    (static layout + batched tiny pairs): far fewer launches, results bit-identical to the pair-by-pair executor, other
    payloads (bitstrings) of the same circuit served by the same plan."""
    import tnc_b200 as tb
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import contract_tensor_network
    c = tb.Context(0)
    try:
        def net(bits):
            return random_circuit_builder(12, 6, 0.5, 0.5, np.random.default_rng(9)).into_amplitude_network(bits)[0]
        tn = net("0" * 12)
        path = greedy(tn)
        c.reset_stats(); a0 = complex(contract_tensor_network(tn, path, ctx=c).to_numpy()); l0 = c.stats()["kernel_launches"]
        c.reset_stats(); a1 = complex(contract_tensor_network(tn, path, ctx=c).to_numpy()); l1 = c.stats()["kernel_launches"]
        c.reset_stats(); a2 = complex(contract_tensor_network(tn, path, ctx=c).to_numpy()); l2 = c.stats()["kernel_launches"]
        assert a0 == a1 == a2
        assert l0 >= len(path.toplevel) and l2 == l1 < l0 // 3, (l0, l1, l2)
        for bits in ("1" * 12, "010101010101"):
            tnb = net(bits)
            got = complex(contract_tensor_network(tnb, path, ctx=c).to_numpy())
            ref = complex(orc.contract_tensor_network(to_oracle(tnb), to_opath(path)).data)
            assert abs(got - ref) <= 1e-12 * abs(ref) + 1e-18
    finally:
        c.close()

