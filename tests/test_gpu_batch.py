"""Instance-batched plan execution (tncb_plan_run_batch / NetworkPlan.run_batch).

Many networks of one structure (other bitstrings, input states, payload matrices) are staged once with stage_slices;
run_batch contracts them each on its own with the instance as a grid dimension of every kernel.  Every launch decision
is the single-network one, so row i must equal run_slices(i, N) bit for bit, on every kernel route:

  1. K0 (level-batched and plain) and K1 in random-circuit amplitude networks, K2 in a 13-qubit statevector network,
     K0 split-K on plan scratch, K1 DMMA in the 64x64, 32x64 and 64x32 tiles, DMMA split-K (also in two groups of
     instances under the 1 GiB partials cap), and bench.py's 36-qubit network (int8 engine, panels) with 3 bitstrings.
  2. Several passes when the static-workspace limit holds only a few workspace copies, and sub-ranges.
  3. One launch per kernel for 64 instances (the instances are a grid dimension, not a host loop).
  4. The plan's own staged leaves and the other executors are untouched by a batch.
  5. Errors, with nothing allocated.
  6. 64 amplitudes of a 20-qubit circuit against its statevector."""
import ctypes as C

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = -1, -9


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


def oracle(tn, path):
    return orc.contract_tensor_network(to_oracle(tn), to_opath(path)).data


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def counted(ctx, fn):
    """(result of fn, engine counts, kernel launches) of one call, synchronised"""
    ctx.reset_stats()
    res = fn()
    ctx.synchronize()
    return res, ctx.engine_counts(), ctx.stats()["kernel_launches"]


def batch_array(plan, first=0, count=None):
    legs, dt = plan.run_batch(first, count)
    return legs, dt.to_numpy()


def check_batch(ctx, plan, nets, path, rel=None, pair_tol=None, oracle_rows=None):
    """run_batch(0, N) against run_slices(i, N) bit for bit and against the oracle; returns the batch's engine counts,
    which must be N times those of one instance"""
    n = len(nets)
    (legs, got), ec, _ = counted(ctx, lambda: batch_array(plan))
    _, ec1, _ = counted(ctx, lambda: plan.run_batch(0, 1))
    assert got.shape[0] == n
    assert ec == {k: n * v for k, v in ec1.items()}, (ec, ec1)
    for i in range(n):
        ref = plan.run_slices(i, n)
        assert ref.legs == legs
        assert np.array_equal(got[i], ref.to_numpy()), i
    for i in (range(n) if oracle_rows is None else oracle_rows):
        exp = oracle(nets[i], path)
        if rel is not None:
            assert abs(complex(got[i]) - complex(exp)) <= rel * abs(complex(exp)), (i, got[i], exp)
        else:
            assert np.abs(got[i] - exp).max() <= pair_tol * np.abs(exp).max(), i
    return ec1


@pytest.fixture(scope="module")
def ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()


# ================================================================================================================
# 1. bit identity on every route
# ================================================================================================================
def amplitude_nets(qubits, rounds, seed, n):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 100)
    bits = ["".join(rng.choice(["0", "1"], qubits)) for _ in range(n)]
    return [c.into_amplitude_network(b)[0] for b in bits]


@pytest.mark.parametrize("qubits,rounds", [(12, 6), (16, 8)])
def test_amplitude_bitstrings(ctx, qubits, rounds):
    """Level-batched K0 (k0_batch_inst_kernel) and plain K0; at 16 qubits and 8 rounds also K1 DMMA."""
    from tnc_b200.tensornetwork import NetworkPlan
    nets = amplitude_nets(qubits, rounds, 5, 8)
    path = greedy(nets[0])
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    assert plan.info()["kernels"] < plan.info()["pairs"]                      # some levels run as one batch launch
    plan.stage_slices(nets)
    ec1 = check_batch(ctx, plan, nets, path, rel=1e-9)
    assert ec1["k0"] > 0
    if qubits == 16:
        assert ec1["k1_dmma"] > 0, ec1


def statevector_nets(n, seed):
    """The 13-qubit statevector network (K0 steps and one K2 step) with random normalised input states"""
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, _ = random_circuit_builder(13, 4, 0.5, 0.5, np.random.default_rng(4)).into_statevector_network()
    rng = np.random.default_rng(seed)
    nets = []
    for _ in range(n):
        out = []
        for t in tn.tensors:
            if len(t.legs) == 1:
                v = rng.standard_normal(2) + 1j * rng.standard_normal(2)
                t = Tensor(t.legs, t.bond_dims)
                t.set_tensor_data(TensorData.Matrix(v / np.linalg.norm(v)))
            out.append(t)
        nets.append(Tensor.new_composite(out))
    return nets


def test_statevector_k2(ctx):
    from tnc_b200.tensornetwork import NetworkPlan
    nets = statevector_nets(6, 1)
    path = greedy(nets[0])
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    plan.stage_slices(nets)
    ec1 = check_batch(ctx, plan, nets, path, pair_tol=1e-12)
    assert ec1["k2"] == 1 and ec1["k0"] > 0, ec1


def pair_nets(a_dims, b_dims, n, seed):
    """Two-leaf networks A[m.., k] x B[k, n..] with random Matrix payloads"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(seed)
    a_legs = list(range(len(a_dims)))
    b_legs = [a_legs[-1]] + list(range(len(a_dims), len(a_dims) + len(b_dims) - 1))
    nets = []
    for _ in range(n):
        ts = []
        for legs, dims in ((a_legs, a_dims), (b_legs, b_dims)):
            t = Tensor(legs, dims)
            t.set_tensor_data(TensorData.Matrix(rng.standard_normal(dims) + 1j * rng.standard_normal(dims)))
            ts.append(t)
        nets.append(Tensor.new_composite(ts))
    return nets, ContractionPath.simple([(0, 1)])


# (A dims, B dims: the last A leg is B's first), instances, the engine the pair must reach
PAIRS = {
    "k1_64x64": ([256, 64], [64, 256], 5, "k1_dmma"),
    "k1_32x64": ([512, 128], [128, 32], 5, "k1_dmma"),          # N <= 32 < M
    "k1_64x32": ([24, 128], [128, 300], 5, "k1_dmma"),          # M <= 32 < N
    "k1_splitk": ([64, 65536], [65536, 64], 4, "k1_dmma_splitk"),
    # 2 x 16 MiB of partials per instance: 64 instances fill the 1 GiB cap, so 66 run in two groups
    "k1_splitk_groups": ([4096, 256], [256, 128], 66, "k1_dmma_splitk"),
}


@pytest.mark.parametrize("name", list(PAIRS))
def test_pair_routes(ctx, name):
    from tnc_b200.tensornetwork import NetworkPlan
    a_dims, b_dims, n, engine = PAIRS[name]
    nets, path = pair_nets(a_dims, b_dims, n, 7)
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    plan.stage_slices(nets)
    ec1 = check_batch(ctx, plan, nets, path, pair_tol=1e-12, oracle_rows=range(min(n, 6)))
    assert ec1[engine] == 1 and sum(ec1.values()) == 1, ec1


def test_k0_splitk_on_plan_scratch(ctx):
    """K = 4096 on a 3 x 5 output: K0 split-K, whose partials live in each instance's copy of the plan scratch"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(11)
    nets = []
    for _ in range(6):
        ts = []
        for legs, dims in (([0, 1, 2], [3, 64, 64]), ([3, 2, 1], [5, 64, 64])):
            t = Tensor(legs, dims)
            t.set_tensor_data(TensorData.Matrix(rng.standard_normal(dims) + 1j * rng.standard_normal(dims)))
            ts.append(t)
        nets.append(Tensor.new_composite(ts))
    path = ContractionPath.simple([(0, 1)])
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    plan.stage_slices(nets)
    ec1 = check_batch(ctx, plan, nets, path, pair_tol=1e-12)
    assert ec1["k0_splitk"] == 1, ec1


def test_bench_network_bitstrings(ctx):
    """bench.py's network (36 qubits, 488 pairs) with 3 bitstrings: the int8 engine instance by instance, the panel path,
    DMMA split-K and K0 split-K, in as many passes as the workspace limit allows"""
    import bench
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    q = bench.NET["qubits"]
    c = random_circuit_builder(q, bench.NET["rounds"], bench.NET["p1"], bench.NET["p2"], np.random.default_rng(bench.NET["seed"]))
    rng = np.random.default_rng(3)
    nets = [c.into_amplitude_network(b)[0] for b in ["0" * q] + ["".join(rng.choice(["0", "1"], q)) for _ in range(2)]]
    path = bench.greedy_path(nets[0])
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    plan.stage_slices(nets)
    ec1 = check_batch(ctx, plan, nets, path, rel=1e-9, oracle_rows=[2])
    assert ec1["k1_tcgen05"] >= 1 and ec1["k1_dmma_splitk"] >= 1 and ec1["k0_splitk"] >= 1, ec1
    del plan
    ctx.trim()


# ================================================================================================================
# 2. several passes, sub-ranges
# ================================================================================================================
def test_passes_and_ranges(ctx, monkeypatch):
    """A 4096 x 128 x 4096 pair: 2 x 8 MiB of operands and a 2^24-element (256 MiB) result, so a 1 GiB workspace limit
    holds 3 workspace copies per pass and 7 instances take 3 passes."""
    from tnc_b200.tensornetwork import NetworkPlan
    nets, path = pair_nets([4096, 128], [128, 4096], 7, 13)
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    plan.stage_slices(nets)
    plan.run_batch(0, 1)                              # builds the K1 offset tables, which later calls of the pair reuse
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    (_, full), ec, launches = counted(ctx, lambda: batch_array(plan))
    _, ec1, launches1 = counted(ctx, lambda: plan.run_batch(0, 1))
    monkeypatch.delenv("TNCB_PLAN_WS_GB")
    _, _, launches_one_pass = counted(ctx, lambda: plan.run_batch(0, 7))
    assert ec == {k: 7 * v for k, v in ec1.items()} and ec1["k1_dmma"] == 1, (ec, ec1)
    assert launches == 3 * launches1 and launches_one_pass == launches1, (launches, launches1, launches_one_pass)
    for i in range(7):
        assert np.array_equal(full[i], plan.run_slices(i, 7).to_numpy()), i
    exp = oracle(nets[4], path)
    assert np.abs(full[4] - exp).max() <= 1e-12 * np.abs(exp).max()
    for first, count in ((2, 3), (6, 1), (0, 1), (4, None), (5, 2)):
        _, part = batch_array(plan, first, count)
        stop = 7 if count is None else first + count
        assert part.shape == (stop - first,) + full.shape[1:]
        assert np.array_equal(part, full[first:stop]), (first, count)


# ================================================================================================================
# 3. the instances are a grid dimension
# ================================================================================================================
def test_one_launch_per_kernel(ctx):
    """A K0/K2-only plan: 64 instances take exactly the launches of one, and every engine counter grows 64-fold."""
    from tnc_b200.tensornetwork import NetworkPlan
    nets = statevector_nets(64, 2)
    plan = NetworkPlan(nets[0], greedy(nets[0]), ctx=ctx)
    plan.stage_slices(nets)
    _, ec1, l1 = counted(ctx, lambda: plan.run_batch(0, 1))
    _, ec64, l64 = counted(ctx, lambda: plan.run_batch(0, 64))
    assert set(k for k, v in ec1.items() if v) == {"k0", "k2"}, ec1
    assert l64 == l1, (l64, l1)
    assert ec64 == {k: 64 * v for k, v in ec1.items()}, (ec64, ec1)


# ================================================================================================================
# 4. state isolation
# ================================================================================================================
def test_batch_leaves_plan_state_alone(ctx):
    from tnc_b200.tensornetwork import NetworkPlan
    nets = statevector_nets(5, 3)
    x, y = statevector_nets(2, 4)
    path = greedy(nets[0])
    plan = NetworkPlan(nets[0], path, ctx=ctx)
    plan.stage_slices(nets)
    slice_ref = [plan.run_slices(i, 5).to_numpy() for i in range(5)]
    y_ref = plan.execute(y).to_numpy()
    plan.stage(x)
    x_ref = plan.run().to_numpy()
    _, batch = batch_array(plan)
    assert np.array_equal(plan.run().to_numpy(), x_ref)                  # the staged leaves in the plan's workspace
    assert np.array_equal(batch[3], slice_ref[3])
    assert np.array_equal(plan.execute(y).to_numpy(), y_ref)
    for i in range(5):
        assert np.array_equal(plan.run_slices(i, 5).to_numpy(), slice_ref[i]), i
    assert np.abs(x_ref - oracle(x, path)).max() <= 1e-12


# ================================================================================================================
# 5. errors
# ================================================================================================================
def raw_run_batch(ctx, plan_handle, first, count):
    out, n_out = C.c_void_p(), C.c_int()
    legs = (C.c_uint64 * 64)()
    return ctx._l.tncb_plan_run_batch(ctx.handle, plan_handle, first, count, C.byref(out), C.byref(n_out), legs)


def test_errors_allocate_nothing(ctx, monkeypatch):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    nets = statevector_nets(3, 5)
    path = greedy(nets[0])
    staged = NetworkPlan(nets[0], path, ctx=ctx)
    staged.stage_slices(nets)
    unstaged = NetworkPlan(nets[0], path, ctx=ctx)
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    not_static = NetworkPlan(nets[0], path, ctx=ctx)
    monkeypatch.delenv("TNCB_NO_STATIC")
    dev = DeviceTensor.from_numpy(ctx, np.eye(2, dtype=np.complex128))
    leaves = list(nets[0].tensors)
    idx = next(i for i, l in enumerate(leaves) if len(l.legs) == 2)          # a single-qubit gate
    t = Tensor(leaves[idx].legs, leaves[idx].bond_dims)
    t.set_tensor_data(TensorData.Matrix(dev))
    leaves[idx] = t
    device_leaf = NetworkPlan(Tensor.new_composite(leaves), path, ctx=ctx)
    other = tb.Context(0)
    try:
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        cases = [(ctx, unstaged.handle, 0, 1, ERR_INVALID),          # nothing staged
                 (other, staged.handle, 0, 1, ERR_INVALID),          # a plan of another context
                 (ctx, staged.handle, 0, 0, ERR_INVALID),            # count = 0
                 (ctx, staged.handle, 3, 1, ERR_INVALID),            # past the end
                 (ctx, staged.handle, 1, 3, ERR_INVALID),
                 (ctx, staged.handle, 2 ** 64 - 1, 2, ERR_INVALID),  # first + count wraps around
                 (ctx, not_static.handle, 0, 1, ERR_UNSUPPORTED),
                 (ctx, device_leaf.handle, 0, 1, ERR_UNSUPPORTED)]
        for c, h, first, count, want in cases:
            assert raw_run_batch(c, h, first, count) == want, (first, count, want)
            assert ctx.stats()["arena_live_bytes"] == live
        with pytest.raises(tb.TncbError) as e:
            unstaged.run_batch()
        assert e.value.status == ERR_INVALID
        assert ctx.stats()["arena_live_bytes"] == live
    finally:
        other.close()
    dev.free()


# ================================================================================================================
# 6. amplitudes against the statevector
# ================================================================================================================
def test_amplitudes_match_statevector(ctx):
    """64 amplitudes of a 20-qubit, 10-round circuit (into_amplitude_network) against the matching entries of its
    statevector (into_statevector_network + Permutor)."""
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan, contract_tensor_network
    q = 20
    c = random_circuit_builder(q, 10, 0.5, 0.5, np.random.default_rng(21))
    rng = np.random.default_rng(22)
    bits = ["".join(rng.choice(["0", "1"], q)) for _ in range(64)]
    nets = [c.into_amplitude_network(b)[0] for b in bits]
    plan = NetworkPlan(nets[0], greedy(nets[0]), ctx=ctx)
    plan.stage_slices(nets)
    _, amps = batch_array(plan)
    sv_tn, perm = c.into_statevector_network()
    sv = perm.apply(contract_tensor_network(sv_tn, greedy(sv_tn), ctx=ctx), ctx=ctx).to_numpy()
    assert sv.shape == (2,) * q and abs(np.vdot(sv, sv) - 1) <= 1e-10
    want = np.array([sv[tuple(int(ch) for ch in b)] for b in bits])
    assert amps.shape == (64,)
    assert np.abs(amps - want).max() <= 1e-12, np.abs(amps - want).max()
