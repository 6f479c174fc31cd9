"""Instance-batched reverse mode (tncb_plan_stage_batch / tncb_plan_vjp_batch, NetworkPlan.vjp_batch, and
network_function(..., batched=...)).

Many networks of one gradient plan's structure run forward and backward in one walk over the schedule, the instance a
grid dimension of every kernel.  Every launch decision is the single-network one, so:

  1. on every route (K0 and its level batches, K1 DMMA in three tiles and split-K, K2 with the long K0 split-K reductions
     of its backward, the int8 engine of bench.py's network) each row of values / gradients equals a fresh
     stage + run + vjp on the same plan bit for bit, the gradient sum equals the left fold of the rows bit for bit, and
     the engine counters grow count-fold;
  2. the rows agree with torch autograd through a CPU replay of the path;
  3. several passes under a small static-workspace limit, and sub-ranges, give the same bits;
  4. 64 instances take the launches of one;
  5. leaves that need more leg groups than the gather holds take K3, per instance;
  6. the plan's own staged leaves and forward state are untouched, and the other batched entry points stay refused;
  7. every error, with the arena's live bytes unchanged;
  8. torch: gradcheck with a batched and a shared input, and the angle gradient of sum_b |psi(b)|^2 over 16 bitstrings
     against finite differences and against 16 unbatched calls."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_OOM, ERR_UNSUPPORTED = -1, -2, -5, -9


@pytest.fixture(scope="module")
def ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()


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


def leaf_array(t):
    td = t.tensordata
    if td.kind == "gate":
        d = orc.OTensor(list(t.legs), list(t.bond_dims), ("gate", td.gate[0], td.gate[1], td.gate[2])).materialise()
    elif td.kind == "matrix":
        d = np.asarray(td.matrix)
    else:
        return None
    return np.asarray(d, dtype=np.complex128).reshape([int(x) for x in t.bond_dims])


def random_seeds(shape, n, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n,) + tuple(shape)) + 1j * rng.standard_normal((n,) + tuple(shape))


# ------------------------------------------------------------------------------------------------ networks
def amplitude_nets(qubits, rounds, seed, n):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 100)
    bits = ["".join(rng.choice(["0", "1"], qubits)) for _ in range(n)]
    return [c.into_amplitude_network(b)[0] for b in bits]


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


def matrix_nets(specs, n, seed):
    """networks of Matrix leaves with random payloads; specs = [(legs, dims)]"""
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(seed)
    nets = []
    for _ in range(n):
        ts = []
        for legs, dims in specs:
            t = Tensor(legs, dims)
            t.set_tensor_data(TensorData.Matrix(rng.standard_normal(dims) + 1j * rng.standard_normal(dims)))
            ts.append(t)
        nets.append(Tensor.new_composite(ts))
    return nets


def pair_nets(a_dims, b_dims, n, seed):
    """Two-leaf networks A[m.., k] x B[k, n..]"""
    from tnc_b200.contractionpath import ContractionPath
    a_legs = list(range(len(a_dims)))
    b_legs = [a_legs[-1]] + list(range(len(a_dims), len(a_dims) + len(b_dims) - 1))
    return matrix_nets([(a_legs, a_dims), (b_legs, b_dims)], n, seed), ContractionPath.simple([(0, 1)])


# ------------------------------------------------------------------------------------------------ the check
def per_instance(ctx, plan, nets, seeds):
    """fresh stage + run + vjp of every instance on the same plan; the engine counts of instance 0"""
    vals, grads, ec1 = [], [], None
    for i, net in enumerate(nets):
        plan.stage(net)
        ctx.synchronize()
        (v, g), ec, _ = counted(ctx, lambda: (plan.run().to_numpy(), plan.vjp(None if seeds is None else seeds[i])))
        if ec1 is None:
            ec1 = ec
        vals.append(v)
        grads.append(g)
    return vals, grads, ec1


def check_batch(ctx, plan, nets, seeds):
    """vjp_batch(0, n) with rows and sum against per-instance runs: values and rows bit for bit, the sum as the left
    fold of the rows bit for bit, the engine counters n-fold.  Returns the counts of one instance."""
    n = len(nets)
    plan.stage_batch(nets)
    (legs, vals, rows, total), ec, _ = counted(ctx, lambda: plan.vjp_batch(0, n, seeds, rows=True, sum=True))
    ref_vals, ref_grads, ec1 = per_instance(ctx, plan, nets, seeds)
    assert legs == plan.result_legs
    assert vals.shape == (n,) + plan.result_dims
    want = {k: n * v for k, v in ec1.items()}
    want["permute"] *= 2                                  # K3 leaves: one permute into the row, one for the sum
    assert ec == want, (ec, ec1)
    assert sorted(rows) == sorted(ref_grads[0]) == sorted(total)
    for i in range(n):
        assert np.array_equal(vals[i], ref_vals[i]), i
        for leaf, g in ref_grads[i].items():
            assert np.array_equal(rows[leaf][i], g), (i, leaf)
    for leaf in rows:
        fold = functools.reduce(np.add, [rows[leaf][i] for i in range(n)], np.zeros(rows[leaf].shape[1:], np.complex128))
        assert np.array_equal(total[leaf], fold), leaf
    return ec1


# ================================================================================================================
# 1. every route
# ================================================================================================================
@pytest.mark.parametrize("qubits,rounds", [(12, 6), (16, 8)])
def test_amplitude_bitstrings(ctx, qubits, rounds):
    """Level-batched and plain K0 in both passes; at 16 qubits and 8 rounds also K1 DMMA.  Per-instance complex seeds."""
    from tnc_b200.tensornetwork import NetworkPlan
    nets = amplitude_nets(qubits, rounds, 5, 6)
    plan = NetworkPlan.for_gradients(nets[0], greedy(nets[0]), ctx=ctx)
    ec1 = check_batch(ctx, plan, nets, random_seeds((), 6, 1))
    assert ec1["k0"] > 0, ec1
    if qubits == 16:
        assert ec1["k1_dmma"] > 0, ec1


def test_statevector_k2(ctx):
    """K2 and the long K0 split-K reductions of its backward (partials on each copy's plan scratch); a [B, 2, .., 2]
    seed"""
    from tnc_b200.tensornetwork import NetworkPlan
    nets = statevector_nets(5, 1)
    plan = NetworkPlan.for_gradients(nets[0], greedy(nets[0]), ctx=ctx)
    ec1 = check_batch(ctx, plan, nets, random_seeds(plan.result_dims, 5, 2))
    assert plan.result_dims == (2,) * 13
    assert ec1["k2"] >= 2 and ec1["k0_splitk"] >= 1, ec1


# (A dims, B dims: the last A leg is B's first), instances, the engine the forward pair reaches
PAIRS = {
    "k1_64x64": ([256, 64], [64, 256], 4, "k1_dmma"),
    "k1_32x64": ([512, 128], [128, 32], 4, "k1_dmma"),          # N <= 32 < M
    "k1_64x32": ([24, 128], [128, 300], 4, "k1_dmma"),          # M <= 32 < N
    "k1_splitk": ([64, 65536], [65536, 64], 3, "k1_dmma_splitk"),
}


@pytest.mark.parametrize("name", list(PAIRS))
def test_pair_routes(ctx, name):
    from tnc_b200.tensornetwork import NetworkPlan
    a_dims, b_dims, n, engine = PAIRS[name]
    nets, path = pair_nets(a_dims, b_dims, n, 7)
    plan = NetworkPlan.for_gradients(nets[0], path, ctx=ctx)
    ec1 = check_batch(ctx, plan, nets, random_seeds(plan.result_dims, n, 3))
    assert ec1[engine] >= 1, ec1


def test_bench_network_bitstrings(ctx):
    """bench.py's network (36 qubits, 489 leaves, every one requested) with 3 bitstrings: the int8 engine instance by
    instance, a 15 GB gradient workspace per copy, in as many passes as the device allows"""
    sys.path.insert(0, ROOT)
    import bench
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    q = bench.NET["qubits"]
    c = random_circuit_builder(q, bench.NET["rounds"], bench.NET["p1"], bench.NET["p2"], np.random.default_rng(bench.NET["seed"]))
    rng = np.random.default_rng(3)
    nets = [c.into_amplitude_network(b)[0] for b in ["0" * q] + ["".join(rng.choice(["0", "1"], q)) for _ in range(2)]]
    plan = NetworkPlan.for_gradients(nets[0], bench.greedy_path(nets[0]), ctx=ctx)
    assert plan.info()["peak_bytes"] > 15e9
    ec1 = check_batch(ctx, plan, nets, random_seeds((), 3, 4))
    assert ec1["k1_tcgen05"] >= 1, ec1
    del plan
    ctx.trim()


# ================================================================================================================
# 2. against an independent reference
# ================================================================================================================
def ttgt(a_legs, A, b_legs, B):
    import torch
    shared = [l for l in a_legs if l in b_legs]
    am = [l for l in a_legs if l not in b_legs]
    bn = [l for l in b_legs if l not in a_legs]
    dim = dict(zip(a_legs, A.shape)) | dict(zip(b_legs, B.shape))
    size = lambda ls: int(np.prod([dim[l] for l in ls], dtype=np.int64))
    At = A.permute([a_legs.index(l) for l in shared + am]).reshape(size(shared), size(am))
    Bt = B.permute([b_legs.index(l) for l in bn + shared]).reshape(size(bn), size(shared))
    return bn + am, torch.matmul(Bt, At).reshape([dim[l] for l in bn + am])


def replay(tn, path, xs):
    it = iter(xs)

    def walk(t, p):
        if not t.tensors:
            return list(t.legs), next(it)
        slots = [walk(c, p.nested.get(i) if c.tensors else None) for i, c in enumerate(t.tensors)]
        for i, j in p.toplevel:
            slots[i] = ttgt(*slots[i], *slots[j])
            slots[j] = None
        return next(s for s in slots if s is not None)
    return walk(tn, path)


def test_rows_against_torch(ctx):
    import torch
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    nets = amplitude_nets(12, 6, 8, 2)
    path = greedy(nets[0])
    plan = NetworkPlan.for_gradients(nets[0], path, ctx=ctx)
    plan.stage_batch(nets)
    seeds = random_seeds((), 2, 5)
    _, vals, rows, _ = plan.vjp_batch(seeds=seeds)
    for i, net in enumerate(nets):
        xs = [torch.tensor(leaf_array(l), requires_grad=True) for l in leaves(net)]
        _, R = replay(net, path, xs)
        gs = torch.autograd.grad(R, xs, grad_outputs=torch.tensor(seeds[i]).conj())
        ref = [g.conj().resolve_conj().numpy() for g in gs]
        assert abs(complex(vals[i]) - complex(R.detach().numpy())) <= 1e-12 * abs(complex(R.detach().numpy()))
        gmax = max(np.abs(g).max() for g in ref)
        assert sorted(rows) == list(range(len(ref)))
        for leaf, g in enumerate(ref):
            assert np.abs(rows[leaf][i] - g).max() <= 1e-12 * gmax, (i, leaf)


# ================================================================================================================
# 3. passes and ranges
# ================================================================================================================
def test_passes_and_ranges(ctx, monkeypatch):
    """A 2048 x 128 x 4096 pair: 12 MiB of leaves, a 128 MiB result and a 128 MiB seed, so a 1 GiB workspace limit holds
    3 gradient workspace copies and 7 instances take 3 passes.  The backward pairs (K = 4096) take the int8 engine,
    which runs its instances one by one; the launch counts are checked on DMMA only, where a pass is one launch per
    kernel."""
    from tnc_b200.tensornetwork import NetworkPlan
    nets, path = pair_nets([2048, 128], [128, 4096], 7, 13)
    plan = NetworkPlan.for_gradients(nets[0], path, ctx=ctx)
    ws = plan.info()["peak_bytes"]
    assert 3 * ws <= 1 << 30 < 4 * ws, ws
    seeds = random_seeds(plan.result_dims, 7, 6)
    plan.stage_batch(nets)
    plan.vjp_batch(0, 1, seeds[:1], rows=True, sum=True)     # builds the K1 offset tables later calls reuse
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    (_, vals, rows, total), ec, launches = counted(ctx, lambda: plan.vjp_batch(0, 7, seeds, rows=True, sum=True))
    _, ec1, _ = counted(ctx, lambda: plan.vjp_batch(0, 1, seeds[:1], rows=True, sum=True))
    monkeypatch.delenv("TNCB_PLAN_WS_GB")
    (_, vals1, rows1, total1), _, launches_one_pass = counted(ctx, lambda: plan.vjp_batch(0, 7, seeds, rows=True, sum=True))
    assert ec == {k: 7 * v for k, v in ec1.items()} and ec1["k1_dmma"] >= 1, (ec, ec1)
    assert launches > launches_one_pass, (launches, launches_one_pass)
    ctx.set_tcgen05_slices(0)
    try:
        plan.vjp_batch(0, 1, seeds[:1], rows=True, sum=True)
        monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
        _, ec_d, l_passes = counted(ctx, lambda: plan.vjp_batch(0, 7, seeds, rows=True, sum=True))
        _, _, l_one = counted(ctx, lambda: plan.vjp_batch(0, 1, seeds[:1], rows=True, sum=True))
        monkeypatch.delenv("TNCB_PLAN_WS_GB")
        _, _, l_one_pass = counted(ctx, lambda: plan.vjp_batch(0, 7, seeds, rows=True, sum=True))
    finally:
        ctx.set_tcgen05_slices(8)
    assert ec_d["k1_tcgen05"] == 0, ec_d
    assert l_passes == 3 * l_one and l_one_pass == l_one, (l_passes, l_one, l_one_pass)
    assert np.array_equal(vals, vals1)
    for leaf in rows:
        assert np.array_equal(rows[leaf], rows1[leaf]) and np.array_equal(total[leaf], total1[leaf]), leaf
    for first, count in ((2, 3), (6, 1), (0, 1), (4, None), (5, 2)):
        stop = 7 if count is None else first + count
        _, v, r, _ = plan.vjp_batch(first, count, seeds[first:stop], rows=True)
        assert np.array_equal(v, vals[first:stop]), (first, count)
        for leaf in rows:
            assert np.array_equal(r[leaf], rows[leaf][first:stop]), (first, count, leaf)


# ================================================================================================================
# 4. the instances are a grid dimension
# ================================================================================================================
def test_one_launch_per_kernel(ctx):
    from tnc_b200.tensornetwork import NetworkPlan
    nets = statevector_nets(64, 2)
    plan = NetworkPlan.for_gradients(nets[0], greedy(nets[0]), ctx=ctx)
    plan.stage_batch(nets)
    seeds = random_seeds(plan.result_dims, 64, 7)
    _, ec1, l1 = counted(ctx, lambda: plan.vjp_batch(0, 1, seeds[:1], rows=True, sum=True))
    _, ec64, l64 = counted(ctx, lambda: plan.vjp_batch(0, 64, seeds, rows=True, sum=True))
    assert ec1["k1_tcgen05"] == 0, ec1
    assert l64 == l1, (l64, l1)
    assert ec64 == {k: 64 * v for k, v in ec1.items()}, (ec64, ec1)


# ================================================================================================================
# 5. the K3 route of the gather
# ================================================================================================================
def test_many_group_leaves(ctx):
    """X (11 legs) and Y (the same legs reversed) plus a matrix on two of them: both adjoints come out in the other
    leaf's order, more leg groups than a gather item holds -> K3 per instance (rows), K3 + add (sum)"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan
    legs = list(range(11))
    nets = matrix_nets([(legs[:10] + [20], [2] * 10 + [3]), ([20, 10], [3, 2]), ([10] + legs[:10][::-1], [2] * 11)], 5, 9)
    path = ContractionPath.simple([(0, 1), (0, 2)])
    plan = NetworkPlan.for_gradients(nets[0], path, ctx=ctx)
    ec1 = check_batch(ctx, plan, nets, random_seeds((), 5, 8))
    assert ec1["permute"] >= 2, ec1


# ================================================================================================================
# 6. state isolation
# ================================================================================================================
def test_batch_leaves_plan_state_alone(ctx):
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    from tnc_b200.tensornetwork.contraction import _Marshal
    nets = statevector_nets(4, 3)
    x = statevector_nets(1, 4)[0]
    plan = NetworkPlan.for_gradients(nets[0], greedy(nets[0]), ctx=ctx)
    seed = random_seeds(plan.result_dims, 1, 9)[0]
    seeds = random_seeds(plan.result_dims, 4, 10)
    plan.stage(x)
    r0 = plan.run().to_numpy()
    g0 = plan.vjp(seed)
    plan.stage(x)
    r1 = plan.run().to_numpy()
    plan.stage_batch(nets)
    _, vals, rows, _ = plan.vjp_batch(seeds=seeds)
    g1 = plan.vjp(seed)                                     # the forward state of run() survived the batch
    assert np.array_equal(r0, r1)
    for leaf in g0:
        assert np.array_equal(g0[leaf], g1[leaf]), leaf
    assert np.array_equal(plan.run().to_numpy(), r0)         # and so did the staged leaves
    _, vals2, rows2, _ = plan.vjp_batch(seeds=seeds)
    assert np.array_equal(vals, vals2)
    for leaf in rows:
        assert np.array_equal(rows[leaf], rows2[leaf]), leaf
    # the batched entry points of plain plans stay refused on a gradient plan
    m = _Marshal()
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(m.tn(nets[0])))
    out, n_out, legs = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)()
    assert ctx._l.tncb_plan_stage_slices(ctx.handle, plan.handle, 1, ptrs) == ERR_UNSUPPORTED
    assert ctx._l.tncb_plan_run_slices(ctx.handle, plan.handle, 0, 1, C.byref(out), C.byref(n_out), legs) == ERR_UNSUPPORTED
    assert ctx._l.tncb_plan_run_batch(ctx.handle, plan.handle, 0, 1, C.byref(out), C.byref(n_out), legs) == ERR_UNSUPPORTED


# ================================================================================================================
# 7. errors
# ================================================================================================================
def raw_vjp_batch(c, handle, first, count, seeds=None, outs=(True, True, True)):
    ptrs = [C.c_void_p() if o else None for o in outs]
    return c._l.tncb_plan_vjp_batch(c.handle, handle, first, count, seeds.handle if seeds is not None else None,
                                    *[C.byref(p) if p is not None else None for p in ptrs])


def rank64_net():
    """A x B over one shared leg, 64 open legs of dimension 1 in the result"""
    from tnc_b200.contractionpath import ContractionPath
    nets = matrix_nets([(list(range(32)) + [100], [1] * 32 + [2]), ([100] + list(range(32, 64)), [2] + [1] * 32)], 1, 12)
    return nets[0], ContractionPath.simple([(0, 1)])


def test_errors(ctx):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    from tnc_b200.tensornetwork.contraction import _Marshal
    amp = amplitude_nets(10, 4, 6, 3)
    amp_path = greedy(amp[0])
    sv = statevector_nets(2, 3)
    g_amp = NetworkPlan.for_gradients(amp[0], amp_path, ctx=ctx)
    g_sv = NetworkPlan.for_gradients(sv[0], greedy(sv[0]), ctx=ctx)
    unstaged = NetworkPlan.for_gradients(amp[0], amp_path, ctx=ctx)
    plain = NetworkPlan(amp[0], amp_path, ctx=ctx)
    plain.stage_slices(amp)
    leg = amp[0].tensors[0].legs[0]
    sliced = SlicedPlan.for_gradients(amp[0], amp_path, [leg], None, ctx=ctx)
    r64, r64_path = rank64_net()
    g64 = NetworkPlan.for_gradients(r64, r64_path, ctx=ctx)
    assert len(g64.result_legs) == 64
    g_amp.stage_batch(amp)
    g_sv.stage_batch(sv)
    g64.stage_batch([r64])
    m = _Marshal()
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(m.tn(amp[0])))
    sv_seeds = DeviceTensor.from_numpy(ctx, random_seeds(g_sv.result_dims, 2, 1))
    short = DeviceTensor.from_numpy(ctx, random_seeds(g_sv.result_dims, 1, 1))
    amp_seeds_wrong = DeviceTensor.from_numpy(ctx, np.ones((3, 2), np.complex128))
    other = tb.Context(0)
    try:
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]

        def expect(rc, want):
            assert rc == want, (rc, want, ctx._l.tncb_last_error())
            assert ctx.stats()["arena_live_bytes"] == live

        expect(raw_vjp_batch(ctx, plain.handle, 0, 1), ERR_INVALID)                  # not a gradient plan
        expect(ctx._l.tncb_plan_stage_batch(ctx.handle, plain.handle, 1, ptrs), ERR_INVALID)
        expect(raw_vjp_batch(ctx, sliced.plan.handle, 0, 1), ERR_UNSUPPORTED)             # sliced x batched
        expect(ctx._l.tncb_plan_stage_batch(ctx.handle, sliced.plan.handle, 1, ptrs), ERR_UNSUPPORTED)
        expect(raw_vjp_batch(ctx, unstaged.handle, 0, 1), ERR_INVALID)               # nothing staged
        expect(raw_vjp_batch(other, g_amp.handle, 0, 1), ERR_INVALID)                # another context
        expect(raw_vjp_batch(ctx, g_amp.handle, 0, 0), ERR_INVALID)                  # count 0
        expect(raw_vjp_batch(ctx, g_amp.handle, 3, 1), ERR_INVALID)                  # past the end
        expect(raw_vjp_batch(ctx, g_amp.handle, 1, 3), ERR_INVALID)
        expect(raw_vjp_batch(ctx, g_amp.handle, 2 ** 64 - 1, 2), ERR_INVALID)        # first + count wraps around
        expect(raw_vjp_batch(ctx, g_amp.handle, 0, 3, outs=(False, False, False)), ERR_INVALID)   # no output
        expect(raw_vjp_batch(ctx, g_sv.handle, 0, 2), ERR_INVALID)                   # no seeds for a rank-13 result
        expect(raw_vjp_batch(ctx, g_sv.handle, 0, 2, short), ERR_SHAPE)              # [1, ..] seeds for 2 instances
        expect(raw_vjp_batch(ctx, g_amp.handle, 0, 3, amp_seeds_wrong), ERR_SHAPE)   # [3, 2] seeds, scalar result
        expect(raw_vjp_batch(ctx, g64.handle, 0, 1), ERR_INVALID)                    # rank 64: no instance dimension
        # the legal calls next to them work
        _, v, rows, total = g_sv.vjp_batch(seeds=sv_seeds, rows=True, sum=True)
        assert v.shape == (2,) + g_sv.result_dims and len(rows) == len(total) == len(sv[0].tensors)
        _, v, rows, total = g_amp.vjp_batch(values=False, rows=False, sum=True)     # NULL seeds: seed 1 each
        assert v is None and rows is None and len(total) == len(amp[0].tensors)
        _, v, rows, total = g_sv.vjp_batch(values=True, rows=False)                  # forward only: no seeds needed
        assert v.shape == (2,) + g_sv.result_dims and rows is None and total is None
    finally:
        other.close()
        for t in (sv_seeds, short, amp_seeds_wrong):
            t.free()
    # not even one workspace copy fits: a 1 MiB arena, 64 KiB of leaves, a 16 MiB outer product inside, a scalar result
    from tnc_b200.contractionpath import ContractionPath
    nets = matrix_nets([([0], [1024]), ([1], [1024]), ([0], [1024]), ([1], [1024])], 2, 14)
    path = ContractionPath.simple([(0, 1), (0, 2), (0, 3)])
    small = tb.Context(0, arena_bytes=1 << 20)
    try:
        plan = NetworkPlan.for_gradients(nets[0], path, ctx=small)
        assert plan.info()["peak_bytes"] > 16 << 20
        plan.stage_batch(nets)
        small.synchronize()
        live = small.stats()["arena_live_bytes"]
        rc = raw_vjp_batch(small, plan.handle, 0, 2)
        assert rc == ERR_OOM, (rc, small._l.tncb_last_error())
        assert small.stats()["arena_live_bytes"] == live
        del plan
    finally:
        small.close()


# ================================================================================================================
# 8. torch
# ================================================================================================================
def as_matrix_leaves(tn, idx):
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    parts = []
    for k, t in enumerate(tn.tensors):
        if k in idx:
            m = Tensor(t.legs, t.bond_dims)
            m.set_tensor_data(TensorData.Matrix(leaf_array(t)))
            t = m
        parts.append(t)
    return Tensor.new_composite(parts)


def test_gradcheck_batched_and_shared(ctx):
    import torch
    from tnc_b200.autograd import network_function
    tn = amplitude_nets(6, 3, 11, 1)[0]
    lv = list(tn.tensors)
    one = [k for k, t in enumerate(lv) if len(t.legs) == 2][0]
    two = [k for k, t in enumerate(lv) if len(t.legs) == 4][0]
    tn = as_matrix_leaves(tn, [one, two])
    f = network_function(tn, greedy(tn), [one, two], ctx=ctx, batched=[one])
    rng = np.random.default_rng(3)
    b = 3
    x1 = torch.tensor(rng.standard_normal((b, 2, 2)) + 1j * rng.standard_normal((b, 2, 2)), requires_grad=True)
    x2 = torch.tensor(rng.standard_normal(lv[two].bond_dims) + 1j * rng.standard_normal(lv[two].bond_dims), requires_grad=True)
    assert f(x1, x2).shape == (b,)
    assert torch.autograd.gradcheck(f, (x1, x2), eps=1e-6, atol=1e-7, rtol=1e-6)
    with pytest.raises(ValueError):
        f(x1, torch.zeros((b,) + tuple(lv[two].bond_dims), dtype=torch.complex128))   # a shared input with a batch dim
    with pytest.raises(ValueError):
        network_function(tn, greedy(tn), [one], ctx=ctx, sliced_legs=[lv[one].legs[0]], batched=[one])


def test_angle_gradient_over_bitstrings(ctx):
    """L = sum_b |psi(b)|^2 over 16 bitstrings of a 10-qubit circuit: the bitstring projectors are batched inputs not
    in wrt, four shared gates are torch-built from angles.  Against central finite differences and against the sum of
    16 unbatched network_function calls."""
    import torch
    from tnc_b200.autograd import network_function
    from tnc_b200.builders import random_circuit_builder
    q, B = 10, 16
    circ = random_circuit_builder(q, 4, 0.5, 0.5, np.random.default_rng(12))
    rng = np.random.default_rng(13)
    bits = ["".join(rng.choice(["0", "1"], q)) for _ in range(B)]
    base = circ.into_amplitude_network("0" * q)[0]
    lv = list(base.tensors)
    proj = list(range(len(lv) - q, len(lv)))                 # the appended bitstring kets, one per qubit
    gates = [k for k, t in enumerate(lv[:len(lv) - q]) if len(t.legs) == 2][:3] + \
            [k for k, t in enumerate(lv[:len(lv) - q]) if len(t.legs) == 4][:1]
    tn = as_matrix_leaves(base, gates + proj)
    path = greedy(tn)
    f = network_function(tn, path, gates, ctx=ctx, batched=proj)
    kets = [torch.tensor(np.array([[1.0, 0.0] if b[j] == "0" else [0.0, 1.0] for b in bits]), dtype=torch.complex128)
            for j in range(q)]
    singles = [network_function(as_matrix_leaves(circ.into_amplitude_network(b)[0], gates), path, gates, ctx=ctx) for b in bits]
    I = torch.eye(2, dtype=torch.complex128)
    X = torch.tensor([[0, 1], [1, 0]], dtype=torch.complex128)
    Y = torch.tensor([[0, -1j], [1j, 0]], dtype=torch.complex128)
    Z = torch.tensor([[1, 0], [0, -1]], dtype=torch.complex128)

    def rot(P, t):
        return torch.cos(t / 2) * I - 1j * torch.sin(t / 2) * P

    def fsim(t, p):
        c, s = torch.cos(t), torch.sin(t)
        m = torch.diag(torch.stack([torch.ones((), dtype=torch.complex128), c + 0j, c + 0j, torch.exp(-1j * p)]))
        e = torch.zeros(4, 4, dtype=torch.complex128)
        e[1, 2] = 1
        e[2, 1] = 1
        return m - 1j * s * e

    def mats(theta):
        ms = [rot(X, theta[0]), rot(Y, theta[1]), rot(Z, theta[2]), fsim(theta[3], theta[4])]
        return [m.reshape(lv[k].bond_dims) for m, k in zip(ms, gates)]

    def loss(theta):
        amps = f(*mats(theta), *kets)
        assert amps.shape == (B,)
        return (amps.abs() ** 2).sum()

    def loss_single(theta):
        ms = mats(theta)
        return sum(g(*ms).abs() ** 2 for g in singles)

    theta = torch.tensor([0.3, -1.1, 0.7, 0.9, 0.4], dtype=torch.float64, requires_grad=True)
    loss(theta).backward()
    grad = theta.grad.numpy().copy()
    theta.grad = None
    loss_single(theta).backward()
    ref = theta.grad.numpy()
    assert np.abs(grad - ref).max() <= 1e-12 * np.abs(ref).max(), (grad, ref)
    h = 1e-5
    fd = []
    with torch.no_grad():
        for k in range(5):
            e = torch.zeros(5, dtype=torch.float64)
            e[k] = h
            fd.append((loss(theta + e) - loss(theta - e)).item() / (2 * h))
    fd = np.array(fd)
    assert np.abs(grad - fd).max() <= 1e-7 * max(1.0, np.abs(fd).max()), (grad, fd)
    assert np.abs(fd).max() > 1e-6
