"""Sliced gradient plans (tncb_plan_create_vjp_sliced / tncb_plan_vjp_sliced, SlicedPlan.for_gradients,
network_function(..., sliced_legs=...)):

  1. every full-shape G_l against torch autograd through a TTGT replay of the UNSLICED network on the CPU (complex128):
     12- and 16-qubit amplitude networks at 1, 2 and 4 sliced legs (one case slices every leg of a two-qubit gate leaf),
     a network whose leaf adjoint needs more leg groups than an accumulate item holds (K3 first), and a 13-qubit
     statevector network with a random seed (K0 and K2 by the engine counters; DMMA by the 16-qubit case);
  2. exactness: 0 sliced legs equals run + vjp element for element, run_slices is bit-identical to SlicedPlan.run, the
     value of vjp_sliced to run_slices, and repeated calls to each other;
  3. partial ranges (world = 2, 3) add up to the whole;
  4. bench.py's network with 2 sliced legs under TNCB_PLAN_WS_GB=8 (the unsliced gradient plan is refused there):
     multilinearity in all 489 leaves, agreement with the unsliced gradient plan, the int8 engine; element by element
     in per-leaf units at 1, 2 and 3 sliced legs, partial ranges against replays of exactly their slices, and the
     512-slice Sycamore-53 depth-12 gradient: test_gpu_vjp_sliced_bench.py;
  5. torch: gradcheck through a sliced network_function, gate-angle gradients equal to the unsliced function's;
  6. the error codes, with the arena's live bytes unchanged."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_UNSUPPORTED = -1, -2, -9


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


def leaf_array(t):
    """the payload of a leaf as an ndarray of its dims (None: no payload)"""
    td = t.tensordata
    if td.kind == "gate":
        d = orc.OTensor(list(t.legs), list(t.bond_dims), ("gate", td.gate[0], td.gate[1], td.gate[2])).materialise()
    elif td.kind == "matrix":
        d = np.asarray(td.matrix)
    else:
        return None
    return np.asarray(d, dtype=np.complex128).reshape([int(x) for x in t.bond_dims])


# ------------------------------------------------------------------------------------------------ reference
def ttgt(a_legs, A, b_legs, B):
    """C[(b\\a) ++ (a\\b)] = sum over the shared legs: transpose, reshape, one GEMM, reshape"""
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
    """contract `tn` along the replace-left `path` in torch; xs = the leaves' torch tensors in leaf order"""
    it = iter(xs)

    def walk(t, p):
        if not t.tensors:
            return list(t.legs), next(it)
        slots = []
        for i, c in enumerate(t.tensors):
            slots.append(walk(c, p.nested.get(i) if c.tensors else None))
        for i, j in p.toplevel:
            slots[i] = ttgt(*slots[i], *slots[j])
            slots[j] = None
        return next(s for s in slots if s is not None)
    return walk(tn, path)


def reference_grads(tn, path, seed=None):
    """(legs, R, [G_l]) of the unsliced network with G_l = sum_r seed[r] dR[r]/dX_l"""
    import torch
    from tnc_b200.tensornetwork import leaves
    xs = [torch.tensor(leaf_array(l), requires_grad=True) for l in leaves(tn)]
    legs, R = replay(tn, path, xs)
    s = torch.ones_like(R) if seed is None else torch.tensor(seed)
    gs = torch.autograd.grad(R, xs, grad_outputs=s.conj())
    return legs, R.detach().numpy(), [g.conj().resolve_conj().numpy() for g in gs]


def counted(ctx, fn):
    ctx.reset_stats()
    res = fn()
    ctx.synchronize()
    return res, ctx.engine_counts()


def amplitude_net(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def statevector_net(seed):
    """13 qubits, 4 rounds, random normalised input states as Matrix leaves"""
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, _ = random_circuit_builder(13, 4, 0.5, 0.5, np.random.default_rng(4)).into_statevector_network()
    rng = np.random.default_rng(seed)
    out = []
    for t in tn.tensors:
        if len(t.legs) == 1:
            v = rng.standard_normal(2) + 1j * rng.standard_normal(2)
            t = Tensor(t.legs, t.bond_dims)
            t.set_tensor_data(TensorData.Matrix(v / np.linalg.norm(v)))
        out.append(t)
    return Tensor.new_composite(out)


def leg_counts(tn):
    from tnc_b200.tensornetwork import leaves
    count = {}
    for l in leaves(tn):
        for x in l.legs:
            count[x] = count.get(x, 0) + 1
    return count


def whole_leaf_legs(tn, rank):
    """the legs of a leaf of `rank` whose legs are all internal (a gate in the middle of the circuit)"""
    count = leg_counts(tn)
    for t in tn.tensors:
        if len(t.legs) == rank and all(count[x] == 2 for x in t.legs):
            return list(t.legs)
    raise AssertionError("no such leaf")


def sliced_plan(ctx, tn, path, legs, wrt=None):
    from tnc_b200.contractionpath.slicing import SlicedPlan
    p = SlicedPlan.for_gradients(tn, path, legs, wrt=wrt, ctx=ctx)
    p.stage(tn)
    return p


def check_against_reference(ctx, tn, path, legs, seed=None):
    from tnc_b200.tensornetwork import leaves
    plan = sliced_plan(ctx, tn, path, legs)
    (res, G), ec = counted(ctx, lambda: plan.vjp(seed))
    rlegs, R, ref = reference_grads(tn, path, seed)
    assert res.legs == rlegs
    assert np.abs(res.to_numpy() - R).max() <= 1e-12 * max(np.abs(R).max(), 1e-300)
    lv = leaves(tn)
    assert sorted(G) == [i for i, l in enumerate(lv) if leaf_array(l) is not None]
    gmax = max(np.abs(g).max() for g in ref)
    for i in G:
        assert G[i].shape == ref[i].shape, i
        assert np.abs(G[i] - ref[i]).max() <= 1e-12 * gmax, (i, np.abs(G[i] - ref[i]).max(), gmax)
    return plan, ec


# ================================================================================================================
# 1. against an independent reference
# ================================================================================================================
@pytest.mark.parametrize("qubits,rounds,n_legs", [(12, 6, 1), (12, 6, 2), (16, 8, 4)])
def test_amplitude_against_torch(ctx, qubits, rounds, n_legs):
    from tnc_b200.contractionpath.slicing import find_slices
    tn = amplitude_net(qubits, rounds, 5)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert len(legs) == n_legs
    plan, ec = check_against_reference(ctx, tn, path, legs)
    assert plan.n_slices == 2 ** n_legs
    assert ec["k0"] > 0, ec
    if qubits == 16:
        assert ec["k1_dmma"] + ec["k1_dmma_splitk"] > 0, ec            # a slice keeps one K1 pair (DMMA at this size)


def test_every_leg_of_a_leaf_sliced(ctx):
    """the four legs of one two-qubit gate: that leaf is rank 0 in every slice, 16 slices"""
    tn = amplitude_net(12, 6, 7)
    path = greedy(tn)
    legs = whole_leaf_legs(tn, 4)
    plan, _ = check_against_reference(ctx, tn, path, legs)
    assert plan.n_slices == 16


def test_many_group_route(ctx):
    """X (11 legs) and Y (the same legs reversed) plus a matrix on two of them: X's adjoint comes out in Y's order, 9
    leg groups after slicing one leg, more than an accumulate item holds -> K3 into the scratch, then the accumulate"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(4)
    legs = list(range(11))

    def leaf(ls, dims):
        t = Tensor(ls, dims)
        t.set_tensor_data(TensorData.Matrix(rng.standard_normal(dims) + 1j * rng.standard_normal(dims)))
        return t
    x = leaf(legs[:10] + [20], [2] * 10 + [3])
    y = leaf([10] + legs[:10][::-1], [2] * 11)
    m = leaf([20, 10], [3, 2])
    tn = Tensor.new_composite([x, m, y])
    path = ContractionPath.simple([(0, 1), (0, 2)])
    _, ec = check_against_reference(ctx, tn, path, [4])
    assert ec["permute"] >= 2, ec                       # one K3 per slice


def test_statevector_against_torch(ctx):
    """a non-scalar result and a random seed over the 2^13 outputs; one sliced leg"""
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import NetworkPlan
    tn = statevector_net(1)
    path = greedy(tn)
    dims = NetworkPlan(tn, path, ctx=ctx).execute(tn).bond_dims
    rng = np.random.default_rng(2)
    seed = rng.standard_normal(dims) + 1j * rng.standard_normal(dims)
    legs = find_slices(tn, path, min_slices=2)
    _, ec = check_against_reference(ctx, tn, path, legs, seed)
    assert ec["k0"] >= 1 and ec["k2"] >= 2, ec                     # the K2 step and its big operand's adjoint


# ================================================================================================================
# 2. exactness invariants
# ================================================================================================================
def test_zero_legs_equal_run_and_vjp(ctx):
    from tnc_b200.tensornetwork import NetworkPlan
    tn = amplitude_net(12, 6, 8)
    path = greedy(tn)
    g = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    g.stage(tn)
    R = g.run().to_numpy()
    G = g.vjp()
    del g
    plan = sliced_plan(ctx, tn, path, [])
    assert plan.n_slices == 1
    res, G2 = plan.vjp()
    assert np.array_equal(res.to_numpy(), R)
    assert sorted(G) == sorted(G2)
    for i in G:
        assert np.array_equal(G[i], G2[i]), i           # == : -0.0 and +0.0 compare equal


def test_bit_identities(ctx):
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    tn = amplitude_net(16, 8, 3)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=8)
    ref = SlicedPlan(tn, path, legs, ctx=ctx).run().to_numpy()
    plan = sliced_plan(ctx, tn, path, legs)
    run = plan.run().to_numpy()
    assert run.tobytes() == ref.tobytes()
    v1, g1 = plan.vjp()
    v2, g2 = plan.vjp()
    assert v1.to_numpy().tobytes() == run.tobytes()
    assert v2.to_numpy().tobytes() == run.tobytes()
    assert plan.run().to_numpy().tobytes() == run.tobytes()
    for i in g1:
        assert g1[i].tobytes() == g2[i].tobytes(), i


# ================================================================================================================
# 3. partial ranges
# ================================================================================================================
def test_partial_ranges_add_up(ctx):
    from tnc_b200.contractionpath.slicing import find_slices
    tn = amplitude_net(12, 6, 9)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    plan = sliced_plan(ctx, tn, path, legs)
    v, G = plan.vjp()
    gmax = max(np.abs(g).max() for g in G.values())
    for world in (2, 3):
        vs, Gs = zip(*[plan.vjp(rank=r, world=world, allreduce=False) for r in range(world)])
        assert abs(sum(complex(x.to_numpy()) for x in vs) - complex(v.to_numpy())) <= 1e-13 * abs(complex(v.to_numpy()))
        for i in G:
            assert np.abs(sum(g[i] for g in Gs) - G[i]).max() <= 1e-13 * gmax, (world, i)
    # more ranks than slices: zeros
    v0, G0 = plan.vjp(rank=plan.n_slices, world=plan.n_slices + 1, allreduce=False)
    assert complex(v0.to_numpy()) == 0 and all(not g.any() for g in G0.values())


# ================================================================================================================
# 4. bench scale, int8 engine
# ================================================================================================================
def test_bench_network_two_legs(ctx, monkeypatch):
    sys.path.insert(0, ROOT)
    import bench
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = bench.build_network()
    path = bench.greedy_path(tn)
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    legs = find_slices(tn, path, min_slices=4)
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "8")
    with pytest.raises(tb.TncbError) as e:
        NetworkPlan.for_gradients(tn, path, ctx=ctx)
    assert e.value.status == ERR_UNSUPPORTED
    plan = sliced_plan(ctx, tn, path, legs)
    (res, G), ec = counted(ctx, plan.vjp)
    assert ec["k1_tcgen05"] >= 1, ec
    assert len(G) == len(lv) == 489
    r = complex(res.to_numpy())
    for i, g in G.items():
        lhs = complex(np.sum(g * xs[i]))
        assert abs(lhs - r) <= 1e-9 * float(np.sum(np.abs(g) * np.abs(xs[i]))), (i, lhs, r)
    del plan
    monkeypatch.delenv("TNCB_PLAN_WS_GB")
    full = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    full.stage(tn)
    R0 = complex(full.run().to_numpy())
    G0 = full.vjp()
    del full
    ctx.trim()
    assert abs(R0 - r) <= 1e-9 * abs(R0)
    gmax = max(np.abs(g).max() for g in G0.values())
    for i in G0:
        assert np.abs(G[i] - G0[i]).max() <= 1e-9 * gmax, i


# ================================================================================================================
# 5. torch
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


def test_gradcheck(ctx):
    import torch
    from tnc_b200.autograd import network_function
    from tnc_b200.contractionpath.slicing import find_slices
    tn = amplitude_net(6, 3, 11)
    lv = list(tn.tensors)
    idx = [k for k, t in enumerate(lv) if len(t.legs) == 2][:2] + [k for k, t in enumerate(lv) if len(t.legs) == 4][:1]
    tn = as_matrix_leaves(tn, idx)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    f = network_function(tn, path, idx, ctx=ctx, sliced_legs=legs)
    rng = np.random.default_rng(3)
    xs = [torch.tensor(rng.standard_normal(lv[k].bond_dims) + 1j * rng.standard_normal(lv[k].bond_dims), requires_grad=True)
          for k in idx]
    assert torch.autograd.gradcheck(f, tuple(xs), eps=1e-6, atol=1e-7, rtol=1e-6)


def test_angle_gradient_equals_unsliced(ctx):
    import torch
    from tnc_b200.autograd import network_function
    tn = amplitude_net(6, 4, 12)
    lv = list(tn.tensors)
    idx = [k for k, t in enumerate(lv) if len(t.legs) == 2][:3] + [k for k, t in enumerate(lv) if len(t.legs) == 4][:1]
    tn = as_matrix_leaves(tn, idx)
    path = greedy(tn)
    from tnc_b200.contractionpath.slicing import find_slices
    legs = find_slices(tn, path, min_slices=8)
    I = torch.eye(2, dtype=torch.complex128)
    X = torch.tensor([[0, 1], [1, 0]], dtype=torch.complex128)
    Y = torch.tensor([[0, -1j], [1j, 0]], dtype=torch.complex128)

    def rot(P, t):
        return torch.cos(t / 2) * I - 1j * torch.sin(t / 2) * P

    def fsim(t, p):
        c, s = torch.cos(t), torch.sin(t)
        m = torch.diag(torch.stack([torch.ones((), dtype=torch.complex128), c + 0j, c + 0j, torch.exp(-1j * p)]))
        e = torch.zeros(4, 4, dtype=torch.complex128)
        e[1, 2] = 1
        e[2, 1] = 1
        return m - 1j * s * e

    grads = []
    for sl in ([], legs):
        f = network_function(tn, path, idx, ctx=ctx, sliced_legs=sl)
        theta = torch.tensor([0.3, -1.1, 0.7, 0.9, 0.4], dtype=torch.float64, requires_grad=True)
        mats = [rot(X, theta[0]), rot(Y, theta[1]), rot(X, theta[2]), fsim(theta[3], theta[4])]
        amp = f(*[m.reshape(lv[k].bond_dims) for m, k in zip(mats, idx)])
        (amp.abs() ** 2).backward()
        grads.append(theta.grad.numpy().copy())
    assert np.abs(grads[0]).max() > 1e-6
    assert np.abs(grads[0] - grads[1]).max() <= 1e-12 * np.abs(grads[0]).max(), grads


# ================================================================================================================
# 6. errors
# ================================================================================================================
def raw_vjp_sliced(c, handle, first=0, stride=1, seed=None):
    v, g = C.c_void_p(), C.c_void_p()
    return c._l.tncb_plan_vjp_sliced(c.handle, handle, first, stride, seed.handle if seed is not None else None, C.byref(v), C.byref(g))


def test_errors(ctx):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath.slicing import SlicedNetwork, SlicedPlan, find_slices
    from tnc_b200.tensornetwork import NetworkPlan
    from tnc_b200.tensornetwork.contraction import _Marshal
    amp = amplitude_net(10, 4, 6)
    path = greedy(amp)
    legs = find_slices(amp, path, min_slices=2)
    sv = statevector_net(3)
    sv_path = greedy(sv)
    sv_legs = find_slices(sv, sv_path, min_slices=2)
    s_amp = SlicedPlan.for_gradients(amp, path, legs, ctx=ctx)
    s_sv = sliced_plan(ctx, sv, sv_path, sv_legs)
    g_amp = NetworkPlan.for_gradients(amp, path, ctx=ctx)
    g_amp.stage(amp)
    wrong = DeviceTensor.from_numpy(ctx, np.ones([2] * 12, dtype=np.complex128))
    other = tb.Context(0)
    try:
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]

        def expect(rc, want):
            assert rc == want, (rc, want, ctx._l.tncb_last_error())
            assert ctx.stats()["arena_live_bytes"] == live

        out, n_out, ol = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)()
        h = s_amp.plan.handle
        expect(raw_vjp_sliced(ctx, h), ERR_INVALID)                                  # not staged
        expect(ctx._l.tncb_plan_run_slices(ctx.handle, h, 0, 1, C.byref(out), C.byref(n_out), ol), ERR_INVALID)
        expect(raw_vjp_sliced(ctx, g_amp.handle), ERR_INVALID)                       # not a sliced gradient plan
        # the structure a stage validates is the full network's: a slice network is refused
        sn = SlicedNetwork(amp, legs)
        m = _Marshal()
        node = m.tn(sn.slice(sn.assignments[0]))
        rc = ctx._l.tncb_plan_stage(ctx.handle, h, C.byref(node))
        assert rc in (ERR_INVALID, ERR_SHAPE), rc
        s_amp.stage(amp)
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        expect(raw_vjp_sliced(ctx, h, stride=0), ERR_INVALID)                        # stride 0
        expect(raw_vjp_sliced(other, h), ERR_INVALID)                                # another context
        scalar_wrong = DeviceTensor.from_numpy(ctx, np.ones(3, dtype=np.complex128))
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        expect(raw_vjp_sliced(ctx, h, seed=scalar_wrong), ERR_SHAPE)                 # a scalar result's seed has rank 0
        expect(raw_vjp_sliced(ctx, s_sv.plan.handle), ERR_INVALID)                   # no seed for a rank-13 result
        expect(raw_vjp_sliced(ctx, s_sv.plan.handle, seed=wrong), ERR_SHAPE)         # seed dims differ
        # one way in: everything else is refused on a sliced gradient plan
        expect(ctx._l.tncb_plan_run(ctx.handle, h, C.byref(out), C.byref(n_out), ol), ERR_UNSUPPORTED)
        node = m.tn(amp)
        expect(ctx._l.tncb_plan_execute(ctx.handle, h, C.byref(node), C.byref(out), C.byref(n_out), ol), ERR_UNSUPPORTED)
        expect(ctx._l.tncb_plan_vjp(ctx.handle, h, None, C.byref(out)), ERR_UNSUPPORTED)
        ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(node))
        expect(ctx._l.tncb_plan_stage_slices(ctx.handle, h, 1, ptrs), ERR_UNSUPPORTED)
        expect(ctx._l.tncb_plan_run_batch(ctx.handle, h, 0, 1, C.byref(out), C.byref(n_out), ol), ERR_UNSUPPORTED)
        # still usable after all of that
        v, G = s_amp.vjp()
        assert len(G) == len(amp.tensors)
        scalar_wrong.free()
        # creation refusals through Python
        for bad in ([legs[0], legs[0]], [10 ** 6]):
            with pytest.raises(tb.TncbError) as e:
                SlicedPlan.for_gradients(amp, path, bad, ctx=ctx)
            assert e.value.status == ERR_INVALID
    finally:
        wrong.free()
        other.close()
