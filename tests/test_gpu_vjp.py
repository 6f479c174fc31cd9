"""Gradients of a contracted network with respect to its leaves (tncb_plan_create_vjp / tncb_plan_vjp,
NetworkPlan.for_gradients, tnc_b200.autograd):

  1. every G_l against torch autograd through a TTGT replay of the same path on the CPU (complex128), on
     random-circuit amplitude networks (K0 and its level batches; K1 DMMA at 16 qubits x 8 rounds) and a 13-qubit
     statevector network with random input states (K2 and the long reductions of its backward; a non-scalar result
     with a random seed);
  2. bench.py's 36-qubit network with every leaf requested (the int8 engine): multilinearity of the amplitude in every
     leaf, fresh forward runs with replaced leaves, agreement with a DMMA-only pass, a forward result bit-identical to a
     plain plan's;
  3. torch: gradcheck, and the gradient of |amp|^2 in gate angles against central finite differences;
  4. the error codes, with the arena's live bytes unchanged."""
import ctypes as C
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
    """(legs, R, [G_l]) with G_l = sum_r seed[r] dR[r]/dX_l: torch returns conj of that for grad_outputs = conj(seed)"""
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


# ================================================================================================================
# 1. against an independent reference
# ================================================================================================================
def amplitude_net(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def statevector_net(seed):
    """13 qubits, 4 rounds, random normalised input states as Matrix leaves: K0 steps and one K2 step"""
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


def check_against_reference(ctx, tn, path, seed=None):
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    plan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    plan.stage(tn)
    (res, fwd_ec) = counted(ctx, plan.run)
    got, bwd_ec = counted(ctx, lambda: plan.vjp(seed))
    legs, R, ref = reference_grads(tn, path, seed)
    assert res.legs == legs
    assert np.abs(res.to_numpy() - R).max() <= 1e-12 * max(np.abs(R).max(), 1e-300)
    lv = leaves(tn)
    assert sorted(got) == [i for i, l in enumerate(lv) if leaf_array(l) is not None]
    gmax = max(np.abs(g).max() for g in ref)
    for i in got:
        assert got[i].shape == ref[i].shape, i
        assert np.abs(got[i] - ref[i]).max() <= 1e-12 * gmax, (i, np.abs(got[i] - ref[i]).max(), gmax)
    return fwd_ec, bwd_ec


@pytest.mark.parametrize("qubits,rounds", [(12, 6), (16, 8)])
def test_amplitude_against_torch(ctx, qubits, rounds):
    """Level-batched and plain K0 in both passes; at 16 qubits and 8 rounds K1 DMMA as well"""
    tn = amplitude_net(qubits, rounds, 5)
    path = greedy(tn)
    fwd, bwd = check_against_reference(ctx, tn, path)
    assert bwd["k0"] > 0, bwd
    if qubits == 16:
        assert fwd["k1_dmma"] > 0 and bwd["k1_dmma"] > 0, (fwd, bwd)


def test_statevector_against_torch(ctx):
    """The K2 step's backward: the big operand's adjoint is again a K2 pair, the small one's a long reduction
    (K0 split-K); a random seed over the 2^13 outputs"""
    tn = statevector_net(1)
    path = greedy(tn)
    from tnc_b200.tensornetwork import NetworkPlan
    legs_dims = NetworkPlan(tn, path, ctx=ctx).execute(tn).bond_dims
    rng = np.random.default_rng(2)
    seed = rng.standard_normal(legs_dims) + 1j * rng.standard_normal(legs_dims)
    fwd, bwd = check_against_reference(ctx, tn, path, seed)
    assert fwd["k2"] >= 1 and bwd["k2"] >= 1, (fwd, bwd)
    assert bwd["k0_splitk"] >= 1, bwd


# ================================================================================================================
# 2. multilinearity at bench scale
# ================================================================================================================
def test_bench_network_multilinear(ctx):
    sys.path.insert(0, ROOT)
    import bench
    from tnc_b200.contractionpath import ContractionPath  # noqa: F401
    from tnc_b200.tensornetwork import NetworkPlan, Tensor, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn = bench.build_network()
    path = bench.greedy_path(tn)
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    plain = NetworkPlan(tn, path, ctx=ctx)
    plain.stage(tn)
    ref = plain.run().to_numpy()
    del plain
    plan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    plan.stage(tn)
    R = plan.run().to_numpy()
    assert np.array_equal(R, ref)                                           # the forward levels are the plain plan's
    G, ec = counted(ctx, plan.vjp)
    assert ec["k1_tcgen05"] >= 1, ec
    assert len(G) == len(lv) == 489
    r = complex(R)
    for i, g in G.items():
        lhs = complex(np.sum(g * xs[i]))
        assert abs(lhs - r) <= 1e-9 * float(np.sum(np.abs(g) * np.abs(xs[i]))), (i, lhs, r)
    # a few leaves replaced by random tensors: a fresh forward run is linear in each of them
    rng = np.random.default_rng(9)
    for i in (0, 200, 488):
        x2 = rng.standard_normal(xs[i].shape) + 1j * rng.standard_normal(xs[i].shape)
        repl = Tensor(lv[i].legs, lv[i].bond_dims)
        repl.set_tensor_data(TensorData.Matrix(x2))
        parts = [repl if k == i else t for k, t in enumerate(tn.tensors)]
        fresh = NetworkPlan(Tensor.new_composite(parts), path, ctx=ctx)
        got = complex(fresh.execute(Tensor.new_composite(parts)).to_numpy())
        want = complex(np.sum(G[i] * x2))
        assert abs(got - want) <= 1e-9 * float(np.sum(np.abs(G[i]) * np.abs(x2))), (i, got, want)
        del fresh
    # the same pass on DMMA only
    ctx.set_tcgen05_slices(0)
    try:
        plan.stage(tn)
        R0 = plan.run().to_numpy()
        G0, ec0 = counted(ctx, plan.vjp)
    finally:
        ctx.set_tcgen05_slices(8)
    assert ec0["k1_tcgen05"] == 0
    assert abs(complex(R0) - r) <= 1e-9 * abs(r)
    gmax = max(np.abs(g).max() for g in G.values())
    for i in G:
        assert np.abs(G[i] - G0[i]).max() <= 1e-9 * gmax, i
    del plan
    ctx.trim()


# ================================================================================================================
# 3. torch
# ================================================================================================================
def as_matrix_leaves(tn, idx):
    """`tn` with the leaves `idx` (top-level children) turned into Matrix leaves of the same payload"""
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
    tn = amplitude_net(6, 3, 11)
    lv = list(tn.tensors)
    one = [k for k, t in enumerate(lv) if len(t.legs) == 2][:2]
    two = [k for k, t in enumerate(lv) if len(t.legs) == 4][:1]
    idx = one + two
    tn = as_matrix_leaves(tn, idx)
    path = greedy(tn)
    f = network_function(tn, path, idx, ctx=ctx)
    rng = np.random.default_rng(3)
    xs = [torch.tensor(rng.standard_normal(lv[k].bond_dims) + 1j * rng.standard_normal(lv[k].bond_dims), requires_grad=True)
          for k in idx]
    assert torch.autograd.gradcheck(f, tuple(xs), eps=1e-6, atol=1e-7, rtol=1e-6)
    out = f(*xs)
    out.abs().backward()
    with pytest.raises(RuntimeError):
        out.abs().backward()                                                # the graph was not retained


def test_angle_gradient(ctx):
    """|amp|^2 of a 6-qubit circuit in which four gates are torch-built rx / ry / rz / fsim matrices of angles theta"""
    import torch
    from tnc_b200.autograd import network_function
    tn = amplitude_net(6, 4, 12)
    lv = list(tn.tensors)
    one = [k for k, t in enumerate(lv) if len(t.legs) == 2][:3]
    two = [k for k, t in enumerate(lv) if len(t.legs) == 4][:1]
    idx = one + two
    tn = as_matrix_leaves(tn, idx)
    f = network_function(tn, greedy(tn), idx, ctx=ctx)
    I = torch.eye(2, dtype=torch.complex128)
    X = torch.tensor([[0, 1], [1, 0]], dtype=torch.complex128)
    Y = torch.tensor([[0, -1j], [1j, 0]], dtype=torch.complex128)
    Z = torch.tensor([[1, 0], [0, -1]], dtype=torch.complex128)

    def rot(P, t):
        return torch.cos(t / 2) * I - 1j * torch.sin(t / 2) * P

    def fsim(t, p):
        c, s = torch.cos(t), torch.sin(t)
        m = torch.zeros(4, 4, dtype=torch.complex128)
        m = m + torch.diag(torch.stack([torch.ones((), dtype=torch.complex128), c + 0j, c + 0j, torch.exp(-1j * p)]))
        e = torch.zeros(4, 4, dtype=torch.complex128)
        e[1, 2] = 1
        e[2, 1] = 1
        return m - 1j * s * e

    def loss(theta):
        mats = [rot(X, theta[0]), rot(Y, theta[1]), rot(Z, theta[2]), fsim(theta[3], theta[4])]
        amp = f(*[m.reshape(lv[k].bond_dims) for m, k in zip(mats, idx)])
        return amp.abs() ** 2

    theta = torch.tensor([0.3, -1.1, 0.7, 0.9, 0.4], dtype=torch.float64, requires_grad=True)
    loss(theta).backward()
    h = 1e-5
    fd = []
    with torch.no_grad():
        for k in range(5):
            e = torch.zeros(5, dtype=torch.float64)
            e[k] = h
            fd.append((loss(theta + e) - loss(theta - e)).item() / (2 * h))
    fd = np.array(fd)
    assert np.abs(theta.grad.numpy() - fd).max() <= 1e-7 * max(1.0, np.abs(fd).max()), (theta.grad, fd)
    assert np.abs(fd).max() > 1e-6


# ================================================================================================================
# 4. errors
# ================================================================================================================
def raw_vjp(ctx, handle, seed=None):
    out = C.c_void_p()
    return ctx._l.tncb_plan_vjp(ctx.handle, handle, seed.handle if seed is not None else None, C.byref(out))


def test_errors(ctx):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    amp = amplitude_net(10, 4, 6)
    amp_path = greedy(amp)
    sv = statevector_net(3)
    sv_path = greedy(sv)
    g_amp = NetworkPlan.for_gradients(amp, amp_path, ctx=ctx)
    g_sv = NetworkPlan.for_gradients(sv, sv_path, ctx=ctx)
    plain = NetworkPlan(amp, amp_path, ctx=ctx)
    plain.stage(amp)
    g_sv.stage(sv)
    res = g_sv.run()
    wrong = DeviceTensor.from_numpy(ctx, np.ones([2] * 12, dtype=np.complex128))
    other = tb.Context(0)
    try:
        g_amp.stage(amp)
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]

        def expect(rc, want):
            assert rc == want, (rc, want, ctx._l.tncb_last_error())
            assert ctx.stats()["arena_live_bytes"] == live

        expect(raw_vjp(ctx, g_amp.handle), ERR_INVALID)                    # staged, no forward run
        expect(raw_vjp(ctx, plain.handle), ERR_INVALID)                    # not a gradient plan
        expect(raw_vjp(other, g_amp.handle), ERR_INVALID)                  # another context
        expect(raw_vjp(ctx, g_sv.handle), ERR_INVALID)                     # no seed for a rank-13 result
        expect(raw_vjp(ctx, g_sv.handle, wrong), ERR_SHAPE)                # seed dims differ from the result's
        seed = DeviceTensor.from_numpy(ctx, np.ones(res.bond_dims, dtype=np.complex128))
        live = ctx.stats()["arena_live_bytes"]
        g = g_sv.vjp(seed)
        assert len(g) == len(sv.tensors)
        ctx.synchronize()
        expect(raw_vjp(ctx, g_sv.handle, seed), ERR_INVALID)              # a second vjp after one
        seed.free()
        wrong.free()
        scalar_wrong = DeviceTensor.from_numpy(ctx, np.ones(3, dtype=np.complex128))
        g_amp.run()
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        expect(raw_vjp(ctx, g_amp.handle, scalar_wrong), ERR_SHAPE)       # a seed for a scalar result has rank 0
        scalar_wrong.free()
        g1 = g_amp.vjp()
        assert len(g1) == len(amp.tensors)
        # slices / batches on a gradient plan
        m_ptr = (C.POINTER(tb._lib.TncbTn) * 1)()
        from tnc_b200.tensornetwork.contraction import _Marshal
        mm = _Marshal()
        node = mm.tn(amp)
        m_ptr[0] = C.pointer(node)
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        expect(ctx._l.tncb_plan_stage_slices(ctx.handle, g_amp.handle, 1, m_ptr), ERR_UNSUPPORTED)
        out, n_out, legs = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)()
        expect(ctx._l.tncb_plan_run_slices(ctx.handle, g_amp.handle, 0, 1, C.byref(out), C.byref(n_out), legs), ERR_UNSUPPORTED)
        expect(ctx._l.tncb_plan_run_batch(ctx.handle, g_amp.handle, 0, 1, C.byref(out), C.byref(n_out), legs), ERR_UNSUPPORTED)
        # creation refusals
        with pytest.raises(tb.TncbError) as e:
            NetworkPlan.for_gradients(amp, amp_path, wrt=[], ctx=ctx)
        assert e.value.status == ERR_INVALID
        one = Tensor([0, 1], [2, 2])
        one.set_tensor_data(TensorData.Matrix(np.eye(2)))
        with pytest.raises(tb.TncbError) as e:
            NetworkPlan.for_gradients(Tensor.new_composite([one]), ContractionPath.simple([]), ctx=ctx)
        assert e.value.status == ERR_UNSUPPORTED
        dev = DeviceTensor.from_numpy(ctx, np.eye(2, dtype=np.complex128))
        parts = list(amp.tensors)
        k = next(i for i, t in enumerate(parts) if len(t.legs) == 2)
        t = Tensor(parts[k].legs, parts[k].bond_dims)
        t.set_tensor_data(TensorData.Matrix(dev))
        parts[k] = t
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        with pytest.raises(tb.TncbError) as e:
            NetworkPlan.for_gradients(Tensor.new_composite(parts), amp_path, ctx=ctx)
        assert e.value.status == ERR_UNSUPPORTED
        assert ctx.stats()["arena_live_bytes"] == live
        dev.free()
    finally:
        other.close()
    # no room for the workspace at run time: OOM, no fallback
    sys.path.insert(0, ROOT)
    import bench
    bn = bench.build_network()
    small = tb.Context(0, arena_bytes=1 << 20)
    try:
        big = NetworkPlan.for_gradients(bn, bench.greedy_path(bn), ctx=small)
        live = small.stats()["arena_live_bytes"]
        with pytest.raises(tb.TncbError) as e:
            big.stage(bn)
        assert e.value.status == ERR_OOM
        assert small.stats()["arena_live_bytes"] == live
        with pytest.raises(tb.TncbError) as e:
            big.execute(bn)
        assert e.value.status == ERR_OOM
        assert small.stats()["arena_live_bytes"] == live
        del big
    finally:
        small.close()
