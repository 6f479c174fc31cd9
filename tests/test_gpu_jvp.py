"""Forward-mode derivatives of a contracted network (tncb_plan_create_jvp / tncb_plan_jvp / tncb_plan_jvp_batch,
NetworkPlan.for_tangents, network_function under torch.autograd.forward_ad and torch.func.jvp):

  1. Ṙ against torch.func.jvp of a TTGT replay of the same path on the CPU (complex128): K0 and its level batches, K1
     DMMA (16 qubits x 8 rounds), K2 (a 13-qubit statevector with random tangents), and a pair that takes the int8
     engine, checked at that engine's error bound;
  2. bench.py's network with every leaf requested: the adjoint identity with the reverse mode, multilinearity
     (Ẋ = X gives n R), a value bit-identical to a plain plan's run, repeated calls bit-identical;
  3. batches: rows bit-identical to single calls across several passes and sub-ranges, stage_instances = stage_batch,
     device tangents = host tangents;
  4. torch: forward_ad and torch.func.jvp through network_function against the replay, unbatched and batched, on the
     host and on the device; reverse mode unchanged; an angle derivative against central finite differences;
  5. every error, with the arena's live bytes unchanged."""
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


def counted(ctx, fn):
    ctx.reset_stats()
    res = fn()
    ctx.synchronize()
    return res, ctx.engine_counts()


def leaf_array(t):
    td = t.tensordata
    if td.kind == "gate":
        d = orc.OTensor(list(t.legs), list(t.bond_dims), ("gate", td.gate[0], td.gate[1], td.gate[2])).materialise()
    elif td.kind == "matrix":
        d = np.asarray(td.matrix)
    else:
        return None
    return np.asarray(d, dtype=np.complex128).reshape([int(x) for x in t.bond_dims])


def crandn(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


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


def reference_jvp(tn, path, xs, ts):
    """(R, Ṙ, scale): torch.func.jvp of the replay; scale bounds sum |terms| of Ṙ elementwise (the replay of |X|, |Ẋ|)"""
    import torch
    f = lambda *ys: replay(tn, path, ys)[1]
    X = [torch.tensor(x) for x in xs]
    T = [torch.tensor(t) for t in ts]
    R, Rd = torch.func.jvp(f, tuple(X), tuple(T))
    _, Sd = torch.func.jvp(f, tuple(torch.abs(x).to(torch.complex128) for x in X), tuple(torch.abs(t).to(torch.complex128) for t in T))
    return R.numpy(), Rd.numpy(), np.abs(Sd.numpy())


def check_against_reference(ctx, tn, path, wrt, seed):
    """tangent plan vs torch.func.jvp of the replay at 1e-12 of the terms' magnitude; returns the engine counts"""
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    rng = np.random.default_rng(seed)
    tans = {i: crandn(rng, xs[i].shape) for i in wrt}
    ts = [tans[i] if i in tans else np.zeros_like(xs[i]) for i in range(len(lv))]
    plan = NetworkPlan.for_tangents(tn, path, wrt, ctx=ctx)
    plan.stage(tn)
    (val, tan), ec = counted(ctx, lambda: plan.jvp(tans))
    R, Rd, scale = reference_jvp(tn, path, xs, ts)
    assert np.abs(val.to_numpy() - R).max() <= 1e-12 * max(np.abs(R).max(), 1e-300)
    assert tan.shape == Rd.shape
    assert (np.abs(tan - Rd) <= 1e-12 * np.maximum(scale, scale.max() * 1e-3)).all(), np.abs(tan - Rd).max()
    plain = NetworkPlan(tn, path, ctx=ctx)
    plain.stage(tn)
    assert np.array_equal(val.to_numpy(), plain.run().to_numpy())            # the forward levels are the plain plan's
    return ec


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
            v = crandn(rng, 2)
            t = Tensor(t.legs, t.bond_dims)
            t.set_tensor_data(TensorData.Matrix(v / np.linalg.norm(v)))
        out.append(t)
    return Tensor.new_composite(out)


def pair_net(rng, m=2048, k=256, n=2048):
    """A[m, k] x B[k, n]: M N K = 2^30 with K = 256, a pair for the int8 engine"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    a = Tensor([0, 1], [m, k])
    a.set_tensor_data(TensorData.Matrix(crandn(rng, (m, k))))
    b = Tensor([1, 2], [k, n])
    b.set_tensor_data(TensorData.Matrix(crandn(rng, (k, n))))
    return Tensor.new_composite([a, b]), ContractionPath.simple([(0, 1)])


@pytest.mark.parametrize("qubits,rounds", [(12, 6), (16, 8)])
def test_amplitude_against_torch(ctx, qubits, rounds):
    from tnc_b200.tensornetwork import leaves
    tn = amplitude_net(qubits, rounds, 5)
    path = greedy(tn)
    n = len(leaves(tn))
    ec = check_against_reference(ctx, tn, path, list(range(n)), 1)
    assert ec["k0"] > 0, ec
    if qubits == 16:
        assert ec["k1_dmma"] > 0, ec
    check_against_reference(ctx, tn, path, [0, n // 2, n - 1], 2)


def test_statevector_against_torch(ctx):
    tn = statevector_net(1)
    path = greedy(tn)
    seed = int(np.random.default_rng().integers(1 << 31))
    ec = check_against_reference(ctx, tn, path, list(range(len(tn.tensors))), seed)
    assert ec["k2"] >= 2, (ec, seed)                                            # the forward K2 pair and its tangent


def test_int8_pair_at_engine_bound(ctx):
    """Ṙ = Ȧ B + A Ḃ, all three pairs on the int8 engine: within its bound of each product plus FP64 rounding"""
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(3)
    tn, path = pair_net(rng)
    A, B = leaf_array(tn.tensors[0]), leaf_array(tn.tensors[1])
    dA, dB = crandn(rng, A.shape), crandn(rng, B.shape)
    plan = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    plan.stage(tn)
    (val, tan), ec = counted(ctx, lambda: plan.jvp({0: dA, 1: dB}))
    assert ec["k1_tcgen05"] == 3, ec
    ref = B.T @ dA.T + (dB.T @ A.T)                                          # result legs (2, 0): C[n, m]
    unit = tb.tcgen05_bound(A.shape[1])["bound"]
    bound = unit * (np.abs(dA).max() * np.abs(B).max() + np.abs(A).max() * np.abs(dB).max())
    err = np.abs(tan - ref).max()
    assert err <= bound + 1e-14 * np.abs(ref).max(), (err, bound)


# ================================================================================================================
# 2. bench.py's network
# ================================================================================================================
def test_bench_network(ctx):
    sys.path.insert(0, ROOT)
    import bench
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = bench.build_network()
    path = bench.greedy_path(tn)
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    rng = np.random.default_rng(17)
    tans = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    plain = NetworkPlan(tn, path, ctx=ctx)
    plain.stage(tn)
    ref = plain.run().to_numpy()
    del plain
    g = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    g.stage(tn)
    g.run()
    S = complex(crandn(rng, ()))
    G = g.vjp(np.asarray(S))
    del g
    ctx.trim()
    plan = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    plan.stage(tn)
    (val, tan), ec = counted(ctx, lambda: plan.jvp(tans))
    assert ec["k1_tcgen05"] >= 1, ec
    assert np.array_equal(val.to_numpy(), ref)                                # the value is the plain plan's, bit for bit
    val2, tan2 = plan.jvp(tans)
    assert np.array_equal(tan2, tan) and np.array_equal(val2.to_numpy(), ref)   # repeatable
    # adjoint identity with the reverse mode: S Ṙ = sum_l <G_l, Ẋ_l>
    lhs = S * complex(tan)
    terms = [np.sum(G[i] * tans[i]) for i in G]
    rhs = complex(np.sum(terms))
    mag = abs(S) * float(sum(np.sum(np.abs(G[i]) * np.abs(tans[i])) for i in G))
    assert abs(lhs - rhs) <= 1e-9 * mag, (lhs, rhs, mag)
    # multilinearity: Ẋ_l = X_l for every leaf gives n R
    _, tan_x = plan.jvp({i: x for i, x in enumerate(xs)})
    r = complex(ref)
    assert abs(complex(tan_x) - len(lv) * r) <= 1e-9 * len(lv) * abs(r), (complex(tan_x), len(lv) * r)
    del plan
    ctx.trim()


# ================================================================================================================
# 3. batches
# ================================================================================================================
def test_batch_bit_identity(ctx, monkeypatch):
    """10 pair networks (int8 engine) on a 1 GiB static-workspace limit: 3 passes; sub-ranges; stage_instances =
    stage_batch; device tangents = host tangents"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(8)
    tn0, path = pair_net(rng)
    A0 = leaf_array(tn0.tensors[0])
    B = leaf_array(tn0.tensors[1])
    n = 10
    As = crandn(rng, (n,) + A0.shape)
    dA, dB = crandn(rng, As.shape), crandn(rng, (n,) + B.shape)
    nets = []
    for i in range(n):
        a = Tensor([0, 1], list(A0.shape))
        a.set_tensor_data(TensorData.Matrix(As[i]))
        nets.append(Tensor.new_composite([a, tn0.tensors[1]]))
    plan = NetworkPlan.for_tangents(tn0, path, ctx=ctx)
    assert plan.info()["peak_bytes"] > (1 << 30) // 5                         # at most 4 copies per pass under 1 GiB
    singles = []
    for i in range(n):
        plan.stage(nets[i])
        v, t = plan.jvp({0: dA[i], 1: dB[i]})
        singles.append((v.to_numpy(), t))
    # device tangents give the bits host tangents give
    dev = {0: torch.from_numpy(dA[n - 1]).cuda(), 1: torch.from_numpy(dB[n - 1]).cuda()}
    vd, td = plan.jvp(dev)
    assert np.array_equal(td, singles[-1][1]) and np.array_equal(vd.to_numpy(), singles[-1][0])
    plan.stage_batch(nets)
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    _, vals, rows = plan.jvp_batch(0, n, {0: dA, 1: dB})
    for i in range(n):
        assert np.array_equal(vals[i], singles[i][0]) and np.array_equal(rows[i], singles[i][1]), i
    _, vals, rows = plan.jvp_batch(3, 5, {0: dA[3:8], 1: dB[3:8]})
    for i in range(5):
        assert np.array_equal(vals[i], singles[3 + i][0]) and np.array_equal(rows[i], singles[3 + i][1]), i
    # stage_instances from device memory: A per instance, B from the template; tangents on the device
    plan.stage_instances(tn0, {0: torch.from_numpy(As).cuda()}, n)
    _, vals2, rows2 = plan.jvp_batch(0, n, {0: torch.from_numpy(dA).cuda(), 1: torch.from_numpy(dB).cuda()})
    for i in range(n):
        assert np.array_equal(vals2[i], singles[i][0]) and np.array_equal(rows2[i], singles[i][1]), i
    monkeypatch.delenv("TNCB_PLAN_WS_GB")
    del plan
    ctx.trim()


def test_directions_of_one_network(ctx):
    """P tangent directions of one statevector network as P stride-0 instances: row p = jvp along direction p; the
    columns of the Jacobian in one call, and a shared leaf's tangent broadcast to every row"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    tn = statevector_net(2)
    path = greedy(tn)
    wrt = [k for k, t in enumerate(tn.tensors) if len(t.legs) == 4][:6]
    plan = NetworkPlan.for_tangents(tn, path, wrt, ctx=ctx)
    plan.stage(tn)
    rng = np.random.default_rng(4)
    P = 8
    shapes = {i: tuple(int(d) for d in tn.tensors[i].bond_dims) for i in wrt}
    tans = {i: crandn(rng, (P,) + shapes[i]) for i in wrt[:-1]}
    tans[wrt[-1]] = crandn(rng, shapes[wrt[-1]])                               # shared by every direction
    first = wrt[0]
    plan.stage_instances(tn, {first: torch.from_numpy(leaf_array(tn.tensors[first])).cuda()}, P)
    _, vals, rows = plan.jvp_batch(0, P, tans)
    for p in range(P):
        v, t = plan.jvp({i: (x[p] if x.ndim > len(shapes[i]) else x) for i, x in tans.items()})
        assert np.array_equal(rows[p], t) and np.array_equal(vals[p], v.to_numpy()), p


# ================================================================================================================
# 4. torch
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


def torch_setup(seed=11):
    tn = amplitude_net(6, 4, seed)
    lv = list(tn.tensors)
    one = [k for k, t in enumerate(lv) if len(t.legs) == 2][:3]
    two = [k for k, t in enumerate(lv) if len(t.legs) == 4][:1]
    idx = one + two
    tn = as_matrix_leaves(tn, idx)
    return tn, greedy(tn), idx, lv


def ref_with(tn, path, idx, xs, ts):
    """torch.func.jvp of the replay with leaves idx replaced by xs (tangents ts)"""
    import torch
    from tnc_b200.tensornetwork import leaves
    base = [torch.tensor(leaf_array(l)) for l in leaves(tn)]

    def f(*ys):
        full = list(base)
        for k, y in zip(idx, ys):
            full[k] = y
        return replay(tn, path, full)[1]
    return torch.func.jvp(f, tuple(x.cpu() for x in xs), tuple(t.cpu() for t in ts))


@pytest.mark.parametrize("on_device", [False, True])
def test_network_function_forward_mode(ctx, on_device):
    import torch
    import torch.autograd.forward_ad as fwAD
    from tnc_b200.autograd import network_function
    tn, path, idx, lv = torch_setup()
    dev = "cuda" if on_device else "cpu"
    f = network_function(tn, path, idx, ctx=ctx, on_device=on_device)
    rng = np.random.default_rng(5)
    xs = [torch.tensor(crandn(rng, lv[k].bond_dims), device=dev) for k in idx]
    ts = [torch.tensor(crandn(rng, lv[k].bond_dims), device=dev) for k in idx]
    with fwAD.dual_level():
        out = f(*[fwAD.make_dual(x, t) for x, t in zip(xs, ts)])
        t_fwd = fwAD.unpack_dual(out).tangent.clone()
    p, t_func = torch.func.jvp(f, tuple(xs), tuple(ts))
    assert t_fwd.device.type == dev and t_func.device.type == dev
    assert torch.equal(t_fwd, t_func)
    _, ref = ref_with(tn, path, idx, xs, ts)
    scale = float(sum(torch.abs(t).sum() * torch.abs(x).sum() for x, t in zip(xs, ts)))
    assert abs(complex(t_func.cpu()) - complex(ref)) <= 1e-12 * max(abs(complex(ref)), 1e-3 * scale)
    # one input without a tangent
    with fwAD.dual_level():
        out = f(*[fwAD.make_dual(xs[0], ts[0])] + xs[1:])
        t1 = fwAD.unpack_dual(out).tangent
    _, ref1 = ref_with(tn, path, idx, xs, [ts[0]] + [torch.zeros_like(x) for x in xs[1:]])
    assert abs(complex(t1.cpu()) - complex(ref1)) <= 1e-12 * max(abs(complex(ref1)), 1e-3 * scale)
    # reverse mode through the same function is unchanged: the gradients of a fresh function, bit for bit
    ys = [x.clone().requires_grad_(True) for x in xs]
    f(*ys).abs().backward()
    fresh = network_function(tn, path, idx, ctx=ctx, on_device=on_device)
    zs = [x.clone().requires_grad_(True) for x in xs]
    fresh(*zs).abs().backward()
    for y, z in zip(ys, zs):
        assert torch.equal(y.grad, z.grad)
    if on_device:                                                             # the host variant gives the same bits
        host = network_function(tn, path, idx, ctx=ctx)
        _, t_host = torch.func.jvp(host, tuple(x.cpu() for x in xs), tuple(t.cpu() for t in ts))
        assert torch.equal(t_host, t_func.cpu())


@pytest.mark.parametrize("on_device", [False, True])
def test_network_function_batched_forward_mode(ctx, on_device):
    """one batched input (tangent per instance) and three shared ones (one tangent for every instance)"""
    import torch
    from tnc_b200.autograd import network_function
    tn, path, idx, lv = torch_setup()
    dev = "cuda" if on_device else "cpu"
    f = network_function(tn, path, idx, ctx=ctx, batched=[idx[0]], on_device=on_device)
    rng = np.random.default_rng(6)
    Bn = 3
    xs = [torch.tensor(crandn(rng, ((Bn,) if k == idx[0] else ()) + tuple(lv[k].bond_dims)), device=dev) for k in idx]
    ts = [torch.tensor(crandn(rng, x.shape), device=dev) for x in xs]
    p, t = torch.func.jvp(f, tuple(xs), tuple(ts))
    assert tuple(t.shape) == (Bn,) and t.device.type == dev
    for b in range(Bn):
        _, ref = ref_with(tn, path, idx, [xs[0][b]] + xs[1:], [ts[0][b]] + ts[1:])
        scale = float(sum(torch.abs(tt).sum() * torch.abs(x).sum() for x, tt in zip(xs, ts)))
        assert abs(complex(t[b].cpu()) - complex(ref)) <= 1e-12 * max(abs(complex(ref)), 1e-3 * scale), b


def test_angle_derivative(ctx):
    """d amp / d theta_k along one angle of torch-built rx / ry / rz gates, against central finite differences"""
    import torch
    from tnc_b200.autograd import network_function
    tn, path, idx, lv = torch_setup(12)
    f = network_function(tn, path, idx, ctx=ctx)
    I = torch.eye(2, dtype=torch.complex128)
    X = torch.tensor([[0, 1], [1, 0]], dtype=torch.complex128)
    Y = torch.tensor([[0, -1j], [1j, 0]], dtype=torch.complex128)
    Z = torch.tensor([[1, 0], [0, -1]], dtype=torch.complex128)
    fourq = torch.tensor(leaf_array(lv[idx[3]]))

    def amp(theta):
        mats = [torch.cos(theta[k] / 2) * I - 1j * torch.sin(theta[k] / 2) * P for k, P in enumerate((X, Y, Z))]
        return f(*[m.reshape(lv[k].bond_dims) for m, k in zip(mats, idx[:3])], fourq)

    theta = torch.tensor([0.3, -1.1, 0.7], dtype=torch.float64)
    h = 1e-5
    for k in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[k] = 1.0
        _, d = torch.func.jvp(amp, (theta,), (e,))
        fd = (complex(amp(theta + h * e)) - complex(amp(theta - h * e))) / (2 * h)
        assert abs(complex(d) - fd) <= 1e-7 * max(1.0, abs(fd)), (k, complex(d), fd)


def test_sliced_forward_mode_refused(ctx):
    import torch
    from tnc_b200.autograd import network_function
    tn, path, idx, lv = torch_setup()
    leg = next(l for l in lv[idx[0]].legs)
    f = network_function(tn, path, idx, ctx=ctx, sliced_legs=[leg])
    xs = [torch.tensor(leaf_array(lv[k])) for k in idx]
    with pytest.raises(NotImplementedError, match="sliced_legs"):
        torch.func.jvp(f, tuple(xs), tuple(torch.ones_like(x) for x in xs))


# ================================================================================================================
# 5. errors
# ================================================================================================================
def raw_jvp(ctx, handle, tangents, outs=(True, True)):
    o = [C.c_void_p() for _ in outs]
    return ctx._l.tncb_plan_jvp(ctx.handle, handle, tangents.handle if tangents is not None else None,
                                *[C.byref(x) if w else None for x, w in zip(o, outs)])


def raw_jvp_batch(ctx, handle, first, count, tangents, outs=(True, True)):
    o = [C.c_void_p() for _ in outs]
    return ctx._l.tncb_plan_jvp_batch(ctx.handle, handle, first, count, tangents.handle if tangents is not None else None,
                                      *[C.byref(x) if w else None for x, w in zip(o, outs)])


def test_errors(ctx, monkeypatch):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.contraction import _Marshal
    from tnc_b200.tensornetwork.tensordata import TensorData
    amp = amplitude_net(10, 4, 6)
    amp_path = greedy(amp)
    t_amp = NetworkPlan.for_tangents(amp, amp_path, ctx=ctx)
    te = sum(int(np.prod(t.bond_dims)) for t in amp.tensors)
    plain = NetworkPlan(amp, amp_path, ctx=ctx)
    plain.stage(amp)
    g_amp = NetworkPlan.for_gradients(amp, amp_path, ctx=ctx)
    a = Tensor(list(range(32)) + [100], [1] * 32 + [2])
    a.set_tensor_data(TensorData.Matrix(np.ones([1] * 32 + [2])))
    b = Tensor([100] + list(range(32, 64)), [2] + [1] * 32)
    b.set_tensor_data(TensorData.Matrix(np.ones([2] + [1] * 32)))
    r64 = Tensor.new_composite([a, b])
    t64 = NetworkPlan.for_tangents(r64, ContractionPath.simple([(0, 1)]), ctx=ctx)
    t64.stage_batch([r64])
    good = DeviceTensor.from_numpy(ctx, np.ones(te, dtype=np.complex128))
    wrong = DeviceTensor.from_numpy(ctx, np.ones(te + 1, dtype=np.complex128))
    rows3 = DeviceTensor.from_numpy(ctx, np.ones((3, te), dtype=np.complex128))
    rows2 = DeviceTensor.from_numpy(ctx, np.ones((2, te), dtype=np.complex128))
    one64 = DeviceTensor.from_numpy(ctx, np.ones((1, 4), dtype=np.complex128))
    ctx.synchronize()
    live = ctx.stats()["arena_live_bytes"]

    def expect(rc, want):
        assert rc == want, (rc, want, ctx._l.tncb_last_error())
        ctx.synchronize()
        assert ctx.stats()["arena_live_bytes"] == live

    expect(raw_jvp(ctx, t_amp.handle, good), ERR_INVALID)                      # nothing staged
    expect(raw_jvp_batch(ctx, t_amp.handle, 0, 3, rows3), ERR_INVALID)
    expect(raw_jvp(ctx, plain.handle, good), ERR_INVALID)                      # not a tangent plan
    expect(raw_jvp(ctx, g_amp.handle, good), ERR_INVALID)
    expect(raw_jvp_batch(ctx, plain.handle, 0, 1, rows3), ERR_INVALID)
    t_amp.stage(amp)
    t_amp.stage_batch([amp] * 3)
    ctx.synchronize()
    live = ctx.stats()["arena_live_bytes"]
    expect(raw_jvp(ctx, t_amp.handle, good, outs=(False, False)), ERR_INVALID)  # no output
    expect(raw_jvp(ctx, t_amp.handle, None), ERR_INVALID)                      # no tangents
    expect(raw_jvp(ctx, t_amp.handle, wrong), ERR_SHAPE)
    expect(raw_jvp(ctx, t_amp.handle, rows3), ERR_SHAPE)
    expect(raw_jvp_batch(ctx, t_amp.handle, 0, 0, rows3), ERR_INVALID)         # count 0
    expect(raw_jvp_batch(ctx, t_amp.handle, 2, 2, rows2), ERR_INVALID)         # past the end
    expect(raw_jvp_batch(ctx, t_amp.handle, 2 ** 64 - 1, 2, rows2), ERR_INVALID)
    expect(raw_jvp_batch(ctx, t_amp.handle, 0, 3, rows3, outs=(False, False)), ERR_INVALID)
    expect(raw_jvp_batch(ctx, t_amp.handle, 0, 3, None), ERR_INVALID)
    expect(raw_jvp_batch(ctx, t_amp.handle, 0, 3, rows2), ERR_SHAPE)
    expect(raw_jvp_batch(ctx, t_amp.handle, 0, 3, good), ERR_SHAPE)
    expect(raw_jvp_batch(ctx, t64.handle, 0, 1, one64), ERR_INVALID)           # rank 64: no instance dimension
    # entry points of other plan kinds
    m = _Marshal()
    node = m.tn(amp)
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(node))
    out, n_out, legs, g = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)(), C.c_void_p()
    expect(ctx._l.tncb_plan_run(ctx.handle, t_amp.handle, C.byref(out), C.byref(n_out), legs), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_execute(ctx.handle, t_amp.handle, C.byref(node), C.byref(out), C.byref(n_out), legs), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_stage_slices(ctx.handle, t_amp.handle, 1, ptrs), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_run_slices(ctx.handle, t_amp.handle, 0, 1, C.byref(out), C.byref(n_out), legs), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_run_batch(ctx.handle, t_amp.handle, 0, 1, C.byref(out), C.byref(n_out), legs), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_vjp(ctx.handle, t_amp.handle, None, C.byref(g)), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_vjp_sliced(ctx.handle, t_amp.handle, 0, 1, None, C.byref(out), C.byref(g)), ERR_UNSUPPORTED)
    expect(ctx._l.tncb_plan_vjp_batch(ctx.handle, t_amp.handle, 0, 1, None, C.byref(out), None, None), ERR_UNSUPPORTED)
    # the legal calls next to them work
    v, t = t_amp.jvp({0: np.ones(amp.tensors[0].bond_dims)})
    _, vals, rows = t_amp.jvp_batch(0, 3, {0: np.ones(amp.tensors[0].bond_dims)})
    assert np.array_equal(rows[2], t) and np.array_equal(vals[1], v.to_numpy())
    for x in (good, wrong, rows3, rows2, one64):
        x.free()
    # creation refusals
    with pytest.raises(tb.TncbError) as e:
        NetworkPlan.for_tangents(amp, amp_path, wrt=[], ctx=ctx)
    assert e.value.status == ERR_INVALID
    one = Tensor([0, 1], [2, 2])
    one.set_tensor_data(TensorData.Matrix(np.eye(2)))
    with pytest.raises(tb.TncbError) as e:
        NetworkPlan.for_tangents(Tensor.new_composite([one]), ContractionPath.simple([]), ctx=ctx)
    assert e.value.status == ERR_UNSUPPORTED
    # not even one workspace copy under the static-workspace limit at run time: OOM
    sys.path.insert(0, ROOT)
    import bench
    bn = bench.build_network()
    big = NetworkPlan.for_tangents(bn, bench.greedy_path(bn), wrt=[0], ctx=ctx)
    big.stage_batch([bn])
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    ctx.synchronize()
    live = ctx.stats()["arena_live_bytes"]
    with pytest.raises(tb.TncbError) as e:
        big.jvp_batch(0, 1, {0: np.ones(bn.tensors[0].bond_dims)})
    assert e.value.status == ERR_OOM
    ctx.synchronize()
    assert ctx.stats()["arena_live_bytes"] == live
