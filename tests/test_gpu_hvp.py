"""Hessian-vector products of a contracted network (tncb_plan_create_hvp / tncb_plan_hvp, NetworkPlan.for_hvp,
second-order torch autograd through network_function):

  1. Ġ and Ṙ against torch.func.jvp of torch.func.vjp of a TTGT replay of the same path on the CPU (complex128), at 1e-12
     of the terms' magnitude: K0 and its level batches, K1 DMMA (16 qubits x 8 rounds), K2 (a 13-qubit statevector with
     a non-scalar seed and seed tangent), and a pair whose nine pairs take the int8 engine, at that engine's bound;
  2. bit identities: R = a plain plan's run, Ṙ = a tangent plan's jvp, G = a gradient plan's run + vjp, Ġ = vjp(Ṡ) for
     zero leaf tangents, repeated calls, host tangents = device tangents;
  3. bench.py's network with every leaf requested: Ẋ = X gives Ġ_l = (k - 1) G_l and Ṙ = k R, and the Hessian is
     symmetric, <W, H V> = <V, H W>;
  4. torch: double backward, torch.autograd.functional.hvp / hessian, torch.func.jvp of torch.func.grad and an angle
     Hessian against central differences, on the host and on the device, each against the same torch code on the CPU
     replay; first-order gradients bit-identical with and without create_graph; batched / sliced refuse create_graph;
  5. every error, with the arena's live bytes unchanged."""
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


def reference_hvp(tn, path, xs, ts, S, Sd, wrt):
    """(Ṙ, [G_l], [Ġ_l]) for l in wrt: torch.func.jvp of the holomorphic vjp of the replay, G = conj(vjp(conj(S)))"""
    import torch
    f = lambda *ys: replay(tn, path, ys)[1]

    def grads(s, *ys):
        _, fn = torch.func.vjp(f, *ys)
        g = fn(torch.conj_physical(s))
        return tuple(torch.conj_physical(g[i]) for i in wrt)

    def run(xs, ts, S, Sd):
        X = tuple(torch.tensor(x) for x in xs)
        T = tuple(torch.tensor(t) for t in ts)
        _, Rd = torch.func.jvp(f, X, T)
        G, Gd = torch.func.jvp(grads, (torch.tensor(S),) + X, (torch.tensor(Sd),) + T)
        return Rd.numpy(), [g.numpy() for g in G], [g.numpy() for g in Gd]
    Rd, G, Gd = run(xs, ts, S, Sd)
    mag = lambda v: [np.abs(x).astype(np.complex128) for x in v]
    sRd, _, sGd = run(mag(xs), mag(ts), np.abs(S).astype(np.complex128), np.abs(Sd).astype(np.complex128))
    return Rd, G, Gd, np.abs(sRd), [np.abs(x) for x in sGd]


def close(got, ref, scale):
    """within 1e-12 of the terms' magnitude (floored at 1e-3 of its largest element)"""
    return bool((np.abs(got - ref) <= 1e-12 * np.maximum(scale, scale.max() * 1e-3) + 1e-300).all())


def check_against_reference(ctx, tn, path, wrt, seed, scalar_seed=True):
    """Hessian-vector plan vs the replay's Ṙ and Ġ, and its G against the replay's; returns the engine counts"""
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    rng = np.random.default_rng(seed)
    tans = {i: crandn(rng, xs[i].shape) for i in wrt}
    ts = [tans[i] if i in tans else np.zeros_like(xs[i]) for i in range(len(lv))]
    plan = NetworkPlan.for_hvp(tn, path, wrt, ctx=ctx)
    rdims = plan.result_dims
    S, Sd = crandn(rng, rdims), crandn(rng, rdims)
    plan.stage(tn)
    (val, tan, G, Gd), ec = counted(ctx, lambda: plan.hvp(tans, S, Sd))
    Rd, Gr, Gdr, sRd, sGd = reference_hvp(tn, path, xs, ts, S, Sd, wrt)
    assert tan.shape == Rd.shape and close(tan, Rd, sRd), np.abs(tan - Rd).max()
    for k, i in enumerate(wrt):
        assert Gd[i].shape == Gdr[k].shape
        assert close(Gd[i], Gdr[k], sGd[k]), (i, np.abs(Gd[i] - Gdr[k]).max(), sGd[k].max())
        assert np.abs(G[i] - Gr[k]).max() <= 1e-12 * max(np.abs(Gr[k]).max(), 1e-300) * 1e3
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
    """A[m, k] x B[k, n]: M N K = 2^30, a pair for the int8 engine"""
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
    check_against_reference(ctx, tn, path, [n // 2], 3)             # one leaf: Ġ comes from Ṡ alone


def test_statevector_against_torch(ctx):
    """a non-scalar result: a seed and a seed tangent with the result's 2^13 entries"""
    tn = statevector_net(1)
    path = greedy(tn)
    ec = check_against_reference(ctx, tn, path, list(range(len(tn.tensors))), 7)
    assert ec["k2"] >= 2, ec


def test_int8_pairs_at_engine_bound(ctx):
    """R = A B: Ġ_A = Ṡ·B + S·Ḃ and Ġ_B = Ṡ·A + S·Ȧ on the int8 engine, within its bound of each product"""
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(3)
    tn, path = pair_net(rng)
    A, B = leaf_array(tn.tensors[0]), leaf_array(tn.tensors[1])
    dA, dB = crandn(rng, A.shape), crandn(rng, B.shape)
    m, k = A.shape
    n = B.shape[1]
    S, Sd = crandn(rng, (n, m)), crandn(rng, (n, m))                        # the result's legs are (2, 0): R[n, m]
    plan = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    plan.stage(tn)
    (val, tan, G, Gd), ec = counted(ctx, lambda: plan.hvp({0: dA, 1: dB}, S, Sd))
    assert ec["k1_tcgen05"] >= 3, ec
    mx = lambda x: np.abs(x).max()
    refs = {0: (Sd.T @ B.T + S.T @ dB.T, tb.tcgen05_bound(n)["bound"] * (mx(Sd) * mx(B) + mx(S) * mx(dB))),
            1: (A.T @ Sd.T + dA.T @ S.T, tb.tcgen05_bound(m)["bound"] * (mx(A) * mx(Sd) + mx(dA) * mx(S)))}
    for i, (ref, bound) in refs.items():
        err = np.abs(Gd[i] - ref).max()
        assert err <= bound + 1e-14 * mx(ref), (i, err, bound)
    ref = B.T @ dA.T + dB.T @ A.T
    assert np.abs(tan - ref).max() <= tb.tcgen05_bound(k)["bound"] * (mx(dA) * mx(B) + mx(A) * mx(dB)) + 1e-14 * mx(ref)


# ================================================================================================================
# 2. bit identities
# ================================================================================================================
@pytest.mark.parametrize("net", ["amp16", "pair"])
def test_bit_identities(ctx, net):
    import torch
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    rng = np.random.default_rng(21)
    if net == "pair":
        tn, path = pair_net(rng)
    else:
        tn = amplitude_net(16, 8, 5)
        path = greedy(tn)
    lv = leaves(tn)
    wrt = list(range(len(lv)))[::2] if net == "amp16" else [0, 1]
    xs = [leaf_array(l) for l in lv]
    tans = {i: crandn(rng, xs[i].shape) for i in wrt}
    h = NetworkPlan.for_hvp(tn, path, wrt, ctx=ctx)
    S, Sd = crandn(rng, h.result_dims), crandn(rng, h.result_dims)
    h.stage(tn)
    val, tan, G, Gd = h.hvp(tans, S, Sd)
    plain = NetworkPlan(tn, path, ctx=ctx)
    plain.stage(tn)
    assert np.array_equal(val, plain.run().to_numpy())                      # R: the plain plan's run
    del plain
    t = NetworkPlan.for_tangents(tn, path, wrt, ctx=ctx)
    t.stage(tn)
    assert np.array_equal(tan, t.jvp(tans)[1])                             # Ṙ: the tangent plan's jvp
    del t
    g = NetworkPlan.for_gradients(tn, path, wrt, ctx=ctx)
    g.stage(tn)
    g.run()
    Gg = g.vjp(S)
    g.run()
    Gs = g.vjp(Sd)
    del g
    for i in wrt:
        assert np.array_equal(G[i], Gg[i]), i                              # G: the gradient plan's run + vjp
    _, _, _, Gd0 = h.hvp({}, S, Sd)                                          # zero leaf tangents: Ġ = vjp(Ṡ)
    for i in wrt:
        assert np.array_equal(Gd0[i], Gs[i]), i
    again = h.hvp(tans, S, Sd)                                               # repeatable
    assert np.array_equal(again[0], val) and np.array_equal(again[1], tan)
    for i in wrt:
        assert np.array_equal(again[2][i], G[i]) and np.array_equal(again[3][i], Gd[i])
    dev = torch.device("cuda", ctx.device)                                   # device tangents, seed and seed tangent
    blocks = h.hvp_blocks({i: torch.tensor(x, device=dev) for i, x in tans.items()}, torch.tensor(S, device=dev),
                          torch.tensor(Sd, device=dev))
    host = [b.to_numpy() for b in blocks]
    offs = h.grad_offsets()
    assert np.array_equal(host[0], val) and np.array_equal(host[1], tan)
    for i in wrt:
        size = xs[i].size
        assert np.array_equal(host[2][offs[i]:offs[i] + size].reshape(xs[i].shape), G[i])
        assert np.array_equal(host[3][offs[i]:offs[i] + size].reshape(xs[i].shape), Gd[i])
    for b in blocks:
        b.free()
    del h
    ctx.trim()


# ================================================================================================================
# 3. bench.py's network
# ================================================================================================================
def test_bench_network(ctx):
    """every leaf requested (the 34 GiB Hessian-vector workspace fits an 80 GB H100): Euler's identity for the
    multilinear R and the symmetry of the Hessian"""
    sys.path.insert(0, ROOT)
    import bench
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = bench.build_network()
    path = bench.greedy_path(tn)
    lv = leaves(tn)
    k = len(lv)
    xs = [leaf_array(l) for l in lv]
    ctx.trim()
    plan = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    plan.stage(tn)
    rng = np.random.default_rng(5)
    S = np.asarray(complex(crandn(rng, ())))
    (val, tan, G, Gd), ec = counted(ctx, lambda: plan.hvp({i: x for i, x in enumerate(xs)}, S))
    assert ec["k1_tcgen05"] >= 1, ec
    r = complex(val)
    assert abs(complex(tan) - k * r) <= 1e-9 * k * abs(r), (complex(tan), k * r)
    gb = np.concatenate([G[i].ravel() for i in range(k)])
    gdb = np.concatenate([Gd[i].ravel() for i in range(k)])
    assert np.linalg.norm(gdb - (k - 1) * gb) <= 1e-9 * (k - 1) * np.linalg.norm(gb)
    V = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    W = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    HV = plan.hvp(V, S)[3]
    HW = plan.hvp(W, S)[3]
    lhs = sum(np.sum(W[i] * HV[i]) for i in range(k))
    rhs = sum(np.sum(V[i] * HW[i]) for i in range(k))
    mag = sum(np.sum(np.abs(W[i]) * np.abs(HV[i])) + np.sum(np.abs(V[i]) * np.abs(HW[i])) for i in range(k))
    assert abs(lhs - rhs) <= 1e-9 * mag, (lhs, rhs, mag)
    del plan
    ctx.trim()


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


def replay_fn(tn, path, idx):
    """the replay on the CPU as a function of the leaves idx (the others fixed)"""
    import torch
    from tnc_b200.tensornetwork import leaves
    base = [torch.tensor(leaf_array(l)) for l in leaves(tn)]

    def f(*ys):
        full = list(base)
        for k, y in zip(idx, ys):
            full[k] = y.cpu()
        return replay(tn, path, full)[1]
    return f


def angle_loss(f, lv, idx, dev):
    """|amp(theta)|^2 with rx / ry / rz gates built by torch from three angles, the fourth input fixed"""
    import torch
    I = torch.eye(2, dtype=torch.complex128)
    X = torch.tensor([[0, 1], [1, 0]], dtype=torch.complex128)
    Y = torch.tensor([[0, -1j], [1j, 0]], dtype=torch.complex128)
    Z = torch.tensor([[1, 0], [0, -1]], dtype=torch.complex128)
    fourq = torch.tensor(leaf_array(lv[idx[3]]), device=dev)

    def loss(theta):
        mats = [torch.cos(theta[k] / 2) * I - 1j * torch.sin(theta[k] / 2) * P for k, P in enumerate((X, Y, Z))]
        amp = f(*[m.reshape(lv[k].bond_dims).to(dev) for m, k in zip(mats, idx[:3])], fourq)
        return (amp.abs() ** 2).sum().cpu()
    return loss


def assert_close(got, ref, rel=1e-10):
    got, ref = got.detach().cpu(), ref.detach().cpu()
    assert got.shape == ref.shape
    err = float((got - ref).abs().max())
    assert err <= rel * max(float(ref.abs().max()), 1e-300), (err, float(ref.abs().max()))


@pytest.mark.parametrize("on_device", [False, True])
def test_network_function_second_order(ctx, on_device):
    import torch
    from tnc_b200.autograd import network_function
    tn, path, idx, lv = torch_setup()
    dev = "cuda" if on_device else "cpu"
    f = network_function(tn, path, idx, ctx=ctx, on_device=on_device)
    ref = replay_fn(tn, path, idx)
    rng = np.random.default_rng(5)
    xs = [torch.tensor(crandn(rng, lv[k].bond_dims), device=dev) for k in idx]
    vs = [torch.tensor(crandn(rng, lv[k].bond_dims), device=dev) for k in idx]

    def double_backward(fn, inputs):
        ys = [x.clone().requires_grad_(True) for x in inputs]
        loss = (fn(*ys).abs() ** 2).sum()
        g = torch.autograd.grad(loss, ys, create_graph=True)
        inner = sum((gi * vi.to(gi.device)).real.sum() for gi, vi in zip(g, vs))
        return g, torch.autograd.grad(inner, ys)

    g, hv = double_backward(f, xs)
    g_ref, hv_ref = double_backward(ref, [x.cpu() for x in xs])
    assert g[0].device.type == dev and hv[0].device.type == dev
    for a, b in zip(g, g_ref):
        assert_close(a, b)
    for a, b in zip(hv, hv_ref):
        assert_close(a, b)
    # first-order gradients: the same bits with and without create_graph
    ys = [x.clone().requires_grad_(True) for x in xs]
    (f(*ys).abs() ** 2).sum().backward()
    for y, a in zip(ys, g):
        assert torch.equal(y.grad, a.detach())
    zs = [x.clone().requires_grad_(True) for x in xs]
    (f(*zs).abs() ** 2).sum().backward(create_graph=True)
    for y, z in zip(ys, zs):
        assert torch.equal(y.grad, z.grad.detach())
    # a real loss over gate angles: functional.hvp / hessian, torch.func.jvp of torch.func.grad, central differences
    loss, loss_ref = angle_loss(f, lv, idx, dev), angle_loss(ref, lv, idx, "cpu")
    theta = torch.tensor([0.3, -1.1, 0.7], dtype=torch.float64)
    v = torch.tensor([0.2, 0.5, -0.4], dtype=torch.float64)
    H = torch.autograd.functional.hessian(loss, theta)
    H_ref = torch.autograd.functional.hessian(loss_ref, theta)
    assert_close(H, H_ref)
    assert_close(H, H.T, rel=1e-12)
    _, hvp = torch.autograd.functional.hvp(loss, theta, v)
    _, hvp_ref = torch.autograd.functional.hvp(loss_ref, theta, v)
    assert_close(hvp, hvp_ref)
    _, fjvp = torch.func.jvp(torch.func.grad(loss), (theta,), (v,))
    assert_close(fjvp, hvp_ref)
    h = 1e-5
    grad = lambda t: torch.autograd.functional.jacobian(loss, t)
    for k in range(3):
        e = torch.zeros(3, dtype=torch.float64)
        e[k] = 1.0
        fd = (grad(theta + h * e) - grad(theta - h * e)) / (2 * h)
        assert float((H[:, k] - fd).abs().max()) <= 1e-6 * max(1.0, float(fd.abs().max())), (k, H[:, k], fd)
    if on_device:                                                             # the host variant gives the same bits
        host = network_function(tn, path, idx, ctx=ctx)
        g_host, hv_host = double_backward(host, [x.cpu() for x in xs])
        for a, b in zip(hv, hv_host):
            assert torch.equal(a.cpu(), b)


def test_second_order_refused_batched_and_sliced(ctx):
    import torch
    from tnc_b200.autograd import network_function
    tn, path, idx, lv = torch_setup()
    xs = [torch.tensor(leaf_array(lv[k])) for k in idx]
    leg = next(l for l in lv[idx[0]].legs)
    sl = network_function(tn, path, idx, ctx=ctx, sliced_legs=[leg])
    bt = network_function(tn, path, idx, ctx=ctx, batched=[idx[0]])
    for fn, ins, what in ((sl, xs, "sliced_legs"), (bt, [xs[0][None]] + xs[1:], "batched")):
        ys = [x.clone().requires_grad_(True) for x in ins]
        loss = (fn(*ys).abs() ** 2).sum()
        with pytest.raises(NotImplementedError, match=what):
            torch.autograd.grad(loss, ys, create_graph=True)
        ys = [x.clone().requires_grad_(True) for x in ins]
        (fn(*ys).abs() ** 2).sum().backward()                                 # first order still works
        assert all(y.grad is not None for y in ys)


# ================================================================================================================
# 5. errors
# ================================================================================================================
def raw_hvp(ctx, handle, tangents, seed=None, seed_tangent=None, outs=(True, True, True, True)):
    o = [C.c_void_p() for _ in outs]
    h = lambda t: t.handle if t is not None else None
    return ctx._l.tncb_plan_hvp(ctx.handle, handle, h(tangents), h(seed), h(seed_tangent),
                                *[C.byref(x) if w else None for x, w in zip(o, outs)])


def test_errors(ctx):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan
    from tnc_b200.tensornetwork.contraction import _Marshal
    sv = statevector_net(2)
    sv_path = greedy(sv)
    h = NetworkPlan.for_hvp(sv, sv_path, ctx=ctx)
    te = sum(int(np.prod(t.bond_dims)) for t in sv.tensors)
    dims = h.result_dims
    plain = NetworkPlan(sv, sv_path, ctx=ctx)
    plain.stage(sv)
    g = NetworkPlan.for_gradients(sv, sv_path, ctx=ctx)
    good = DeviceTensor.from_numpy(ctx, np.ones(te, dtype=np.complex128))
    wrong = DeviceTensor.from_numpy(ctx, np.ones(te + 1, dtype=np.complex128))
    seed = DeviceTensor.from_numpy(ctx, np.ones(dims, dtype=np.complex128))
    bad_seed = DeviceTensor.from_numpy(ctx, np.ones(dims[:-1] + (dims[-1] * 2,), dtype=np.complex128))
    ctx.synchronize()
    live = ctx.stats()["arena_live_bytes"]

    def expect(rc, want):
        assert rc == want, (rc, want, ctx._l.tncb_last_error())
        ctx.synchronize()
        assert ctx.stats()["arena_live_bytes"] == live

    expect(raw_hvp(ctx, h.handle, good, seed), ERR_INVALID)                   # nothing staged
    expect(raw_hvp(ctx, plain.handle, good, seed), ERR_INVALID)               # not a Hessian-vector plan
    expect(raw_hvp(ctx, g.handle, good, seed), ERR_INVALID)
    h.stage(sv)
    ctx.synchronize()
    live = ctx.stats()["arena_live_bytes"]
    expect(raw_hvp(ctx, h.handle, good, seed, outs=(False,) * 4), ERR_INVALID)   # no output
    expect(raw_hvp(ctx, h.handle, None, seed), ERR_INVALID)                   # no tangents
    expect(raw_hvp(ctx, h.handle, good, None), ERR_INVALID)                   # no seed for a rank-13 result
    expect(raw_hvp(ctx, h.handle, wrong, seed), ERR_SHAPE)
    expect(raw_hvp(ctx, h.handle, good, bad_seed), ERR_SHAPE)
    expect(raw_hvp(ctx, h.handle, good, seed, bad_seed), ERR_SHAPE)
    # the other entry points refuse a Hessian-vector plan
    m = _Marshal()
    node = m.tn(sv)
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(node))
    out, n_out, legs, gg = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)(), C.c_void_p()
    L, cx, p = ctx._l, ctx.handle, h.handle
    for rc in (L.tncb_plan_run(cx, p, C.byref(out), C.byref(n_out), legs),
               L.tncb_plan_execute(cx, p, C.byref(node), C.byref(out), C.byref(n_out), legs),
               L.tncb_plan_stage_slices(cx, p, 1, ptrs),
               L.tncb_plan_run_slices(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs),
               L.tncb_plan_run_batch(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs),
               L.tncb_plan_vjp(cx, p, seed.handle, C.byref(gg)),
               L.tncb_plan_vjp_sliced(cx, p, 0, 1, seed.handle, C.byref(out), C.byref(gg)),
               L.tncb_plan_stage_batch(cx, p, 1, ptrs),
               L.tncb_plan_vjp_batch(cx, p, 0, 1, None, C.byref(out), None, None),
               L.tncb_plan_jvp(cx, p, good.handle, C.byref(out), None),
               L.tncb_plan_jvp_batch(cx, p, 0, 1, good.handle, C.byref(out), None)):
        expect(rc, ERR_UNSUPPORTED)
    # the legal call next to them works, with every output alone
    v, t, G, Gd = h.hvp({0: np.ones(sv.tensors[0].bond_dims)}, np.ones(dims))
    for k in range(4):
        outs = [C.c_void_p() for _ in range(4)]
        assert L.tncb_plan_hvp(cx, p, good.handle, seed.handle, None,
                               *[C.byref(o) if j == k else None for j, o in enumerate(outs)]) == 0
        DeviceTensor.adopt(ctx, outs[k]).free()
    for x in (good, wrong, seed, bad_seed):
        x.free()
    with pytest.raises(tb.TncbError) as e:
        NetworkPlan.for_hvp(sv, sv_path, wrt=[], ctx=ctx)
    assert e.value.status == ERR_INVALID
