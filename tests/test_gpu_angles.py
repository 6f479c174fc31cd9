"""Derivatives with respect to gate angles on the H100 (tncb_angles_*, tnc_b200.angles, autograd.circuit_function).

References: tncb_gate_matrix for the gate rows; a CPU torch replay that builds every gate from θ with torch ops for
values, gradients, tangents and Hessians; exact parameter shifts of existing plans at bench.py's scale; bit identities of
the rows, folds, batched instances and repeated calls; the C ABI's argument errors with the arena unchanged."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE = -1, -2


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


def cuda(x):
    import torch
    return torch.as_tensor(np.asarray(x, dtype=np.float64)).cuda()


# ------------------------------------------------------------------------------------------------ CPU torch replay
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


def torch_gate(name, a, adjoint):
    """the gate matrix from the angle tensors `a` with torch ops (differentiable), row-major [d, d]"""
    import torch
    one, zero = torch.ones((), dtype=torch.complex128), torch.zeros((), dtype=torch.complex128)
    e = lambda x: torch.exp(1j * x.to(torch.complex128))
    c = lambda x: torch.cos(x).to(torch.complex128)
    s = lambda x: torch.sin(x).to(torch.complex128)
    if name == "u":
        m = [[c(a[0] / 2), -e(a[2]) * s(a[0] / 2)], [e(a[1]) * s(a[0] / 2), e(a[1] + a[2]) * c(a[0] / 2)]]
    elif name == "rx":
        m = [[c(a[0] / 2), -1j * s(a[0] / 2)], [-1j * s(a[0] / 2), c(a[0] / 2)]]
    elif name == "ry":
        m = [[c(a[0] / 2), -s(a[0] / 2)], [s(a[0] / 2), c(a[0] / 2)]]
    elif name == "rz":
        m = [[e(-a[0] / 2), zero], [zero, e(a[0] / 2)]]
    elif name == "cp":
        m = [[one, zero, zero, zero], [zero, one, zero, zero], [zero, zero, one, zero], [zero, zero, zero, e(a[0])]]
    else:
        m = [[one, zero, zero, zero], [zero, c(a[0]), -1j * s(a[0]), zero], [zero, -1j * s(a[0]), c(a[0]), zero],
             [zero, zero, zero, e(-a[1])]]
    M = torch.stack([torch.stack(list(r)) for r in m])
    return M.conj().T if adjoint else M


def replay_fn(tn, path, amap):
    """θ (CPU float64 torch) -> R of the network with every mapped gate built from θ"""
    import torch
    from tnc_b200.gates import load_gate, load_gate_adjoint
    from tnc_b200.tensornetwork import leaves
    lv = leaves(tn)
    refs = {}
    for l, s, p, c in amap.refs:
        refs.setdefault(l, []).append((s, p, c))
    fixed = []
    for i, t in enumerate(lv):
        td = t.tensordata
        if td.kind == "gate":
            arr = (load_gate_adjoint if td.gate[2] else load_gate)(td.gate[0], td.gate[1])
        else:
            arr = np.asarray(td.matrix, dtype=np.complex128)
        fixed.append(torch.tensor(np.asarray(arr, dtype=np.complex128).reshape([int(d) for d in t.bond_dims])))

    def f(theta):
        xs = list(fixed)
        for l, rs in refs.items():
            name, own, adj = lv[l].tensordata.gate
            a = [torch.tensor(float(x), dtype=torch.float64) for x in own]
            for s, p, c in rs:
                a[s] = c * theta[p]
            xs[l] = torch_gate(name, a, adj).reshape(fixed[l].shape)
        return replay(tn, path, xs)[1]
    return f


def mixed_circuit(qubits=8, seed=3):
    """all six angle gates, adjoint flags, a tied rx(2β) layer and an angle used twice with different scales"""
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    from tnc_b200.tensornetwork import leaves
    rng = np.random.default_rng(seed)
    c = Circuit()
    q = c.allocate_register(qubits)
    plan = []                                    # (gate, qubits, adjoint, [(slot, param, scale)])
    for i in range(qubits):
        plan.append(("h", [i], False, []))
    for layer in range(2):
        for i in range(qubits):
            plan.append(("rx", [i], False, [(0, 0, 2.0)]))               # rx(2β), β = θ[0], on every qubit
        for i in range(0, qubits - 1, 2):
            plan.append(("fsim", [i, i + 1], layer == 1, [(0, 1 + 2 * (i // 2), 1.0), (1, 2 + 2 * (i // 2), 1.0)]))
        k = 1 + qubits
        plan.append(("u", [0], layer == 0, [(0, k, 1.0), (1, k + 1, 0.5), (2, k + 2, -1.5)]))
        plan.append(("ry", [1], False, [(0, k + 3, 1.0)]))
        plan.append(("rz", [2], True, [(0, k + 4, 3.0)]))
        plan.append(("cp", [3, 4], layer == 1, [(0, k + 5, 1.0)]))
        plan.append(("rz", [5], False, [(0, k + 5, -0.7)]))                 # θ[k+5] used by cp and rz
        plan.append(("u", [6], False, [(1, k + 6, 1.0)]))                   # slots 0 and 2 keep their own angle
    n_params = 1 + qubits + 7
    theta = rng.uniform(-math.pi, math.pi, n_params)
    own = {"u": 3, "rx": 1, "ry": 1, "rz": 1, "cp": 1, "fsim": 2}
    for g, qs, adj, _ in plan:
        c.append_gate(g, list(rng.uniform(-2, 2, own.get(g, 0))), [q[x] for x in qs], adjoint=adj)
    tn = c.into_amplitude_network("0" * qubits)[0]
    gate_leaves = [i for i, t in enumerate(leaves(tn)) if t.tensordata.kind == "gate"]
    assert len(gate_leaves) == len(plan)
    refs = [(l, s, p, sc) for l, (_, _, _, rs) in zip(gate_leaves, plan) for s, p, sc in rs]
    return tn, AngleMap(refs, n_params, theta)


# ------------------------------------------------------------------------------------------------ 1. gates
SWEEP = [0.0, -0.0, math.pi, -math.pi, math.pi / 2, -math.pi / 2, 0.3, 0.2, -1.7, 2.5, 1e3, -1e3, 123.456, -999.9, 7.0]


def ulps(got, want):
    """|got - want| in units of the last place of want (0 where equal, signed zeros included)"""
    return np.where(got == want, 0.0, np.abs(got - want) / np.spacing(np.abs(want)))


def test_gate_rows_against_host_table(ctx):
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.gates import load_gate, load_gate_adjoint
    from tnc_b200.tensornetwork import leaves
    from tnc_b200.builders import Circuit
    c = Circuit()
    q = c.allocate_register(2)
    gates = [("u", 3, False), ("u", 3, True), ("rx", 1, False), ("ry", 1, True), ("rz", 1, False), ("rz", 1, True),
             ("cp", 1, False), ("cp", 1, True), ("fsim", 2, False), ("fsim", 2, True)]
    for g, n, adj in gates:
        c.append_gate(g, [0.1] * n, [q[0]] if g in ("u", "rx", "ry", "rz") else [q[0], q[1]], adjoint=adj)
    tn = c.into_amplitude_network("00")[0]
    lv = leaves(tn)
    gl = [i for i, t in enumerate(lv) if t.tensordata.kind == "gate"]
    refs, P = [], 0
    for l, (g, n, adj) in zip(gl, gates):
        for s in range(n):
            refs.append((l, s, P, 1.0))
            P += 1
    amap = AngleMap(refs, P)
    ang = Angles(ctx, tn, amap)
    n = len(SWEEP)                               # every triple of SWEEP values on three consecutive slots
    theta = np.array([[SWEEP[(i // n ** (k % 3)) % n] for k in range(P)] for i in range(n ** 3)])
    got = ang.gates(cuda(theta)).to_numpy()
    worst = 0.0
    for i, th in enumerate(theta):
        p = 0
        for l, (g, n, adj) in zip(gl, gates):
            want = (load_gate_adjoint if adj else load_gate)(g, list(th[p:p + n])).reshape(-1)
            off = ang.offsets[l]
            row = got[i, off:off + want.size]
            worst = max(worst, ulps(row.real, want.real).max(), ulps(row.imag, want.imag).max())
            p += n
    assert worst <= 4, worst


def test_set_leaves_matches_host_staging(ctx):
    import torch
    from tnc_b200.angles import Angles
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, amap = mixed_circuit()
    path = greedy(tn)
    plan = NetworkPlan(tn, path, ctx=ctx)
    plan.stage(tn)
    ang = Angles(ctx, tn, amap)
    for seed in range(3):
        th = np.random.default_rng(seed).uniform(-4, 4, amap.n_params)
        ang.set_leaves(plan, cuda(th))
        got = complex(plan.run().to_numpy())
        # host staging of the Gate network at those angles
        lv = leaves(tn)
        saved = {}
        for l, s, p, c in amap.refs:
            name, own, adj = lv[l].tensordata.gate if l not in saved else saved[l]
            a = list(saved[l][1]) if l in saved else list(own)
            a[s] = c * th[p]
            saved[l] = (name, tuple(a), adj)
        old = {l: lv[l].tensordata for l in saved}
        for l, g in saved.items():
            lv[l].set_tensor_data(TensorData.Gate(*g))
        try:
            ref = complex(NetworkPlan(tn, path, ctx=ctx).execute(tn).to_numpy())
        finally:
            for l, td in old.items():
                lv[l].set_tensor_data(td)
        assert abs(got - ref) <= 1e-14 * abs(ref), (got, ref)


# ------------------------------------------------------------------------------------------------ 2. against torch
def test_against_torch_replay(ctx):
    import torch
    from tnc_b200.angles import Angles
    from tnc_b200.tensornetwork import NetworkPlan
    tn, amap = mixed_circuit()
    path = greedy(tn)
    f = replay_fn(tn, path, amap)
    th = torch.tensor(amap.theta0)
    R = f(th)
    gr = torch.autograd.functional.jacobian(lambda t: f(t).real, th) + 1j * torch.autograd.functional.jacobian(lambda t: f(t).imag, th)
    Hre = torch.func.hessian(lambda t: f(t).real)(th)
    Him = torch.func.hessian(lambda t: f(t).imag)(th)
    v = np.random.default_rng(1).standard_normal(amap.n_params)
    Hv = (Hre.numpy() + 1j * Him.numpy()) @ v
    tdot = np.random.default_rng(2).standard_normal(amap.n_params)
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()
    wrt = amap.leaves()
    # vjp + pullback
    gp = NetworkPlan.for_gradients(tn, path, wrt=wrt, ctx=ctx)
    gp.stage(tn)
    ang = Angles(ctx, tn, amap, gp)
    T = cuda(amap.theta0)
    ang.set_leaves(gp, T)
    assert rel(gp.run().to_numpy(), R.numpy()) < 1e-12
    G = gp.vjp_block()
    g = ang.pullback(T, G)[0].to_numpy()[0]
    assert rel(g, gr.numpy()) < 1e-12
    # tangents + jvp
    tp = NetworkPlan.for_tangents(tn, path, wrt=wrt, ctx=ctx)
    tp.stage(tn)
    at = Angles(ctx, tn, amap, tp)
    at.set_leaves(tp, T)
    tan = at.tangents(T, cuda(tdot))
    out = C.c_void_p()
    assert ctx._l.tncb_plan_jvp(ctx.handle, tp.handle, tan.handle, None, C.byref(out)) == 0
    from tnc_b200 import DeviceTensor
    rdot = DeviceTensor.adopt(ctx, out).to_numpy()
    assert rel(rdot, gr.numpy() @ tdot) < 1e-12
    # hvp + pullback(G, Ġ, v)
    hp = NetworkPlan.for_hvp(tn, path, wrt=wrt, ctx=ctx)
    hp.stage(tn)
    ah = Angles(ctx, tn, amap, hp)
    ah.set_leaves(hp, T)
    tv = ah.tangents(T, cuda(v))
    _, _, Gh, Ghd = hvp_blocks(ctx, hp, tv)
    hv = ah.pullback(T, Gh, Ghd, cuda(v))[0].to_numpy()[0]
    assert rel(hv, Hv) < 1e-12
    # the full angle Hessian: P directions through hvp_batch (rows), one pullback with the direction rows
    P = amap.n_params
    eye = np.eye(P)
    trows = ah.tangents(T, cuda(eye))
    Grows, Gdrows = hvp_batch_rows(ctx, hp, P, trows)
    H = ah.pullback(T, Grows, Gdrows, cuda(eye))[0].to_numpy()
    assert rel(H, Hre.numpy() + 1j * Him.numpy()) < 1e-12


def hvp_blocks(ctx, plan, tangents):
    from tnc_b200 import DeviceTensor
    outs = [C.c_void_p() for _ in range(4)]
    assert ctx._l.tncb_plan_hvp(ctx.handle, plan.handle, tangents.handle, None, None, *[C.byref(o) for o in outs]) == 0, \
        ctx._l.tncb_last_error()
    return [DeviceTensor.adopt(ctx, o) for o in outs]


def hvp_batch_rows(ctx, plan, count, tangents):
    from tnc_b200 import DeviceTensor
    g, gd = C.c_void_p(), C.c_void_p()
    assert ctx._l.tncb_plan_hvp_batch(ctx.handle, plan.handle, count, 0, None, None, None, tangents.handle, None, None,
                                      None, None, C.byref(g), None, C.byref(gd), None) == 0, ctx._l.tncb_last_error()
    return DeviceTensor.adopt(ctx, g), DeviceTensor.adopt(ctx, gd)


# ------------------------------------------------------------------------------------------------ 3. benchmark scale
@pytest.fixture(scope="module")
def bench_net(built_lib):
    sys.path.insert(0, ROOT)
    import bench
    tn = bench.build_network()
    return tn, bench.greedy_path(tn)


def test_bench_parameter_shift(ctx, bench_net):
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, path = bench_net
    amap = AngleMap.every_angle(tn)
    gp = NetworkPlan.for_gradients(tn, path, wrt=amap.leaves(), ctx=ctx)
    gp.stage(tn)
    ang = Angles(ctx, tn, amap, gp)
    T = cuda(amap.theta0)
    ang.set_leaves(gp, T)
    R0 = complex(gp.run().to_numpy())
    G = gp.vjp_block()
    g = ang.pullback(T, G)[0].to_numpy()[0]
    # exact shifts through a plain plan on host-staged Gate networks
    lv = leaves(tn)
    plain = NetworkPlan(tn, path, ctx=ctx)
    rng = np.random.default_rng(0)
    for p in rng.choice(amap.n_params, 16, replace=False):
        l, s, _, _ = amap.refs[p]
        name, own, adj = lv[l].tensordata.gate
        vals = []
        for sign in (1, -1):
            a = list(own)
            a[s] = own[s] + sign * math.pi / 2
            lv[l].set_tensor_data(TensorData.Gate(name, tuple(a), adj))
            plain.stage(tn)
            vals.append(complex(plain.run().to_numpy()))
        lv[l].set_tensor_data(TensorData.Gate(name, own, adj))
        ref = (vals[0] - vals[1]) / 2
        assert abs(g[p] - ref) <= 1e-12 * max(abs(vals[0]), abs(vals[1])), (p, g[p], ref)
    # the transpose identity sum_p θ̇_p g_p = Ṙ
    tp = NetworkPlan.for_tangents(tn, path, wrt=amap.leaves(), ctx=ctx)
    tp.stage(tn)
    at = Angles(ctx, tn, amap, tp)
    at.set_leaves(tp, T)
    tdot = rng.standard_normal(amap.n_params)
    from tnc_b200 import DeviceTensor
    out = C.c_void_p()
    tan = at.tangents(T, cuda(tdot))
    assert ctx._l.tncb_plan_jvp(ctx.handle, tp.handle, tan.handle, None, C.byref(out)) == 0
    rdot = complex(DeviceTensor.adopt(ctx, out).to_numpy())
    assert abs(rdot - g @ tdot) <= 1e-12 * np.abs(g).sum() * np.abs(tdot).max()
    assert abs(R0) > 0


# ------------------------------------------------------------------------------------------------ 4. bit identities
def test_bit_identities(ctx):
    from tnc_b200.angles import Angles
    from tnc_b200.tensornetwork import NetworkPlan
    tn, amap = mixed_circuit(seed=5)
    path = greedy(tn)
    rng = np.random.default_rng(4)
    B, P = 5, amap.n_params
    TH = rng.uniform(-3, 3, (B, P))
    gp = NetworkPlan.for_gradients(tn, path, wrt=amap.leaves(), ctx=ctx)
    gp.stage(tn)
    ang = Angles(ctx, tn, amap, gp)
    rows = ang.gates(cuda(TH)).to_numpy()
    for i in range(B):
        assert np.array_equal(rows[i], ang.gates(cuda(TH[i])).to_numpy()[0])
    assert np.array_equal(rows, ang.gates(cuda(TH)).to_numpy())                       # repeats
    D = rng.standard_normal((B, P))
    trows = ang.tangents(cuda(TH), cuda(D)).to_numpy()
    for i in range(B):
        assert np.array_equal(trows[i], ang.tangents(cuda(TH[i]), cuda(D[i])).to_numpy())
    # B angle sets as instances: vjp_batch + pullback, row i against set_leaves + run + vjp + pullback
    ang.stage_instances(gp, tn, cuda(TH))
    _, G = gp.vjp_batch_blocks(0, B, rows=True, sum=False, values=False)[:2]
    prow, psum = ang.pullback(cuda(TH), G, rows=True, sum=True)
    prow, psum = prow.to_numpy(), psum.to_numpy()
    fold = np.zeros(P, dtype=np.complex128)
    for i in range(B):
        fold = fold + prow[i]
    assert np.array_equal(psum, fold)
    for i in range(B):
        ang.set_leaves(gp, cuda(TH[i]))
        gp.run()
        Gi = gp.vjp_block()
        assert np.array_equal(prow[i], ang.pullback(cuda(TH[i]), Gi)[0].to_numpy()[0])
        assert np.array_equal(prow[i], ang.pullback(cuda(TH[i]), Gi)[0].to_numpy()[0])    # repeats
    # P hvp_batch directions against P hvp calls
    hp = NetworkPlan.for_hvp(tn, path, wrt=amap.leaves(), ctx=ctx)
    hp.stage(tn)
    ah = Angles(ctx, tn, amap, hp)
    T = cuda(TH[0])
    ah.set_leaves(hp, T)
    V = rng.standard_normal((P, P))
    tv = ah.tangents(T, cuda(V))
    Gr, Gdr = hvp_batch_rows(ctx, hp, P, tv)
    Hb = ah.pullback(T, Gr, Gdr, cuda(V))[0].to_numpy()
    for k in range(P):
        t1 = ah.tangents(T, cuda(V[k]))
        _, _, g1, gd1 = hvp_blocks(ctx, hp, t1)
        assert np.array_equal(Hb[k], ah.pullback(T, g1, gd1, cuda(V[k]))[0].to_numpy()[0])


# ------------------------------------------------------------------------------------------------ 5. sliced
@pytest.mark.parametrize("legs", [1, 2])
def test_sliced_against_unsliced(ctx, bench_net, legs):
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = bench_net
    amap = AngleMap.every_angle(tn)
    T = cuda(amap.theta0)
    gp = NetworkPlan.for_gradients(tn, path, wrt=amap.leaves(), ctx=ctx)
    gp.stage(tn)
    ang = Angles(ctx, tn, amap, gp)
    ang.set_leaves(gp, T)
    gp.run()
    ref = ang.pullback(T, gp.vjp_block())[0].to_numpy()[0]
    del gp
    sp = SlicedPlan.for_gradients(tn, path, [149, 156][:legs], wrt=amap.leaves(), ctx=ctx)
    sp.stage(tn)
    asl = Angles(ctx, tn, amap, sp)
    asl.set_leaves(sp, T)
    value, G = sp.vjp_blocks()
    got = asl.pullback(T, G)[0].to_numpy()[0]
    assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------ 6. expectation network
def test_expectation_tied(ctx):
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.builders.random_circuit import random_circuit_with_set_observable
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    # <ψ|U† O U|ψ> with Hermitian Paulis: no single-qubit gates (the builder mirrors sy and sz with sx†, as the
    # reference does) and real closing states (the builder puts the same vector on both sides, not its conjugate)
    tn = random_circuit_with_set_observable(8, 5, 0.0, 0.5, [2, 5], np.random.default_rng(9))
    lv = leaves(tn)
    for t in lv:
        if t.tensordata.kind == "matrix":
            t.set_tensor_data(TensorData.Matrix(np.ascontiguousarray(np.asarray(t.tensordata.matrix).real + 0j)))
    fs = [i for i, t in enumerate(lv) if t.tensordata.kind == "gate" and t.tensordata.gate[0] == "fsim"]
    ket = [i for i in fs if not lv[i].tensordata.gate[2]]
    bra = [i for i in fs if lv[i].tensordata.gate[2]]
    assert len(ket) == len(bra) > 0
    path = greedy(tn)
    # untied: every occurrence its own θ and φ; tied: one (θ, φ) for all
    untied = AngleMap.every_angle(tn)
    tied = AngleMap([(l, s, s, 1.0) for l in fs for s in (0, 1)], 2, [0.3, 0.2])
    gp = NetworkPlan.for_gradients(tn, path, wrt=sorted(fs), ctx=ctx)
    gp.stage(tn)
    au, at = Angles(ctx, tn, untied, gp), Angles(ctx, tn, tied, gp)
    Tu, Tt = cuda(untied.theta0), cuda([0.3, 0.2])
    at.set_leaves(gp, Tt)
    gp.run()
    G = gp.vjp_block()
    gt = at.pullback(Tt, G)[0].to_numpy()[0]
    gu = au.pullback(Tu, G)[0].to_numpy()[0]
    assert np.abs(gt.imag).max() <= 1e-13 * np.abs(gt).max()
    sums = np.zeros(2, dtype=np.complex128)
    for (l, s, p, _) in untied.refs:
        sums[s] += gu[p]
    assert np.abs(gt - sums).max() <= 1e-13 * np.abs(gt).max()


# ------------------------------------------------------------------------------------------------ 7. torch
def test_circuit_function(ctx):
    import torch
    from tnc_b200.autograd import circuit_function
    tn, amap = mixed_circuit(seed=7)
    path = greedy(tn)
    f = circuit_function(tn, path, amap, ctx=ctx)
    ref = replay_fn(tn, path, amap)
    rng = np.random.default_rng(3)
    P = amap.n_params
    rel = lambda a, b: (a - b).abs().max().item() / b.abs().max().item()
    # [P]: value, gradient of a real loss, forward-mode tangent
    th = rng.uniform(-3, 3, P)
    w = complex(0.3, -1.2)
    T = cuda(th).requires_grad_()
    R = f(T)
    (R * w).real.backward()
    Tc = torch.tensor(th, requires_grad=True)
    Rc = ref(Tc)
    (Rc * w).real.backward()
    assert rel(R.detach().cpu(), Rc.detach()) < 1e-12
    assert rel(T.grad.cpu(), Tc.grad) < 1e-12
    tdot = rng.standard_normal(P)
    _, rd = torch.func.jvp(f, (cuda(th),), (cuda(tdot),))
    _, rdc = torch.func.jvp(ref, (torch.tensor(th),), (torch.tensor(tdot),))
    assert rel(rd.cpu(), rdc) < 1e-12
    # [B, P]
    B = 3
    TH = rng.uniform(-3, 3, (B, P))
    TB = cuda(TH).requires_grad_()
    RB = f(TB)
    W = torch.tensor(rng.standard_normal(B) + 1j * rng.standard_normal(B))
    (RB * W.cuda()).real.sum().backward()
    for i in range(B):
        Ti = torch.tensor(TH[i], requires_grad=True)
        Ri = ref(Ti)
        (Ri * W[i]).real.backward()
        assert rel(RB[i].detach().cpu(), Ri.detach()) < 1e-12
        assert rel(TB.grad[i].cpu(), Ti.grad) < 1e-12
    DT = rng.standard_normal((B, P))
    _, rdb = torch.func.jvp(f, (cuda(TH),), (cuda(DT),))
    for i in range(B):
        _, rdi = torch.func.jvp(ref, (torch.tensor(TH[i]),), (torch.tensor(DT[i]),))
        assert rel(rdb[i].cpu(), rdi) < 1e-12
    # refusals
    for bad, msg in [(torch.tensor(th), "CUDA"), (cuda(th).float(), "float64"), (cuda(th[:-1]), "shape"),
                     (cuda(np.zeros((2, 2, P))), "shape")]:
        with pytest.raises(ValueError, match=msg):
            f(bad)
    T2 = cuda(th).requires_grad_()
    with pytest.raises(NotImplementedError):
        torch.autograd.grad(f(T2).real, T2, create_graph=True)


def test_circuit_function_sliced(ctx, bench_net):
    import torch
    from tnc_b200.angles import AngleMap
    from tnc_b200.autograd import circuit_function
    tn, path = bench_net
    amap = AngleMap.every_angle(tn)
    f = circuit_function(tn, path, amap, ctx=ctx)
    fs = circuit_function(tn, path, amap, ctx=ctx, sliced_legs=[149])
    T1, T2 = cuda(amap.theta0).requires_grad_(), cuda(amap.theta0).requires_grad_()
    R1, R2 = f(T1), fs(T2)
    assert abs(complex(R1.detach().cpu()) - complex(R2.detach().cpu())) <= 1e-13 * abs(complex(R1.detach().cpu()))
    R1.real.backward()
    R2.real.backward()
    assert (T1.grad - T2.grad).abs().max().item() <= 1e-13 * T1.grad.abs().max().item()
    with pytest.raises(NotImplementedError):
        torch.func.jvp(fs, (cuda(amap.theta0),), (cuda(np.ones(amap.n_params)),))


# ------------------------------------------------------------------------------------------------ 8. C ABI errors
def test_abi_errors(ctx):
    import torch
    from tnc_b200 import DeviceTensor
    from tnc_b200.angles import Angles
    from tnc_b200.tensornetwork import NetworkPlan
    tn, amap = mixed_circuit(seed=2)
    path = greedy(tn)
    gp = NetworkPlan.for_gradients(tn, path, wrt=amap.leaves(), ctx=ctx)
    gp.stage(tn)
    ang = Angles(ctx, tn, amap, gp)
    P, E = amap.n_params, ang.block_elems
    l = ctx._l
    th = cuda(amap.theta0)
    ang.gates(th).free()                      # tables uploaded
    ctx.synchronize()
    G = DeviceTensor.from_numpy(ctx, np.zeros(E, dtype=np.complex128))
    Gbad = DeviceTensor.from_numpy(ctx, np.zeros(E + 1, dtype=np.complex128))
    host = np.zeros(P)
    big = torch.zeros(P, dtype=torch.float64, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())
    out, out2 = C.c_void_p(), C.c_void_p()
    ab = C.c_void_p(th.data_ptr() + 4)
    cases = [
        (lambda: l.tncb_angles_gates(ctx.handle, ang.handle, p(th), 0, 0, C.byref(out)), ERR_INVALID, "count is 0"),
        (lambda: l.tncb_angles_gates(ctx.handle, ang.handle, None, 0, 1, C.byref(out)), ERR_INVALID, "theta is null"),
        (lambda: l.tncb_angles_gates(ctx.handle, ang.handle, ab, 0, 1, C.byref(out)), ERR_INVALID, "theta is not 8-byte aligned"),
        (lambda: l.tncb_angles_gates(ctx.handle, ang.handle, host.ctypes.data_as(C.c_void_p), 0, 1, C.byref(out)), ERR_INVALID,
         "theta is not device memory"),
        (lambda: l.tncb_angles_gates(ctx.handle, ang.handle, p(th), P - 1, 2, C.byref(out)), ERR_INVALID,
         f"theta: row stride {P - 1} is below the {P} parameters"),
        (lambda: l.tncb_angles_gates(ctx.handle, ang.handle, p(big), 1 << 40, 2, C.byref(out)), ERR_INVALID,
         f"theta: its {8 * ((1 << 40) + P)} bytes run past the end of its allocation"),
        (lambda: l.tncb_angles_tangents(ctx.handle, ang.handle, p(th), 0, None, 0, 1, C.byref(out)), ERR_INVALID, "theta_dot is null"),
        (lambda: l.tncb_angles_pullback(ctx.handle, ang.handle, p(th), 0, 1, G.handle, None, None, 0, None, None), ERR_INVALID,
         "no output requested"),
        (lambda: l.tncb_angles_pullback(ctx.handle, ang.handle, p(th), 0, 1, None, None, None, 0, C.byref(out), None), ERR_INVALID,
         "grads is null"),
        (lambda: l.tncb_angles_pullback(ctx.handle, ang.handle, p(th), 0, 1, Gbad.handle, None, None, 0, C.byref(out), None),
         ERR_SHAPE, f"grads must be [{E}] or [1, {E}]"),
        (lambda: l.tncb_angles_pullback(ctx.handle, ang.handle, p(th), 0, 1, G.handle, G.handle, None, 0, C.byref(out), None),
         ERR_INVALID, "grad_tangents and direction come together"),
        (lambda: l.tncb_angles_pullback(ctx.handle, ang.handle, p(th), 0, 1, G.handle, G.handle, None, 0, C.byref(out), C.byref(out2)),
         ERR_INVALID, "grad_tangents and direction come together"),
    ]
    before = ctx.stats()
    for call, status, msg in cases:
        assert call() == status
        assert l.tncb_last_error().decode() == msg
    ctx.synchronize()
    after = ctx.stats()
    assert after["arena_live_bytes"] == before["arena_live_bytes"]
    assert after["kernel_launches"] == before["kernel_launches"]
