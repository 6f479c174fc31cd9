"""Expectation values of Pauli sums on the H100 (tncb_plan_expect, tnc_b200.Expectation).

  1. values: every term's value row bit-identical to the host-staged per-term network with `run`, the energy to numpy's
     left fold of those rows, the same bits for batch = 1, 3 and 0 and on a repeated call, plan.run() unchanged;
  2. gradients: on a gradient plan, values and grad_sum bit-identical to vjp_batch(seeds = c) over the host-staged
     per-term networks;
  3. independent references: the energy against the oracle state vector's <H> (QAOA MaxCut on 14 qubits, an Ising
     ansatz), value_and_grad against central differences and, for untied rx / ry / rz, the exact parameter-shift rule,
     params whose refs were all pruned at exactly 0, and torch.autograd.gradcheck of expectation_function;
  4. scale: bench.py's 36-qubit circuit family (six rounds) with a Hamiltonian on qubits 0-3, against the host recipe;
  5. every refusal of the C ABI, with the arena and the staged plan unchanged."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = -1, -9
ONE_Q = [("h", 0), ("t", 0), ("x", 0), ("y", 0), ("sx", 0), ("rx", 1), ("ry", 1), ("rz", 1), ("u", 3)]
TWO_Q = [("cx", 0), ("cz", 0), ("fsim", 2), ("cp", 1), ("iswap", 0)]


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


def to_oracle(t):
    if t.is_composite():
        return orc.OTensor(children=[to_oracle(c) for c in t.tensors])
    td = t.tensordata
    d = ("gate", td.gate[0], td.gate[1], td.gate[2]) if td.kind == "gate" else np.asarray(td.matrix)
    return orc.OTensor(list(t.legs), list(t.bond_dims), d)


def to_opath(p):
    return orc.OPath(list(p.toplevel), {i: to_opath(q) for i, q in p.nested.items()})


def random_circuit(n, depth, seed):
    from tnc_b200.builders import Circuit
    rng = np.random.default_rng(seed)
    c = Circuit()
    c.allocate_register(n)
    for _ in range(depth):
        for q in range(n):
            g, k = ONE_Q[rng.integers(len(ONE_Q))]
            c.append_gate(g, list(rng.uniform(-3, 3, k)), [q])
        perm = rng.permutation(n)
        for a, b in zip(perm[0::2][: n // 3], perm[1::2][: n // 3]):
            g, k = TWO_Q[rng.integers(len(TWO_Q))]
            c.append_gate(g, list(rng.uniform(-3, 3, k)), [int(a), int(b)])
    return c


def random_hamiltonian(n, k, seed, qubits=None):
    from tnc_b200 import PauliSum
    rng = np.random.default_rng(seed)
    qubits = list(range(n)) if qubits is None else qubits
    terms = []
    for _ in range(k):
        w = int(rng.integers(1, min(4, len(qubits)) + 1))
        qs = rng.choice(qubits, w, replace=False)
        terms.append((float(rng.normal()), {int(q): "XYZ"[rng.integers(3)] for q in qs}))
    terms.append((0.75, {int(qubits[0]): "Y"}))           # an odd number of Y's
    return PauliSum(terms, n_qubits=n)


def term_networks(exp):
    """the host-staged network of every term: the layer leaves hold pauli_layer_matrix payloads"""
    from tnc_b200 import pauli_layer_matrix
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    pn = exp.network
    x, z, _ = exp.hamiltonian.masks()
    nets = []
    for xk, zk in zip(x.tolist(), z.tolist()):
        leaves = list(pn.tn.tensors)
        for leaf, q in zip(pn.layer_leaf, pn.layer_qubit):
            t = Tensor(list(leaves[leaf].legs), list(leaves[leaf].bond_dims))
            t.set_tensor_data(TensorData.Matrix(pauli_layer_matrix((xk >> q) & 1, (zk >> q) & 1)))
            leaves[leaf] = t
        nets.append(Tensor.new_composite(leaves))
    return nets


def left_fold(coeff, rows):
    re = im = 0.0
    for c, r in zip(coeff, rows):
        re = re + c * r.real
        im = im + c * r.imag
    return complex(re, im)


def bits(a):
    return np.asarray(a, dtype=np.complex128).reshape(-1).view(np.uint64)


def expect_raw(exp, outputs, batch=0):
    """tncb_plan_expect on the plan as staged (no θ): DeviceTensors, None where not requested"""
    return exp._expect(None, outputs, batch)


# ------------------------------------------------------------------------------------------------ 1. values
def test_values_bit_identical(ctx):
    from tnc_b200 import Expectation
    from tnc_b200.tensornetwork import NetworkPlan
    c = random_circuit(10, 3, 11)
    h = random_hamiltonian(10, 11, 12, qubits=[1, 2, 4, 5, 8])
    exp = Expectation(c, h, ctx=ctx)
    before = exp.plan.run().to_numpy()
    ref_plan = NetworkPlan(exp.network.tn, exp.path, ctx=ctx)
    rows = []
    for net in term_networks(exp):
        ref_plan.stage(net)
        rows.append(complex(ref_plan.run().to_numpy().reshape(())))
    _, _, coeff = h.masks()
    want_e = left_fold(coeff.tolist(), rows)
    for batch in (1, 3, None, None):
        e, vals = exp.values(batch=batch)
        assert np.array_equal(bits(vals.cpu().numpy()), bits(rows)), batch
        assert np.array_equal(bits([e]), bits([want_e])), (batch, e, want_e)
    assert np.array_equal(bits(exp.plan.run().to_numpy()), bits(before))
    assert abs(complex(before.reshape(())) - 1.0) < 1e-12          # the staged identities: <psi|psi>


# ------------------------------------------------------------------------------------------------ 2. gradients
def test_grad_sum_bit_identical(ctx):
    from tnc_b200 import Expectation
    from tnc_b200.angles import AngleMap
    from tnc_b200.tensornetwork import NetworkPlan
    c = random_circuit(9, 3, 21)
    h = random_hamiltonian(9, 9, 22, qubits=[0, 3, 4, 7])
    exp = Expectation(c, h, angle_map=AngleMap.every_angle(c.into_statevector_network()[0]), ctx=ctx)
    wrt = exp.angle_map.leaves()
    ref = NetworkPlan.for_gradients(exp.network.tn, exp.path, wrt=wrt, ctx=ctx)
    ref.stage_batch(term_networks(exp))
    _, _, coeff = h.masks()
    rv, _, rs = ref.vjp_batch_blocks(0, len(h), seeds=coeff.astype(np.complex128), rows=False, sum=True)
    want_v, want_s = rv.to_numpy(), rs.to_numpy()
    for batch in (1, 3, 0):
        vals, energy, gs = expect_raw(exp, (True, True, True), batch)
        assert np.array_equal(bits(vals.to_numpy()), bits(want_v)), batch
        assert np.array_equal(bits(gs.to_numpy()), bits(want_s)), batch
        assert np.array_equal(bits(energy.to_numpy().reshape(1)), bits([left_fold(coeff.tolist(), want_v)])), batch
        for t in (vals, energy, gs):
            t.free()


# ------------------------------------------------------------------------------------------------ 3. references
def state_vector(c):
    tn, perm = c.into_statevector_network()
    res = orc.contract_tensor_network(to_oracle(tn), to_opath(greedy(tn)))
    return np.asarray(orc.permute_to(res, perm.target_leg_order).data).reshape(-1)


def oracle_energy(c, h):
    n = c.num_qubits()
    psi = state_vector(c)
    mats = {"X": np.array([[0, 1], [1, 0]], complex), "Y": np.array([[0, -1j], [1j, 0]]), "Z": np.diag([1.0 + 0j, -1.0])}
    e = 0.0
    for coeff, paulis in h.terms:
        t = psi.reshape([2] * n)
        for q, letter in paulis.items():
            t = np.moveaxis(np.tensordot(mats[letter], t, axes=([1], [q])), 0, q)
        e += coeff * np.vdot(psi, t.reshape(-1))
    return e


def regular3(n, seed):
    """a random 3-regular graph on n qubits (pairing model, retried until simple)"""
    rng = np.random.default_rng(seed)
    while True:
        stubs = rng.permutation(np.repeat(np.arange(n), 3))
        edges = {tuple(sorted((int(a), int(b)))) for a, b in stubs.reshape(-1, 2)}
        if len(edges) == 3 * n // 2 and all(a != b for a, b in edges):
            return sorted(edges)


def qaoa(n, p, seed, theta=None):
    """QAOA MaxCut on a random 3-regular graph: cx rz(2γ) cx per edge, rx(2β) mixers; γ_l, β_l tied through scales 2"""
    from tnc_b200 import PauliSum
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    edges = regular3(n, seed)
    theta = np.random.default_rng(seed + 1).uniform(-1, 1, 2 * p) if theta is None else np.asarray(theta)
    c = Circuit()
    c.allocate_register(n)
    for q in range(n):
        c.append_gate("h", [], [q])
    refs = []
    for l in range(p):
        for a, b in edges:
            c.append_gate("cx", [], [a, b])
            refs.append((len(c.tensors), 0, 2 * l, 2.0))
            c.append_gate("rz", [2 * theta[2 * l]], [b])
            c.append_gate("cx", [], [a, b])
        for q in range(n):
            refs.append((len(c.tensors), 0, 2 * l + 1, 2.0))
            c.append_gate("rx", [2 * theta[2 * l + 1]], [q])
    h = PauliSum([(0.5, f"Z{a} Z{b}") for a, b in edges], n_qubits=n)
    return c, h, AngleMap(refs, 2 * p, theta)


def ising(n, depth, seed, theta=None, gates=("ry",)):
    """a transverse-field Ising chain, H = -sum Z_q Z_q+1 - 0.7 sum X_q, on an ry + cz ansatz (the rotations cycle
    through `gates`), every rotation its own param"""
    from tnc_b200 import PauliSum
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    theta = np.random.default_rng(seed).uniform(-math.pi, math.pi, n * depth) if theta is None else np.asarray(theta)
    c = Circuit()
    c.allocate_register(n)
    refs = []
    for d in range(depth):
        for q in range(n):
            refs.append((len(c.tensors), 0, d * n + q, 1.0))
            c.append_gate(gates[(d * n + q) % len(gates)], [theta[d * n + q]], [q])
        for q in range(d % 2, n - 1, 2):
            c.append_gate("cz", [], [q, q + 1])
    h = PauliSum([(-1.0, f"Z{q} Z{q + 1}") for q in range(n - 1)] + [(-0.7, f"X{q}") for q in range(n)], n_qubits=n)
    return c, h, AngleMap(refs, n * depth, theta)


@pytest.mark.parametrize("case", ["qaoa14", "ising10"])
def test_energy_against_state_vector(ctx, case):
    import torch
    from tnc_b200 import Expectation
    c, h, amap = qaoa(14, 2, 3) if case == "qaoa14" else ising(10, 4, 4)
    exp = Expectation(c, h, angle_map=amap, ctx=ctx)
    want = oracle_energy(c, h)
    scale = max(1.0, sum(abs(x) for x, _ in h.terms))
    e, vals = exp.values()
    assert abs(e - want) <= 1e-12 * scale, (e, want)
    theta = torch.tensor(amap.theta0, dtype=torch.float64, device="cuda")
    e2, g = exp.value_and_grad(theta)
    assert abs(e2 - want.real) <= 1e-12 * scale and exp.max_imag < 1e-12 * scale
    assert g.shape == (amap.n_params,) and g.dtype == torch.float64


def test_gradient_against_finite_differences_and_parameter_shift(ctx):
    import torch
    from tnc_b200 import Expectation
    c, h, amap = ising(8, 3, 5, gates=("rx", "ry", "rz", "ry"))
    exp = Expectation(c, h, angle_map=amap, ctx=ctx)
    theta = torch.tensor(amap.theta0, dtype=torch.float64, device="cuda")
    e, g = exp.value_and_grad(theta)
    g = g.cpu().numpy()
    E = lambda t: exp.values(torch.tensor(t, dtype=torch.float64, device="cuda"))[0].real
    t0 = np.asarray(amap.theta0)
    for p in range(amap.n_params):
        up, dn = t0.copy(), t0.copy()
        up[p] += math.pi / 2
        dn[p] -= math.pi / 2
        shift = (E(up) - E(dn)) / 2
        assert abs(g[p] - shift) <= 1e-12 * max(1.0, abs(shift)), (p, g[p], shift)
        eps = 1e-5
        up, dn = t0.copy(), t0.copy()
        up[p] += eps
        dn[p] -= eps
        fd = (E(up) - E(dn)) / (2 * eps)
        assert abs(g[p] - fd) <= 1e-6 * max(1.0, abs(fd)), (p, g[p], fd)
    # QAOA: tied angles through scales, against central differences
    c, h, amap = qaoa(12, 2, 7)
    exp = Expectation(c, h, angle_map=amap, ctx=ctx)
    t0 = np.asarray(amap.theta0)
    e, g = exp.value_and_grad(torch.tensor(t0, dtype=torch.float64, device="cuda"))
    E = lambda t: exp.values(torch.tensor(t, dtype=torch.float64, device="cuda"))[0].real
    for p in range(amap.n_params):
        up, dn = t0.copy(), t0.copy()
        up[p] += 1e-5
        dn[p] -= 1e-5
        fd = (E(up) - E(dn)) / 2e-5
        assert abs(float(g[p]) - fd) <= 1e-6 * max(1.0, abs(fd)), (p, float(g[p]), fd)


def test_pruned_params_get_zero(ctx):
    import torch
    from tnc_b200 import Expectation, PauliSum
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    c = Circuit()
    c.allocate_register(4)
    c.append_gate("ry", [0.3], [0])
    c.append_gate("ry", [0.4], [3])          # outside the cone of qubits 0, 1
    c.append_gate("cx", [], [0, 1])
    c.append_gate("rx", [0.5], [1])
    c.append_gate("rz", [0.6], [2])          # outside too
    amap = AngleMap([(4, 0, 0, 1.0), (5, 0, 1, 1.0), (7, 0, 2, 1.0), (8, 0, 3, 1.0)], 4, [0.3, 0.4, 0.5, 0.6])
    exp = Expectation(c, PauliSum([(1.0, "Z0 Y1"), (0.5, "X1")], n_qubits=4), angle_map=amap, ctx=ctx)
    assert exp.network.kept == [0, 1, 4, 6, 7]
    e, g = exp.value_and_grad(torch.tensor([0.3, 0.4, 0.5, 0.6], dtype=torch.float64, device="cuda"))
    g = g.cpu().numpy()
    assert g[1] == 0.0 and g[3] == 0.0
    assert abs(e - oracle_energy(c, exp.hamiltonian).real) < 1e-12


def test_gradcheck(ctx):
    import torch
    from tnc_b200 import Expectation
    from tnc_b200.autograd import expectation_function
    c, h, amap = ising(8, 2, 9)
    f = expectation_function(Expectation(c, h, angle_map=amap, ctx=ctx))
    theta = torch.tensor(amap.theta0, dtype=torch.float64, device="cuda", requires_grad=True)
    assert torch.autograd.gradcheck(f, (theta,), eps=1e-6, atol=1e-7, rtol=1e-6)
    y = f(theta)
    assert y.dtype == torch.float64 and y.dim() == 0 and y.is_cuda
    with pytest.raises(NotImplementedError):
        f(theta.detach().unsqueeze(0).repeat(2, 1))
    with pytest.raises(NotImplementedError):
        import torch.autograd.forward_ad as fwAD
        with fwAD.dual_level():
            f(fwAD.make_dual(theta.detach(), torch.ones_like(theta)))
    with pytest.raises(NotImplementedError):
        (gr,) = torch.autograd.grad(f(theta), theta, create_graph=True)


# ------------------------------------------------------------------------------------------------ 4. scale
def test_bench_scale(ctx):
    from tnc_b200 import Expectation, PauliSum
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders.random_circuit import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    # bench.py's 36-qubit circuit family; at its ten rounds the light cone of qubits 0-3 is the whole circuit and the
    # doubled network does not fit, at six it spans all 36 qubits and the plan needs 64 MiB
    c = random_circuit_builder(36, 6, 0.5, 0.5, np.random.default_rng(1))
    h = PauliSum([(0.5, "Z0 Z1"), (-0.3, "X2 Y3"), (0.2, "Y0"), (1.1, "X1 X2 Z3"), (-0.4, "Y1 Y2")], n_qubits=36)
    amap = AngleMap.every_angle(c.into_statevector_network()[0])
    exp = Expectation(c, h, angle_map=amap, ctx=ctx)
    assert set(q for i in exp.network.kept for q in c.tensor_qubits()[i]) == set(range(36))
    ref = NetworkPlan.for_gradients(exp.network.tn, exp.path, wrt=exp.angle_map.leaves(), ctx=ctx)
    ref.stage_batch(term_networks(exp))
    _, _, coeff = h.masks()
    rv, _, rs = ref.vjp_batch_blocks(0, len(h), seeds=coeff.astype(np.complex128), rows=False, sum=True)
    vals, energy, gs = expect_raw(exp, (True, True, True))
    assert np.array_equal(bits(vals.to_numpy()), bits(rv.to_numpy()))
    assert np.array_equal(bits(gs.to_numpy()), bits(rs.to_numpy()))
    assert np.array_equal(bits(energy.to_numpy().reshape(1)), bits([left_fold(coeff.tolist(), rv.to_numpy())]))


# ------------------------------------------------------------------------------------------------ 5. refusals
def test_refusals(ctx, monkeypatch):
    import torch
    from tnc_b200 import Expectation, PauliSum
    from tnc_b200._lib import TncbPauliLayer, u64_array
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    l = ctx._l
    c = random_circuit(6, 2, 31)
    h = PauliSum([(1.0, "Z0 X2"), (0.5, "Y2")], n_qubits=6)
    exp = Expectation(c, h, ctx=ctx)
    pn = exp.network
    want = exp.plan.run().to_numpy()
    tn, path = pn.tn, exp.path
    grad = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    grad.stage(tn)
    jvp = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    jvp.stage(tn)
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    loose = NetworkPlan(tn, path, ctx=ctx)
    loose.stage(tn)
    monkeypatch.delenv("TNCB_NO_STATIC")
    unstaged = NetworkPlan(tn, path, ctx=ctx)
    a = Tensor([0, 1], [2, 3])
    a.set_tensor_data(TensorData.Matrix(np.arange(6, dtype=np.complex128).reshape(2, 3)))
    b = Tensor([0], [2])
    b.set_tensor_data(TensorData.Matrix(np.array([1, 0], dtype=np.complex128)))
    vec = Tensor.new_composite([a, b])
    open_plan = NetworkPlan(vec, ContractionPath.simple([(0, 1)]), ctx=ctx)
    open_plan.stage(vec)
    gate_leaf = next(i for i, t in enumerate(tn.tensors) if len(t.legs) == 4)
    ket_leaf = 0

    def layer(n=6, leaves=None, qubits=None):
        leaves = list(pn.layer_leaf) if leaves is None else leaves
        qubits = list(pn.layer_qubit) if qubits is None else qubits
        keep = (u64_array(leaves), (C.c_int * max(len(qubits), 1))(*qubits))
        ly = TncbPauliLayer(n, len(leaves), *keep)
        ly._keep = keep
        return ly

    x, z, cf = h.masks()

    def call(plan=None, ly=None, k=2, xs=None, zs=None, cs=None, out=(True, True, False), null=None):
        xs = x.tolist() if xs is None else xs
        zs = z.tolist() if zs is None else zs
        cs = cf.tolist() if cs is None else cs
        args = [ctx.handle, (plan or exp.plan).handle, C.byref(ly or layer()), k, u64_array(xs), u64_array(zs),
                (C.c_double * len(cs))(*cs), 0]
        if null is not None:
            args[null] = None
        outs = [C.c_void_p() if w else None for w in out]
        rc = l.tncb_plan_expect(*args, *[C.byref(o) if o is not None else None for o in outs])
        for o in outs:
            if o is not None and o.value:
                l.tncb_tensor_free(ctx.handle, o)
        return rc

    cases = [
        (ERR_INVALID, "null argument", dict(null=2)),
        (ERR_INVALID, "null argument", dict(null=4)),
        (ERR_INVALID, "null argument", dict(null=6)),
        (ERR_INVALID, "n_terms is 0", dict(k=0)),
        (ERR_INVALID, "n_qubits 0 is outside 1..64", dict(ly=layer(n=0))),
        (ERR_INVALID, "n_qubits 65 is outside 1..64", dict(ly=layer(n=65))),
        (ERR_INVALID, f"layer leaf 9999 is out of range ({len(tn.tensors)} leaves)", dict(ly=layer(leaves=[9999, pn.layer_leaf[1]]))),
        (ERR_INVALID, f"layer leaf {pn.layer_leaf[0]} is listed twice", dict(ly=layer(leaves=[pn.layer_leaf[0]] * 2))),
        (ERR_INVALID, f"layer leaf {gate_leaf} is not a rank-2 leaf with dims [2, 2]", dict(ly=layer(leaves=[gate_leaf, pn.layer_leaf[1]]))),
        (ERR_INVALID, f"layer leaf {ket_leaf} is not a rank-2 leaf with dims [2, 2]", dict(ly=layer(leaves=[ket_leaf, pn.layer_leaf[1]]))),
        (ERR_INVALID, "layer qubit 1 is qubit 6, outside 0..5", dict(ly=layer(qubits=[0, 6]))),
        (ERR_INVALID, "qubit 0 is listed twice (layer qubit 1)", dict(ly=layer(qubits=[0, 0]))),
        (ERR_INVALID, "term 1 acts on qubit 3, which has no layer leaf", dict(xs=[1, 1 << 3])),
        (ERR_INVALID, "term 0 acts on qubit 40, which has no layer leaf", dict(zs=[1 << 40, 0])),
        (ERR_INVALID, "the coefficient of term 1 is not finite", dict(cs=[1.0, float("nan")])),
        (ERR_INVALID, "the coefficient of term 0 is not finite", dict(cs=[float("-inf"), 1.0])),
        (ERR_INVALID, "the network does not contract to a scalar (1 result legs)", dict(plan=open_plan, ly=layer(leaves=[], qubits=[]), xs=[0, 0], zs=[0, 0])),
        (ERR_INVALID, "no output requested", dict(out=(False, False, False))),
        (ERR_INVALID, "grad_sum needs a gradient plan (tncb_plan_create_vjp)", dict(out=(False, False, True))),
        (ERR_INVALID, "tncb_plan_stage has not been called on this plan and context", dict(plan=unstaged)),
        (ERR_UNSUPPORTED, "tncb_plan_expect takes a plain or a gradient plan (tncb_plan_create / _vjp)", dict(plan=jvp)),
        (ERR_UNSUPPORTED, "expectation values need a plan with a static layout (no device leaves)", dict(plan=loose)),
    ]
    assert [pn.layer_qubit, pn.layer_leaf[0] != ket_leaf] == [[0, 2], True]
    live = ctx.stats()["arena_live_bytes"]
    for status, msg, kw in cases:
        assert call(**kw) == status, msg
        assert l.tncb_last_error().decode() == msg, (msg, l.tncb_last_error().decode())
        assert ctx.stats()["arena_live_bytes"] == live, msg
    assert np.array_equal(exp.plan.run().to_numpy(), want)
    assert call() == 0 and call(plan=grad, out=(True, True, True)) == 0
    assert ctx.stats()["arena_live_bytes"] == live
