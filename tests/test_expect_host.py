"""Expectation values of Pauli sums without a GPU: PauliSum's parsing, masks, order and refusals; the pruned expectation
network with pauli_layer_matrix payloads, contracted by the oracle, against <psi|P|psi> from the oracle's state vector
(odd numbers of Y's, pruned gates and joined wires included); the full-support network leaf for leaf against
into_expectation_value_network; PauliNetwork.angle_map; the expect cell of the kind table on host-only plans of all
seven kinds; and what Expectation passes to the library, with every later entry answered by a recorder."""
import ctypes as C
import math
import types

import numpy as np
import pytest

from oracle import tnc_oracle as orc

ERR_INVALID, ERR_UNSUPPORTED = -1, -9
KINDS = ["plain", "vjp", "jvp", "hvp", "sliced vjp", "sliced jvp", "sliced hvp"]
ONE_Q = [("h", 0), ("t", 0), ("x", 0), ("y", 0), ("sx", 0), ("rx", 1), ("ry", 1), ("rz", 1), ("u", 3)]
TWO_Q = [("cx", 0), ("cz", 0), ("fsim", 2), ("cp", 1), ("iswap", 0)]


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def to_oracle(t, payloads=None):
    """the oracle's copy of `t`; payloads: {leaf index: array} replacing leaves' data"""
    from tnc_b200.tensornetwork.contraction import leaves
    payloads = payloads or {}
    index = {id(l): i for i, l in enumerate(leaves(t))}

    def conv(x):
        if x.is_composite():
            return orc.OTensor(children=[conv(c) for c in x.tensors])
        td = x.tensordata
        if index[id(x)] in payloads:
            d = np.asarray(payloads[index[id(x)]], dtype=np.complex128)
        else:
            d = ("gate", td.gate[0], td.gate[1], td.gate[2]) if td.kind == "gate" else np.asarray(td.matrix)
        return orc.OTensor(list(x.legs), list(x.bond_dims), d)
    return conv(t)


def oracle_path(p):
    return orc.OPath(toplevel=list(p.toplevel), nested={i: oracle_path(q) for i, q in p.nested.items()})


def contract(tn, payloads=None):
    res = orc.contract_tensor_network(to_oracle(tn, payloads), oracle_path(greedy(tn)))
    return complex(np.asarray(res.data).reshape(()))


def random_circuit(n, depth, seed):
    """a circuit of `depth` layers: a random one-qubit gate on every qubit, then two-qubit gates on random pairs"""
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


def state_vector(c):
    tn, perm = c.into_statevector_network()
    res = orc.contract_tensor_network(to_oracle(tn), oracle_path(greedy(tn)))
    return np.asarray(orc.permute_to(res, perm.target_leg_order).data).reshape(-1)


def apply_pauli(psi, n, paulis):
    """P psi for the state vector psi (qubit 0 the most significant index) and paulis {qubit: letter}"""
    mats = {"X": np.array([[0, 1], [1, 0]], complex), "Y": np.array([[0, -1j], [1j, 0]]), "Z": np.diag([1.0 + 0j, -1.0])}
    t = psi.reshape([2] * n)
    for q, letter in paulis.items():
        t = np.moveaxis(np.tensordot(mats[letter], t, axes=([1], [q])), 0, q)
    return t.reshape(-1)


# ------------------------------------------------------------------------------------------------ PauliSum
def test_pauli_sum_parsing_masks_order():
    from tnc_b200 import PauliSum
    h = PauliSum([(0.5, "X0 Z3 Y7"), (-2, {1: "Y", 2: "Z"}), (1.5, ""), (0.5, "X0 Z3 Y7"), (np.float32(0.25), "I4 Z5"),
                  (3 + 0j, {})], n_qubits=8)
    x, z, c = h.masks()
    assert x.dtype == np.uint64 and z.dtype == np.uint64 and c.dtype == np.float64
    assert x.tolist() == [(1 << 0) | (1 << 7), 1 << 1, 0, (1 << 0) | (1 << 7), 0, 0]
    assert z.tolist() == [(1 << 3) | (1 << 7), (1 << 1) | (1 << 2), 0, (1 << 3) | (1 << 7), 1 << 5, 0]
    assert c.tolist() == [0.5, -2.0, 1.5, 0.5, 0.25, 3.0]
    assert len(h) == 6 and h.support() == [0, 1, 2, 3, 5, 7]
    big = PauliSum([(1.0, "X63 Y0")], n_qubits=64)
    assert big.masks()[0].tolist() == [(1 << 63) | 1] and big.masks()[1].tolist() == [1]


@pytest.mark.parametrize("terms, n, message", [
    ([(1j, "X0")], 4, "the coefficient of term 0 is not real"),
    ([(1.0, "X0"), (float("nan"), "Z1")], 4, "the coefficient of term 1 is not finite"),
    ([(float("inf"), "Z1")], 4, "the coefficient of term 0 is not finite"),
    ([("1", "Z1")], 4, "the coefficient of term 0 is not a number"),
    ([(1.0, "X4")], 4, "term 0: qubit 4 is outside the 4-qubit circuit"),
    ([(1.0, {-1: "X"})], 4, "term 0: qubit -1 is outside the 4-qubit circuit"),
    ([(1.0, "W1")], 4, "term 0: unknown Pauli 'W'"),
    ([(1.0, {0: "x"})], 4, "term 0: unknown Pauli 'x'"),
    ([(1.0, "X")], 4, "term 0: 'X' is not a letter followed by a qubit"),
    ([(1.0, "X1 Z1")], 4, "term 0: qubit 1 is named twice"),
    ([(1.0, 3)], 4, "term 0: the Paulis must be a string or a {qubit: letter} dict"),
    ([], 4, "a Pauli sum needs at least one term"),
    ([(1.0, "X0")], 65, "a Pauli sum acts on 1..64 qubits, not 65"),
])
def test_pauli_sum_refusals(terms, n, message):
    from tnc_b200 import PauliSum
    with pytest.raises(ValueError, match=message.replace("(", r"\(").replace("{", r"\{").replace(".", r"\.")):
        PauliSum(terms, n_qubits=n)


def test_pauli_layer_matrix():
    from tnc_b200 import pauli_layer_matrix
    paulis = {(0, 0): np.eye(2), (1, 0): np.array([[0, 1], [1, 0]]), (0, 1): np.diag([1, -1]),
              (1, 1): np.array([[0, -1j], [1j, 0]])}
    for (x, z), p in paulis.items():
        m = pauli_layer_matrix(x, z)
        assert m.dtype == np.complex128 and m.shape == (2, 2)
        assert np.array_equal(m, np.asarray(p, dtype=np.complex128).T)
        assert not np.signbit(m.real[m.real == 0]).any() and not np.signbit(m.imag[m.imag == 0]).any()   # the device's +0.0


# ------------------------------------------------------------------------------------------------ the network
@pytest.mark.parametrize("n, seed, support, terms", [
    (10, 1, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9], [{0: "Y", 3: "X", 7: "Z"}, {2: "Y", 5: "Y", 9: "Y"}, {1: "X"}, {}]),
    (11, 2, [4, 6], [{4: "Y"}, {4: "Z", 6: "X"}, {6: "Y", 4: "Y"}, {4: "X", 6: "Y"}]),
    (12, 3, [0], [{0: "Y"}, {0: "X"}, {0: "Z"}]),
    (12, 4, [2, 9, 11], [{2: "Y", 9: "X", 11: "Z"}, {9: "Y"}, {2: "X", 11: "X"}]),
])
def test_network_against_state_vector(n, seed, support, terms):
    c = random_circuit(n, 2 if len(support) < n else 3, seed)
    psi = state_vector(c)
    from tnc_b200 import pauli_layer_matrix
    from tnc_b200.tensornetwork.contraction import leaves
    pn = c.into_pauli_expectation_network(support)
    lv = leaves(pn.tn)
    n_kept = len(pn.kept)
    assert len(lv) == 2 * n_kept + len(support) and pn.layer_qubit == sorted(support)
    if len(support) < 3:   # the light cone of one or two qubits after two layers leaves gates out and joins wires
        assert n_kept < len(c.tensors)
        offset = c.next_edge
        joined = [t for t in lv[n_kept:2 * n_kept] if any(l < offset for l in t.legs)]
        assert joined
    count = {}
    for t in lv:
        for l in t.legs:
            count[l] = count.get(l, 0) + 1
    assert set(count.values()) == {2}
    for paulis in terms:
        payloads = {leaf: pauli_layer_matrix(int(paulis.get(q, "I") in "XY"), int(paulis.get(q, "I") in "ZY"))
                    for leaf, q in zip(pn.layer_leaf, pn.layer_qubit)}
        got = contract(pn.tn, payloads)
        want = np.vdot(psi, apply_pauli(psi, n, paulis))
        assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (paulis, got, want)
    # the staged identity layer: <psi|psi>
    assert abs(contract(pn.tn) - 1.0) <= 1e-12


def test_full_support_matches_expectation_value_network():
    from tnc_b200.tensornetwork.contraction import leaves
    c = random_circuit(10, 3, 8)
    pn = c.into_pauli_expectation_network(range(10))
    ref = leaves(c.into_expectation_value_network())
    got = leaves(pn.tn)
    assert len(got) == len(ref) and pn.kept == list(range(len(c.tensors)))
    n_layer = c.num_qubits()
    for i, (a, b) in enumerate(zip(got, ref)):
        assert list(a.legs) == list(b.legs) and list(a.bond_dims) == list(b.bond_dims), i
        if i >= len(ref) - n_layer:
            assert a.tensordata.kind == "matrix" and np.array_equal(np.asarray(a.tensordata.matrix), np.eye(2))
            continue
        assert a.tensordata.kind == b.tensordata.kind, i
        if a.tensordata.kind == "gate":
            assert a.tensordata.gate == b.tensordata.gate, i
        else:
            assert np.array_equal(np.asarray(a.tensordata.matrix), np.asarray(b.tensordata.matrix)), i
    assert pn.layer_leaf == list(range(len(ref) - n_layer, len(ref))) and pn.layer_qubit == list(range(10))
    k = len(c.tensors)
    assert pn.ket_of == {k + j: j for j in range(k)}


def test_support_refusals():
    c = random_circuit(4, 1, 0)
    for bad in ([], [4], [-1]):
        with pytest.raises(ValueError, match="must be a non-empty set of qubits of the 4-qubit circuit"):
            c.into_pauli_expectation_network(bad)


def test_angle_map_translation():
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    c = Circuit()
    c.allocate_register(4)
    c.append_gate("rx", [0.1], [0])      # tensor 4
    c.append_gate("ry", [0.2], [3])      # tensor 5: outside the cone of qubit 0
    c.append_gate("cx", [], [0, 1])      # tensor 6
    c.append_gate("rz", [0.3], [1])      # tensor 7: after the cone's last gate on qubit 1, pruned
    c.append_gate("u", [0.1, 0.2, 0.3], [0])   # tensor 8
    amap = AngleMap([(4, 0, 0, 2.0), (5, 0, 1, 1.0), (7, 0, 2, -1.0), (8, 2, 0, 0.5), (8, 0, 3, 1.0)], 4, [1, 2, 3, 4])
    pn = c.into_pauli_expectation_network([0])
    assert pn.kept == [0, 1, 4, 6, 8]
    k = len(pn.kept)
    m = pn.angle_map(amap)
    assert m.n_params == 4 and m.theta0.tolist() == [1, 2, 3, 4]
    assert m.refs == [(2, 0, 0, 2.0), (2 + k, 0, 0, 2.0), (4, 2, 0, 0.5), (4 + k, 2, 0, 0.5), (4, 0, 3, 1.0), (4 + k, 0, 3, 1.0)]
    assert all(pn.ket_of[b] == kk for kk, b in [(2, 2 + k), (4, 4 + k)])
    assert m.leaves() == [2, 4, 2 + k, 4 + k]


# ------------------------------------------------------------------------------------------------ the route cell
def test_expect_route_cell(built_lib):
    from tnc_b200._lib import TncbPauliLayer, u64_array
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork.contraction import _Marshal
    l = built_lib
    c = random_circuit(8, 2, 5)
    pn = c.into_pauli_expectation_network([0, 1])
    tn = pn.tn
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    fake_ctx = C.create_string_buffer(1 << 16)
    cx = C.cast(fake_ctx, C.c_void_p)
    layer = TncbPauliLayer(8, 2, u64_array(pn.layer_leaf), (C.c_int * 2)(0, 1))
    one = u64_array([1])
    coeff = (C.c_double * 1)(1.0)
    got = []
    for kind in KINDS:
        m = _Marshal()
        ct, cp = m.tn(tn), m.path(path)
        h = C.c_void_p()
        if kind == "plain":
            rc = l.tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h))
        elif kind.startswith("sliced "):
            rc = getattr(l, f"tncb_plan_create_{kind[7:]}_sliced")(None, C.byref(ct), C.byref(cp), len(legs), u64_array(legs),
                                                                  None, C.byref(h))
        else:
            rc = getattr(l, f"tncb_plan_create_{kind}")(None, C.byref(ct), C.byref(cp), None, C.byref(h))
        assert rc == 0, l.tncb_last_error()
        e = C.c_void_p()
        rc = l.tncb_plan_expect(cx, h, C.byref(layer), 1, one, one, coeff, 0, None, C.byref(e), None)
        got.append((rc, l.tncb_last_error().decode()))
        l.tncb_plan_destroy(h)
    staged = (ERR_INVALID, "tncb_plan_stage has not been called on this plan and context")
    refuse = (ERR_UNSUPPORTED, "tncb_plan_expect takes a plain or a gradient plan (tncb_plan_create / _vjp)")
    assert got == [staged, staged] + [refuse] * 5


def test_null_arguments(built_lib):
    from tnc_b200._lib import TncbPauliLayer
    l = built_lib
    layer = TncbPauliLayer(1, 0, None, None)
    one = (C.c_uint64 * 1)(0)
    coeff = (C.c_double * 1)(1.0)
    e = C.c_void_p()
    for args in [(None, None), (C.c_void_p(1), None)]:
        assert l.tncb_plan_expect(*args, C.byref(layer), 1, one, one, coeff, 0, None, C.byref(e), None) == ERR_INVALID
        assert l.tncb_last_error().decode() == "null argument"


# ------------------------------------------------------------------------------------------------ Expectation's arguments
class Recorder:
    """Stands in for the library: plan creation and metadata pass through, every other entry is logged"""

    def __init__(self, lib, log):
        self._lib, self._log = lib, log

    def __getattr__(self, name):
        if name in ("tncb_network_out_legs", "tncb_plan_destroy", "tncb_last_error", "tncb_plan_grad_offsets",
                    "tncb_angles_create", "tncb_angles_layout", "tncb_angles_destroy", "tncb_plan_info") or \
                name.startswith("tncb_plan_create"):
            return getattr(self._lib, name)
        return lambda *args: self._log.append((name,) + args) or 0


@pytest.fixture
def recorded(built_lib, monkeypatch):
    log = []
    ctx = types.SimpleNamespace(_l=Recorder(built_lib, log), handle=None, device=0)
    made = []
    yield ctx, log, made
    for e in made:
        built_lib.tncb_plan_destroy(e.plan.handle)
        e.plan.handle = None


def qaoa(n, seed, p=1):
    """a QAOA MaxCut circuit on a ring of n qubits with an extra chord; rz angles at refs (leaf, 0, γ_l, 2), rx at
    (leaf, 0, β_l, 2)"""
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    rng = np.random.default_rng(seed)
    edges = [(q, (q + 1) % n) for q in range(n)] + [(0, n // 2)]
    c = Circuit()
    c.allocate_register(n)
    for q in range(n):
        c.append_gate("h", [], [q])
    refs, theta = [], rng.uniform(-1, 1, 2 * p)
    for layer in range(p):
        for a, b in edges:
            c.append_gate("cx", [], [a, b])
            refs.append((len(c.tensors), 0, 2 * layer, 2.0))
            c.append_gate("rz", [2 * theta[2 * layer]], [b])
            c.append_gate("cx", [], [a, b])
        for q in range(n):
            refs.append((len(c.tensors), 0, 2 * layer + 1, 2.0))
            c.append_gate("rx", [2 * theta[2 * layer + 1]], [q])
    return c, edges, AngleMap(refs, 2 * p, theta)


def test_expectation_calls(recorded, monkeypatch):
    import tnc_b200.observables as obs
    from tnc_b200 import Expectation, PauliSum
    ctx, log, made = recorded
    c, edges, amap = qaoa(8, 1)
    h = PauliSum([(0.5, f"Z{a} Z{b}") for a, b in edges[:3]] + [(-0.25, "Y2")], n_qubits=8)
    calls = []

    def fake_call(cx, fn, args, outputs=(), keep=None, temps=()):
        calls.append((fn, args, outputs))
        return [None] * len(outputs)
    monkeypatch.setattr(obs, "_library_call", fake_call)
    exp = Expectation(c, h, ctx=ctx)
    made.append(exp)
    assert [r[0] for r in log] == ["tncb_plan_stage"]
    assert exp.network.layer_qubit == h.support() == [0, 1, 2, 3]
    with pytest.raises(ValueError, match="theta needs an angle_map"):
        exp.values(theta=object())
    with pytest.raises(ValueError, match="value_and_grad needs an angle_map"):
        exp.value_and_grad(object())
    with pytest.raises(AttributeError):        # the recorder returns no tensors: the arguments are what matters here
        exp.values(batch=3)
    ((fn, args, outputs),) = calls
    assert fn == "tncb_plan_expect" and outputs == (True, True, False)
    assert args[0] is None and args[1] is exp.plan.handle and args[3] == 4 and args[7] == 3
    layer = args[2]._obj
    assert layer.n_qubits == 8 and layer.n_layer == 4
    assert [layer.layer_leaf[j] for j in range(4)] == exp.network.layer_leaf
    assert [layer.layer_qubit[j] for j in range(4)] == [0, 1, 2, 3]
    x, z, coeff = h.masks()
    assert [args[4][k] for k in range(4)] == x.tolist() and [args[5][k] for k in range(4)] == z.tolist()
    assert [args[6][k] for k in range(4)] == coeff.tolist()
    # with an angle map: a gradient plan on the translated map's leaves, support widened on request
    del log[:]
    exp2 = Expectation(c, h, angle_map=amap, support=[0, 1, 2, 3, 7], ctx=ctx)
    made.append(exp2)
    assert exp2.network.layer_qubit == [0, 1, 2, 3, 7]
    assert [r[0] for r in log] == ["tncb_plan_stage"]
    offs = exp2.plan.grad_offsets()
    assert [i for i, o in enumerate(offs) if o >= 0] == exp2.angle_map.leaves()
    assert exp2.angles.n_params == 2
    with pytest.raises(ValueError, match=r"support \[0, 1\] does not hold the terms' qubits \[0, 1, 2, 3\]"):
        Expectation(c, h, support=[0, 1], ctx=ctx)
    with pytest.raises(ValueError, match="the Pauli sum acts on 9 qubits, the circuit has 8"):
        Expectation(c, PauliSum([(1.0, "Z0")], n_qubits=9), ctx=ctx)
    with pytest.raises(ValueError, match="every term is the identity"):
        Expectation(c, PauliSum([(1.0, "")], n_qubits=8), ctx=ctx)
