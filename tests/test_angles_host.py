"""Gate angles without a GPU: the one angle table of gate_angles.h (tncb_gate_matrix unchanged bit for bit, its first and
second derivatives), every refusal of tncb_angles_create and the layouts it compiles against host-only gradient plans."""
import ctypes as C
import hashlib
import itertools
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_GATE = -1, -2, -7
N_ANG = {"u": 3, "rx": 1, "ry": 1, "rz": 1, "cp": 1, "fsim": 2}
SWEEP = [0.0, -0.0, math.pi, -math.pi, math.pi / 2, -math.pi / 2, 0.3, 0.2, -1.7, 2.5, 1e3, -1e3, 123.456, -999.9, 1e-300, 7.0]
# sha256 of the raw tncb_gate_matrix output over all 18 gates, both adjoint flags and every tuple of SWEEP angles, as
# produced by the table before the six angle gates moved to gate_angles.h
MATRIX_DIGEST = "8b889515e253ff281100876b511fb44d67a7cf13b1d67b0e0947d53b116fd876"


def _lib():
    from tnc_b200._lib import lib
    return lib()


def _err():
    return _lib().tncb_last_error().decode()


def test_gate_matrix_bits_unchanged(built_lib):
    from tnc_b200.gates import KNOWN_GATES
    h, calls = hashlib.sha256(), 0
    for g in KNOWN_GATES:
        n = N_ANG.get(g, 0)
        for adj in (0, 1):
            for ang in itertools.product(SWEEP, repeat=n):
                a, out, r = (C.c_double * 3)(*ang), (C.c_double * 32)(), C.c_int()
                assert _lib().tncb_gate_matrix(g.encode(), a, n, adj, out, C.byref(r)) == 0
                h.update(bytes(out)[:8 * 2 * (4 if r.value == 2 else 16)])
                calls += 1
    assert calls == 8856
    assert h.hexdigest() == MATRIX_DIGEST


def _mat(g, a, adj):
    from tnc_b200.gates import load_gate, load_gate_adjoint
    return (load_gate_adjoint if adj else load_gate)(g, a).reshape(-1)


def _d(g, a, s, t=-1, adj=False):
    from tnc_b200.gates import load_gate_derivative
    return load_gate_derivative(g, a, s, t, adj).reshape(-1)


@pytest.mark.parametrize("gate", sorted(N_ANG))
@pytest.mark.parametrize("adj", [False, True])
def test_derivatives_against_central_differences(built_lib, gate, adj):
    rng = np.random.default_rng(len(gate) + 7 * adj)
    h = 1e-5
    for _ in range(4):
        a = rng.uniform(-4, 4, N_ANG[gate])
        for s in range(N_ANG[gate]):
            e = np.eye(N_ANG[gate])[s] * h
            fd = (_mat(gate, a + e, adj) - _mat(gate, a - e, adj)) / (2 * h)
            assert np.abs(_d(gate, a, s, -1, adj) - fd).max() < 1e-9
            for t in range(N_ANG[gate]):
                et = np.eye(N_ANG[gate])[t] * h
                fd2 = (_d(gate, a + et, s, -1, adj) - _d(gate, a - et, s, -1, adj)) / (2 * h)
                assert np.abs(_d(gate, a, s, t, adj) - fd2).max() < 1e-9
                assert np.array_equal(_d(gate, a, s, t, adj), _d(gate, a, t, s, adj))   # symmetric
            # the adjoint's derivative is the derivative's adjoint
            d = 2 if _d(gate, a, s).size == 4 else 4
            assert np.array_equal(_d(gate, a, s, -1, True), _d(gate, a, s).reshape(d, d).conj().T.reshape(-1))


def test_exact_identities(built_lib):
    for a in (0.7, -2.1, math.pi):
        for g in ("rx", "ry", "rz"):
            assert np.array_equal(_d(g, [a], 0, 0), -_mat(g, [a], False) / 4)
        cp = _mat("cp", [a], False)
        dcp = _d("cp", [a], 0)
        assert np.array_equal(dcp[:15], np.zeros(15)) and dcp[15] == 1j * cp[15]
        assert np.array_equal(_d("cp", [a], 0, 0)[:15], np.zeros(15)) and _d("cp", [a], 0, 0)[15] == -cp[15]
        f = _mat("fsim", [0.3, a], False)
        dphi = _d("fsim", [0.3, a], 1)
        assert np.count_nonzero(dphi) == 1 and dphi[15] == -1j * f[15]
        assert np.array_equal(_d("fsim", [0.3, a], 0, 1), np.zeros(16))      # no mixed θ, φ entry
        u = _mat("u", [0.4, 0.9, a], False)
        assert _d("u", [0.4, 0.9, a], 1, 2)[3] == -u[3]                      # d²/dφ dλ e^{i(φ+λ)} c
        assert np.array_equal(_d("u", [0.4, 0.9, a], 1, 2)[:3], np.zeros(3))


def test_derivative_errors(built_lib):
    lib = _lib()
    out, r = (C.c_double * 32)(), C.c_int()
    a = (C.c_double * 3)(0.1, 0.2, 0.3)
    cases = [("fsim", 1, 0, -1, ERR_GATE, "Expected 2 angles, but got 1."),
             ("nope", 0, 0, -1, ERR_GATE, "Gate 'nope' not found."),
             ("x", 0, 0, -1, ERR_GATE, "slot out of range for this gate: 'x' takes 0 angles, slots 0, -1"),
             ("rx", 1, 1, -1, ERR_GATE, "slot out of range for this gate: 'rx' takes 1 angles, slots 1, -1"),
             ("fsim", 2, 0, 2, ERR_GATE, "slot out of range for this gate: 'fsim' takes 2 angles, slots 0, 2"),
             ("u", 3, -1, -1, ERR_GATE, "slot out of range for this gate: 'u' takes 3 angles, slots -1, -1")]
    for name, n, s, t, status, msg in cases:
        assert lib.tncb_gate_derivative(name.encode(), a, n, 0, s, t, out, C.byref(r)) == status
        assert _err() == msg
    assert lib.tncb_gate_derivative(None, a, 1, 0, 0, -1, out, C.byref(r)) == ERR_INVALID
    assert lib.tncb_gate_derivative(b"rx", None, 1, 0, 0, -1, out, C.byref(r)) == ERR_INVALID


# ---- angle maps ----
def _circuit():
    """3 qubits: u, rx, ry, rz, cp, fsim, an adjointed fsim and gates without angles; leaves in collect order"""
    from tnc_b200.builders import Circuit
    c = Circuit()
    q = c.allocate_register(3)
    c.append_gate("u", [0.1, 0.2, 0.3], [q[0]])
    c.append_gate("rx", [0.4], [q[1]])
    c.append_gate("h", [], [q[2]])
    c.append_gate("ry", [0.5], [q[2]])
    c.append_gate("cp", [0.6], [q[0], q[1]])
    c.append_gate("fsim", [0.7, 0.8], [q[1], q[2]])
    c.append_gate("rz", [0.9], [q[0]])
    c.append_gate("fsim", [1.0, 1.1], [q[0], q[2]], adjoint=True)
    return c.into_amplitude_network("000")[0]


def _gate_leaves(tn):
    from tnc_b200.tensornetwork import leaves
    return {i: leaf.tensordata.gate for i, leaf in enumerate(leaves(tn)) if leaf.tensordata.kind == "gate"}


def _create(tn, n_params, refs, offsets=None, block=0):
    from tnc_b200.angles import _Ref
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct = m.tn(tn)
    arr = (_Ref * max(len(refs), 1))(*[_Ref(*r) for r in refs])
    offs = None if offsets is None else (C.c_int64 * len(offsets))(*offsets)
    h = C.c_void_p()
    rc = _lib().tncb_angles_create(C.byref(ct), n_params, len(refs), arr, offs, block, C.byref(h))
    return rc, h


def _layout(h, n_leaves):
    n_p, n_b = C.c_size_t(), C.c_size_t()
    offs = (C.c_int64 * n_leaves)()
    assert _lib().tncb_angles_layout(h, C.byref(n_p), C.byref(n_b), offs) == 0
    return n_p.value, n_b.value, list(offs)


def test_creation_refusals(built_lib):
    from tnc_b200.tensornetwork import leaves
    tn = _circuit()
    gl = _gate_leaves(tn)
    names = {gl[i][0]: i for i in sorted(gl, reverse=True)}      # first leaf of each gate name
    n = len(leaves(tn))
    ket = next(i for i in range(n) if i not in gl)
    fs, rx, h = names["fsim"], names["rx"], names["h"]
    packed = [-1] * n
    packed[fs] = 0
    cases = [
        (1, [(n, 0, 0, 1.0)], None, 0, ERR_INVALID, f"ref 0: leaf {n} is out of range ({n} leaves)"),
        (1, [(ket, 0, 0, 1.0)], None, 0, ERR_INVALID, f"ref 0: leaf {ket} is not a Gate leaf"),
        (1, [(h, 0, 0, 1.0)], None, 0, ERR_GATE, f"ref 0: leaf {h}: gate 'h' takes no angles"),
        (1, [(fs, 0, 0, 1.0), (rx, 1, 0, 1.0)], None, 0, ERR_GATE, f"ref 1: leaf {rx}: slot 1 is past the 1 angles of gate 'rx'"),
        (2, [(fs, 0, 2, 1.0)], None, 0, ERR_INVALID, f"ref 0: leaf {fs}: param 2 >= n_params 2"),
        (2, [(fs, 1, 0, 1.0), (rx, 0, 1, 1.0), (fs, 1, 1, 2.0)], None, 0, ERR_INVALID,
         f"ref 2: leaf {fs}, slot 1 is already set by ref 0"),
        (1, [(fs, 0, 0, float("nan"))], None, 0, ERR_INVALID, f"ref 0: leaf {fs}: the scale is not finite"),
        (1, [(fs, 0, 0, float("inf"))], None, 0, ERR_INVALID, f"ref 0: leaf {fs}: the scale is not finite"),
        (1, [(fs, 0, 0, 1.0), (rx, 0, 0, 1.0)], packed, 16, ERR_INVALID, f"ref 1: leaf {rx} has offset -1 (not in the block)"),
        (1, [(fs, 0, 0, 1.0)], packed, 15, ERR_INVALID, f"ref 0: leaf {fs}: its 16 elements at offset 0 run past block_elems 15"),
        (1, [(fs, 0, 0, 1.0)], None, 8, ERR_INVALID, f"ref 0: leaf {fs}: its 16 elements at offset 0 run past block_elems 8"),
        (0, [(fs, 0, 0, 1.0)], None, 0, ERR_INVALID, "n_params is 0"),
        (1, [], None, 0, ERR_INVALID, "no refs"),
    ]
    for n_params, refs, offs, block, status, msg in cases:
        rc, hd = _create(tn, n_params, refs, offs, block)
        assert (rc, _err()) == (status, msg), (refs, offs, block)
    over = [-1] * n
    over[fs], over[rx] = 0, 12
    rc, _ = _create(tn, 1, [(fs, 0, 0, 1.0), (rx, 0, 0, 1.0)], over, 32)
    assert (rc, _err()) == (ERR_INVALID, f"leaves {fs} and {rx} overlap in the block")


def test_packed_layout(built_lib):
    from tnc_b200.angles import AngleMap
    from tnc_b200.tensornetwork import leaves
    tn = _circuit()
    amap = AngleMap.every_angle(tn)
    gl = _gate_leaves(tn)
    assert amap.n_params == 3 + 1 + 1 + 1 + 2 + 1 + 2
    assert list(amap.theta0) == [a for i in sorted(gl) for a in gl[i][1]]
    rc, h = _create(tn, amap.n_params, amap.refs)
    assert rc == 0, _err()
    n = len(leaves(tn))
    n_p, block, offs = _layout(h, n)
    want, pos = [-1] * n, 0
    for i in sorted(gl):
        if gl[i][1]:
            want[i], pos = pos, pos + (4 if len(leaves(tn)[i].legs) == 2 else 16)
    assert (n_p, block, offs) == (amap.n_params, pos, want)
    assert _lib().tncb_angles_destroy(h) == 0


def _grad_offsets(tn, path, wrt):
    from tnc_b200.tensornetwork import leaves
    from tnc_b200.tensornetwork.contraction import _Marshal
    n = len(leaves(tn))
    mask = (C.c_uint8 * n)(*[1 if i in wrt else 0 for i in range(n)])
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    assert _lib().tncb_plan_create_vjp(None, C.byref(ct), C.byref(cp), mask, C.byref(h)) == 0, _err()
    offs = (C.c_int64 * n)()
    assert _lib().tncb_plan_grad_offsets(h, offs) == 0
    _lib().tncb_plan_destroy(h)
    return list(offs)


def _greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


@pytest.mark.parametrize("net", ["q12", "bench"])
def test_layout_against_grad_offsets(built_lib, net):
    from tnc_b200.angles import AngleMap, _block_size
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import leaves
    if net == "q12":
        tn = random_circuit_builder(12, 6, 0.5, 0.5, np.random.default_rng(5)).into_amplitude_network("0" * 12)[0]
    else:
        sys.path.insert(0, ROOT)
        import bench
        tn = bench.build_network()
    amap = AngleMap.every_angle(tn)
    gl = _gate_leaves(tn)
    fsims = [i for i in gl if gl[i][0] == "fsim"]
    assert len(amap.refs) == 2 * len(fsims) and amap.leaves() == sorted(fsims)   # two refs per fsim leaf
    if net == "bench":
        assert len(fsims) > 100
    offs = _grad_offsets(tn, _greedy(tn), set(amap.leaves()))
    shapes = [tuple(l.bond_dims) for l in leaves(tn)]
    block = _block_size(offs, shapes)
    rc, h = _create(tn, amap.n_params, amap.refs, offs, block)
    assert rc == 0, _err()
    assert _layout(h, len(offs)) == (amap.n_params, block, offs)
    assert _lib().tncb_angles_destroy(h) == 0
