"""CPU-side tests: the C-ABI library loads and exports every symbol include/tncb.h declares,
the host logic (leg algebra, gate table, fan-in mapping, path helpers) matches the oracle /
the reference's KATs.  No compute calls (no GPU here)."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from oracle import tnc_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_exported(built_lib):
    from tnc_b200._lib import SIGNATURES
    hdr = open(os.path.join(ROOT, "include", "tncb.h")).read()
    declared = set(re.findall(r"\b(tncb_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(built_lib, name), f"{name} declared in tncb.h but not exported"
    assert declared == set(SIGNATURES), declared ^ set(SIGNATURES)
    assert b"sm_90a" in built_lib.tncb_version()


def test_no_gpu_fails_loudly(built_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import tnc_b200 as tb
    with pytest.raises(tb.TncbError) as e:
        tb.Context(0)
    assert e.value.status == -6 and "no CPU fallback" in str(e.value)


def test_product_never_imports_oracle():
    for dp, _, fs in os.walk(os.path.join(ROOT, "tnc_b200")):
        for f in fs:
            if f.endswith((".py", ".cpp", ".cu", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "tnc_oracle" not in src and "from oracle" not in src and "import oracle" not in src, f


def _out_legs(lib, a_legs, a_dims, b_legs, b_dims):
    from tnc_b200._lib import u64_array
    n = C.c_int(); ol = u64_array([0] * 64); od = u64_array([0] * 64)
    m, nn, k = C.c_uint64(), C.c_uint64(), C.c_uint64()
    rc = lib.tncb_pair_out_legs(len(a_legs), u64_array(a_legs), u64_array(a_dims), len(b_legs), u64_array(b_legs),
                                u64_array(b_dims), C.byref(n), ol, od, C.byref(m), C.byref(nn), C.byref(k))
    return rc, [ol[i] for i in range(n.value)], [od[i] for i in range(n.value)], (m.value, nn.value, k.value)


def test_pair_leg_algebra_matches_reference(built_lib, kat):
    # contraction.rs:121-178: legs of AxB = [3,4,0,1] shape [8,6,3,2]; BxC = [0,5,2,4] shape [3,5,7,6]
    rc, legs, dims, mnk = _out_legs(built_lib, kat["A"]["legs"], kat["A"]["shape"], kat["B"]["legs"], kat["B"]["shape"])
    assert rc == 0 and legs == kat["AxB"]["legs"] and dims == kat["AxB"]["shape"] and mnk == (6, 48, 7)
    rc, legs, dims, mnk = _out_legs(built_lib, kat["B"]["legs"], kat["B"]["shape"], kat["C"]["legs"], kat["C"]["shape"])
    assert rc == 0 and legs == kat["BxC"]["legs"] and dims == kat["BxC"]["shape"] and mnk == (42, 15, 8)
    # tensor.rs doc example: [1,2,3]^[4,2,5] (self=tensor1) = [1,3,4,5]; here self=b
    rc, legs, dims, _ = _out_legs(built_lib, [4, 2, 5], [3, 4, 9], [1, 2, 3], [2, 4, 6])
    assert rc == 0 and legs == [1, 3, 4, 5] and dims == [2, 6, 3, 9]
    # random cross-check against the oracle's symmetric difference
    rng = np.random.default_rng(0)
    for _ in range(50):
        ids = list(rng.permutation(12))
        a_legs = [int(x) for x in ids[: rng.integers(0, 7)]]
        pool = [int(x) for x in rng.permutation(12)]
        b_legs = pool[: rng.integers(0, 7)]
        dim_of = {i: int(rng.integers(1, 5)) for i in range(12)}
        a_dims = [dim_of[l] for l in a_legs]; b_dims = [dim_of[l] for l in b_legs]
        rc, legs, dims, mnk = _out_legs(built_lib, a_legs, a_dims, b_legs, b_dims)
        exp_l, exp_d = orc.sym_diff_legs(b_legs, b_dims, a_legs, a_dims)
        assert rc == 0 and legs == exp_l and dims == exp_d
        assert mnk == orc.pair_mnk(a_legs, a_dims, b_legs, b_dims)


def test_pair_errors(built_lib):
    rc, *_ = _out_legs(built_lib, [0, 1], [2, 3], [1, 2], [4, 2])
    assert rc == -2  # bond dimension mismatch
    rc, *_ = _out_legs(built_lib, [0, 0], [2, 2], [1], [2])
    assert rc == -1


def test_kernel_class(built_lib):
    from tnc_b200._lib import u64_array
    def cls(a_legs, b_legs, d):
        return built_lib.tncb_pair_kernel_class(len(a_legs), u64_array(a_legs), u64_array([d] * len(a_legs)),
                                                len(b_legs), u64_array(b_legs), u64_array([d] * len(b_legs)))
    assert cls([0, 1], [1, 2], 2) == 0          # tiny -> K0
    assert cls(list(range(12)), [12, 1, 13, 3, 14, 5, 15, 7, 16, 9, 17, 11], 4) == 1  # C2 -> K1
    assert cls(list(range(20)), list(range(20)), 2) == 0  # full inner product -> K0 split-K


GATES = ["x", "y", "z", "h", "t", "u", "sx", "sy", "sz", "rx", "ry", "rz", "cx", "cz", "swap", "cp", "iswap", "fsim"]
NPAR = {"u": 3, "rx": 1, "ry": 1, "rz": 1, "cp": 1, "fsim": 2}


def test_gate_table_matches_oracle(built_lib):
    from tnc_b200 import gates
    rng = np.random.default_rng(42)
    for g in GATES:
        a = list(rng.uniform(-math.pi, math.pi, NPAR.get(g, 0)))
        assert np.array_equal(gates.load_gate(g, a), orc.load_gate(g, a)), g
        assert np.array_equal(gates.load_gate_adjoint(g, a), orc.load_gate(g, a, True)), g
    assert gates.is_gate_known("fsim") and not gates.is_gate_known("foo")


def test_gate_errors(built_lib):
    import tnc_b200 as tb
    from tnc_b200 import gates
    with pytest.raises(tb.TncbError, match="Gate 'foo' not found."):
        gates.load_gate("foo")
    with pytest.raises(tb.TncbError, match="Expected 0 angles, but got 2."):
        gates.load_gate("x", [2.0, 4.0])


def test_fanin_mapping_kat(built_lib):
    """mpi/communication.rs:257-279 test_tensor_mapping."""
    from tnc_b200._lib import u64_array
    ranks = (C.c_int * 3)()
    rc = built_lib.tncb_fanin_mapping(3, u64_array([0, 1, 2]), 2, u64_array([0, 2, 0, 1]), 4, ranks)
    assert rc == 0
    # the reference's assertions verbatim: rank(0) == 0, rank(1) == 2, rank(2) == 1 (FxHashMap walk order 0, 2, 1)
    assert list(ranks) == [0, 2, 1]
    rc = built_lib.tncb_fanin_mapping(3, u64_array([0, 1, 2]), 2, u64_array([1, 0, 2, 1]), 4, ranks)
    assert rc == 0 and list(ranks) == [1, 2, 0]
    rc = built_lib.tncb_fanin_mapping(3, u64_array([0, 1, 2]), 2, u64_array([0, 2, 0, 1]), 2, ranks)
    assert rc == -1  # not enough ranks


def test_python_path_helpers():
    from tnc_b200.contractionpath import ContractionPath, path, ssa_ordering, ssa_replace_ordering, validate_path
    assert ssa_ordering([(0, 3, 15), (1, 2, 44), (6, 4, 8), (5, 15, 22), (8, 44, 12), (12, 22, 99)], 7).toplevel == \
        [(0, 3), (1, 2), (6, 4), (5, 7), (9, 8), (11, 10)]
    p = path((0, 3), (1, 2), (6, 4), (5, 7), (9, 8), (11, 10), nested={1: [(2, 1), (0, 3)], 6: [(0, 2), (1, 3), (4, 5)]})
    r = ssa_replace_ordering(p)
    assert r.toplevel == [(0, 3), (1, 2), (6, 4), (5, 0), (6, 1), (6, 5)]
    assert r.nested[1].toplevel == [(2, 1), (0, 2)] and r.nested[6].toplevel == [(0, 2), (1, 3), (0, 1)]
    assert validate_path(path((0, 1), (0, 2))) and not validate_path(path((0, 1), (1, 2)))
    assert ContractionPath.single(0, 1).toplevel == [(0, 1)]


def test_python_tensor_algebra():
    from tnc_b200.tensornetwork import Tensor
    bd = {1: 2, 2: 4, 3: 6, 4: 3, 5: 9}
    t1, t2 = Tensor.new_from_map([1, 2, 3], bd), Tensor.new_from_map([4, 2, 5], bd)
    assert (t1 - t2).legs == [1, 3] and (t1 | t2).legs == [1, 2, 3, 4, 5] and (t1 & t2).legs == [2]
    assert (t1 ^ t2).legs == [1, 3, 4, 5] and (t1 ^ t2).bond_dims == [2, 6, 3, 9]
    tn = Tensor.new_composite([t1, t2])
    assert tn.external_tensor().legs == [1, 3, 4, 5] and tn.is_connected()
    tn.push_tensor(Tensor.new_from_const([7], 2))
    assert not tn.is_connected()


def test_python_circuit_matches_oracle_structure():
    from tnc_b200.builders import Circuit
    c = Circuit(); q = c.allocate_register(3)
    c.append_gate("h", [], [q[0]]); c.append_gate("cx", [], [q[0], q[1]]); c.append_gate("cx", [], [q[1], q[2]])
    tn, perm = c.into_statevector_network()
    o = orc.OCircuit(); oq = o.allocate_register(3)
    o.append_gate("h", [], [oq[0]]); o.append_gate("cx", [], [oq[0], oq[1]]); o.append_gate("cx", [], [oq[1], oq[2]])
    otn, ofinal = o.into_statevector_network()
    assert [t.legs for t in tn.tensors] == [t.legs for t in otn.children]
    assert perm.target_leg_order == ofinal == [4, 6, 7]
    with pytest.raises(ValueError, match="Qubit arguments must be unique"):
        c.append_gate("cx", [], [q[1], q[1]])


def test_marshalled_tree_round_trips(built_lib):
    """The C tree handed to tncb_contract_tensor_network (tncb_tn, include/tncb.h) read back field by field equals the
    Python `Tensor` tree it was built from: gate / matrix / file / empty leaves, nested composites, angle packing."""
    from tnc_b200.builders import random_circuit
    from tnc_b200.tensornetwork import Tensor, TensorData
    from tnc_b200.tensornetwork import contraction as ct

    def read(addr, n, keep):
        rec = np.frombuffer((C.c_char * (n * ct._TN_DTYPE.itemsize)).from_address(addr), dtype=ct._TN_DTYPE)
        out = []
        for r in rec:
            rk = int(r["rank"])
            d = {"legs": [int(x) for x in np.frombuffer((C.c_char * (8 * rk)).from_address(int(r["legs"])), dtype=np.uint64)] if rk else [],
                 "dims": [int(x) for x in np.frombuffer((C.c_char * (8 * rk)).from_address(int(r["dims"])), dtype=np.uint64)] if rk else [],
                 "kind": int(r["kind"])}
            if d["kind"] == 2:
                na = int(r["n_gate_angles"])
                ang = tuple(np.frombuffer((C.c_char * (8 * na)).from_address(int(r["gate_angles"])), dtype=np.float64)) if na else ()
                d["gate"] = (C.string_at(int(r["gate_name"])).decode(), ang, bool(r["gate_adjoint"]))
            if d["kind"] == 1:
                d["host"] = int(r["host_re_im"])
            if d["kind"] == 4:
                d["file"] = (C.string_at(int(r["file_path"])).decode(), bool(r["file_adjoint"]))
            if r["n_children"]:
                d["children"] = read(int(r["children"]), int(r["n_children"]), keep)
            out.append(d)
        return out

    def expect(t, host_ptrs):
        if t.tensors:
            return {"legs": [], "dims": [], "kind": 0, "children": [expect(c, host_ptrs) for c in t.tensors]}
        td = t.tensordata
        d = {"legs": list(t.legs), "dims": list(t.bond_dims), "kind": {"uncontracted": 0, "matrix": 1, "gate": 2, "file": 4}[td.kind]}
        if td.kind == "gate":
            d["gate"] = (td.gate[0], tuple(td.gate[1]), td.gate[2])
        if td.kind == "matrix":
            d["host"] = host_ptrs[id(td.matrix)]
        if td.kind == "file":
            d["file"] = td.file
        return d

    rc = random_circuit(12, 8, 0.5, 0.5, np.random.default_rng(9))
    n = len(rc.tensors)
    a = np.arange(8, dtype=np.complex128).reshape(2, 4)
    ta = Tensor.new([0, 1], [2, 4]); ta.set_tensor_data(TensorData.Matrix(a))
    tf = Tensor.new([1, 2], [4, 3]); tf.set_tensor_data(TensorData.File("/tmp/some file.h5", True))
    nested = Tensor.new_composite([Tensor.new_composite(rc.tensors[:n // 3]), Tensor.new_composite(rc.tensors[n // 3:]),
                                   Tensor.new_composite([ta, tf, Tensor.new([], [])])])
    for tn in (rc, nested):
        m = ct._Marshal()
        c_tn = m.tn(tn)
        got = read(C.addressof(c_tn), 1, m.keep)[0]
        host_ptrs = {}
        def walk(t):
            for c in t.tensors:
                walk(c)
            if not t.tensors and t.tensordata.kind == "matrix":
                host_ptrs[id(t.tensordata.matrix)] = np.asarray(t.tensordata.matrix).__array_interface__["data"][0]
        walk(tn)
        assert got == expect(tn, host_ptrs)


def test_network_out_legs_matches_the_python_replay(built_lib):
    """tncb_network_out_legs (metadata only, no GPU) == dist.communication.contracted_legs == the oracle's result legs, for
    flat and nested paths; errors are the real call's"""
    from tnc_b200 import TncbError
    from tnc_b200._lib import check, u64_array
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.contractionpath.paths import Cotengrust
    from tnc_b200.dist.communication import contracted_legs
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork import contraction as ct

    def native(tn, path):
        m = ct._Marshal()
        c_tn, c_path = m.tn(tn), m.path(path)
        n = C.c_int()
        legs, dims = u64_array([0] * 64), u64_array([0] * 64)
        check(built_lib.tncb_network_out_legs(C.byref(c_tn), C.byref(c_path), C.byref(n), legs, dims))
        return [int(legs[i]) for i in range(n.value)], [int(dims[i]) for i in range(n.value)]

    def greedy(tn):
        o = Cotengrust(tn); o.find_path()
        return o.get_best_replace_path()

    sv, _ = random_circuit_builder(8, 5, 0.6, 0.6, np.random.default_rng(4)).into_statevector_network()     # 8 open legs
    p = greedy(sv)
    assert native(sv, p) == contracted_legs(sv, p) and len(native(sv, p)[0]) == 8
    n = len(sv.tensors)
    nested = Tensor.new_composite([Tensor.new_composite(sv.tensors[:n // 2]), Tensor.new_composite(sv.tensors[n // 2:])])
    pn = greedy(nested)
    assert sorted(pn.nested) == [0, 1]
    assert native(nested, pn) == contracted_legs(nested, pn)
    for i in (0, 1):      # a partition on its own: what the receiver of the fan-in is told
        assert native(nested.tensor(i), pn.nested[i]) == contracted_legs(nested.tensor(i), pn.nested[i])
    with pytest.raises(TncbError) as e:          # not fully contracted (contraction.rs:50)
        native(sv, ContractionPath.simple(p.toplevel[:-1]))
    assert e.value.status == -4


def test_null_arguments_never_crash(built_lib):
    """every exported entry point called with zero / NULL for every argument returns (a status, 0 or NULL) instead of
    dereferencing: the Rust shim turns statuses into panics, a segfault would take the host down.  One child process, so
    that a crash is seen as one (the name of the call in flight is the last line it printed)."""
    import subprocess
    import sys
    code = r"""
import sys, ctypes as C
sys.path.insert(0, %r)
from tnc_b200._lib import SIGNATURES, lib
l = lib()
for name in sorted(SIGNATURES):
    res, args = SIGNATURES[name]
    vals = [0 if a in (C.c_int, C.c_size_t, C.c_longlong, C.c_uint64, C.c_int64) else 0.0 if a is C.c_double else None for a in args]
    print(name, flush=True)
    getattr(l, name)(*vals)
print("SWEEP_OK", len(SIGNATURES))
""" % ROOT
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "SWEEP_OK" in r.stdout, (r.returncode, r.stdout.strip().splitlines()[-1:], r.stderr[-500:])
