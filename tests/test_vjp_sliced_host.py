"""Sliced gradient plans compiled without a device (tncb_plan_create_vjp_sliced with a NULL context): one slice's
schedule and workspace are those of a gradient plan of the host-sliced slice network, the gradients pack the full
leaves' shapes, the refusals, and networks whose gradient workspace only fits sliced."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = -1, -9
D12_LEGS = [157, 1115, 231, 606, 1084, 986, 1088, 155, 515]     # the committed 6 + three from find_slices (peak 2^27)


def _lib():
    from tnc_b200._lib import lib
    return lib()


def _mask(tn, wrt):
    from tnc_b200.tensornetwork import leaves
    if wrt is None:
        return None
    mask = (C.c_uint8 * max(len(leaves(tn)), 1))()
    for i in wrt:
        mask[i] = 1
    return mask


def create(tn, path, wrt=None):
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    return _lib().tncb_plan_create_vjp(None, C.byref(ct), C.byref(cp), _mask(tn, wrt), C.byref(h)), h


def create_sliced(tn, path, legs, wrt=None):
    from tnc_b200._lib import u64_array
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    arr = u64_array(list(legs) or [0])
    return _lib().tncb_plan_create_vjp_sliced(None, C.byref(ct), C.byref(cp), len(legs), arr, _mask(tn, wrt), C.byref(h)), h


def ok(rc_h):
    rc, h = rc_h
    assert rc == 0, _lib().tncb_last_error()
    return h


def info(h):
    n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fl, by = C.c_double(), C.c_double()
    assert _lib().tncb_plan_info(h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
    return {"pairs": n.value, "flops": fl.value, "bytes": by.value, "peak_bytes": pk.value, "kernels": k.value}


def offsets(h, n):
    arr = (C.c_int64 * n)()
    assert _lib().tncb_plan_grad_offsets(h, arr) == 0
    return list(arr)


def destroy(*hs):
    for h in hs:
        _lib().tncb_plan_destroy(h)


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def amplitude(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


@pytest.fixture(scope="module")
def q12(built_lib):
    tn = amplitude(12, 6, 5)
    return tn, greedy(tn)


@pytest.fixture(scope="module")
def bench_net(built_lib):
    sys.path.insert(0, ROOT)
    import bench
    tn = bench.build_network()
    return tn, bench.greedy_path(tn)


def check_matches_host_sliced(tn, path, legs):
    """pairs, flops and per-slice workspace equal tncb_plan_create_vjp on host-sliced slices; extract + accumulate are
    the only extra launches"""
    from tnc_b200.contractionpath.slicing import SlicedNetwork
    hs = ok(create_sliced(tn, path, legs))
    got = info(hs)
    sn = SlicedNetwork(tn, legs)
    assert len(sn.assignments) == 2 ** len(legs)
    for a in (sn.assignments[0], sn.assignments[-1]):
        h = ok(create(sn.slice(a), path))
        want = info(h)
        destroy(h)
        assert (got["pairs"], got["flops"], got["bytes"], got["peak_bytes"]) == \
            (want["pairs"], want["flops"], want["bytes"], want["peak_bytes"]), (legs, a, got, want)
        assert got["kernels"] == want["kernels"] + 1, (got, want)       # + the extract launch
    destroy(hs)
    return got


@pytest.mark.parametrize("n_legs", [1, 2, 3])
def test_q12_matches_host_sliced(q12, n_legs):
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = q12
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert len(legs) == n_legs
    check_matches_host_sliced(tn, path, legs)


@pytest.mark.parametrize("n_legs", [1, 2, 3])
def test_bench_matches_host_sliced(bench_net, n_legs):
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = bench_net
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert len(legs) == n_legs
    got = check_matches_host_sliced(tn, path, legs)
    # the issue's table: 7.99 / 4.37 / 2.56 GB per slice
    assert got["peak_bytes"] / 1e9 == pytest.approx({1: 7.99, 2: 4.37, 3: 2.56}[n_legs], abs=0.01)


def test_offsets_pack_full_leaves(q12):
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    tn, path = q12
    lv = leaves(tn)
    legs = find_slices(tn, path, min_slices=4)
    full = [int(np.prod(l.bond_dims)) for l in lv]
    h = ok(create_sliced(tn, path, legs))
    assert offsets(h, len(lv)) == list(np.cumsum([0] + full[:-1]))
    destroy(h)
    want = [0, 3, len(lv) - 1] + [i for i, l in enumerate(lv) if set(l.legs) & set(legs)][:2]
    h = ok(create_sliced(tn, path, legs, wrt=want))
    offs, pos = offsets(h, len(lv)), 0
    for i in range(len(lv)):
        if i in want:
            assert offs[i] == pos, i
            pos += full[i]
        else:
            assert offs[i] == -1, i
    destroy(h)


def test_zero_legs_is_the_gradient_plan(q12):
    from tnc_b200.tensornetwork import leaves
    tn, path = q12
    n = len(leaves(tn))
    for wrt in (None, [2, 7]):
        a, b = ok(create(tn, path, wrt)), ok(create_sliced(tn, path, [], wrt))
        ia, ib = info(a), info(b)
        assert ia == ib, (ia, ib)          # no sliced leaf: no extract launch; the accumulate replaces the gather
        assert offsets(a, n) == offsets(b, n)
        destroy(a, b)


def test_refusals(q12, monkeypatch):
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, path = q12
    lv = leaves(tn)
    count = {}
    for l in lv:
        for x in l.legs:
            count[x] = count.get(x, 0) + 1
    inner = [x for x, c in count.items() if c == 2]
    absent = max(count) + 1000

    def refused(legs, status, words, wrt=None, net=tn, p=path):
        rc, _ = create_sliced(net, p, legs, wrt)
        msg = _lib().tncb_last_error().decode()
        assert rc == status, (legs, rc, msg)
        assert words in msg, msg

    refused([absent], ERR_INVALID, "does not occur")
    from tnc_b200.builders import random_circuit_builder
    sv, _ = random_circuit_builder(6, 2, 0.5, 0.5, np.random.default_rng(1)).into_statevector_network()
    sv_count = {}
    for l in leaves(sv):
        for x in l.legs:
            sv_count[x] = sv_count.get(x, 0) + 1
    open_leg = next(x for x, c in sv_count.items() if c == 1)
    sv_inner = next(x for x, c in sv_count.items() if c == 2)
    refused([sv_inner, open_leg], ERR_INVALID, "open leg", net=sv, p=greedy(sv))
    refused([inner[0], inner[1], inner[0]], ERR_INVALID, "listed twice")
    assert len(inner) >= 64
    refused(inner[:64], ERR_INVALID, "overflows 64 bits")
    # everything tncb_plan_create_vjp refuses: wrt selecting nothing, no pairs, device leaves
    refused([inner[0]], ERR_INVALID, "selects no leaf", wrt=[])
    one = Tensor([0, 1], [2, 2])
    one.set_tensor_data(TensorData.Matrix(np.eye(2)))
    refused([], ERR_UNSUPPORTED, "at least one pair", net=Tensor.new_composite([one]), p=ContractionPath.simple([]))
    from tnc_b200 import DeviceTensor
    fake = DeviceTensor.__new__(DeviceTensor)
    fake.handle, fake.shape, fake.ctx = C.c_void_p(0x1000), tuple(lv[1].bond_dims), None
    t = Tensor(lv[1].legs, lv[1].bond_dims)
    t.set_tensor_data(TensorData.Matrix(fake))
    parts = list(tn.tensors)
    parts[1] = t
    refused([inner[0]], ERR_UNSUPPORTED, "device leaves", net=Tensor.new_composite(parts))
    fake.handle = None
    # the per-slice workspace above the static-workspace limit
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    sys.path.insert(0, ROOT)
    import bench
    big = bench.build_network()
    refused([], ERR_UNSUPPORTED, "static-workspace limit", net=big, p=bench.greedy_path(big))


def test_leaf_with_too_many_sliced_legs(built_lib):
    """a leaf carrying 9 sliced legs does not fit an item: refused, not mis-addressed"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(0)
    legs = list(range(10))
    a = Tensor(legs, [2] * 10)
    a.set_tensor_data(TensorData.Matrix(rng.standard_normal([2] * 10) + 0j))
    b = Tensor(legs[::-1], [2] * 10)
    b.set_tensor_data(TensorData.Matrix(rng.standard_normal([2] * 10) + 0j))
    tn = Tensor.new_composite([a, b])
    path = ContractionPath.simple([(0, 1)])
    rc, _ = create_sliced(tn, path, legs[:9])
    assert rc == ERR_UNSUPPORTED and "sliced legs" in _lib().tncb_last_error().decode()
    destroy(ok(create_sliced(tn, path, legs[:8])))


def test_workspace_limit_8_gb(bench_net, monkeypatch):
    """at TNCB_PLAN_WS_GB=8 bench.py's network (15.24 GB) has no gradient plan, but a 2-leg sliced one (4.37 GB)"""
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = bench_net
    legs = find_slices(tn, path, min_slices=4)
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "8")
    rc, _ = create(tn, path)
    assert rc == ERR_UNSUPPORTED and "15" in _lib().tncb_last_error().decode()
    h = ok(create_sliced(tn, path, legs))
    assert info(h)["peak_bytes"] <= 8 << 30
    destroy(h)


def test_sycamore_d12_nine_legs(built_lib):
    """the committed depth-12 tree: its 6 committed legs need 218 GB per slice (refused); with 3 more legs a slice's
    gradient fits the 46 GiB of a device-less compile, 512 slices"""
    from tnc_b200.builders import sycamore_circuit
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.contractionpath.slicing import path_cost, _flat
    with open(os.path.join(ROOT, "bench_inputs", "sycamore53_d12.json")) as f:
        d = json.load(f)
    tn = sycamore_circuit(53, 12, np.random.default_rng(1)).into_amplitude_network("0" * 53)[0]
    path = ContractionPath.simple([tuple(x) for x in d["toplevel"]])
    assert sorted(D12_LEGS[:6]) == sorted(d["sliced_legs"])
    rc, _ = create_sliced(tn, path, d["sliced_legs"])
    assert rc == ERR_UNSUPPORTED and "static-workspace limit" in _lib().tncb_last_error().decode()
    h = ok(create_sliced(tn, path, D12_LEGS))
    got = info(h)
    assert got["peak_bytes"] <= 46 << 30, got
    fl, _, _ = path_cost([(t.legs, t.bond_dims) for t in _flat(tn)], path, D12_LEGS)
    assert got["flops"] >= fl                          # forward + backward pairs of one slice
    from tnc_b200.contractionpath.slicing import slice_assignments
    assert len(slice_assignments(tn, D12_LEGS)) == 512
    destroy(h)
