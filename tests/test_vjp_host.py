"""Gradient plans compiled without a device (tncb_plan_create_vjp with a NULL context): the backward schedule, the
packing of the leaf gradients, the refusals, and forward-only plans keeping their peak bytes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = -1, -9


def _lib():
    from tnc_b200._lib import lib
    return lib()


def create(tn, path, wrt=None, grad=True):
    """(status, handle) of a host-only plan; wrt = leaf indices or None"""
    from tnc_b200.tensornetwork import leaves
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if not grad:
        return _lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)), h
    mask = None
    if wrt is not None:
        mask = (C.c_uint8 * max(len(leaves(tn)), 1))()
        for i in wrt:
            mask[i] = 1
    return _lib().tncb_plan_create_vjp(None, C.byref(ct), C.byref(cp), mask, C.byref(h)), h


def info(h):
    n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fl, by = C.c_double(), C.c_double()
    assert _lib().tncb_plan_info(h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
    return {"pairs": n.value, "flops": fl.value, "peak_bytes": pk.value, "kernels": k.value}


def offsets(h, n):
    arr = (C.c_int64 * n)()
    assert _lib().tncb_plan_grad_offsets(h, arr) == 0
    return list(arr)


def plans(tn, path, **kw):
    rc, h = create(tn, path, **kw)
    assert rc == 0, _lib().tncb_last_error()
    return h


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def amplitude(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def ancestors(tn, path, leaf):
    """number of forward pairs whose subtree holds `leaf` (replay of the replace-left path on leaf sets)"""
    from tnc_b200.tensornetwork import leaves
    counter = [0]

    def walk(t, p):
        if not t.tensors:
            counter[0] += 1
            return {counter[0] - 1}, 0
        sets, hits = [], 0
        for i, c in enumerate(t.tensors):
            if c.tensors and (p is None or i not in p.nested):
                sets.append(set(range(counter[0], counter[0] + len(leaves(c)))))
                counter[0] += len(leaves(c))
                continue
            s, h = walk(c, p.nested.get(i) if p is not None and c.tensors else None)
            sets.append(s)
            hits += h
        for i, j in (p.toplevel if p is not None else []):
            sets[i] = sets[i] | sets[j]
            sets[j] = set()
            hits += leaf in sets[i]
        return set().union(*sets), hits
    return walk(tn, path)[1]


@pytest.fixture(scope="module")
def small(built_lib):
    tn = amplitude(10, 5, 3)
    return tn, greedy(tn)


def test_all_leaves_triple_pairs_and_flops(small):
    tn, path = small
    fwd = info(plans(tn, path, grad=False))
    g = info(plans(tn, path))
    assert g["pairs"] == 3 * fwd["pairs"]
    assert g["flops"] == pytest.approx(3 * fwd["flops"], rel=1e-15)


def test_one_leaf_ancestors(small):
    from tnc_b200.tensornetwork import leaves
    tn, path = small
    fwd = info(plans(tn, path, grad=False))["pairs"]
    n = len(leaves(tn))
    for leaf in (0, n // 3, n - 1):
        got = info(plans(tn, path, wrt=[leaf]))["pairs"] - fwd
        assert got == ancestors(tn, path, leaf) and got >= 1, leaf


def test_offsets_pack_in_leaf_order(small):
    from tnc_b200.tensornetwork import leaves
    tn, path = small
    lv = leaves(tn)
    want = [1, 4, 5, len(lv) - 1]
    offs = offsets(plans(tn, path, wrt=want), len(lv))
    pos = 0
    for i, leaf in enumerate(lv):
        if i in want:
            assert offs[i] == pos, i
            pos += int(np.prod(leaf.bond_dims))
        else:
            assert offs[i] == -1, i
    all_offs = offsets(plans(tn, path), len(lv))
    assert all_offs == list(np.cumsum([0] + [int(np.prod(l.bond_dims)) for l in lv[:-1]]))


def test_refusals(small, monkeypatch):
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, path = small
    # a device leaf (the handle is never dereferenced: the plan is refused first)
    lv = list(tn.tensors)
    from tnc_b200 import DeviceTensor
    fake = DeviceTensor.__new__(DeviceTensor)
    fake.handle, fake.shape, fake.ctx = C.c_void_p(0x1000), tuple(lv[1].bond_dims), None
    t = Tensor(lv[1].legs, lv[1].bond_dims)
    t.set_tensor_data(TensorData.Matrix(fake))
    lv[1] = t
    rc, _ = create(Tensor.new_composite(lv), path)
    fake.handle = None
    assert rc == ERR_UNSUPPORTED
    # no pairs
    one = Tensor([0, 1], [2, 2])
    one.set_tensor_data(TensorData.Matrix(np.eye(2)))
    assert create(Tensor.new_composite([one]), ContractionPath.simple([]))[0] == ERR_UNSUPPORTED
    # wrt selecting nothing
    assert create(tn, path, wrt=[])[0] == ERR_INVALID
    # a gradient workspace above TNCB_PLAN_WS_GB: bench.py's network at 1 GiB
    sys.path.insert(0, ROOT)
    import bench
    big = bench.build_network()
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    rc, _ = create(big, bench.greedy_path(big))
    assert rc == ERR_UNSUPPORTED
    assert "bytes" in _lib().tncb_last_error().decode()
    assert len(leaves(big)) == 489


# forward-only plans of bench.py's network and of the config-4 partitions (bench_inputs/c4_partitions.json): their peak
# bytes from before gradient plans generalised the static layout, which must not move
FORWARD_PEAK = {
    "bench": 7248097472,
    "c4_2": 2147561664, "c4_2_part0": 1276155712, "c4_2_part1": 981506432,
    "c4_4": 1345400768, "c4_4_part0": 536907264, "c4_4_part1": 671122784, "c4_4_part2": 2150240, "c4_4_part3": 1576448,
    "c4_8": 957723072, "c4_8_part0": 805321504, "c4_8_part1": 1069120, "c4_8_part2": 269518368, "c4_8_part3": 69213248,
    "c4_8_part4": 25310528, "c4_8_part5": 284800, "c4_8_part6": 44704, "c4_8_part7": 672,
}


def test_forward_peak_bytes_unchanged(built_lib):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench
    import plan_partitions as pp
    tn = bench.build_network()
    got = {"bench": info(plans(tn, bench.greedy_path(tn), grad=False))["peak_bytes"]}
    for n in (2, 4, 8):
        net, path, _ = pp.load(tn, n)
        got[f"c4_{n}"] = info(plans(net, path, grad=False))["peak_bytes"]
        for i, part in enumerate(net.tensors):
            if i in path.nested:
                got[f"c4_{n}_part{i}"] = info(plans(part, path.nested[i], grad=False))["peak_bytes"]
    assert got == FORWARD_PEAK


def test_bench_gradient_plan_fits(built_lib):
    """bench.py's network with every leaf requested: 488 forward + 976 backward pairs in a workspace under the
    46 GiB static-workspace limit of a plan compiled without a device"""
    sys.path.insert(0, ROOT)
    import bench
    tn = bench.build_network()
    g = info(plans(tn, bench.greedy_path(tn)))
    assert g["pairs"] == 3 * 488
    assert g["peak_bytes"] <= 46 << 30, g
