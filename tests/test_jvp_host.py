"""Tangent plans compiled without a device (tncb_plan_create_jvp with a NULL context): the tangent schedule on top of the
forward one, the packing of the leaf tangents, the refusals, and the Python / torch-side checks that run before any
device work."""
import ctypes as C
import os
import re
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = -1, -9


def _lib():
    from tnc_b200._lib import lib
    return lib()


def mask_of(tn, wrt):
    from tnc_b200.tensornetwork import leaves
    if wrt is None:
        return None
    mask = (C.c_uint8 * max(len(leaves(tn)), 1))()
    for i in wrt:
        mask[i] = 1
    return mask


def create(tn, path, wrt=None, kind="jvp"):
    """(status, handle) of a host-only plan: kind = "jvp", "vjp" or "plain"; wrt = leaf indices or None"""
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if kind == "plain":
        return _lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)), h
    fn = _lib().tncb_plan_create_jvp if kind == "jvp" else _lib().tncb_plan_create_vjp
    return fn(None, C.byref(ct), C.byref(cp), mask_of(tn, wrt), C.byref(h)), h


def plan(tn, path, wrt=None, kind="jvp"):
    rc, h = create(tn, path, wrt, kind)
    assert rc == 0, _lib().tncb_last_error()
    return h


def info(h):
    n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fl, by = C.c_double(), C.c_double()
    assert _lib().tncb_plan_info(h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
    return {"pairs": n.value, "flops": fl.value, "peak_bytes": pk.value, "kernels": k.value}


def offsets(h, n):
    arr = (C.c_int64 * n)()
    assert _lib().tncb_plan_grad_offsets(h, arr) == 0
    return list(arr)


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def amplitude(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def ancestor_flops(tn, path, wrt):
    """(tangent pairs, their flops) by replaying the replace-left path on leaf sets: a forward pair gets one tangent pair
    per operand whose subtree holds a requested leaf, each with the forward pair's 8 M N K"""
    from tnc_b200.tensornetwork import leaves
    counter = [0]
    want = set(wrt)

    def walk(t, p):
        if not t.tensors:
            counter[0] += 1
            return ({counter[0] - 1}, list(t.legs), dict(zip(t.legs, t.bond_dims))), 0, 0.0
        slots, pairs, flops = [], 0, 0.0
        for i, c in enumerate(t.tensors):
            if c.tensors and (p is None or i not in p.nested):
                counter[0] += len(leaves(c))
                slots.append(None)
                continue
            s, n, f = walk(c, p.nested.get(i) if p is not None and c.tensors else None)
            slots.append(s)
            pairs += n
            flops += f
        for i, j in (p.toplevel if p is not None else []):
            (sa, la, da), (sb, lb, db) = slots[i], slots[j]
            dims = da | db
            out = [l for l in lb if l not in la] + [l for l in la if l not in lb]
            mnk = float(np.prod([dims[l] for l in set(la) | set(lb)], dtype=np.float64))
            sides = int(bool(sa & want)) + int(bool(sb & want))
            pairs += sides
            flops += sides * 8.0 * mnk
            slots[i], slots[j] = (sa | sb, out, dims), None
        return next(s for s in slots if s is not None), pairs, flops
    return walk(tn, path)[1:]


@pytest.fixture(scope="module")
def small(built_lib):
    tn = amplitude(12, 6, 3)
    return tn, greedy(tn)


@pytest.fixture(scope="module")
def bench_net(built_lib):
    sys.path.insert(0, ROOT)
    import bench
    tn = bench.build_network()
    return tn, bench.greedy_path(tn)


# C parameter types of include/tncb.h -> the ctypes the binding declares
CTYPES = {"tncb_ctx*": C.c_void_p, "tncb_plan*": C.c_void_p, "size_t": C.c_size_t, "const tncb_tn*": "tn*",
          "const tncb_path*": "path*", "const uint8_t*": "u8p", "tncb_plan**": "vpp", "const tncb_tensor*": C.c_void_p,
          "tncb_tensor**": "vpp"}


def header_params(name):
    with open(os.path.join(ROOT, "include", "tncb.h")) as f:
        text = f.read()
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\w+$", "", p).replace(" *", "*") for p in params]


@pytest.mark.parametrize("name", ["tncb_plan_create_jvp", "tncb_plan_jvp", "tncb_plan_jvp_batch"])
def test_signatures_match_header(name):
    from tnc_b200._lib import SIGNATURES, TncbPath, TncbTn, vpp
    resolve = {"vpp": vpp, "tn*": C.POINTER(TncbTn), "path*": C.POINTER(TncbPath), "u8p": C.POINTER(C.c_uint8)}
    want = [resolve.get(CTYPES[p], CTYPES[p]) for p in header_params(name)]
    res, args = SIGNATURES[name]
    assert res is C.c_int
    assert args == want, (args, want)


@pytest.mark.parametrize("net", ["small", "bench_net"])
def test_pairs_and_flops(net, request):
    """forward + tangent pairs, forward + tangent flops, with every leaf, a third of them and one leaf requested"""
    from tnc_b200.tensornetwork import leaves
    tn, path = request.getfixturevalue(net)
    fwd = info(plan(tn, path, kind="plain"))
    n = len(leaves(tn))
    every = [i for i, l in enumerate(leaves(tn)) if l.tensordata.kind != "uncontracted"]
    for wrt in (None, every[::3], [every[0]], [every[-1]]):
        got = info(plan(tn, path, wrt))
        pairs, flops = ancestor_flops(tn, path, every if wrt is None else wrt)
        assert got["pairs"] == fwd["pairs"] + pairs, (wrt, got, fwd, pairs)
        assert got["flops"] == pytest.approx(fwd["flops"] + flops, rel=1e-12)
        if wrt is None:                              # every leaf: two tangent pairs per forward pair
            assert got["pairs"] == 3 * fwd["pairs"]
            assert got["flops"] == pytest.approx(3 * fwd["flops"], rel=1e-12)
        if wrt is not None and len(wrt) == 1:        # one leaf: one tangent pair per ancestor step, no sums
            assert 1 <= pairs < n
    if net == "bench_net":
        assert fwd["pairs"] == 488 and n == 489


def test_offsets_equal_gradient_plan(small):
    from tnc_b200.tensornetwork import leaves
    tn, path = small
    n = len(leaves(tn))
    for wrt in (None, [1, 4, 5, n - 1], [n // 2]):
        assert offsets(plan(tn, path, wrt), n) == offsets(plan(tn, path, wrt, kind="vjp"), n), wrt


def test_plain_and_gradient_layouts_unchanged(bench_net):
    """bench.py's network: the plain and gradient plans' pairs, kernels and bytes from before tangent plans shared the
    static layout, which must not move (a gradient plan's peak_bytes is its static workspace)"""
    tn, path = bench_net
    assert info(plan(tn, path, kind="plain")) == {"pairs": 488, "flops": 6689291543832.0, "peak_bytes": 7248097472, "kernels": 70}
    assert info(plan(tn, path, kind="vjp")) == {"pairs": 1464, "flops": 20067874631496.0, "peak_bytes": 15244053248, "kernels": 155}


def test_tangent_workspace_fits(bench_net):
    """bench.py's network with every leaf requested fits one static workspace under the 46 GiB limit of a plan compiled
    without a device, and is larger than the gradient plan's (tangent slots live next to the forward ones)"""
    tn, path = bench_net
    t = info(plan(tn, path))
    g = info(plan(tn, path, kind="vjp"))
    assert g["peak_bytes"] < t["peak_bytes"] <= 46 << 30, (t, g)


def test_refusals(small, bench_net, monkeypatch):
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, path = small
    # a device leaf (the handle is never dereferenced: the plan is refused first)
    lv = list(tn.tensors)
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
    # wrt selecting nothing, a leaf without a payload
    assert create(tn, path, wrt=[])[0] == ERR_INVALID
    bare = Tensor([0, 1], [2, 2])
    other = Tensor([1, 0], [2, 2])
    other.set_tensor_data(TensorData.Matrix(np.eye(2)))
    assert create(Tensor.new_composite([bare, other]), ContractionPath.simple([(0, 1)]), wrt=[0])[0] != 0
    # a workspace above TNCB_PLAN_WS_GB: the message states the bytes
    big, big_path = bench_net
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    rc, _ = create(big, big_path)
    assert rc == ERR_UNSUPPORTED
    msg = _lib().tncb_last_error().decode()
    assert "tangent workspace needs" in msg and "bytes" in msg
    assert len(leaves(big)) == 489


def test_tangent_block_refusals(small):
    """NetworkPlan._tangent_block checks every tangent before anything reaches the device"""
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn, path = small
    lv = leaves(tn)
    p = NetworkPlan.__new__(NetworkPlan)
    p.handle = plan(tn, path, wrt=[0, 3])
    p.ctx = types.SimpleNamespace(_l=_lib(), device=0)
    p.leaf_shapes = [tuple(int(d) for d in l.bond_dims) for l in lv]
    try:
        with pytest.raises(ValueError, match="not requested"):
            p._tangent_block({1: np.zeros(p.leaf_shapes[1])})
        with pytest.raises(IndexError):
            p._tangent_block({len(lv): np.zeros(2)})
        with pytest.raises(ValueError, match="shape"):
            p._tangent_block({0: np.zeros(p.leaf_shapes[0] + (1,))})
        with pytest.raises(ValueError, match="shape"):
            p._tangent_block({3: np.zeros((4,) + p.leaf_shapes[3])}, count=3)
    finally:
        _lib().tncb_plan_destroy(p.handle)
        p.handle = None


def test_network_function_sliced_forward_mode_refused():
    """forward mode through a sliced network_function: NotImplementedError, before any device work"""
    torch = pytest.importorskip("torch")
    from tnc_b200.autograd import NetworkFunction
    f = NetworkFunction.__new__(NetworkFunction)
    f.sliced = True
    with pytest.raises(NotImplementedError, match="sliced_legs"):
        f._jvp((torch.zeros(2),), (torch.ones(2),), ((), torch.device("cpu")))
