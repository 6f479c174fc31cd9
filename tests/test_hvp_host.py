"""Hessian-vector plans compiled without a device (tncb_plan_create_hvp with a NULL context): the forward, tangent,
backward and backward-tangent pairs on top of one another, the gradient offsets, the pinned layouts of the other plan
kinds, and the refusals between plan kinds that happen before any device work."""
import ctypes as C
import os
import re
import sys

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


CREATE = {"hvp": "tncb_plan_create_hvp", "jvp": "tncb_plan_create_jvp", "vjp": "tncb_plan_create_vjp"}


def create(tn, path, wrt=None, kind="hvp"):
    """(status, handle) of a host-only plan: kind = "hvp", "jvp", "vjp" or "plain"; wrt = leaf indices or None"""
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if kind == "plain":
        return _lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)), h
    return getattr(_lib(), CREATE[kind])(None, C.byref(ct), C.byref(cp), mask_of(tn, wrt), C.byref(h)), h


class Plan:
    """a host-only plan handle, destroyed with the object"""

    def __init__(self, tn, path, wrt=None, kind="hvp"):
        rc, self.h = create(tn, path, wrt, kind)
        assert rc == 0, _lib().tncb_last_error()

    def __del__(self):
        if self.h:
            _lib().tncb_plan_destroy(self.h)

    def info(self):
        n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
        fl, by = C.c_double(), C.c_double()
        assert _lib().tncb_plan_info(self.h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
        return {"pairs": n.value, "flops": fl.value, "peak_bytes": pk.value, "kernels": k.value}

    def offsets(self, n):
        arr = (C.c_int64 * n)()
        assert _lib().tncb_plan_grad_offsets(self.h, arr) == 0
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


def forward_sides(tn, path, wrt):
    """per forward pair of the replace-left path: (s, M N K), s = the number of operands whose subtree holds a requested
    leaf"""
    from tnc_b200.tensornetwork import leaves
    counter = [0]
    want = set(wrt)
    pairs = []

    def walk(t, p):
        if not t.tensors:
            counter[0] += 1
            return {counter[0] - 1}, list(t.legs), dict(zip(t.legs, t.bond_dims))
        slots = []
        for i, c in enumerate(t.tensors):
            if c.tensors and (p is None or i not in p.nested):
                counter[0] += len(leaves(c))
                slots.append(None)
                continue
            slots.append(walk(c, p.nested.get(i) if p is not None and c.tensors else None))
        for i, j in (p.toplevel if p is not None else []):
            (sa, la, da), (sb, lb, db) = slots[i], slots[j]
            dims = da | db
            out = [l for l in lb if l not in la] + [l for l in la if l not in lb]
            mnk = float(np.prod([dims[l] for l in set(la) | set(lb)], dtype=np.float64))
            pairs.append((int(bool(sa & want)) + int(bool(sb & want)), mnk))
            slots[i], slots[j] = (sa | sb, out, dims), None
        return next(s for s in slots if s is not None)
    walk(tn, path)
    return pairs


def expected(tn, path, wrt):
    """(pairs, flops, sums) of a Hessian-vector plan: a forward pair with s sided operands gets s tangent pairs, s
    backward pairs and s * s backward-tangent pairs (each backward pair: dC̄·O, plus C̄·dO when O has a tangent), all of
    its M N K; a two-sided pair adds one tangent sum and two backward-tangent sums"""
    fs = forward_sides(tn, path, wrt)
    pairs = sum((1 + s) ** 2 for s, _ in fs)
    flops = sum(8.0 * mnk * (1 + s) ** 2 for s, mnk in fs)
    sums = 3 * sum(1 for s, _ in fs if s == 2)
    return pairs, flops, sums


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
CTYPES = {"tncb_ctx*": C.c_void_p, "tncb_plan*": C.c_void_p, "const tncb_tn*": "tn*", "const tncb_path*": "path*",
          "const uint8_t*": "u8p", "tncb_plan**": "vpp", "const tncb_tensor*": C.c_void_p, "tncb_tensor**": "vpp"}


def header_params(name):
    with open(os.path.join(ROOT, "include", "tncb.h")) as f:
        text = f.read()
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\w+$", "", p).replace(" *", "*") for p in params]


@pytest.mark.parametrize("name", ["tncb_plan_create_hvp", "tncb_plan_hvp"])
def test_signatures_match_header(name):
    from tnc_b200._lib import SIGNATURES, TncbPath, TncbTn, vpp
    resolve = {"vpp": vpp, "tn*": C.POINTER(TncbTn), "path*": C.POINTER(TncbPath), "u8p": C.POINTER(C.c_uint8)}
    want = [resolve.get(CTYPES[p], CTYPES[p]) for p in header_params(name)]
    res, args = SIGNATURES[name]
    assert res is C.c_int
    assert args == want, (args, want)


def test_expected_counts_model():
    """the count model: every leaf requested on a tree of F pairs gives 9 F pairs and 3 F sums"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    a, b, c = Tensor([0, 1], [2, 3]), Tensor([1, 2], [3, 4]), Tensor([2, 5], [4, 2])
    for t in (a, b, c):
        t.set_tensor_data(TensorData.Matrix(np.ones(t.bond_dims)))
    tn = Tensor.new_composite([a, b, c])
    path = ContractionPath.simple([(0, 1), (0, 2)])
    assert expected(tn, path, [0, 1, 2]) == (18, 8.0 * 9 * (24 + 16), 6)
    assert expected(tn, path, [2]) == (1 + 4, 8.0 * (24 + 4 * 16), 0)


@pytest.mark.parametrize("net", ["small", "bench_net"])
def test_pairs_and_flops(net, request):
    """forward + tangent + backward + backward-tangent pairs and flops, with every leaf, a third of them and one leaf"""
    from tnc_b200.tensornetwork import leaves
    tn, path = request.getfixturevalue(net)
    fwd = Plan(tn, path, kind="plain").info()
    every = [i for i, l in enumerate(leaves(tn)) if l.tensordata.kind != "uncontracted"]
    for wrt in (None, every[::3], [every[0]], [every[-1]]):
        got = Plan(tn, path, wrt).info()
        pairs, flops, sums = expected(tn, path, every if wrt is None else wrt)
        assert got["pairs"] == pairs, (wrt, got, pairs)
        assert got["flops"] == pytest.approx(flops, rel=1e-12)
        if wrt is None:                              # every leaf: nine pairs of the forward volume per forward pair
            assert got["pairs"] == 9 * fwd["pairs"]
            assert got["flops"] == pytest.approx(9 * fwd["flops"], rel=1e-12)
            assert sums == 3 * fwd["pairs"]
        if wrt is not None and len(wrt) == 1:        # one leaf: one pair of each kind per ancestor step, no sums
            assert sums == 0
    if net == "bench_net":
        assert fwd["pairs"] == 488 and len(leaves(tn)) == 489


def test_offsets_equal_gradient_plan(small):
    from tnc_b200.tensornetwork import leaves
    tn, path = small
    n = len(leaves(tn))
    for wrt in (None, [1, 4, 5, n - 1], [n // 2]):
        assert Plan(tn, path, wrt).offsets(n) == Plan(tn, path, wrt, kind="vjp").offsets(n), wrt


def test_other_layouts_unchanged(bench_net):
    """bench.py's network: the plain, gradient and tangent plans keep their pairs, flops, workspace bytes and kernel
    counts from before Hessian-vector plans shared the compiler"""
    tn, path = bench_net
    assert Plan(tn, path, kind="plain").info() == {"pairs": 488, "flops": 6689291543832.0, "peak_bytes": 7248097472, "kernels": 70}
    assert Plan(tn, path, kind="vjp").info() == {"pairs": 1464, "flops": 20067874631496.0, "peak_bytes": 15244053248, "kernels": 155}
    assert Plan(tn, path, kind="jvp").info() == {"pairs": 1464, "flops": 20067874631496.0, "peak_bytes": 23476130560, "kernels": 207}


def test_hvp_workspace_pinned(bench_net):
    """bench.py's network with every leaf requested: 34 GiB of static workspace, under the 46 GiB limit of a plan
    compiled without a device (and the 0.62 share of an 80 GB H100)"""
    tn, path = bench_net
    h = Plan(tn, path).info()
    assert h == {"pairs": 4392, "flops": 60203623894488.0, "peak_bytes": 36487643136, "kernels": 443}
    assert h["peak_bytes"] <= 46 << 30


def test_creation_refusals(small, bench_net, monkeypatch):
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, path = small
    lv = list(tn.tensors)
    fake = DeviceTensor.__new__(DeviceTensor)                  # a device leaf: refused before its handle is read
    fake.handle, fake.shape, fake.ctx = C.c_void_p(0x1000), tuple(lv[1].bond_dims), None
    t = Tensor(lv[1].legs, lv[1].bond_dims)
    t.set_tensor_data(TensorData.Matrix(fake))
    lv[1] = t
    rc, _ = create(Tensor.new_composite(lv), path)
    fake.handle = None
    assert rc == ERR_UNSUPPORTED
    one = Tensor([0, 1], [2, 2])
    one.set_tensor_data(TensorData.Matrix(np.eye(2)))
    assert create(Tensor.new_composite([one]), ContractionPath.simple([]))[0] == ERR_UNSUPPORTED   # no pairs
    assert create(tn, path, wrt=[])[0] == ERR_INVALID
    bare = Tensor([0, 1], [2, 2])
    other = Tensor([1, 0], [2, 2])
    other.set_tensor_data(TensorData.Matrix(np.eye(2)))
    assert create(Tensor.new_composite([bare, other]), ContractionPath.simple([(0, 1)]), wrt=[0])[0] != 0
    big, big_path = bench_net
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "20")
    rc, _ = create(big, big_path)
    assert rc == ERR_UNSUPPORTED
    msg = _lib().tncb_last_error().decode()
    assert "Hessian-vector workspace needs 36487643136 bytes" in msg, msg


def test_refusals_between_plan_kinds(small):
    """every other entry point refuses a Hessian-vector plan (TNCB_ERR_UNSUPPORTED) and tncb_plan_hvp refuses the other
    plan kinds (TNCB_ERR_INVALID), before the context is used: a zeroed block stands in for it"""
    from tnc_b200.tensornetwork.contraction import _Marshal
    import tnc_b200 as tb
    tn, path = small
    l = _lib()
    fake_ctx = C.create_string_buffer(1 << 16)
    cx = C.cast(fake_ctx, C.c_void_p)
    h = Plan(tn, path)
    m = _Marshal()
    node = m.tn(tn)
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(node))
    out, n_out, legs, g = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)(), C.c_void_p()
    t = C.c_void_p(0x1000)                                      # never read: the plan kind is refused first
    calls = {
        "run": lambda p: l.tncb_plan_run(cx, p, C.byref(out), C.byref(n_out), legs),
        "execute": lambda p: l.tncb_plan_execute(cx, p, C.byref(node), C.byref(out), C.byref(n_out), legs),
        "stage_slices": lambda p: l.tncb_plan_stage_slices(cx, p, 1, ptrs),
        "run_slices": lambda p: l.tncb_plan_run_slices(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs),
        "run_batch": lambda p: l.tncb_plan_run_batch(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs),
        "vjp": lambda p: l.tncb_plan_vjp(cx, p, None, C.byref(g)),
        "vjp_sliced": lambda p: l.tncb_plan_vjp_sliced(cx, p, 0, 1, None, C.byref(out), C.byref(g)),
        "stage_batch": lambda p: l.tncb_plan_stage_batch(cx, p, 1, ptrs),
        "vjp_batch": lambda p: l.tncb_plan_vjp_batch(cx, p, 0, 1, None, C.byref(out), None, None),
        "jvp": lambda p: l.tncb_plan_jvp(cx, p, t, C.byref(out), None),
        "jvp_batch": lambda p: l.tncb_plan_jvp_batch(cx, p, 0, 1, t, C.byref(out), None),
        "stage_instances": lambda p: l.tncb_plan_stage_instances(cx, p, C.byref(node), 1, 0, None, None, None),
    }
    for name, call in calls.items():
        assert call(h.h) == ERR_UNSUPPORTED, (name, l.tncb_last_error())
        assert "tncb_plan_hvp" in l.tncb_last_error().decode(), name
    for kind in ("plain", "vjp", "jvp"):
        p = Plan(tn, path, kind=kind)
        rc = l.tncb_plan_hvp(cx, p.h, t, None, None, C.byref(out), None, None, None)
        assert rc == ERR_INVALID, (kind, l.tncb_last_error())
        assert "not a Hessian-vector plan" in l.tncb_last_error().decode()
