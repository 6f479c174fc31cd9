"""Sliced tangent and Hessian-vector plans compiled without a device (tncb_plan_create_jvp_sliced / _hvp_sliced with a
NULL context): one slice's schedule and workspace are those of a tangent / Hessian-vector plan of the host-sliced slice
network, the offsets pack the full leaves' shapes, the refusals, and bench.py's network past the memory wall."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_UNSUPPORTED = -1, -2, -9
KINDS = ["jvp", "hvp"]
NOUN = {"vjp": "gradient", "jvp": "tangent", "hvp": "Hessian-vector"}
# the committed depth-12 tree: its 9-leg gradient set plus one more leg from find_slices (max_peak_elements = 2^26)
D12_HVP_LEGS = [157, 1115, 231, 606, 1084, 986, 1088, 155, 515, 424]


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


def create(kind, tn, path, wrt=None):
    """(status, handle) of a host-only unsliced plan of `kind` ("plain", "vjp", "jvp" or "hvp")"""
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if kind == "plain":
        return _lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)), h
    return getattr(_lib(), f"tncb_plan_create_{kind}")(None, C.byref(ct), C.byref(cp), _mask(tn, wrt), C.byref(h)), h


def create_sliced(kind, tn, path, legs, wrt=None):
    from tnc_b200._lib import u64_array
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    arr = u64_array(list(legs) or [0])
    return getattr(_lib(), f"tncb_plan_create_{kind}_sliced")(None, C.byref(ct), C.byref(cp), len(legs), arr,
                                                              _mask(tn, wrt), C.byref(h)), h


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


def check_matches_host_sliced(kind, tn, path, legs):
    """pairs, flops, bytes and per-slice workspace equal the unsliced plan of the host-sliced first and last slices.
    Kernels: the tangent extract replaces the tangent staging, the G / Ġ accumulates replace the G / Ġ gathers, and the
    extract of the leaves with a sliced leg is the one extra launch"""
    from tnc_b200.contractionpath.slicing import SlicedNetwork
    hs = ok(create_sliced(kind, tn, path, legs))
    got = info(hs)
    sn = SlicedNetwork(tn, legs)
    assert len(sn.assignments) == 2 ** len(legs)
    for a in (sn.assignments[0], sn.assignments[-1]):
        h = ok(create(kind, sn.slice(a), path))
        want = info(h)
        destroy(h)
        assert (got["pairs"], got["flops"], got["bytes"], got["peak_bytes"]) == \
            (want["pairs"], want["flops"], want["bytes"], want["peak_bytes"]), (kind, legs, a, got, want)
        assert got["kernels"] == want["kernels"] + 1, (got, want)
    destroy(hs)
    return got


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n_legs", [1, 2, 3])
def test_q12_matches_host_sliced(q12, kind, n_legs):
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = q12
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert len(legs) == n_legs
    check_matches_host_sliced(kind, tn, path, legs)


# per-slice workspace of bench.py's network with every leaf requested, bytes (unsliced: 23476130560 / 36487643136)
BENCH_PEAK = {"jvp": {1: 12865060352, 2: 6221283072, 3: 3704689408},
              "hvp": {1: 18775095552, 2: 10248070144, 3: 5852428288}}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n_legs", [1, 2, 3])
def test_bench_matches_host_sliced(bench_net, kind, n_legs):
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = bench_net
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert legs == [149, 156, 160][:n_legs]
    got = check_matches_host_sliced(kind, tn, path, legs)
    assert got["peak_bytes"] == BENCH_PEAK[kind][n_legs]


@pytest.mark.parametrize("kind", KINDS)
def test_zero_legs_is_the_unsliced_plan(q12, kind):
    from tnc_b200.tensornetwork import leaves
    tn, path = q12
    n = len(leaves(tn))
    for wrt in (None, [2, 7]):
        a, b = ok(create(kind, tn, path, wrt)), ok(create_sliced(kind, tn, path, [], wrt))
        ia, ib = info(a), info(b)
        assert ia == ib, (ia, ib)          # no sliced leaf: no extract launch; extract / accumulate replace stage / gather
        assert offsets(a, n) == offsets(b, n)
        destroy(a, b)


@pytest.mark.parametrize("kind", KINDS)
def test_offsets_pack_full_leaves(q12, kind):
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    tn, path = q12
    lv = leaves(tn)
    legs = find_slices(tn, path, min_slices=4)
    full = [int(np.prod(l.bond_dims)) for l in lv]
    h = ok(create_sliced(kind, tn, path, legs))
    assert offsets(h, len(lv)) == list(np.cumsum([0] + full[:-1]))
    destroy(h)
    want = [0, 3, len(lv) - 1] + [i for i, l in enumerate(lv) if set(l.legs) & set(legs)][:2]
    h = ok(create_sliced(kind, tn, path, legs, wrt=want))
    offs, pos = offsets(h, len(lv)), 0
    for i in range(len(lv)):
        if i in want:
            assert offs[i] == pos, i
            pos += full[i]
        else:
            assert offs[i] == -1, i
    # the same packing as a sliced gradient plan with the same wrt
    g = ok(create_sliced("vjp", tn, path, legs, wrt=want))
    assert offsets(g, len(lv)) == offs
    destroy(h, g)


@pytest.mark.parametrize("kind", KINDS)
def test_creation_refusals(q12, bench_net, kind, monkeypatch):
    """the sliced-leg checks of tncb_plan_create_vjp_sliced with its messages, the plan kind's own refusals, and the
    per-slice workspace limit naming the bytes"""
    from tnc_b200 import DeviceTensor
    from tnc_b200.builders import random_circuit_builder
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

    def refused(legs, status, words, wrt=None, net=tn, p=path, k=kind):
        rc, _ = create_sliced(k, net, p, legs, wrt)
        msg = _lib().tncb_last_error().decode()
        assert rc == status, (legs, rc, msg)
        assert words in msg, msg
        return msg

    # byte for byte the sliced gradient plan's messages
    for k in ("vjp", kind):
        assert refused([absent], ERR_INVALID, "does not occur", k=k) == f"sliced leg {absent} does not occur in the network"
        assert refused([inner[0], inner[1], inner[0]], ERR_INVALID, "listed twice", k=k) == f"sliced leg {inner[0]} is listed twice"
        assert refused(inner[:64], ERR_INVALID, "overflows", k=k) == "the slice count overflows 64 bits"
    sv, _ = random_circuit_builder(6, 2, 0.5, 0.5, np.random.default_rng(1)).into_statevector_network()
    sv_count = {}
    for l in leaves(sv):
        for x in l.legs:
            sv_count[x] = sv_count.get(x, 0) + 1
    open_leg = next(x for x, c in sv_count.items() if c == 1)
    sv_inner = next(x for x, c in sv_count.items() if c == 2)
    assert refused([sv_inner, open_leg], ERR_INVALID, "open leg", net=sv, p=greedy(sv)) == \
        f"sliced leg {open_leg} occurs once: it is an open leg of the result"
    a, b = Tensor([0, 1], [2, 0]), Tensor([1, 0], [0, 2])           # a leg of dimension 0
    for t in (a, b):
        t.set_tensor_data(TensorData.Matrix(np.zeros(t.bond_dims)))
    refused([1], ERR_INVALID, "sliced leg 1 has dimension 0", net=Tensor.new_composite([a, b]), p=ContractionPath.simple([(0, 1)]))
    refused([inner[0]], ERR_INVALID, "selects no leaf", wrt=[])
    one = Tensor([0, 1], [2, 2])
    one.set_tensor_data(TensorData.Matrix(np.eye(2)))
    refused([], ERR_UNSUPPORTED, "at least one pair", net=Tensor.new_composite([one]), p=ContractionPath.simple([]))
    fake = DeviceTensor.__new__(DeviceTensor)
    fake.handle, fake.shape, fake.ctx = C.c_void_p(0x1000), tuple(lv[1].bond_dims), None
    t = Tensor(lv[1].legs, lv[1].bond_dims)
    t.set_tensor_data(TensorData.Matrix(fake))
    parts = list(tn.tensors)
    parts[1] = t
    assert refused([inner[0]], ERR_UNSUPPORTED, "device leaves", net=Tensor.new_composite(parts)) == \
        f"{NOUN[kind]} plans do not take device leaves (they are consumed per call)"
    fake.handle = None
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    big, big_path = bench_net
    need = BENCH_PEAK[kind][3]
    assert refused([149, 156, 160], ERR_UNSUPPORTED, "static-workspace limit", net=big, p=big_path) == \
        f"the {NOUN[kind]} workspace of one slice needs {need} bytes, above the static-workspace limit of {1 << 30} bytes (TNCB_PLAN_WS_GB)"


@pytest.mark.parametrize("kind", KINDS)
def test_leaf_with_too_many_sliced_legs(built_lib, kind):
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
    rc, _ = create_sliced(kind, tn, path, legs[:9])
    assert rc == ERR_UNSUPPORTED and "carries more than 8 sliced legs" in _lib().tncb_last_error().decode()
    destroy(ok(create_sliced(kind, tn, path, legs[:8])))


def test_refusals_between_plan_kinds(q12):
    """every entry point but stage / run_slices / info / grad_offsets refuses the new plans naming their call, before
    the context is used (a zeroed block stands in for it); the _sliced calls refuse every other plan kind"""
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    from tnc_b200.tensornetwork.contraction import _Marshal
    import tnc_b200 as tb
    tn, path = q12
    legs = find_slices(tn, path, min_slices=4)
    l = _lib()
    fake_ctx = C.create_string_buffer(1 << 16)
    cx = C.cast(fake_ctx, C.c_void_p)
    m = _Marshal()
    node = m.tn(tn)
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(node))
    out, n_out, legs_out, g = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)(), C.c_void_p()
    t = C.c_void_p(0x1000)                                      # never read: the plan kind is refused first
    idx, src = (C.c_uint64 * 1)(0), (C.c_void_p * 1)(0x1000)
    calls = {
        "run": lambda p: l.tncb_plan_run(cx, p, C.byref(out), C.byref(n_out), legs_out),
        "execute": lambda p: l.tncb_plan_execute(cx, p, C.byref(node), C.byref(out), C.byref(n_out), legs_out),
        "stage_slices": lambda p: l.tncb_plan_stage_slices(cx, p, 1, ptrs),
        "run_batch": lambda p: l.tncb_plan_run_batch(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs_out),
        "vjp": lambda p: l.tncb_plan_vjp(cx, p, None, C.byref(g)),
        "vjp_sliced": lambda p: l.tncb_plan_vjp_sliced(cx, p, 0, 1, None, C.byref(out), C.byref(g)),
        "stage_batch": lambda p: l.tncb_plan_stage_batch(cx, p, 1, ptrs),
        "vjp_batch": lambda p: l.tncb_plan_vjp_batch(cx, p, 0, 1, None, C.byref(out), None, None),
        "jvp": lambda p: l.tncb_plan_jvp(cx, p, t, C.byref(out), None),
        "jvp_batch": lambda p: l.tncb_plan_jvp_batch(cx, p, 0, 1, t, C.byref(out), None),
        "hvp": lambda p: l.tncb_plan_hvp(cx, p, t, None, None, C.byref(out), None, None, None),
        "stage_instances": lambda p: l.tncb_plan_stage_instances(cx, p, C.byref(node), 1, 0, None, None, None),
        "set_leaves": lambda p: l.tncb_plan_set_leaves(cx, p, 1, idx, src),
    }
    jvp_sliced = lambda p: l.tncb_plan_jvp_sliced(cx, p, 0, 1, t, C.byref(out), None)
    hvp_sliced = lambda p: l.tncb_plan_hvp_sliced(cx, p, 0, 1, t, None, None, C.byref(out), None, None, None)
    plans = {k: ok(create_sliced(k, tn, path, legs)) for k in ("vjp", "jvp", "hvp")}
    for k in ("plain", "vjp", "jvp", "hvp"):
        plans["unsliced " + k] = ok(create(k, tn, path))
    for kind, name in (("jvp", "tncb_plan_jvp_sliced"), ("hvp", "tncb_plan_hvp_sliced")):
        for call_name, call in calls.items():
            assert call(plans[kind]) == ERR_UNSUPPORTED, (kind, call_name, l.tncb_last_error())
            msg = l.tncb_last_error().decode()
            assert msg == f"a sliced {NOUN[kind]} plan runs through {name} / tncb_plan_run_slices", (call_name, msg)
    # the _sliced calls take their own plan kind only
    for k, h in plans.items():
        if k != "jvp":
            assert jvp_sliced(h) == ERR_INVALID, k
            assert l.tncb_last_error().decode() == "not a sliced tangent plan (tncb_plan_create_jvp_sliced)"
        if k != "hvp":
            assert hvp_sliced(h) == ERR_INVALID, k
            assert l.tncb_last_error().decode() == "not a sliced Hessian-vector plan (tncb_plan_create_hvp_sliced)"
    # their own plan, but nothing staged on this context: a tensor header with the tangent block's dims stands in for
    # the tangents (its storage is never read); a wrong tangent size; stride 0
    class Header(C.Structure):
        _fields_ = [("ptr", C.c_void_p), ("rank", C.c_int), ("dims", C.c_uint64 * 64)]
    lvs = leaves(tn)
    n_leaves = len(lvs)
    for k in ("jvp", "hvp"):
        hd = Header(0x1000, 1)
        hd.dims[0] = sum(int(np.prod(lf.bond_dims)) for lf in lvs)
        assert offsets(plans[k], n_leaves)[-1] + int(np.prod(lvs[-1].bond_dims)) == hd.dims[0]
        ht = C.cast(C.pointer(hd), C.c_void_p)
        rc = (l.tncb_plan_jvp_sliced(cx, plans[k], 0, 1, ht, C.byref(out), None) if k == "jvp" else
              l.tncb_plan_hvp_sliced(cx, plans[k], 0, 1, ht, None, None, C.byref(out), None, None, None))
        assert rc == ERR_INVALID and "tncb_plan_stage has not been called" in l.tncb_last_error().decode()
        hd.dims[0] -= 1
        rc = (l.tncb_plan_jvp_sliced(cx, plans[k], 0, 1, ht, C.byref(out), None) if k == "jvp" else
              l.tncb_plan_hvp_sliced(cx, plans[k], 0, 1, ht, None, None, C.byref(out), None, None, None))
        assert rc == ERR_SHAPE and "the tangents' dims differ" in l.tncb_last_error().decode()
    assert l.tncb_plan_jvp_sliced(cx, plans["jvp"], 0, 0, t, C.byref(out), None) == ERR_INVALID
    assert l.tncb_plan_jvp_sliced(cx, plans["jvp"], 0, 1, t, None, None) == ERR_INVALID        # no output
    assert "no output requested" in l.tncb_last_error().decode()
    assert l.tncb_plan_hvp_sliced(cx, plans["hvp"], 0, 1, None, None, None, C.byref(out), None, None, None) == ERR_INVALID
    assert "tangents are needed" in l.tncb_last_error().decode()
    # run_slices takes them (and asks for staging here)
    for k in ("jvp", "hvp"):
        assert l.tncb_plan_run_slices(cx, plans[k], 0, 1, C.byref(out), C.byref(n_out), legs_out) == ERR_INVALID
        assert "tncb_plan_stage has not been called" in l.tncb_last_error().decode()
    # the existing plan kinds keep their messages
    assert calls["run"](plans["vjp"]) == ERR_UNSUPPORTED
    assert l.tncb_last_error().decode() == "a sliced gradient plan runs through tncb_plan_run_slices / tncb_plan_vjp_sliced"
    assert calls["jvp"](plans["unsliced hvp"]) == ERR_UNSUPPORTED
    assert l.tncb_last_error().decode() == "a Hessian-vector plan runs through tncb_plan_hvp"
    destroy(*plans.values())


def test_memory_wall(bench_net, monkeypatch):
    """at TNCB_PLAN_WS_GB=20 bench.py's network (36.49 GB) has no Hessian-vector plan, but a 2-leg sliced one
    (10.25 GB per slice); likewise at 12 GB for tangents (23.48 GB unsliced, 6.22 GB per slice)"""
    tn, path = bench_net
    for kind, gb in (("hvp", 20), ("jvp", 12)):
        monkeypatch.setenv("TNCB_PLAN_WS_GB", str(gb))
        rc, _ = create(kind, tn, path)
        assert rc == ERR_UNSUPPORTED and "static-workspace limit" in _lib().tncb_last_error().decode()
        h = ok(create_sliced(kind, tn, path, [149, 156]))
        assert info(h)["peak_bytes"] == BENCH_PEAK[kind][2] <= gb << 30
        destroy(h)


def test_sycamore_d12_hvp_legs(built_lib):
    """the committed depth-12 tree: the 9 legs that fit its sliced gradient leave a 61.2 GB Hessian-vector slice
    (refused at 46 GiB); one more leg from find_slices gives 1024 slices of 33.0 GB each"""
    from tnc_b200.builders import sycamore_circuit
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.contractionpath.slicing import find_slices, slice_assignments
    with open(os.path.join(ROOT, "bench_inputs", "sycamore53_d12.json")) as f:
        d = json.load(f)
    tn = sycamore_circuit(53, 12, np.random.default_rng(1)).into_amplitude_network("0" * 53)[0]
    path = ContractionPath.simple([tuple(x) for x in d["toplevel"]])
    rc, _ = create_sliced("hvp", tn, path, D12_HVP_LEGS[:9])
    assert rc == ERR_UNSUPPORTED and "needs 61237166080 bytes" in _lib().tncb_last_error().decode()
    assert find_slices(tn, path, max_peak_elements=2 ** 26) == D12_HVP_LEGS
    h = ok(create_sliced("hvp", tn, path, D12_HVP_LEGS))
    got = info(h)
    assert got["peak_bytes"] == 33017808896 <= 46 << 30, got
    assert len(slice_assignments(tn, D12_HVP_LEGS)) == 1024
    destroy(h)


@pytest.mark.parametrize("name", ["tncb_plan_create_jvp_sliced", "tncb_plan_jvp_sliced", "tncb_plan_create_hvp_sliced",
                                  "tncb_plan_hvp_sliced"])
def test_signatures_match_header(name):
    import re
    from tnc_b200._lib import SIGNATURES, TncbPath, TncbTn, u64p, vpp
    ctypes_of = {"tncb_ctx*": C.c_void_p, "tncb_plan*": C.c_void_p, "const tncb_tn*": C.POINTER(TncbTn),
                 "const tncb_path*": C.POINTER(TncbPath), "const uint8_t*": C.POINTER(C.c_uint8), "tncb_plan**": vpp,
                 "const tncb_tensor*": C.c_void_p, "tncb_tensor**": vpp, "size_t": C.c_size_t, "const uint64_t*": u64p}
    with open(os.path.join(ROOT, "include", "tncb.h")) as f:
        text = f.read()
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    params = [re.sub(r"\s*\w+$", "", " ".join(p.split())).replace(" *", "*") for p in m.group(1).split(",")]
    res, args = SIGNATURES[name]
    assert res is C.c_int
    assert args == [ctypes_of[p] for p in params], (args, params)
