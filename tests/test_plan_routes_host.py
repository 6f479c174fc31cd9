"""Which call takes which plan kind, without a GPU: all 19 plan-taking calls on host-only plans of all 7 kinds, with a
zeroed block standing in for the context, against the kind x call table of include/tncb.h; and what the creators of the
six derivative kinds answer (device leaves, the static-workspace limit) and compile (tncb_plan_info, gradient offsets)."""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_UNSUPPORTED = -1, -2, -9
KINDS = ["plain", "vjp", "jvp", "hvp", "sliced vjp", "sliced jvp", "sliced hvp"]
NOUN = {"vjp": "gradient", "jvp": "tangent", "hvp": "Hessian-vector"}
ACCEPTED = "accepted"       # passes the kind check and goes on to use the context: not called with a fake one

HVP = (ERR_UNSUPPORTED, "a Hessian-vector plan runs through tncb_plan_hvp")
SJ = (ERR_UNSUPPORTED, "a sliced tangent plan runs through tncb_plan_jvp_sliced / tncb_plan_run_slices")
SH = (ERR_UNSUPPORTED, "a sliced Hessian-vector plan runs through tncb_plan_hvp_sliced / tncb_plan_run_slices")
SV_RUN = (ERR_UNSUPPORTED, "a sliced gradient plan runs through tncb_plan_run_slices / tncb_plan_vjp_sliced")
SV_NO_BATCH = (ERR_UNSUPPORTED, "a sliced gradient plan has no batched gradients")
TAN_JVP = (ERR_UNSUPPORTED, "a tangent plan runs through tncb_plan_jvp")
TAN_BATCH = (ERR_UNSUPPORTED, "a tangent plan runs through tncb_plan_jvp_batch")
GRAD_ONE = (ERR_UNSUPPORTED, "gradient plans run one staged network at a time")
NOT_GRAD = (ERR_INVALID, "not a gradient plan (tncb_plan_create_vjp)")
NOT_TAN = (ERR_INVALID, "not a tangent plan (tncb_plan_create_jvp)")
NOT_HVP = (ERR_INVALID, "not a Hessian-vector plan (tncb_plan_create_hvp)")
NOT_SJ = (ERR_INVALID, "not a sliced tangent plan (tncb_plan_create_jvp_sliced)")
NOT_SH = (ERR_INVALID, "not a sliced Hessian-vector plan (tncb_plan_create_hvp_sliced)")
NOT_SV = (ERR_INVALID, "not a sliced gradient plan (tncb_plan_create_vjp_sliced)")
NOT_STAGED = (ERR_INVALID, "tncb_plan_stage has not been called on this context")
NOT_STAGED_PLAN = (ERR_INVALID, "tncb_plan_stage has not been called on this plan and context")
TANGENTS = (ERR_SHAPE, "the tangents' dims differ from [760]")
TANGENT_ROWS = (ERR_SHAPE, "the tangents' dims differ from [1, 760]")
OK = (0, None)

# the columns are KINDS; recorded from the library before its routing became one table
ROUTES = {
    "stage": [ACCEPTED] * 7,
    "run": [NOT_STAGED, NOT_STAGED, TAN_JVP, HVP, SV_RUN, SJ, SH],
    "execute": [ACCEPTED, ACCEPTED, TAN_JVP, HVP, SV_RUN, SJ, SH],
    "stage_slices": [ACCEPTED, (ERR_UNSUPPORTED, "gradient plans run one staged network at a time"),
                     (ERR_UNSUPPORTED, "tangent plans stage many networks with tncb_plan_stage_batch"), HVP,
                     (ERR_UNSUPPORTED, "a sliced gradient plan stages its full network once (tncb_plan_stage)"), SJ, SH],
    "run_slices": [(ERR_INVALID, "tncb_plan_stage_slices has not been called on this context"), GRAD_ONE,
                   (ERR_UNSUPPORTED, "a tangent plan runs through tncb_plan_jvp / tncb_plan_jvp_batch"), HVP,
                   NOT_STAGED, NOT_STAGED, NOT_STAGED],
    "run_batch": [(ERR_INVALID, "tncb_plan_stage_slices has not been called on this context"), GRAD_ONE, TAN_BATCH, HVP,
                  SV_RUN, SJ, SH],
    "vjp": [NOT_GRAD, (ERR_INVALID, "tncb_plan_vjp needs a forward run (tncb_plan_run / tncb_plan_execute) of the plan on "
                                    "this context since its leaves were staged or its last tncb_plan_vjp"),
            TAN_JVP, HVP, (ERR_UNSUPPORTED, "a sliced gradient plan runs through tncb_plan_vjp_sliced"), SJ, SH],
    "vjp_sliced": [NOT_SV, NOT_SV, TAN_JVP, HVP, NOT_STAGED, SJ, SH],
    "stage_batch": [(ERR_INVALID, "not a gradient or tangent plan (plain plans stage many networks with tncb_plan_stage_slices)"),
                    ACCEPTED, ACCEPTED, HVP, SV_NO_BATCH, SJ, SH],
    "vjp_batch": [NOT_GRAD, (ERR_INVALID, "tncb_plan_stage_batch has not been called on this context"), TAN_BATCH, HVP,
                  SV_NO_BATCH, SJ, SH],
    "jvp": [NOT_TAN, NOT_TAN, TANGENTS, HVP, NOT_TAN, SJ, SH],
    "jvp_batch": [NOT_TAN, NOT_TAN,
                  (ERR_INVALID, "tncb_plan_stage_batch / tncb_plan_stage_instances has not been called on this context"),
                  HVP, NOT_TAN, SJ, SH],
    "jvp_sliced": [NOT_SJ] * 5 + [TANGENTS, NOT_SJ],
    "hvp": [NOT_HVP] * 3 + [TANGENTS, NOT_HVP, SJ, SH],
    "hvp_batch": [NOT_HVP] * 3 + [TANGENT_ROWS, NOT_HVP, SJ, SH],
    "hvp_sliced": [NOT_SH] * 6 + [TANGENTS],
    "stage_instances": [ACCEPTED, ACCEPTED, ACCEPTED, HVP,
                        (ERR_UNSUPPORTED, "a sliced gradient plan takes device payloads through tncb_plan_set_leaves"), SJ, SH],
    "set_leaves": [NOT_STAGED_PLAN] * 5 + [SJ, SH],
    "grad_offsets": [(ERR_INVALID, "not a gradient or tangent plan (tncb_plan_create_vjp / _jvp)")] + [OK] * 6,
}


def _lib():
    from tnc_b200._lib import lib
    return lib()


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def amplitude(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def create(kind, tn, path, legs=None):
    """(status, handle) of a host-only plan of `kind` ("plain", "vjp", "jvp", "hvp", or one of the last three sliced on
    `legs`)"""
    from tnc_b200._lib import u64_array
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if kind == "plain":
        return _lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)), h
    if kind.startswith("sliced "):
        return getattr(_lib(), f"tncb_plan_create_{kind[7:]}_sliced")(None, C.byref(ct), C.byref(cp), len(legs),
                                                                       u64_array(list(legs)), None, C.byref(h)), h
    return getattr(_lib(), f"tncb_plan_create_{kind}")(None, C.byref(ct), C.byref(cp), None, C.byref(h)), h


def ok(rc_h):
    rc, h = rc_h
    assert rc == 0, _lib().tncb_last_error()
    return h


def info(h):
    n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fl, by = C.c_double(), C.c_double()
    assert _lib().tncb_plan_info(h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
    return (n.value, fl.value, by.value, pk.value, k.value)


def offsets_digest(h, n):
    """(count, sha256 prefix) of the plan's gradient offsets as little-endian int64"""
    arr = (C.c_int64 * n)()
    assert _lib().tncb_plan_grad_offsets(h, arr) == 0
    return n, hashlib.sha256(np.array(list(arr), dtype="<i8").tobytes()).hexdigest()[:16]


@pytest.fixture(scope="module")
def q12(built_lib):
    from tnc_b200.contractionpath.slicing import find_slices
    tn = amplitude(12, 6, 5)
    path = greedy(tn)
    return tn, path, find_slices(tn, path, min_slices=4)


@pytest.fixture(scope="module")
def bench_net(built_lib):
    sys.path.insert(0, ROOT)
    import bench
    tn = bench.build_network()
    return tn, bench.greedy_path(tn), [149, 156]


def route_matrix(tn, path, legs):
    """{call: [per kind: ACCEPTED, or (status, message)]}; ACCEPTED cells are not called"""
    from tnc_b200.tensornetwork.contraction import _Marshal
    import tnc_b200 as tb
    l = _lib()
    fake_ctx = C.create_string_buffer(1 << 16)
    cx = C.cast(fake_ctx, C.c_void_p)
    m = _Marshal()
    node = m.tn(tn)
    ptrs = (C.POINTER(tb._lib.TncbTn) * 1)(C.pointer(node))
    out, n_out, legs_out, g = C.c_void_p(), C.c_int(), (C.c_uint64 * 64)(), C.c_void_p()

    class Header(C.Structure):   # the head of a tncb_tensor: a rank-1 tangent block of 1 element fits no plan here
        _fields_ = [("ptr", C.c_void_p), ("rank", C.c_int), ("dims", C.c_uint64 * 64)]
    hd = Header(0x1000, 1)
    hd.dims[0] = 1
    t = C.cast(C.pointer(hd), C.c_void_p)
    idx, src = (C.c_uint64 * 1)(0), (C.c_void_p * 1)(0x1000)
    offs = (C.c_int64 * 4096)()
    calls = {
        "stage": lambda p: l.tncb_plan_stage(cx, p, C.byref(node)),
        "run": lambda p: l.tncb_plan_run(cx, p, C.byref(out), C.byref(n_out), legs_out),
        "execute": lambda p: l.tncb_plan_execute(cx, p, C.byref(node), C.byref(out), C.byref(n_out), legs_out),
        "stage_slices": lambda p: l.tncb_plan_stage_slices(cx, p, 1, ptrs),
        "run_slices": lambda p: l.tncb_plan_run_slices(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs_out),
        "run_batch": lambda p: l.tncb_plan_run_batch(cx, p, 0, 1, C.byref(out), C.byref(n_out), legs_out),
        "vjp": lambda p: l.tncb_plan_vjp(cx, p, None, C.byref(g)),
        "vjp_sliced": lambda p: l.tncb_plan_vjp_sliced(cx, p, 0, 1, None, C.byref(out), C.byref(g)),
        "stage_batch": lambda p: l.tncb_plan_stage_batch(cx, p, 1, ptrs),
        "vjp_batch": lambda p: l.tncb_plan_vjp_batch(cx, p, 0, 1, None, C.byref(out), None, None),
        "jvp": lambda p: l.tncb_plan_jvp(cx, p, t, C.byref(out), None),
        "jvp_batch": lambda p: l.tncb_plan_jvp_batch(cx, p, 0, 1, t, C.byref(out), None),
        "jvp_sliced": lambda p: l.tncb_plan_jvp_sliced(cx, p, 0, 1, t, C.byref(out), None),
        "hvp": lambda p: l.tncb_plan_hvp(cx, p, t, None, None, C.byref(out), None, None, None),
        "hvp_batch": lambda p: l.tncb_plan_hvp_batch(cx, p, 1, 0, None, None, None, t, None, None, C.byref(out),
                                                     None, None, None, None, None),
        "hvp_sliced": lambda p: l.tncb_plan_hvp_sliced(cx, p, 0, 1, t, None, None, C.byref(out), None, None, None),
        "stage_instances": lambda p: l.tncb_plan_stage_instances(cx, p, C.byref(node), 1, 0, None, None, None),
        "set_leaves": lambda p: l.tncb_plan_set_leaves(cx, p, 1, idx, src),
        "grad_offsets": lambda p: l.tncb_plan_grad_offsets(p, offs),
    }
    plans = [ok(create(k, tn, path, legs)) for k in KINDS]
    got = {}
    for name, call in calls.items():
        got[name] = []
        for k, p in zip(KINDS, plans):
            if ROUTES[name][KINDS.index(k)] == ACCEPTED:
                got[name].append(ACCEPTED)
                continue
            rc = call(p)
            got[name].append((rc, l.tncb_last_error().decode() if rc else None))
    for p in plans:
        l.tncb_plan_destroy(p)
    return got


def test_routes(q12):
    """every cell of the kind x call matrix: the exact status and message, or accepted"""
    got = route_matrix(*q12)
    assert list(got) == list(ROUTES)
    for name in ROUTES:
        for k, want, have in zip(KINDS, ROUTES[name], got[name]):
            assert have == want, (name, k, have, want)
    cells = [c for row in ROUTES.values() for c in row]
    assert len(cells) == 133 and cells.count(ACCEPTED) == 15


# (pairs, flops, bytes, peak bytes, kernels) of each kind with every leaf requested, and the (count, digest) of its
# gradient offsets; sliced on q12's find_slices(min_slices=4) legs and on [149, 156] for bench.py's network
INFO = {
    "q12": {"plain": (90, 88536.0, 95824.0, 25472, 15),
            "vjp": (270, 265608.0, 287472.0, 67072, 31),
            "jvp": (270, 265608.0, 287472.0, 67072, 31),
            "hvp": (810, 796824.0, 862416.0, 145408, 63),
            "sliced vjp": (270, 140232.0, 208368.0, 49152, 32),
            "sliced jvp": (270, 140232.0, 208368.0, 63488, 32),
            "sliced hvp": (810, 420696.0, 625104.0, 113152, 64)},
    "bench": {"plain": (488, 6689291543832.0, 19749401616.0, 7248097472, 70),
              "vjp": (1464, 20067874631496.0, 59248204848.0, 15244053248, 155),
              "jvp": (1464, 20067874631496.0, 59248204848.0, 23476130560, 207),
              "hvp": (4392, 60203623894488.0, 177744614544.0, 36487643136, 443),
              "sliced vjp": (1464, 5064986991816.0, 18153106224.0, 4368338432, 155),
              "sliced jvp": (1464, 5064986991816.0, 18153106224.0, 6221283072, 208),
              "sliced hvp": (4392, 15194960975448.0, 54459318672.0, 10248070144, 441)},
}
OFFSETS = {"q12": (91, "2db9e8044e92731c"), "bench": (489, "d7db7239d3283fd2")}


@pytest.mark.parametrize("net", ["q12", "bench"])
def test_created_plans(request, net):
    from tnc_b200.tensornetwork import leaves
    tn, path, legs = request.getfixturevalue("q12" if net == "q12" else "bench_net")
    if net == "q12":
        assert legs == [26, 81]
    for k in KINDS:
        h = ok(create(k, tn, path, legs))
        assert info(h) == INFO[net][k], k
        if k != "plain":
            assert offsets_digest(h, len(leaves(tn))) == OFFSETS[net], k
        _lib().tncb_plan_destroy(h)


@pytest.mark.parametrize("kind", KINDS[1:])
def test_creation_refusals(q12, bench_net, kind, monkeypatch):
    """a device leaf, and bench.py's network above a 1 GiB static-workspace limit"""
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import Tensor, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, path, legs = q12
    lv = leaves(tn)
    fake = DeviceTensor.__new__(DeviceTensor)
    fake.handle, fake.shape, fake.ctx = C.c_void_p(0x1000), tuple(lv[1].bond_dims), None
    t = Tensor(lv[1].legs, lv[1].bond_dims)
    t.set_tensor_data(TensorData.Matrix(fake))
    parts = list(tn.tensors)
    parts[1] = t
    rc, _ = create(kind, Tensor.new_composite(parts), path, legs)
    fake.handle = None
    noun = NOUN[kind.split()[-1]]
    assert (rc, _lib().tncb_last_error().decode()) == \
        (ERR_UNSUPPORTED, f"{noun} plans do not take device leaves (they are consumed per call)")
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    big, big_path, big_legs = bench_net
    rc, _ = create(kind, big, big_path, big_legs)
    what = "workspace of one slice" if kind.startswith("sliced") else "workspace"
    assert (rc, _lib().tncb_last_error().decode()) == \
        (ERR_UNSUPPORTED, f"the {noun} {what} needs {INFO['bench'][kind][3]} bytes, above the static-workspace limit of "
                          f"{1 << 30} bytes (TNCB_PLAN_WS_GB)")
