"""Batched Hessian-vector products without a GPU (tncb_plan_hvp_batch on host-only plans, a zeroed block standing in for
the context): the refusals between plan kinds, which happen before the context is touched, the declared signature, and
NetworkPlan.hvp_batch_blocks' handling of its tangent, seed and seed-tangent arguments up to the library call."""
import ctypes as C
import os
import re
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = -1, -9
NOUN = {"jvp": "tangent", "hvp": "Hessian-vector"}


def _lib():
    from tnc_b200._lib import lib
    return lib()


def amplitude(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


@pytest.fixture(scope="module")
def q10(built_lib):
    tn = amplitude(10, 4, 3)
    return tn, greedy(tn)


def create(kind, tn, path, legs=None):
    """(status, handle) of a host-only plan of `kind` ("plain", "vjp", "jvp" or "hvp"), sliced on `legs` if given"""
    from tnc_b200._lib import u64_array
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if kind == "plain":
        return _lib().tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)), h
    if legs is None:
        return getattr(_lib(), f"tncb_plan_create_{kind}")(None, C.byref(ct), C.byref(cp), None, C.byref(h)), h
    return getattr(_lib(), f"tncb_plan_create_{kind}_sliced")(None, C.byref(ct), C.byref(cp), len(legs), u64_array(legs),
                                                              None, C.byref(h)), h


def ok(rc_h):
    rc, h = rc_h
    assert rc == 0, _lib().tncb_last_error()
    return h


def test_refusals_between_plan_kinds(q10):
    """plain, gradient, tangent and sliced gradient plans are not Hessian-vector plans (TNCB_ERR_INVALID); sliced
    tangent and Hessian-vector plans name their own call (TNCB_ERR_UNSUPPORTED); all before the context is read"""
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = q10
    l = _lib()
    fake_ctx = C.create_string_buffer(1 << 16)
    cx = C.cast(fake_ctx, C.c_void_p)
    t = C.c_void_p(0x1000)                                      # never read: the plan kind is refused first
    out = C.c_void_p()

    def hvp_batch(p):
        return l.tncb_plan_hvp_batch(cx, p, 1, 0, None, None, None, t, None, None, C.byref(out), None, None, None, None, None)
    legs = find_slices(tn, path, min_slices=4)
    plans = {k: ok(create(k, tn, path)) for k in ("plain", "vjp", "jvp", "hvp")}
    for k in ("vjp", "jvp", "hvp"):
        plans["sliced " + k] = ok(create(k, tn, path, legs))
    for k in ("plain", "vjp", "jvp", "sliced vjp"):
        assert hvp_batch(plans[k]) == ERR_INVALID, (k, l.tncb_last_error())
        assert l.tncb_last_error().decode() == "not a Hessian-vector plan (tncb_plan_create_hvp)", k
    for k, call in (("jvp", "tncb_plan_jvp_sliced"), ("hvp", "tncb_plan_hvp_sliced")):
        assert hvp_batch(plans["sliced " + k]) == ERR_UNSUPPORTED, (k, l.tncb_last_error())
        assert l.tncb_last_error().decode() == f"a sliced {NOUN[k]} plan runs through {call} / tncb_plan_run_slices", k
    # a Hessian-vector plan that was never staged: refused as such, still without reading the context
    class Header(C.Structure):
        _fields_ = [("ptr", C.c_void_p), ("rank", C.c_int), ("dims", C.c_uint64 * 64)]
    offs = (C.c_int64 * len(tn.tensors))()
    assert l.tncb_plan_grad_offsets(plans["hvp"], offs) == 0
    hd = Header(0x1000, 2)
    hd.dims[0], hd.dims[1] = 3, offs[len(tn.tensors) - 1] + int(np.prod(tn.tensors[-1].bond_dims))
    ht = C.cast(C.pointer(hd), C.c_void_p)
    rc = l.tncb_plan_hvp_batch(cx, plans["hvp"], 3, 0, None, None, None, ht, None, None, C.byref(out), None, None, None, None, None)
    assert rc == ERR_INVALID and "tncb_plan_stage has not been called" in l.tncb_last_error().decode()
    for args, msg in (((0, ht), "count is 0"), ((3, None), "tangents are needed")):
        rc = l.tncb_plan_hvp_batch(cx, plans["hvp"], args[0], 0, None, None, None, args[1], None, None, C.byref(out),
                                   None, None, None, None, None)
        assert rc == ERR_INVALID and msg in l.tncb_last_error().decode(), msg
    rc = l.tncb_plan_hvp_batch(cx, plans["hvp"], 3, 0, None, None, None, ht, None, None, None, None, None, None, None, None)
    assert rc == ERR_INVALID and "no output requested" in l.tncb_last_error().decode()
    hd.dims[0] = 2                                             # rows for another count
    rc = l.tncb_plan_hvp_batch(cx, plans["hvp"], 3, 0, None, None, None, ht, None, None, C.byref(out), None, None, None, None, None)
    assert rc == -2 and "the tangents' dims differ" in l.tncb_last_error().decode()
    for h in plans.values():
        l.tncb_plan_destroy(h)


def test_signature_matches_header():
    from tnc_b200._lib import SIGNATURES, u64p, vpp
    ctypes_of = {"tncb_ctx*": C.c_void_p, "tncb_plan*": C.c_void_p, "size_t": C.c_size_t, "const uint64_t*": u64p,
                 "const void* const*": vpp, "const tncb_tensor*": C.c_void_p, "tncb_tensor**": vpp}
    with open(os.path.join(ROOT, "include", "tncb.h")) as f:
        text = f.read()
    m = re.search(r"int\s+tncb_plan_hvp_batch\s*\(([^)]*)\)\s*;", text)
    assert m
    params = [re.sub(r"\s*\w+$", "", " ".join(p.split())).replace(" *", "*") for p in m.group(1).split(",")]
    res, args = SIGNATURES["tncb_plan_hvp_batch"]
    assert res is C.c_int
    assert args == [ctypes_of[p] for p in params], (args, params)


@pytest.fixture
def host_plan(q10, monkeypatch):
    """a host-only Hessian-vector plan behind a NetworkPlan whose context has no device: every upload is recorded
    instead of made, and the library call then refuses the NULL context"""
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = q10
    fake = types.SimpleNamespace(_l=_lib(), handle=None, device=0)
    plan = NetworkPlan._derivative_plan("tncb_plan_create_hvp", tn, path, None, fake)
    uploads = []

    def record(cls, ctx, arr):
        uploads.append(np.array(arr, dtype=np.complex128))
        t = DeviceTensor.__new__(DeviceTensor)
        t.ctx, t.handle, t.shape = ctx, None, tuple(np.shape(arr))
        return t
    monkeypatch.setattr(DeviceTensor, "from_numpy", classmethod(record))
    yield plan, uploads
    plan.ctx._l.tncb_plan_destroy(plan.handle)
    plan.handle = None


def reaches_library(plan, *args, **kwargs):
    from tnc_b200 import TncbError
    with pytest.raises(TncbError) as e:
        plan.hvp_batch_blocks(*args, **kwargs)
    return e.value.status == ERR_INVALID and "null argument" in str(e.value)


def test_tangent_arguments(host_plan):
    plan, uploads = host_plan
    offs = plan.grad_offsets()
    sizes = [int(np.prod(s)) for s in plan.leaf_shapes]
    te = sum(sz for off, sz in zip(offs, sizes) if off >= 0)
    count = 3
    rng = np.random.default_rng(1)
    # a dict: per-instance rows and a shared leaf-shaped tangent, packed at the gradient offsets, the rest zero
    rows = rng.standard_normal((count,) + plan.leaf_shapes[0])
    shared = rng.standard_normal(plan.leaf_shapes[2])
    assert reaches_library(plan, count, {0: rows, 2: shared})
    want = np.zeros((count, te), dtype=np.complex128)
    want[:, offs[0]:offs[0] + sizes[0]] = rows.reshape(count, -1)
    want[:, offs[2]:offs[2] + sizes[2]] = shared.reshape(-1)
    assert len(uploads) == 1 and np.array_equal(uploads[0], want)
    # an already packed block: a Hessian block of P = count directions, uploaded as it is
    uploads.clear()
    block = np.eye(te)[[0, te // 2, te - 1]]
    assert reaches_library(plan, count, block)
    assert len(uploads) == 1 and np.array_equal(uploads[0], block)
    # seeds and seed tangents shaped [count, *result dims] (a scalar result: [count])
    uploads.clear()
    assert plan.result_dims == ()
    assert reaches_library(plan, count, block, seeds=np.ones(count), seed_tangents=np.zeros(count))
    assert [u.shape for u in uploads] == [(count, te), (count,), (count,)]
    # refused before the refused argument is uploaded
    uploads.clear()
    for bad in (np.zeros((count, te + 1)), np.zeros(te), np.zeros((count + 1, te)), np.zeros((1, count, te))):
        with pytest.raises(ValueError, match="the tangents have shape"):
            plan.hvp_batch_blocks(count, bad)
    with pytest.raises(ValueError, match="the tangent of leaf 0 has shape"):
        plan.hvp_batch_blocks(count, {0: np.zeros((count + 1,) + plan.leaf_shapes[0])})
    with pytest.raises(IndexError):
        plan.hvp_batch_blocks(count, {len(sizes): np.zeros(1)})
    assert uploads == []
    for kw, what in ((dict(seeds=np.ones(count + 1)), "seeds"), (dict(seeds=np.ones((count, 1))), "seeds"),
                     (dict(seed_tangents=np.ones(1)), "seed tangents")):
        with pytest.raises(ValueError, match=f"the {what} have shape"):
            plan.hvp_batch_blocks(count, block, **kw)
        assert all(u.shape == (count, te) or u.shape == (count,) for u in uploads)
