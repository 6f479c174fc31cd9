"""Leaf payloads staged from device memory (tncb_plan_set_leaves / tncb_plan_stage_instances, NetworkPlan.set_leaves /
stage_instances, SlicedPlan.set_leaves, DeviceTensor.to_torch / from_torch, network_function(on_device=True)).

  1. on every route (a static graphed plain plan, a static plan with int8-engine steps, TNCB_NO_STATIC=1, a gradient
     plan, a sliced gradient plan, stage_instances against stage_slices and stage_batch) device staging gives the bits
     host staging gives for the same payloads;
  2. network_function(on_device=True) gives the CPU-input path's values and gradients bit for bit, as CUDA tensors;
  3. its steady state makes no host round trip;
  4. stream ordering both ways, and the source's memory stays protected after the call;
  5. more than 65535 instances;
  6. every refusal, before any launch, with the staged state untouched."""
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = -1, -9


@pytest.fixture(scope="module")
def ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def matrixify(tn):
    """the flat network `tn` (or a list of leaves) with every leaf a Matrix leaf holding its materialised payload"""
    from tnc_b200.contractionpath.slicing import _leaf_array
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    out = []
    for t in (tn if isinstance(tn, list) else tn.tensors):
        m = Tensor(list(t.legs), list(t.bond_dims))
        m.set_tensor_data(TensorData.Matrix(np.ascontiguousarray(_leaf_array(t), dtype=np.complex128)))
        out.append(m)
    return Tensor.new_composite(out)


def amplitude(qubits, rounds, seed, bits=None):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return matrixify(c.into_amplitude_network(bits or "0" * qubits)[0])


def perturbed(tn, idx, rng):
    """{leaf: its payload scaled by 1 + 0.1 * complex noise}"""
    from tnc_b200.contractionpath.slicing import _leaf_array
    from tnc_b200.tensornetwork import leaves
    lv = leaves(tn)
    out = {}
    for i in idx:
        a = _leaf_array(lv[i])
        out[i] = a * (1 + 0.1 * (rng.standard_normal(a.shape) + 1j * rng.standard_normal(a.shape)))
    return out


def host_net(tn, pay):
    from tnc_b200.autograd import _with_payloads
    return _with_payloads(tn, pay, [0])


def cuda(pay):
    import torch
    return {i: torch.from_numpy(np.ascontiguousarray(a)).cuda() for i, a in pay.items()}


def launches(ctx):
    ctx.synchronize()
    return ctx.stats()["kernel_launches"]


# ================================================================================================================
# 1. bit identity with host staging, route by route
# ================================================================================================================
def check_plain(ctx, tn, path, idx, seed):
    """stage(tn) + set_leaves(P) + run == stage(tn with P) + run, twice with other payloads; engine counts of a run"""
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(seed)
    plan = NetworkPlan(tn, path, ctx=ctx)
    plan.stage(tn)
    for _ in range(2):
        pay = perturbed(tn, idx, rng)
        plan.set_leaves(cuda(pay))
        ctx.reset_stats()
        dev = plan.run().to_numpy()
        counts = ctx.engine_counts()
        again = plan.run().to_numpy()              # the payloads stay in place
        plan.stage(host_net(tn, pay))
        ref = plan.run().to_numpy()
        plan.stage(tn)
        assert np.array_equal(dev, ref) and np.array_equal(again, ref)
    return counts


def test_static_graphed_plan(ctx):
    """K0 / K2 steps only: the plan replays its graph, which reads the leaf block set_leaves writes"""
    tn = amplitude(12, 6, 3)
    counts = check_plain(ctx, tn, greedy(tn), range(0, len(tn.tensors), 3), 1)
    assert counts["k1_dmma"] == counts["k1_tcgen05"] == 0, counts


def test_static_plan_int8_engine(ctx):
    """a pair large enough for the int8 engine (K1')"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(2)
    a, b = Tensor([0, 1], [1536, 1408]), Tensor([1, 2], [1408, 1536])
    a.set_tensor_data(TensorData.Matrix(rng.standard_normal((1536, 1408)) + 0j))
    b.set_tensor_data(TensorData.Matrix(rng.standard_normal((1408, 1536)) + 0j))
    tn = Tensor.new_composite([a, b])
    counts = check_plain(ctx, tn, ContractionPath.simple([(0, 1)]), [0, 1], 3)
    assert counts["k1_tcgen05"] == 1, counts


def test_no_static_plan(ctx, monkeypatch):
    """TNCB_NO_STATIC=1: the resident leaf block of the pair-by-pair executor"""
    tn = amplitude(12, 6, 4)
    path = greedy(tn)
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    check_plain(ctx, tn, path, range(1, len(tn.tensors), 2), 5)


def check_gradient(ctx, tn, path, idx, seed):
    from tnc_b200._lib import TncbError
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(seed)
    plan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    plan.stage(tn)
    for k in range(2):                              # the second set_leaves follows a vjp
        pay = perturbed(tn, idx, rng)
        plan.set_leaves(cuda(pay))
        if k == 1:
            with pytest.raises(TncbError):          # new payloads need a new forward run
                plan.vjp()
        dev_v, dev_g = plan.run().to_numpy(), plan.vjp()
        plan.stage(host_net(tn, pay))
        ref_v, ref_g = plan.run().to_numpy(), plan.vjp()
        plan.stage(tn)
        plan.set_leaves(cuda(pay))
        assert np.array_equal(dev_v, ref_v)
        assert sorted(dev_g) == sorted(ref_g)
        for leaf in ref_g:
            assert np.array_equal(dev_g[leaf], ref_g[leaf]), leaf


def test_gradient_plan(ctx):
    tn = amplitude(14, 8, 6)
    check_gradient(ctx, tn, greedy(tn), range(len(tn.tensors)), 7)


def test_gradient_plan_bench_network(ctx):
    """bench.py's network (36 qubits, 489 leaves, the int8 engine, a 15 GB gradient workspace), every leaf set from the
    device in one call"""
    sys.path.insert(0, ROOT)
    import bench
    from tnc_b200.builders import random_circuit_builder
    q = bench.NET["qubits"]
    c = random_circuit_builder(q, bench.NET["rounds"], bench.NET["p1"], bench.NET["p2"], np.random.default_rng(bench.NET["seed"]))
    tn = matrixify(c.into_amplitude_network("0" * q)[0])
    check_gradient(ctx, tn, bench.greedy_path(tn), range(len(tn.tensors)), 8)
    ctx.trim()


def test_sliced_gradient_plan(ctx):
    """set_leaves into the full leaf block: run_slices and vjp_sliced, the full range and two halves"""
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    tn = amplitude(12, 6, 9)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    plan = SlicedPlan.for_gradients(tn, path, legs, ctx=ctx)
    rng = np.random.default_rng(10)
    pay = perturbed(tn, range(0, len(tn.tensors), 2), rng)
    plan.stage(host_net(tn, pay))
    ranges = [(0, 1), (0, 2), (1, 2)]
    ref = [(plan.run(r, w, allreduce=False).to_numpy(), plan.vjp(None, r, w, allreduce=False)) for r, w in ranges]
    plan.stage(tn)
    plan.set_leaves(cuda(pay))
    for (r, w), (rv, (rval, rg)) in zip(ranges, ref):
        val, g = plan.vjp(None, r, w, allreduce=False)
        assert np.array_equal(plan.run(r, w, allreduce=False).to_numpy(), rv)
        assert np.array_equal(val.to_numpy(), rval.to_numpy())
        for leaf in rg:
            assert np.array_equal(g[leaf], rg[leaf]), (r, w, leaf)


def bra_sources(nets, q):
    """the bitstring projectors of every instance in ONE device tensor [B, q, 2]: leaf j's payload is the padded-stride
    view [:, j, :]"""
    import torch
    from tnc_b200.contractionpath.slicing import _leaf_array
    X = np.stack([np.stack([_leaf_array(t) for t in net.tensors[-q:]]) for net in nets])
    return torch.from_numpy(X).cuda()


@pytest.mark.parametrize("qubits,count", [(12, 9), (16, 512)])
def test_stage_instances(ctx, qubits, count):
    """stage_instances against stage_slices (run_batch, run_slices) and stage_batch (vjp_batch values, rows, sum): the
    bras from one device tensor (padded stride), one gate packed per instance, one shared (stride 0)"""
    import torch
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    from tnc_b200.tensornetwork import Tensor
    c = random_circuit_builder(qubits, 10 if qubits == 16 else 6, 0.5, 0.5, np.random.default_rng(qubits))
    rng = np.random.default_rng(11)
    base = matrixify(c.into_amplitude_network("0" * qubits)[0])
    n = len(base.tensors)
    packed = np.stack([perturbed(base, [0], rng)[0] for _ in range(count)])
    shared = perturbed(base, [1], rng)[1]
    nets = []
    for i in range(count):
        bits = "".join(rng.choice(["0", "1"], qubits))
        bras = matrixify(c.into_amplitude_network(bits)[0].tensors[-qubits:]).tensors   # (only the bras differ)
        nets.append(host_net(Tensor.new_composite(base.tensors[:n - qubits] + bras), {0: packed[i], 1: shared}))
    X = bra_sources(nets, qubits)
    pay = {n - qubits + j: X[:, j, :] for j in range(qubits)}
    pay[0] = torch.from_numpy(packed).cuda()
    pay[1] = torch.from_numpy(shared).cuda()
    assert pay[n - 1].stride(0) == 2 * qubits
    path = greedy(base)
    plain = NetworkPlan(base, path, ctx=ctx)
    plain.stage_slices(nets)
    ref_rows, ref_sum = plain.run_batch()[1].to_numpy(), plain.run_slices(0, 1).to_numpy()
    plain.stage_instances(base, pay, count)
    assert plain.n_staged == count
    assert np.array_equal(plain.run_batch()[1].to_numpy(), ref_rows)
    assert np.array_equal(plain.run_slices(0, 1).to_numpy(), ref_sum)
    grad = NetworkPlan.for_gradients(base, path, ctx=ctx)
    seeds = rng.standard_normal(count) + 1j * rng.standard_normal(count)
    grad.stage_batch(nets)
    _, rv, rr, rs = grad.vjp_batch(0, count, seeds, rows=True, sum=True)
    grad.stage_instances(base, pay, count)
    _, v, r, s = grad.vjp_batch(0, count, seeds, rows=True, sum=True)
    assert np.array_equal(v, rv)
    for leaf in rr:
        assert np.array_equal(r[leaf], rr[leaf]) and np.array_equal(s[leaf], rs[leaf]), leaf


def test_more_than_65535_instances(ctx):
    """a 3-leaf network, 70,000 instances: several launches along the instance dimension"""
    import torch
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(12)
    count = 70000
    A = rng.standard_normal((count, 2, 2)) + 1j * rng.standard_normal((count, 2, 2))
    B = rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2))
    Cm = rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2))

    def net(a):
        ts = []
        for legs, m in (([0, 1], a), ([1, 2], B), ([2, 0], Cm)):
            t = Tensor(legs, [2, 2])
            t.set_tensor_data(TensorData.Matrix(m))
            ts.append(t)
        return Tensor.new_composite(ts)
    plan = NetworkPlan(net(A[0]), ContractionPath.simple([(0, 1), (0, 2)]), ctx=ctx)
    plan.stage_slices([net(A[i]) for i in range(count)])
    ref = plan.run_batch()[1].to_numpy()
    plan.stage_instances(net(np.zeros((2, 2))), {0: torch.from_numpy(A).cuda(), 1: torch.from_numpy(B).cuda()}, count)
    assert np.array_equal(plan.run_batch()[1].to_numpy(), ref)


# ================================================================================================================
# 2. - 4. network_function(on_device=True)
# ================================================================================================================
def big_leaf_net(rng):
    """a 1024-element (16 KiB) state leaf [legs 0..9] projected by ten 2-vectors, and one 2x2 matrix on leg 0"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    ts = []
    psi = Tensor(list(range(10)), [2] * 10)
    psi.set_tensor_data(TensorData.Matrix(rng.standard_normal((2,) * 10) + 1j * rng.standard_normal((2,) * 10)))
    ts.append(psi)
    u = Tensor([0, 10], [2, 2])
    u.set_tensor_data(TensorData.Matrix(rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2))))
    ts.append(u)
    for j in range(10):
        v = Tensor([10 if j == 0 else j], [2])
        v.set_tensor_data(TensorData.Matrix(rng.standard_normal(2) + 1j * rng.standard_normal(2)))
        ts.append(v)
    pairs = [(0, 1)] + [(0, j) for j in range(2, 12)]
    return Tensor.new_composite(ts), ContractionPath.simple(pairs)


def step(f, xs):
    """forward + backward of sum Re(w f(xs)) for a fixed w; (value, grads).  The loss is linear so that its gradient,
    the seed, has the same bits whether torch computes it on the CPU or on the GPU."""
    import torch
    xs = [x.detach().clone().requires_grad_(True) for x in xs]
    out = f(*xs)
    (out * torch.full(out.shape, complex(0.3, -0.7), dtype=out.dtype, device=out.device)).real.sum().backward()
    return out.detach(), [x.grad for x in xs]


@pytest.mark.parametrize("variant", ["unbatched", "sliced", "batched"])
def test_network_function_on_device(ctx, variant):
    import torch
    from tnc_b200.autograd import network_function
    rng = np.random.default_rng(13)
    tn, path = big_leaf_net(rng)
    kw = {"unbatched": {}, "sliced": {"sliced_legs": [3]}, "batched": {"batched": [2, 3]}}[variant]
    wrt = [0, 1, 2]
    f_host = network_function(tn, path, wrt, ctx=ctx, **kw)
    f_dev = network_function(tn, path, wrt, ctx=ctx, on_device=True, **kw)
    for k in range(2):
        xs = [torch.from_numpy(rng.standard_normal((2,) * 10) + 1j * rng.standard_normal((2,) * 10)),
              torch.from_numpy(rng.standard_normal((2, 2)) + 1j * rng.standard_normal((2, 2)))]
        if variant == "batched":
            xs += [torch.from_numpy(rng.standard_normal((5, 2)) + 0j), torch.from_numpy(rng.standard_normal((5, 2)) + 0j)]
        else:
            xs += [torch.from_numpy(rng.standard_normal(2) + 0j)]
        hv, hg = step(f_host, xs)
        dv, dg = step(f_dev, [x.cuda() for x in xs])
        assert dv.is_cuda and dv.device.index == ctx.device and not hv.is_cuda
        assert torch.equal(dv.cpu(), hv)
        for a, b in zip(dg, hg):
            if b is None:
                assert a is None
                continue
            assert a.is_cuda and torch.equal(a.cpu(), b)


def test_network_function_refusals(ctx):
    import torch
    from tnc_b200.autograd import network_function
    tn, path = big_leaf_net(np.random.default_rng(14))
    f = network_function(tn, path, [1], ctx=ctx, on_device=True)
    with pytest.raises(ValueError, match="CUDA"):
        f(torch.zeros((2, 2), dtype=torch.complex128))
    with pytest.raises(ValueError, match="shape"):
        f(torch.zeros((2, 3), dtype=torch.complex128, device="cuda"))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            f(torch.zeros((2, 2), dtype=torch.complex128, device=f"cuda:{1 - ctx.device}"))


@pytest.mark.parametrize("variant", ["unbatched", "batched"])
def test_no_host_round_trip(ctx, monkeypatch, variant):
    """after the first step, a step with .cpu / .numpy / host staging / host tensor transfers patched to raise succeeds,
    and its trace holds no host<->device copy as large as the 16 KiB input leaf"""
    import torch
    import tnc_b200 as tb
    from tnc_b200.autograd import network_function
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(15)
    tn, path = big_leaf_net(rng)
    kw = {"batched": [2]} if variant == "batched" else {}
    f = network_function(tn, path, [0, 1], ctx=ctx, on_device=True, **kw)
    xs = [torch.randn((2,) * 10, dtype=torch.complex128, device="cuda"), torch.randn((2, 2), dtype=torch.complex128, device="cuda")]
    if variant == "batched":
        xs.append(torch.randn((8, 2), dtype=torch.complex128, device="cuda"))
    step(f, xs)

    def refuse(*a, **k):
        raise AssertionError("host round trip")
    for owner, name in [(torch.Tensor, "cpu"), (torch.Tensor, "numpy"), (NetworkPlan, "stage"), (NetworkPlan, "stage_batch"),
                        (tb.DeviceTensor, "to_numpy"), (tb.DeviceTensor, "from_numpy")]:
        monkeypatch.setattr(owner, name, refuse)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        v, g = step(f, xs)
        torch.cuda.synchronize()
    monkeypatch.undo()
    assert v.is_cuda and all(x.is_cuda for x in g[:2])
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "trace.json")
        prof.export_chrome_trace(p)
        with open(p) as fh:
            events = json.load(fh)["traceEvents"]
    copies = [e for e in events if "Memcpy" in e.get("name", "") and ("HtoD" in e["name"] or "DtoH" in e["name"])]
    big = [e for e in copies if int(e.get("args", {}).get("bytes", 0)) >= 16 * 1024]
    assert not big, big


def test_ordering(ctx):
    """inputs written behind a long op on torch's current stream; a staging source freed right after the call while
    the allocator churns"""
    import torch
    from tnc_b200.autograd import network_function
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(16)
    tn, path = big_leaf_net(rng)
    f_host = network_function(tn, path, [0, 1], ctx=ctx)
    f_dev = network_function(tn, path, [0, 1], ctx=ctx, on_device=True)
    a = torch.from_numpy(rng.standard_normal((2,) * 10) + 1j * rng.standard_normal((2,) * 10))
    b = torch.from_numpy(rng.standard_normal((2, 2)) + 0j)
    ref = f_host(a, b)
    xa, xb = torch.zeros_like(a, device="cuda"), torch.zeros_like(b, device="cuda")
    ac, bc = a.cuda(), b.cuda()
    f_dev(xa, xb)
    torch.cuda._sleep(200_000_000)                   # ~0.1 s on the current stream, then the inputs are written there
    xa.copy_(ac)
    xb.copy_(bc)
    assert torch.equal(f_dev(xa, xb).cpu(), ref)
    # a temporary source, freed as soon as set_leaves returns, its block wanted by the next allocations
    plan = NetworkPlan(tn, path, ctx=ctx)
    plan.stage(tn)
    pay = perturbed(tn, [0], rng)
    plan.stage(host_net(tn, pay))
    want = plan.run().to_numpy()
    plan.stage(tn)
    src = torch.from_numpy(pay[0]).cuda()
    torch.cuda._sleep(200_000_000)
    plan.set_leaves({0: src * 1})                    # the product lives only through the call
    junk = [torch.full((1024,), float(i), dtype=torch.complex128, device="cuda") for i in range(64)]
    del junk
    assert np.array_equal(plan.run().to_numpy(), want)


# ================================================================================================================
# 6. refusals
# ================================================================================================================
def test_refusals(ctx):
    """every refusal returns its status before any launch, and the next run returns the staged result bit for bit"""
    import torch
    import tnc_b200 as tb
    from tnc_b200._lib import TncbError, TncbTn, u64_array
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.contraction import PreparedNetwork
    from tnc_b200.tensornetwork.tensordata import TensorData
    l = ctx._l
    tn = amplitude(10, 4, 17)
    path = greedy(tn)
    plan = NetworkPlan(tn, path, ctx=ctx)
    x = torch.randn((2, 2), dtype=torch.complex128, device="cuda")
    ptr = lambda *ps: (C.c_void_p * len(ps))(*ps)

    def status(fn):
        before = launches(ctx)
        rc = fn()
        assert launches(ctx) == before, "a refused call launched"
        return rc
    assert status(lambda: l.tncb_plan_set_leaves(ctx.handle, plan.handle, 1, u64_array([0]), ptr(x.data_ptr()))) == ERR_INVALID
    plan.stage(tn)
    want = plan.run().to_numpy()
    two = next(i for i, t in enumerate(tn.tensors) if list(t.bond_dims) == [2, 2])
    xp = x.data_ptr()
    cases = [
        ([len(tn.tensors)], [xp]),                  # out of range
        ([two, two], [xp, xp]),                     # listed twice
        ([two], [None]),                            # null
        ([two], [xp + 8]),                          # misaligned
        ([two], [np.zeros(4, np.complex128).ctypes.data]),   # host memory
        ([two], [torch.zeros(4, dtype=torch.complex128).pin_memory().data_ptr()]),
    ]
    for idx, ps in cases:
        assert status(lambda: l.tncb_plan_set_leaves(ctx.handle, plan.handle, len(idx), u64_array(idx), ptr(*ps))) == ERR_INVALID, idx
        assert np.array_equal(plan.run().to_numpy(), want)
    # instances: 0 instances, a stride below the leaf, a range past the end of the source's allocation
    gp = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    gp.stage_batch([tn, tn])
    vals = gp.vjp_batch(0, 2, None, rows=False, values=True)[1]
    tmpl = PreparedNetwork(tn)
    small = torch.zeros(4, dtype=torch.complex128, device="cuda")
    for n_inst, stride in [(0, 4), (4, 3), (1 << 20, 4), (2, 1 << 40)]:
        rc = status(lambda: l.tncb_plan_stage_instances(ctx.handle, gp.handle, C.byref(tmpl.node), n_inst, 1, u64_array([two]),
                                                        ptr(small.data_ptr()), u64_array([stride])))
        assert rc == ERR_INVALID, (n_inst, stride)
        assert gp.n_staged == 2 and np.array_equal(gp.vjp_batch(0, 2, None, rows=False, values=True)[1], vals)
    # plans with device leaves, sliced gradient plans
    lv = list(tn.tensors)
    d = Tensor(list(lv[0].legs), list(lv[0].bond_dims))
    d.set_tensor_data(TensorData.Matrix(tb.DeviceTensor.from_numpy(ctx, np.asarray(lv[0].tensordata.matrix))))
    dplan = NetworkPlan(Tensor.new_composite([d] + lv[1:]), path, ctx=ctx)
    assert l.tncb_plan_set_leaves(ctx.handle, dplan.handle, 0, None, None) == ERR_UNSUPPORTED
    sp = SlicedPlan.for_gradients(tn, path, [tn.tensors[two].legs[0]], ctx=ctx)
    assert l.tncb_plan_stage_instances(ctx.handle, sp.plan.handle, C.byref(tmpl.node), 1, 0, None, None, None) == ERR_UNSUPPORTED
    with pytest.raises(TypeError):
        SlicedPlan(tn, path, [tn.tensors[two].legs[0]], ctx=ctx).set_leaves({})
    # refusals in Python
    with pytest.raises(ValueError, match="CUDA"):
        plan.set_leaves({two: x.cpu()})
    with pytest.raises(ValueError, match="shape"):
        plan.set_leaves({two: torch.zeros((4,), dtype=torch.complex128, device="cuda")})
    with pytest.raises(ValueError, match="shape"):
        plan.stage_instances(tn, {two: torch.zeros((3, 2, 3), dtype=torch.complex128, device="cuda")}, 3)
    assert np.array_equal(plan.run().to_numpy(), want)


def test_device_tensor_torch_round_trip(ctx):
    import torch
    import tnc_b200 as tb
    t = torch.randn((3, 4, 5), dtype=torch.complex128, device="cuda")
    d = tb.DeviceTensor.from_torch(ctx, t)
    assert d.shape == (3, 4, 5)
    back = d.to_torch()
    assert back.is_cuda and torch.equal(back, t)
    assert np.array_equal(d.to_numpy(), t.cpu().numpy())
    s = tb.DeviceTensor.from_torch(ctx, torch.tensor(2.5, device="cuda"))      # 0-d, cast from float64
    assert s.shape == () and s.to_torch().item() == 2.5
    with pytest.raises(ValueError):
        tb.DeviceTensor.from_torch(ctx, t.cpu())
