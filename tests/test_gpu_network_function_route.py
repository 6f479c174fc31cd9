"""How network_function delivers its inputs to the device and its outputs back, and payloads with a conj or neg bit.

  1. lazily conjugated (x.conj()) or negated payloads give the bits of their resolved copies: NetworkPlan.set_leaves,
     stage_instances, hvp_batch_blocks and network_function with on_device True and False;
  2. with on_device=False, the value comes back on the CPU and each gradient on its input's device;
  3. a step with CPU inputs moves the inputs to the device in one copy and the gradients back in one copy;
  4. a function whose results and gradients are released is freed at once, with its plans' device memory: no
     reference cycle leaves that to the garbage collector."""
import gc
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from test_gpu_device_stage import big_leaf_net, step

pytestmark = pytest.mark.gpu

W = complex(0.3, -0.7)


def crandn(rng, shape):
    import torch
    return torch.from_numpy(rng.standard_normal(shape) + 1j * rng.standard_normal(shape))


# ================================================================================================================
# 1. conj and neg bits
# ================================================================================================================
def test_set_leaves_conj_and_neg_views(ctx):
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(20)
    tn, path = big_leaf_net(rng)
    psi, u = crandn(rng, (2,) * 10).cuda(), crandn(rng, (2, 2)).cuda()
    plan = NetworkPlan(tn, path, ctx=ctx)
    plan.stage(tn)
    plan.set_leaves({0: psi.conj(), 1: torch._neg_view(u)})
    lazy = plan.run().to_numpy()
    plan.set_leaves({0: psi.conj().resolve_conj(), 1: -u})
    assert np.array_equal(lazy, plan.run().to_numpy())


def test_stage_instances_conj_views(ctx):
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(21)
    tn, path = big_leaf_net(rng)
    U, v = crandn(rng, (3, 2, 2)).cuda(), crandn(rng, (2,)).cuda()
    plan = NetworkPlan(tn, path, ctx=ctx)
    plan.stage_instances(tn, {1: U.conj(), 2: v.conj()}, 3)
    lazy = plan.run_batch()[1].to_numpy()
    plan.stage_instances(tn, {1: U.conj().resolve_conj(), 2: v.conj().resolve_conj()}, 3)
    assert np.array_equal(lazy, plan.run_batch()[1].to_numpy())


def test_hvp_batch_blocks_conj_views(ctx):
    from tnc_b200.tensornetwork import NetworkPlan
    rng = np.random.default_rng(22)
    tn, path = big_leaf_net(rng)
    plan = NetworkPlan.for_hvp(tn, path, [0, 1], ctx=ctx)
    plan.stage(tn)
    U = crandn(rng, (3, 2, 2)).cuda()
    tangents = {0: crandn(rng, (2,) * 10).cuda(), 1: crandn(rng, (3, 2, 2)).cuda()}
    out = []
    for pay in ({1: U.conj()}, {1: U.conj().resolve_conj()}):
        blocks = plan.hvp_batch_blocks(3, tangents, payloads=pay)
        out.append([b.to_numpy() for b in blocks])
        for b in blocks:
            b.free()
    for lazy, resolved in zip(*out):
        assert np.array_equal(lazy, resolved)


@pytest.mark.parametrize("on_device", [True, False])
def test_network_function_conj_inputs(ctx, on_device):
    """a conj view of a leaf as input: value and gradients equal those of its resolved copy (with on_device=False this
    used to raise, as numpy refuses conj views)"""
    import torch
    from tnc_b200.autograd import network_function
    rng = np.random.default_rng(23)
    tn, path = big_leaf_net(rng)
    f = network_function(tn, path, [0, 1], ctx=ctx, on_device=on_device)
    dev = "cuda" if on_device else "cpu"
    psi, u = crandn(rng, (2,) * 10).to(dev), crandn(rng, (2, 2)).to(dev)
    res = []
    for resolve in (False, True):
        a, b = psi.clone().requires_grad_(True), u.clone().requires_grad_(True)
        x = a.conj().resolve_conj() if resolve else a.conj()
        out = f(x, b)
        (out * W).real.sum().backward()
        res.append((out.detach(), a.grad, b.grad))
    for lazy, resolved in zip(*res):
        assert torch.equal(lazy, resolved)


# ================================================================================================================
# 2. output devices with on_device=False
# ================================================================================================================
@pytest.mark.parametrize("variant", ["unbatched", "sliced", "batched"])
def test_output_devices(ctx, variant):
    """CPU inputs: CPU value and gradients; CUDA inputs: CPU value, CUDA gradients; one of each: each gradient on its
    input's device.  All with the same bits."""
    import torch
    from tnc_b200.autograd import network_function
    rng = np.random.default_rng(24)
    tn, path = big_leaf_net(rng)
    kw = {"unbatched": {}, "sliced": {"sliced_legs": [3]}, "batched": {"batched": [2, 3]}}[variant]
    f = network_function(tn, path, [0, 1, 2], ctx=ctx, **kw)
    xs = [crandn(rng, (2,) * 10), crandn(rng, (2, 2))]
    xs += [crandn(rng, (5, 2)), crandn(rng, (5, 2))] if variant == "batched" else [crandn(rng, (2,))]
    ref_v, ref_g = step(f, xs)
    assert ref_v.device.type == "cpu" and all(g is None or g.device.type == "cpu" for g in ref_g)
    for devs in (["cuda"] * len(xs), ["cuda", "cpu"] + ["cuda"] * (len(xs) - 2)):
        v, g = step(f, [x.to(d) for x, d in zip(xs, devs)])
        assert v.device.type == "cpu" and torch.equal(v, ref_v)
        for gi, ri, d in zip(g, ref_g, devs):
            if ri is None:
                assert gi is None
                continue
            assert gi.device.type == d and torch.equal(gi.cpu(), ri)


# ================================================================================================================
# 3. one copy each way
# ================================================================================================================
def cpu_input_step_copies():
    """(bytes of the inputs, [(name, bytes)] of every memcpy in the trace of a forward + backward() with CPU inputs (a
    16 KiB state and a 2x2 matrix) after a first step)"""
    import torch
    import tnc_b200 as tb
    from tnc_b200.autograd import network_function
    rng = np.random.default_rng(25)
    tn, path = big_leaf_net(rng)
    f = network_function(tn, path, [0, 1], ctx=tb.default_context())
    xs = [crandn(rng, (2,) * 10), crandn(rng, (2, 2))]
    step(f, xs)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        _, g = step(f, xs)
        torch.cuda.synchronize()
    assert all(x.device.type == "cpu" for x in g)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "trace.json")
        prof.export_chrome_trace(p)
        with open(p) as fh:
            events = json.load(fh)["traceEvents"]
    return sum(x.numel() * 16 for x in xs), [(e["name"], int(e.get("args", {}).get("bytes", 0)))
                                             for e in events if "Memcpy" in e.get("name", "")]


def test_cpu_inputs_one_copy_each_way(built_lib):
    """one host-to-device copy of at least 16 KiB, holding both inputs, and one device-to-host copy, holding both
    gradients.  The step is traced in a process of its own: in a process that has run other profiled tests before, the
    trace can lack copy records."""
    code = ("import json, sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; import test_gpu_network_function_route as t; "
            "print('COPIES', json.dumps(t.cpu_input_step_copies()))")
    tests = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-s", "-c", code, os.path.dirname(tests), tests], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    line = [l for l in r.stdout.splitlines() if l.startswith("COPIES ")]
    assert r.returncode == 0 and line, r.stdout[-3000:]
    nbytes, copies = json.loads(line[0][len("COPIES "):])
    h2d = [n for name, n in copies if "HtoD" in name and n >= 16 * 1024]
    d2h = [n for name, n in copies if "DtoH" in name and n >= 16 * 1024]
    assert h2d == [nbytes], copies
    assert d2h == [nbytes], copies


# ================================================================================================================
# 4. no reference cycle
# ================================================================================================================
@pytest.mark.parametrize("on_device", [False, True])
def test_released_function_is_freed(ctx, on_device):
    """with the cyclic garbage collector off, dropping a function after a training step and after a forward whose graph
    is still alive frees it"""
    import weakref
    from tnc_b200.autograd import network_function
    rng = np.random.default_rng(26)
    tn, path = big_leaf_net(rng)
    dev = "cuda" if on_device else "cpu"
    xs = [crandn(rng, (2,) * 10).to(dev), crandn(rng, (2, 2)).to(dev)]
    f = network_function(tn, path, [0, 1], ctx=ctx, on_device=on_device)
    gc.collect()
    gc.disable()
    try:
        v, g = step(f, xs)
        out = f(*[x.clone().requires_grad_(True) for x in xs])
        freed = weakref.ref(f)
        del f, v, g, out
        assert freed() is None
    finally:
        gc.enable()
