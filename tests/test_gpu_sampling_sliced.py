"""Sampling sliced circuits on the H100 (tncb_plan_sample_slices, Sampler(..., sliced_legs=...)).

  1. one staged network: sample_slices after stage_slices([tn]) equals sample after stage(tn) bit for bit;
  2. the wiring, exactly: every candidate's amplitudes from the host route (its network sliced on the host,
     stage_slices + run_slices on the same plan), p = |a|^2 bit for bit, the pick of a numpy restatement of the kernel's
     prefix sum, the closed bits of numpy's Philox, and u < r for every accept decision;
  3. the distribution: chi-square and acceptance rate against the oracle's state vector for k = 0, 4, 12;
  4. reproducibility: seeds, pass sizes, a call split in two, and the staged slices left alone;
  5. the in-place pass: with device memory held so that no workspace copy fits, the same samples, and the plan's
     staged leaves documented as gone;
  6. the committed Sycamore-53 depth-12 tree, 64 slices, ten qubits open, against the host route;
  7. every refusal of the C ABI, with the arena and the staged slices unchanged."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = -1, -9
D12_OPEN = [2, 8, 12, 13, 16, 18, 22, 29, 32, 35]


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


def to_oracle(t):
    if t.is_composite():
        return orc.OTensor(children=[to_oracle(c) for c in t.tensors])
    td = t.tensordata
    d = ("gate", td.gate[0], td.gate[1], td.gate[2]) if td.kind == "gate" else np.asarray(td.matrix)
    return orc.OTensor(list(t.legs), list(t.bond_dims), d)


def circuit(n, seed, rounds=5):
    from tnc_b200.builders.random_circuit import random_circuit_builder
    return random_circuit_builder(n, rounds, 0.5, 0.5, np.random.default_rng(seed))


def statevector(c):
    """the oracle's state vector of circuit c, shaped [2] * n with axis q = qubit q"""
    tn, _ = c.into_statevector_network()
    res = orc.contract_tensor_network(to_oracle(tn), orc.OPath(list(greedy(tn).toplevel), {}))
    return orc.permute_to(res, list(c.open_edges)).data


def inner_legs(c, count):
    """`count` legs shared by two of the circuit's gates, spread over the circuit"""
    seen = {}
    for t in c.tensors:
        for leg in t.legs:
            seen[leg] = seen.get(leg, 0) + 1
    legs = sorted(l for l, k in seen.items() if k == 2 and l not in c.open_edges)
    return [legs[(i + 1) * len(legs) // (count + 1)] for i in range(count)]


def numpy_candidate(seed, i):
    g = np.random.Philox(key=np.array([seed, 0], dtype=np.uint64), counter=(i - 1) % (1 << 256))
    w = [int(x) for x in g.random_raw(4)]
    return w, (w[1] >> 11) * 2.0 ** -53, (w[2] >> 11) * 2.0 ** -53


def host(s):
    return [int(w) & ((1 << 64) - 1) for w in s.bits.cpu().tolist()], s.probabilities.cpu().tolist()


def same(a, b):
    return host(a) == host(b) and (a.candidates, a.clipped, a.max_ratio, a.passes) == (b.candidates, b.clipped, b.max_ratio, b.passes)


def host_route(c, s, closed):
    """candidate `closed` ({qubit: bit}) through the host: its amplitude network sliced on the host, stage_slices +
    run_slices on the sampler's plan.  Returns the amplitudes in the row-major order of the result legs."""
    from tnc_b200.contractionpath.slicing import SlicedNetwork
    n = c.num_qubits()
    tn, _ = c.into_amplitude_network("".join("*" if q in s.open_qubits else str(closed[q]) for q in range(n)))
    sn = SlicedNetwork(tn, s.sliced_legs)
    s.plan.stage_slices([sn.slice(a) for a in sn.assignments])
    r = s.plan.run_slices(0, 1)
    assert [int(l) for l in r.legs] == [int(l) for l in s.plan.result_legs]
    return r.to_numpy().reshape(-1)


def kernel_pick(p, v):
    """the select kernel's pick restated: T = min(256, 2^k) chunks, each summed left to right, the chunk sums scanned
    left to right; y is the first outcome whose prefix exceeds v q.  Returns (y or None, q)."""
    K = len(p)
    T = min(256, K)
    L = K // T
    excl = [0.0]
    for t in range(T):
        s = 0.0
        for y in range(t * L, (t + 1) * L):
            s = s + float(p[y])
        excl.append(excl[-1] + s)
    q = excl[T]
    target = v * q
    for t in range(T):
        if excl[t] <= target < excl[t + 1]:
            s, y = 0.0, t * L
            while y < (t + 1) * L - 1:
                s = s + float(p[y])
                if excl[t] + s > target:
                    break
                y += 1
            return y, q
    return None, q


# ------------------------------------------------------------------------------------------------ 1. one staged network
def test_one_staged_network(ctx):
    from tnc_b200 import Sampler
    c = circuit(10, 21)
    opened = [2, 5, 8]
    tn, _ = c.into_amplitude_network("".join("*" if q in opened else "0" for q in range(10)))
    path = greedy(tn)
    plain = Sampler(c, opened, path=path, ctx=ctx)
    one = Sampler(c, opened, path=path, ctx=ctx, sliced_legs=[])
    assert one.n_slices == 1
    for batch in (1, 7, None):
        for m in (1e-9, 1.5):
            a = plain.sample(60, m, seed=3, first=11, max_candidates=300, batch=batch)
            b = one.sample(60, m, seed=3, first=11, max_candidates=300, batch=batch)
            assert same(a, b), (batch, m)
            assert a.bits.numel() > 0


# ------------------------------------------------------------------------------------------------ 2. the wiring
def test_wiring_exact(ctx):
    from tnc_b200 import Sampler
    n, k = 12, 3
    c = circuit(n, 22)
    opened = [1, 6, 10]
    for legs in (inner_legs(c, 2), inner_legs(c, 3)):
        s = Sampler(c, opened, ctx=ctx, sliced_legs=legs)
        assert s.n_slices == 1 << len(legs)
        seed, first, count = 5, 300, 48
        tiny = s.sample(count, 1e-9, seed=seed, first=first, max_candidates=count)   # every candidate with q > 0
        m = 1.5
        real = s.sample(count, m, seed=seed, first=first, max_candidates=count)
        bits, probs = host(tiny)
        got, got_p = host(real)
        at = acc = 0
        for i in range(count):
            w, u, v = numpy_candidate(seed, first + i)
            closed = {q: (w[0] >> j) & 1 for j, q in enumerate(s.closed_qubits)}
            a = host_route(c, s, closed)
            p = a.real * a.real + a.imag * a.imag
            y, q = kernel_pick(p, v)
            r = (q * 2.0 ** (n - k)) / m
            if u < r:                                    # accepted with m: the next sample of the realistic call
                word = sum(b << qb for qb, b in closed.items()) | sum(((y >> (k - 1 - j)) & 1) << qb
                                                                      for j, qb in enumerate(s.result_qubits))
                assert got[acc] == word and got_p[acc] == float(p[y]), i
                acc += 1
            if y is None:                                # q == 0: never accepted
                continue
            word = sum(b << qb for qb, b in closed.items())
            word |= sum(((y >> (k - 1 - j)) & 1) << qb for j, qb in enumerate(s.result_qubits))
            assert bits[at] == word, (i, bits[at], word)
            assert probs[at] == float(p[y]), i
            at += 1
        assert at == len(bits) == tiny.clipped and tiny.candidates == count and at > count // 2
        assert acc == len(got) and 0 < acc < count and real.candidates == count


# ------------------------------------------------------------------------------------------------ 3. the distribution
@pytest.mark.parametrize("k", [0, 4, 12])
def test_distribution(ctx, k):
    from scipy import stats
    from tnc_b200 import Sampler
    n = 12
    c = circuit(n, 31)
    psi = statevector(c)
    p = (psi.real ** 2 + psi.imag ** 2).reshape(-1)       # index: qubit 0 is the most significant bit
    opened = list(range(0, n, n // k)) if 0 < k < n else list(range(k))
    s = Sampler(c, opened, ctx=ctx, sliced_legs=inner_legs(c, 2))
    q_c = (psi.real ** 2 + psi.imag ** 2).sum(axis=tuple(opened)) if opened else p.reshape(psi.shape)
    m = 1.01 * float(np.max(q_c)) * 2.0 ** (n - k)
    N = 200_000
    out = s.sample(N, m, seed=5, max_candidates=N)
    assert out.candidates == N and out.clipped == 0 and out.max_ratio <= 1.0
    words, probs = host(out)
    S = len(words)
    frac, want = S / N, 1.0 / m * p.sum()
    assert abs(frac - want) <= 5 * math.sqrt(want * (1 - want) / N), (frac, want)
    index = np.array([sum(((w >> q) & 1) << (n - 1 - q) for q in range(n)) for w in words])
    np.testing.assert_allclose(np.asarray(probs), p[index], rtol=1e-10, atol=0)
    counts = np.bincount(index, minlength=1 << n).astype(np.float64)
    expect = S * p / p.sum()
    small = expect < 5
    obs = np.append(counts[~small], counts[small].sum())
    exp = np.append(expect[~small], expect[small].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    pval = stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue
    assert pval > 1e-6, pval


# ------------------------------------------------------------------------------------------------ 4. reproducibility
def test_reproducible(ctx):
    from tnc_b200 import Sampler
    c = circuit(10, 41)
    s = Sampler(c, [1, 6], ctx=ctx, sliced_legs=inner_legs(c, 2))
    before = s.plan.run_slices(0, 1).to_numpy()
    m = 2.0
    a = s.sample(40, m, seed=9)
    assert same(a, s.sample(40, m, seed=9))
    assert host(s.sample(40, m, seed=10)) != host(a)
    for batch in (1, 7):
        x = s.sample(40, m, seed=9, batch=batch)
        assert host(x) == host(a) and (x.candidates, x.clipped, x.max_ratio) == (a.candidates, a.clipped, a.max_ratio)
    one = s.sample(15, m, seed=9)
    two = s.sample(25, m, seed=9, first=one.next_candidate)
    wa, pa = host(a)
    w1, p1 = host(one)
    w2, p2 = host(two)
    assert w1 + w2 == wa and p1 + p2 == pa
    assert one.candidates + two.candidates == a.candidates and two.next_candidate == a.next_candidate
    assert one.clipped + two.clipped == a.clipped and max(one.max_ratio, two.max_ratio) == a.max_ratio
    assert np.array_equal(s.plan.run_slices(0, 1).to_numpy(), before)


# ------------------------------------------------------------------------------------------------ 5. the in-place pass
def test_in_place_pass(built_lib):
    """Device memory is held by a torch tensor until the device has no room for one workspace copy beside the plan's
    (the arena keeps 1 GiB free): the call then runs in the plan's own workspace.  This exercises a documented memory
    path; the tensor is released in `finally`."""
    import torch
    import tnc_b200 as tb
    from tnc_b200 import Sampler, TncbError
    from tnc_b200.contractionpath.slicing import SlicedNetwork
    own = tb.Context(0)                     # a fresh arena: at most one 256 MiB slab of slack
    try:
        c = circuit(10, 71)
        s = Sampler(c, [0, 4, 7], ctx=own, sliced_legs=inner_legs(c, 2))
        tn, _ = c.into_amplitude_network("".join("*" if q in s.open_qubits else "0" for q in range(10)))
        net0 = SlicedNetwork(tn, s.sliced_legs).slice((0, 0))
        s.plan.stage(net0)
        staged = s.plan.run().to_numpy()
        sums = s.plan.run_slices(0, 1).to_numpy()
        s.plan.stage(net0)
        copies = s.sample(30, 1.5, seed=4, max_candidates=400)
        assert np.array_equal(s.plan.run().to_numpy(), staged)       # the copies route leaves the staged leaves alone
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info()
        hold = None
        try:
            hold = torch.empty(max(free - (256 << 20), 0), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info()[0] < (1 << 30)
            inplace = s.sample(30, 1.5, seed=4, max_candidates=400)
            torch.cuda.synchronize()
        finally:
            del hold
            torch.cuda.empty_cache()
        assert host(inplace) == host(copies)
        assert (inplace.candidates, inplace.clipped, inplace.max_ratio) == (copies.candidates, copies.clipped, copies.max_ratio)
        assert inplace.passes == inplace.candidates > copies.passes          # one candidate per pass: in place
        with pytest.raises(TncbError) as e:
            s.plan.run()
        assert e.value.status == ERR_INVALID and "tncb_plan_stage has not been called" in str(e.value)
        assert np.array_equal(s.plan.run_slices(0, 1).to_numpy(), sums)
        s.plan.stage(net0)
        assert np.array_equal(s.plan.run().to_numpy(), staged)
        del s
    finally:
        own.close()


# ------------------------------------------------------------------------------------------------ 6. benchmark scale
def test_sycamore_d12(ctx, record_property):
    """the committed depth-12 tree with its 64 slices and ten qubits open, two candidates at tiny m: each p and pick
    against the host route on the same plan, run after sampling (two 32.5 GiB workspaces do not fit together)"""
    import json
    import os
    import torch
    from tnc_b200 import Sampler
    from tnc_b200.builders import sycamore_circuit
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.sampling import open_path
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "bench_inputs", "sycamore53_d12.json")) as f:
        d = json.load(f)
    n, k = 53, len(D12_OPEN)
    c = sycamore_circuit(n, 12, np.random.default_rng(1))
    path = open_path(c, ContractionPath.simple([tuple(x) for x in d["toplevel"]]), D12_OPEN)
    s = Sampler(c, D12_OPEN, path=path, ctx=ctx, sliced_legs=d["sliced_legs"])
    assert s.n_slices == 64
    free, _ = torch.cuda.mem_get_info()
    record_property("copy_fits_beside_plan", free > s.plan.info()["peak_bytes"] + ((1 << 30) + (12 << 30)))
    out = s.sample(2, 1e-12, seed=1, max_candidates=2, batch=1)
    assert out.candidates == 2 and out.passes == out.candidates
    bits, probs = host(out)
    assert len(bits) == out.clipped
    at = 0
    for i in range(2):
        w, u, v = numpy_candidate(1, i)
        closed = {q: (w[0] >> j) & 1 for j, q in enumerate(s.closed_qubits)}
        a = host_route(c, s, closed)
        p = a.real * a.real + a.imag * a.imag
        y, q = kernel_pick(p, v)
        if y is None:
            continue
        word = sum(b << qb for qb, b in closed.items())
        word |= sum(((y >> (k - 1 - j)) & 1) << qb for j, qb in enumerate(s.result_qubits))
        assert bits[at] == word and probs[at] == float(p[y]), i
        at += 1
    assert at == len(bits) == 2


# ------------------------------------------------------------------------------------------------ 7. refusals
def test_refusals(ctx, monkeypatch):
    import torch
    from tnc_b200 import Sampler
    from tnc_b200._lib import TncbSampleSpec, TncbSampleStats, u64_array
    from tnc_b200.contractionpath.slicing import SlicedNetwork
    from tnc_b200.tensornetwork import NetworkPlan
    l = ctx._l
    c = circuit(6, 61)
    s = Sampler(c, [1, 4], ctx=ctx, sliced_legs=inner_legs(c, 1))
    want = s.plan.run_slices(0, 1).to_numpy()
    tn, _ = c.into_amplitude_network("".join("*" if q in s.open_qubits else "0" for q in range(6)))
    path = greedy(tn)

    def spec(n=6, leaves=None, closed=None, result=None):
        leaves = list(s.closed_leaves) if leaves is None else leaves
        closed = list(s.closed_qubits) if closed is None else closed
        result = list(s.result_qubits) if result is None else result
        keep = (u64_array(leaves), (C.c_int * max(len(closed), 1))(*closed), (C.c_int * max(len(result), 1))(*result))
        sp = TncbSampleSpec(n, len(closed), *keep)
        sp._keep = keep
        return sp

    torch.cuda.empty_cache()
    words = 1 << 21           # 16 MiB: above 10 MiB the caching allocator gives a block its own allocation of this size
    bits = torch.empty(words, dtype=torch.int64, device="cuda")
    probs = torch.empty(words, dtype=torch.float64, device="cuda")
    stats = TncbSampleStats()

    def call(plan=None, sp=None, m=2.0, max_samples=8, b=None, p=None, st=True):
        return l.tncb_plan_sample_slices(ctx.handle, (plan or s.plan).handle, None if sp is False else C.byref(sp or spec()),
                                         1, 0, 100, max_samples, m, 0, bits.data_ptr() if b is None else b,
                                         probs.data_ptr() if p is None else p, C.byref(stats) if st else None)

    grad = NetworkPlan.for_gradients(tn, path, ctx=ctx)
    grad.stage(tn)
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    loose = NetworkPlan(tn, path, ctx=ctx)
    loose.stage(tn)
    monkeypatch.delenv("TNCB_NO_STATIC")
    only_staged = NetworkPlan(tn, path, ctx=ctx)
    only_staged.stage(tn)                   # staged, but no slices
    bra = c.open_edges[s.closed_qubits[0]]
    sn = SlicedNetwork(tn, [bra])           # a sliced leg on a closed bra: that bra becomes a rank-0 leaf
    on_bra = NetworkPlan(sn.slice((0,)), path, ctx=ctx)
    on_bra.stage_slices([sn.slice(a) for a in sn.assignments])
    host_words = np.zeros(8, dtype=np.uint64)
    gate_leaf = next(i for i, t in enumerate(c.tensors) if len(t.legs) == 4)
    cases = [
        (ERR_INVALID, "null argument", dict(sp=False)),
        (ERR_INVALID, "null argument", dict(st=False)),
        (ERR_INVALID, "null argument", dict(b=0)),
        (ERR_INVALID, "n_qubits 0 is outside 1..64", dict(sp=spec(n=0))),
        (ERR_INVALID, "n_qubits 65 is outside 1..64", dict(sp=spec(n=65))),
        (ERR_INVALID, "closed leaf 999 is out of range", dict(sp=spec(leaves=[999] + s.closed_leaves[1:]))),
        (ERR_INVALID, "is listed twice", dict(sp=spec(leaves=[s.closed_leaves[0]] * 4))),
        (ERR_INVALID, f"closed leaf {gate_leaf} is not a rank-1 leaf of dimension 2",
         dict(sp=spec(leaves=[gate_leaf] + s.closed_leaves[1:]))),
        (ERR_INVALID, f"closed leaf {s.closed_leaves[0]} is not a rank-1 leaf of dimension 2", dict(plan=on_bra)),
        (ERR_INVALID, "qubit 4 is listed twice", dict(sp=spec(closed=s.closed_qubits[:-1] + [4]))),
        (ERR_INVALID, "qubit 5 is neither closed nor on a result leg",
         dict(sp=spec(leaves=s.closed_leaves[:-1], closed=s.closed_qubits[:-1]))),
        (ERR_INVALID, "m must be finite and > 0", dict(m=float("nan"))),
        (ERR_INVALID, "m must be finite and > 0", dict(m=0.0)),
        (ERR_INVALID, "max_samples is 0", dict(max_samples=0)),
        (ERR_INVALID, "bits: the buffer is not device memory", dict(b=host_words.ctypes.data)),
        (ERR_INVALID, "bits: the buffer is not 8-byte aligned", dict(b=bits.data_ptr() + 4)),
        (ERR_INVALID, f"probs: the buffer's {8 * 9} bytes run past the end of its allocation",
         dict(max_samples=9, p=probs.data_ptr() + 8 * (words - 8))),
        (ERR_INVALID, "tncb_plan_stage_slices has not been called on this context", dict(plan=only_staged)),
        (ERR_UNSUPPORTED, "tncb_plan_sample_slices takes a plain plan (tncb_plan_create)", dict(plan=grad)),
        (ERR_UNSUPPORTED, "static layout", dict(plan=loose)),
    ]
    live = ctx.stats()["arena_live_bytes"]
    for status, msg, kw in cases:
        assert call(**kw) == status, msg
        assert msg in l.tncb_last_error().decode(), (msg, l.tncb_last_error().decode())
        assert ctx.stats()["arena_live_bytes"] == live, msg
    assert np.array_equal(s.plan.run_slices(0, 1).to_numpy(), want)
    assert call() == 0 and stats.samples == 8
    assert np.array_equal(s.plan.run_slices(0, 1).to_numpy(), want)
