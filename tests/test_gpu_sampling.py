"""Sampling on the H100 (tncb_plan_sample, tnc_b200.Sampler).

  1. the random stream's wiring, exactly: closed bits = numpy Philox's w0, open bits = the inverse-CDF pick recomputed
     from the oracle's state vector with numpy's v, accept / reject = u < r with numpy's u;
  2. the distribution: a chi-square test of 2e5 candidates against p, and the accepted fraction against 1/M;
  3. reproducibility: seeds, pass sizes, calls split in two, and the plan's staged leaves left alone;
  4. every returned p against |amplitude|^2 of its bitstring, contracted closed;
  5. bench.py's 36-qubit circuit with qubits 0-3 open, each p against an independent closed contraction;
  6. every refusal of the C ABI, with the arena and the staged plan unchanged."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

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


def to_oracle(t):
    if t.is_composite():
        return orc.OTensor(children=[to_oracle(c) for c in t.tensors])
    td = t.tensordata
    d = ("gate", td.gate[0], td.gate[1], td.gate[2]) if td.kind == "gate" else np.asarray(td.matrix)
    return orc.OTensor(list(t.legs), list(t.bond_dims), d)


def to_opath(p):
    return orc.OPath(list(p.toplevel), {i: to_opath(q) for i, q in p.nested.items()})


def circuit(n, seed, rounds=5):
    from tnc_b200.builders.random_circuit import random_circuit_builder
    return random_circuit_builder(n, rounds, 0.5, 0.5, np.random.default_rng(seed))


def statevector(c):
    """the oracle's state vector of circuit c, shaped [2] * n with axis q = qubit q"""
    tn, _ = c.into_statevector_network()
    res = orc.contract_tensor_network(to_oracle(tn), to_opath(greedy(tn)))
    return orc.permute_to(res, list(c.open_edges)).data


def outcome_probs(psi, s, closed):
    """p(c, y) over y in the row-major order of s's result legs, for the closed assignment {qubit: bit} `closed`"""
    n = psi.ndim
    idx = [slice(None)] * n
    for q, b in closed.items():
        idx[q] = b
    sub = psi[tuple(idx)]                          # remaining axes: the open qubits in ascending order
    opened = sorted(s.result_qubits)
    sub = np.transpose(sub, [opened.index(q) for q in s.result_qubits])
    return (sub.real * sub.real + sub.imag * sub.imag).reshape(-1)


def numpy_candidate(seed, i):
    g = np.random.Philox(key=np.array([seed, 0], dtype=np.uint64), counter=(i - 1) % (1 << 256))
    w = [int(x) for x in g.random_raw(4)]
    return w, (w[1] >> 11) * 2.0 ** -53, (w[2] >> 11) * 2.0 ** -53


def host(s):
    return [int(w) & ((1 << 64) - 1) for w in s.bits.cpu().tolist()], s.probabilities.cpu().tolist()


# ------------------------------------------------------------------------------------------------ 1. the stream's wiring
def test_stream_wiring(ctx):
    from tnc_b200 import Sampler
    c = circuit(10, 21)
    psi = statevector(c)
    s = Sampler(c, [2, 5, 8], ctx=ctx)
    seed, first, count = 77, 1000, 300
    n, k = 10, 3
    out = s.sample(count, 1e-9, seed=seed, first=first, max_candidates=count)      # every candidate with q > 0 accepted
    bits, probs = host(out)
    at = checked = 0
    for i in range(count):
        w, u, v = numpy_candidate(seed, first + i)
        closed = {q: (w[0] >> j) & 1 for j, q in enumerate(s.closed_qubits)}
        p = outcome_probs(psi, s, closed)
        cdf = np.cumsum(p)
        q = cdf[-1]
        if q == 0:                                     # r = 0: never accepted
            continue
        for qb, b in closed.items():
            assert (bits[at] >> qb) & 1 == b, (i, qb)
        target = v * q
        if np.min(np.abs(cdf - target)) >= 1e-12 * q:
            y = int(np.argmax(cdf > target))
            for r, qb in enumerate(s.result_qubits):
                assert (bits[at] >> qb) & 1 == (y >> (k - 1 - r)) & 1, (i, r)
            assert abs(probs[at] - p[y]) <= 1e-12 * q
            checked += 1
        at += 1
    assert at == len(bits) == out.clipped and out.candidates == count and checked >= at - 3 and at > count // 3
    # accept / reject with a realistic M: sample i comes from the i-th accepted candidate
    m = 1.3
    out = s.sample(count, m, seed=seed, first=first, max_candidates=count)
    got, _ = host(out)
    accepted = []
    for i in range(count):
        w, u, v = numpy_candidate(seed, first + i)
        closed = {q: (w[0] >> j) & 1 for j, q in enumerate(s.closed_qubits)}
        r = outcome_probs(psi, s, closed).sum() * 2.0 ** (n - k) / m
        accepted.append((i, w[0], abs(u - r) < 1e-12 * r, u < r))
    assert 0 < len(got) < count
    # the accepted candidates, in candidate order; a decision within 1e-12 r of the boundary may go either way
    closed_of = lambda word: [(word >> q) & 1 for q in s.closed_qubits]
    at = 0
    for i, w0, near, acc in accepted:
        mine = at < len(got) and closed_of(got[at]) == [(w0 >> j) & 1 for j in range(len(s.closed_qubits))]
        if near:
            at += mine
            continue
        assert acc == mine, i
        at += acc
    assert at == len(got)
    assert out.candidates == count and out.max_ratio > 0


# ------------------------------------------------------------------------------------------------ 2. the distribution
@pytest.mark.parametrize("k", [0, 4, 12])
def test_distribution(ctx, k):
    from scipy import stats
    from tnc_b200 import Sampler
    n = 12
    c = circuit(n, 31)
    psi = statevector(c)
    p = (psi.real ** 2 + psi.imag ** 2).reshape(-1)       # index: qubit 0 is the most significant bit
    opened = list(range(0, n, n // k)) if 0 < k < n else list(range(k))
    s = Sampler(c, opened, ctx=ctx)
    closed_axes = [q for q in range(n) if q not in opened]
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
    assert pval > 1e-6, (pval, closed_axes)


# ------------------------------------------------------------------------------------------------ 3. reproducibility
def test_reproducible(ctx):
    from tnc_b200 import Sampler
    c = circuit(10, 41)
    s = Sampler(c, [1, 6], ctx=ctx)
    before = s.plan.run().to_numpy()
    m = 2.0
    a = s.sample(40, m, seed=9)
    b = s.sample(40, m, seed=9)
    assert host(a) == host(b) and a.candidates == b.candidates and a.clipped == b.clipped and a.max_ratio == b.max_ratio
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
    assert np.array_equal(s.plan.run().to_numpy(), before)
    # an unreachable target ends after max_candidates
    few = s.sample(1000, m, seed=9, max_candidates=50)
    assert few.candidates == 50 and few.bits.numel() < 1000 and host(few)[0] == wa[:few.bits.numel()]


# ------------------------------------------------------------------------------------------------ 4. probabilities
def test_probabilities(ctx):
    from tnc_b200 import Sampler
    from tnc_b200.tensornetwork import contract_tensor_network
    c = circuit(11, 51)
    s = Sampler(c, [0, 3, 4, 9], ctx=ctx)
    out = s.sample(24, 2.0, seed=3)
    _, probs = host(out)
    strings = out.bitstrings()
    path = None
    for st, p in zip(strings, probs):
        tn, _ = c.into_amplitude_network(st)
        path = path or greedy(tn)
        amp = complex(contract_tensor_network(tn, path, ctx=ctx).to_numpy().reshape(()))
        want = amp.real ** 2 + amp.imag ** 2
        assert abs(p - want) <= 1e-12 * want, (st, p, want)


# ------------------------------------------------------------------------------------------------ 5. benchmark scale
def test_bench_scale(ctx):
    from tnc_b200 import Sampler
    from tnc_b200.builders.random_circuit import random_circuit_builder
    from tnc_b200.tensornetwork import NetworkPlan
    c = random_circuit_builder(36, 10, 0.5, 0.5, np.random.default_rng(1))
    s = Sampler(c, [0, 1, 2, 3], ctx=ctx)
    out = s.sample(32, 3.0, seed=1)
    assert out.bits.numel() == 32
    assert math.isfinite(out.max_ratio) and out.max_ratio > 0
    assert 32 <= out.candidates and out.clipped <= out.candidates
    _, probs = host(out)
    tn0, _ = c.into_amplitude_network("0" * 36)
    plan = NetworkPlan(tn0, greedy(tn0), ctx=ctx)
    for st, p in zip(out.bitstrings(), probs):
        tn, _ = c.into_amplitude_network(st)
        amp = complex(plan.execute(tn).to_numpy().reshape(()))
        want = amp.real ** 2 + amp.imag ** 2
        assert abs(p - want) <= 1e-10 * want, (st, p, want)


# ------------------------------------------------------------------------------------------------ 6. refusals
def test_refusals(ctx, monkeypatch):
    import torch
    from tnc_b200 import Sampler
    from tnc_b200._lib import TncbSampleSpec, TncbSampleStats, u64_array
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    l = ctx._l
    c = circuit(6, 61)
    s = Sampler(c, [1, 4], ctx=ctx)
    want = s.plan.run().to_numpy()
    n_gates = len(c.tensors)

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

    def call(plan=None, sp=None, m=2.0, max_samples=8, b=None, p=None, st=True, ctxh=None):
        return l.tncb_plan_sample(ctx.handle if ctxh is None else ctxh, (plan or s.plan).handle, None if sp is False else C.byref(sp or spec()),
                                  1, 0, 100, max_samples, m, 0, bits.data_ptr() if b is None else b,
                                  probs.data_ptr() if p is None else p, C.byref(stats) if st else None)

    grad = NetworkPlan.for_gradients(*_amplitude(c, s), ctx=ctx)
    grad.stage(_amplitude(c, s)[0])
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    loose = NetworkPlan(*_amplitude(c, s), ctx=ctx)
    loose.stage(_amplitude(c, s)[0])
    monkeypatch.delenv("TNCB_NO_STATIC")
    unstaged = NetworkPlan(*_amplitude(c, s), ctx=ctx)
    odd = _odd_plan(ctx)
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
        (ERR_INVALID, "qubit 4 is listed twice", dict(sp=spec(closed=s.closed_qubits[:-1] + [4]))),
        (ERR_INVALID, "qubit 5 is neither closed nor on a result leg",
         dict(sp=spec(leaves=s.closed_leaves[:-1], closed=s.closed_qubits[:-1]))),
        (ERR_INVALID, "closed qubit 0 is qubit 9, outside 0..5", dict(sp=spec(closed=[9] + s.closed_qubits[1:]))),
        (ERR_INVALID, "m must be finite and > 0", dict(m=float("nan"))),
        (ERR_INVALID, "m must be finite and > 0", dict(m=float("inf"))),
        (ERR_INVALID, "m must be finite and > 0", dict(m=0.0)),
        (ERR_INVALID, "max_samples is 0", dict(max_samples=0)),
        (ERR_INVALID, "bits: the buffer is not device memory", dict(b=host_words.ctypes.data)),
        (ERR_INVALID, "bits: the buffer is not 8-byte aligned", dict(b=bits.data_ptr() + 4)),
        (ERR_INVALID, f"bits: the buffer's {8 * (words + 1)} bytes run past the end of its allocation",
         dict(max_samples=words + 1, p=probs.data_ptr())),
        (ERR_INVALID, f"probs: the buffer's {8 * 9} bytes run past the end of its allocation",
         dict(max_samples=9, p=probs.data_ptr() + 8 * (words - 8))),
        (ERR_INVALID, "tncb_plan_stage has not been called", dict(plan=unstaged)),
        (ERR_UNSUPPORTED, "tncb_plan_sample takes a plain plan", dict(plan=grad)),
        (ERR_UNSUPPORTED, "static layout", dict(plan=loose)),
        (ERR_INVALID, "result leg 0 has dimension 3, not 2", dict(plan=odd[0], sp=odd[1])),
    ]
    live = ctx.stats()["arena_live_bytes"]
    for status, msg, kw in cases:
        assert call(**kw) == status, msg
        assert msg in l.tncb_last_error().decode(), (msg, l.tncb_last_error().decode())
        assert ctx.stats()["arena_live_bytes"] == live, msg
    assert np.array_equal(s.plan.run().to_numpy(), want)
    # a valid call through the same arguments
    assert call() == 0 and stats.samples == 8


def _amplitude(c, s):
    tn, _ = c.into_amplitude_network("".join("*" if q in s.open_qubits else "0" for q in range(c.num_qubits())))
    return tn, greedy(tn)


def _odd_plan(ctx):
    """a staged plain plan whose one result leg has dimension 3, and a spec naming it"""
    from tnc_b200._lib import TncbSampleSpec
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import NetworkPlan, Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    a = Tensor([0, 1], [2, 3])
    a.set_tensor_data(TensorData.Matrix(np.arange(6, dtype=np.complex128).reshape(2, 3)))
    b = Tensor([0], [2])
    b.set_tensor_data(TensorData.Matrix(np.array([1, 0], dtype=np.complex128)))
    tn = Tensor.new_composite([a, b])
    plan = NetworkPlan(tn, ContractionPath.simple([(0, 1)]), ctx=ctx)
    plan.stage(tn)
    result = (C.c_int * 1)(0)
    sp = TncbSampleSpec(1, 0, None, None, result)
    sp._keep = result
    return plan, sp
