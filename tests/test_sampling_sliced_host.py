"""Sampling sliced circuits without a GPU: the sample_slices cell of the kind table on host-only plans of all seven kinds;
what Sampler(..., sliced_legs=...) passes to the library (the plan created by the real library on a NULL context, every
later entry answered by a recorder); every ValueError of sliced_legs and of open_path; open_path against the oracle's
state vector; and the cost of the committed Sycamore-53 depth-12 tree with ten qubits open."""
import ctypes as C
import json
import os
import types

import numpy as np
import pytest

from oracle import tnc_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_UNSUPPORTED = -1, -9
KINDS = ["plain", "vjp", "jvp", "hvp", "sliced vjp", "sliced jvp", "sliced hvp"]
D12_OPEN = [2, 8, 12, 13, 16, 18, 22, 29, 32, 35]


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def circuit(n, seed, rounds=4):
    from tnc_b200.builders.random_circuit import random_circuit_builder
    return random_circuit_builder(n, rounds, 0.5, 0.5, np.random.default_rng(seed))


def to_oracle(t):
    if t.is_composite():
        return orc.OTensor(children=[to_oracle(c) for c in t.tensors])
    td = t.tensordata
    d = ("gate", td.gate[0], td.gate[1], td.gate[2]) if td.kind == "gate" else np.asarray(td.matrix)
    return orc.OTensor(list(t.legs), list(t.bond_dims), d)


def open_network(c, opened, closed_bits=None):
    n = c.num_qubits()
    bit = lambda q: "*" if q in opened else ("0" if closed_bits is None else str(closed_bits[q]))
    return c.into_amplitude_network("".join(bit(q) for q in range(n)))[0]


# ------------------------------------------------------------------------------------------------ the route cell
def test_sample_slices_route_cell(built_lib):
    from tnc_b200._lib import TncbSampleSpec, TncbSampleStats, u64_array
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork.contraction import _Marshal
    l = built_lib
    c = circuit(12, 5, rounds=6)
    tn = c.into_amplitude_network("0" * 12)[0]
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    fake_ctx = C.create_string_buffer(1 << 16)
    cx = C.cast(fake_ctx, C.c_void_p)
    result = (C.c_int * 1)(0)
    spec = TncbSampleSpec(12, 0, None, None, result)
    stats = TncbSampleStats()
    got = []
    for kind in KINDS:
        m = _Marshal()
        ct, cp = m.tn(tn), m.path(path)
        h = C.c_void_p()
        if kind == "plain":
            rc = l.tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h))
        elif kind.startswith("sliced "):
            rc = getattr(l, f"tncb_plan_create_{kind[7:]}_sliced")(None, C.byref(ct), C.byref(cp), len(legs), u64_array(legs),
                                                                  None, C.byref(h))
        else:
            rc = getattr(l, f"tncb_plan_create_{kind}")(None, C.byref(ct), C.byref(cp), None, C.byref(h))
        assert rc == 0, l.tncb_last_error()
        rc = l.tncb_plan_sample_slices(cx, h, C.byref(spec), 1, 0, 10, 1, 2.0, 0, C.c_void_p(0x1000), None, C.byref(stats))
        got.append((rc, l.tncb_last_error().decode()))
        l.tncb_plan_destroy(h)
    refuse = (ERR_UNSUPPORTED, "tncb_plan_sample_slices takes a plain plan (tncb_plan_create)")
    assert got == [(ERR_INVALID, "tncb_plan_stage_slices has not been called on this context")] + [refuse] * 6


# ------------------------------------------------------------------------------------------------ Sampler's arguments
class Recorder:
    """Stands in for the library: plan creation and metadata pass through, every other entry is logged; the sample
    entries report `stats`"""

    def __init__(self, lib, log, stats):
        self._lib, self._log, self._stats = lib, log, stats

    def __getattr__(self, name):
        if name in ("tncb_network_out_legs", "tncb_plan_destroy", "tncb_last_error") or name.startswith("tncb_plan_create"):
            return getattr(self._lib, name)
        return lambda *args: self._call(name, args)

    def _call(self, name, args):
        row = [name]
        for a in args[1:]:
            if type(a).__name__ == "CArgObject":
                obj = a._obj
                if type(obj).__name__ == "TncbSampleSpec":
                    k = obj.n_qubits - obj.n_closed
                    row.append({"n_qubits": obj.n_qubits, "closed_leaf": [obj.closed_leaf[j] for j in range(obj.n_closed)],
                                "closed_qubit": [obj.closed_qubit[j] for j in range(obj.n_closed)],
                                "result_qubit": [obj.result_qubit[r] for r in range(k)]})
                elif type(obj).__name__ == "TncbSampleStats":
                    for f, v in self._stats.items():
                        setattr(obj, f, v)
                    row.append("stats")
                else:
                    row.append(type(obj).__name__)
            elif isinstance(a, C.c_void_p):
                row.append("handle" if a.value else None)
            elif isinstance(a, C.Array):
                row.append(("array", len(a)))
            else:
                row.append(a)
        self._log.append(tuple(row))
        return 0


@pytest.fixture
def recorded(built_lib, monkeypatch):
    import torch
    import tnc_b200 as tb
    log = []
    stats = {"candidates": 40, "samples": 3, "clipped": 2, "passes": 2, "max_ratio": 1.5}
    ctx = types.SimpleNamespace(_l=Recorder(built_lib, log, stats), handle=None, device=0)

    class Stream:
        def __init__(self, name):
            self.name = name

        def wait_stream(self, other):
            log.append(("wait", self.name, other.name))

    cpu_empty = torch.empty
    monkeypatch.setattr(tb, "torch_streams", lambda ctx: (Stream("torch"), Stream("ctx")))
    monkeypatch.setattr(torch, "empty", lambda *shape, dtype=None, device=None: cpu_empty(*shape, dtype=dtype))
    samplers = []
    yield ctx, log, samplers
    for s in samplers:
        built_lib.tncb_plan_destroy(s.plan.handle)
        s.plan.handle = None


def _sample_row(log, name):
    (row,) = [r for r in log if r[0] == name]
    return row[:1] + row[1:3] + row[3:9] + row[11:]       # without the two output addresses


def test_sampler_sliced_calls(recorded):
    from tnc_b200 import Sampler
    from tnc_b200.contractionpath.slicing import SlicedNetwork
    ctx, log, samplers = recorded
    c = circuit(8, 3)
    opened = [6, 1]
    tn = open_network(c, opened)
    path = greedy(tn)
    closed_bra_legs = {c.open_edges[q] for q in range(8) if q not in opened}
    shared = {}
    for t in tn.tensors:
        for leg in t.legs:
            shared[leg] = shared.get(leg, 0) + 1
    legs = [l for l in sorted(shared) if shared[l] == 2 and l not in closed_bra_legs][3:6]
    plain = Sampler(c, opened, path=path, ctx=ctx)
    samplers.append(plain)
    assert [row[0] for row in log] == ["tncb_plan_stage"] and plain.n_slices == 1 and plain.sliced_legs is None
    plain.sample(7, 2.5, seed=11, first=100, max_candidates=5000, batch=9)
    want = _sample_row(log, "tncb_plan_sample")
    del log[:]
    s = Sampler(c, opened, path=path, ctx=ctx, sliced_legs=legs)
    samplers.append(s)
    assert s.n_slices == 8 and s.sliced_legs == legs
    assert log == [("tncb_plan_stage_slices", "handle", 8, ("array", 8))]
    assert (s.closed_leaves, s.closed_qubits, s.result_qubits) == (plain.closed_leaves, plain.closed_qubits, plain.result_qubits)
    # one slice's structure: the sliced legs are gone from the plan's leaves
    assert [list(t.legs) for t in SlicedNetwork(tn, legs).slice((0, 0, 0)).tensors] == [
        [l for l in t.legs if l not in legs] for t in tn.tensors]
    del log[:]
    out = s.sample(7, 2.5, seed=11, first=100, max_candidates=5000, batch=9)
    assert [row[0] for row in log if row[0].startswith("tncb")] == ["tncb_plan_sample_slices"]
    assert _sample_row(log, "tncb_plan_sample_slices")[1:] == want[1:]
    assert log[0] == ("wait", "ctx", "torch") and log[-1] == ("wait", "torch", "ctx")
    assert (out.candidates, out.clipped, out.max_ratio, out.next_candidate, out.passes) == (40, 2, 1.5, 140, 2)


def test_sliced_legs_refusals(recorded):
    from tnc_b200 import Sampler
    ctx, log, samplers = recorded
    c = circuit(6, 4)
    opened = [1, 4]
    tn = open_network(c, opened)
    inner = next(l for l in tn.tensors[0].legs if sum(l in t.legs for t in tn.tensors) == 2
                 and l not in c.open_edges)
    cases = [
        ([inner, inner], f"sliced leg {inner} is listed twice"),
        ([c.open_edges[0]], f"sliced leg {c.open_edges[0]} lies on the bra of closed qubit 0"),
        ([c.open_edges[4]], f"sliced leg {c.open_edges[4]} is the open leg of qubit 4"),
        ([10 ** 6], "sliced leg 1000000 is not shared by two leaves"),
    ]
    for legs, msg in cases:
        with pytest.raises(ValueError, match=msg):
            Sampler(c, opened, ctx=ctx, sliced_legs=legs)
    assert log == []


# ------------------------------------------------------------------------------------------------ open_path
def test_open_path_refusals():
    from tnc_b200.contractionpath import ContractionPath, path
    from tnc_b200.sampling import open_path
    c = circuit(6, 4)
    closed = greedy(c.into_amplitude_network("0" * 6)[0])
    with pytest.raises(ValueError, match="nested paths"):
        open_path(c, path((0, 1), nested={1: [(0, 1)]}), [1])
    with pytest.raises(ValueError, match="open qubits"):
        open_path(c, closed, [1, 1])
    with pytest.raises(ValueError, match="open qubits"):
        open_path(c, closed, [6])
    with pytest.raises(ValueError, match="outside the closed network"):
        open_path(c, ContractionPath.simple([(0, 999)]), [1])


@pytest.mark.parametrize("n,seed,opened", [(8, 11, [0, 5]), (9, 12, [2, 3, 8]), (10, 13, [9]), (10, 14, [1, 4, 6, 7])])
def test_open_path_oracle(built_lib, n, seed, opened):
    """the derived path contracts the open network to the state vector's slice of the open qubits, for several closed
    assignments; the library compiles it"""
    from tnc_b200.sampling import open_path
    from tnc_b200.tensornetwork.contraction import _Marshal
    c = circuit(n, seed)
    closed_tn = c.into_amplitude_network("0" * n)[0]
    p = open_path(c, greedy(closed_tn), opened)
    assert p.is_simple() and len(p.toplevel) == len(closed_tn.tensors) - len(opened) - 1
    sv_tn, _ = c.into_statevector_network()
    psi = orc.permute_to(orc.contract_tensor_network(to_oracle(sv_tn), orc.OPath(list(greedy(sv_tn).toplevel), {})),
                         list(c.open_edges)).data
    rng = np.random.default_rng(seed)
    for _ in range(4):
        bits = {q: int(rng.integers(2)) for q in range(n) if q not in opened}
        tn = open_network(c, opened, bits)
        res = orc.contract_tensor_network(to_oracle(tn), orc.OPath(list(p.toplevel), {}))
        got = orc.permute_to(res, [c.open_edges[q] for q in sorted(opened)]).data
        want = psi[tuple(bits.get(q, slice(None)) for q in range(n))]
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    m = _Marshal()
    ct, cp = m.tn(open_network(c, opened)), m.path(p)
    h = C.c_void_p()
    assert built_lib.tncb_plan_create(None, C.byref(ct), C.byref(cp), C.byref(h)) == 0, built_lib.tncb_last_error()
    built_lib.tncb_plan_destroy(h)


def test_open_path_d12_cost(built_lib):
    """the committed depth-12 tree, its six sliced legs and ten open qubits: a slice costs at most 5 % more flops than a
    slice of the closed tree, and the largest intermediate stays 2^30"""
    from tnc_b200.builders import sycamore_circuit
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.contractionpath.slicing import path_cost
    from tnc_b200.sampling import _check_sliced_legs, open_path
    with open(os.path.join(ROOT, "bench_inputs", "sycamore53_d12.json")) as f:
        d = json.load(f)
    c = sycamore_circuit(53, 12, np.random.default_rng(1))
    closed = c.into_amplitude_network("0" * 53)[0]
    p = ContractionPath.simple([tuple(x) for x in d["toplevel"]])
    legs = d["sliced_legs"]
    f0, peak0, _ = path_cost([(t.legs, t.bond_dims) for t in closed.tensors], p, legs)
    tn = open_network(c, D12_OPEN)
    assert _check_sliced_legs(c, tn, D12_OPEN, legs) == legs
    q = open_path(c, p, D12_OPEN)
    f1, peak1, _ = path_cost([(t.legs, t.bond_dims) for t in tn.tensors], q, legs)
    assert peak0 == peak1 == 2.0 ** 30
    assert f0 <= f1 <= 1.05 * f0, (f0, f1)
