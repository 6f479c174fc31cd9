"""Sampling without a GPU: the random stream's Philox header, compiled for the host, against numpy's Philox; and what
Sampler passes to tncb_plan_sample (spec, seed, range, output pointers) for a circuit with scattered open qubits, with
the plan created by the real library on a NULL context and every later entry answered by a recorder."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASK = (1 << 64) - 1


def numpy_block(key, counter):
    """the Philox4x64-10 block at the 256-bit counter `counter` of key (key, 0): numpy increments before it generates"""
    g = np.random.Philox(key=np.array([key, 0], dtype=np.uint64), counter=(counter - 1) % (1 << 256))
    return [int(x) for x in g.random_raw(4)]


@pytest.fixture(scope="module")
def stream(tmp_path_factory):
    """runs the host build of csrc/philox.h on lines of input, one output line each"""
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    exe = str(tmp_path_factory.mktemp("philox") / "philox_stream")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "tnc_b200", "csrc"),
                    os.path.join(ROOT, "tests", "cpp", "philox_stream.cpp"), "-o", exe], check=True)

    def run(lines):
        r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True)
        return [[int(x) for x in row.split()] for row in r.stdout.splitlines()]
    return run


def test_philox_blocks_match_numpy(stream):
    rng = np.random.default_rng(5)
    keys = [0, 1, 12345, MASK] + [int(x) for x in rng.integers(0, 1 << 63, 4, dtype=np.uint64)]
    counters = [0, 1, 7, (1 << 64) - 1, 1 << 64, (1 << 128) - 1, 1 << 128, 1 << 192, (1 << 256) - 1,
                (5 << 64) + 3, (1 << 64) + (1 << 130) + 99]
    counters += [int.from_bytes(rng.bytes(32), "little") for _ in range(6)]
    cases = [(k, c) for k in keys for c in counters]
    words = lambda c: [(c >> (64 * j)) & MASK for j in range(4)]
    got = stream([f"key {k} " + " ".join(map(str, words(c))) for k, c in cases])
    for (k, c), row in zip(cases, got):
        assert row == numpy_block(k, c), (k, hex(c))


def test_candidate_stream(stream):
    """candidate i of seed s: counter (i, 0, 0, 0) of key (s, 0); u, v the top 53 bits of w1, w2 times 2^-53"""
    rng = np.random.default_rng(6)
    cases = [(s, i) for s in (0, 3, MASK) for i in (0, 1, 2, 1000, (1 << 64) - 1)]
    cases += [(int(s), int(i)) for s, i in zip(rng.integers(0, 1 << 63, 20, dtype=np.uint64),
                                               rng.integers(0, 1 << 63, 20, dtype=np.uint64))]
    got = stream([f"cand {s} {i}" for s, i in cases])
    for (s, i), row in zip(cases, got):
        w = numpy_block(s, i)
        assert row[:4] == w, (s, i)
        u, v = (struct.unpack("<d", struct.pack("<Q", b))[0] for b in row[4:])
        assert u == (w[1] >> 11) * 2.0 ** -53 and v == (w[2] >> 11) * 2.0 ** -53, (s, i)
        assert 0.0 <= u < 1.0 and 0.0 <= v < 1.0


# ------------------------------------------------------------------------------------------------ Sampler's arguments
def circuit(n=6):
    from tnc_b200.builders.random_circuit import random_circuit_builder
    return random_circuit_builder(n, 4, 0.5, 0.5, np.random.default_rng(3))


class Recorder:
    """Stands in for the library: plan creation and metadata pass through, every other entry is logged; the sample
    entry reports `stats`"""

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

    made = []
    cpu_empty = torch.empty

    def empty(*shape, dtype=None, device=None):
        t = cpu_empty(*shape, dtype=dtype)
        made.append(t)
        return t

    monkeypatch.setattr(tb, "torch_streams", lambda ctx: (Stream("torch"), Stream("ctx")))
    monkeypatch.setattr(torch, "empty", empty)
    samplers = []
    yield ctx, log, made, samplers
    for s in samplers:
        built_lib.tncb_plan_destroy(s.plan.handle)
        s.plan.handle = None


def test_sampler_spec(recorded):
    from tnc_b200 import Sampler
    from tnc_b200.tensornetwork.contraction import leaves
    ctx, log, made, samplers = recorded
    c = circuit()
    opened = [4, 1]
    s = Sampler(c, opened, ctx=ctx)
    samplers.append(s)
    assert [row[0] for row in log] == ["tncb_plan_stage"]
    # the bras of the closed qubits 0, 2, 3, 5 follow the circuit's tensors, in qubit order
    tn, _ = c.into_amplitude_network("0*00*0")
    lv = leaves(tn)
    n_gates = len(c.tensors)
    assert len(lv) == n_gates + 4
    for j, q in enumerate([0, 2, 3, 5]):
        assert lv[n_gates + j].legs == [c.open_edges[q]] and lv[n_gates + j].bond_dims == [2]
    del log[:]
    out = s.sample(7, 2.5, seed=11, first=100, max_candidates=5000, batch=9)
    (call,) = [row for row in log if row[0] == "tncb_plan_sample"]
    spec = call[2]
    assert spec["n_qubits"] == 6
    assert spec["closed_leaf"] == [n_gates + j for j in range(4)]
    assert spec["closed_qubit"] == [0, 2, 3, 5]
    assert sorted(spec["result_qubit"]) == [1, 4]
    assert [c.open_edges[q] for q in spec["result_qubit"]] == s.plan.result_legs
    bits, probs = made
    assert call[1] == "handle" and call[3:] == (11, 100, 5000, 7, 2.5, 9, bits.data_ptr(), probs.data_ptr(), "stats")
    import torch
    assert bits.dtype == torch.int64 and probs.dtype == torch.float64
    assert bits.shape == (7,) and probs.shape == (7,)
    # ordered after torch's current stream, which then waits for the library
    assert log[0] == ("wait", "ctx", "torch") and log[-1] == ("wait", "torch", "ctx")
    assert out.bits.shape == (3,) and out.probabilities.shape == (3,)
    assert (out.candidates, out.clipped, out.max_ratio, out.next_candidate) == (40, 2, 1.5, 140)
    # defaults: every candidate slot the library picks, the documented candidate budget
    del log[:], made[:]
    s.sample(3, 4.0)
    (call,) = [row for row in log if row[0] == "tncb_plan_sample"]
    assert call[3:8] == (0, 0, 16 * 4 * 3 + 1024, 3, 4.0) and call[8] == 0


def test_sampler_refusals(recorded):
    from tnc_b200 import Sampler
    ctx, log, made, samplers = recorded
    c = circuit()
    for bad in ([1, 1], [6], [-1]):
        with pytest.raises(ValueError, match="open qubits"):
            Sampler(c, bad, ctx=ctx)
    s = Sampler(c, [], ctx=ctx)
    samplers.append(s)
    with pytest.raises(ValueError, match="n_samples"):
        s.sample(0, 2.0)


def test_bitstrings_decode():
    """bit q of a word is character q, the order of into_amplitude_network's bitstring"""
    import torch
    from tnc_b200 import Samples
    strings = ["1" + "0" * 62 + "1", "0" * 63 + "1", "01" * 32, "1" * 64, "0" * 64]
    words = [sum(1 << q for q, ch in enumerate(st) if ch == "1") for st in strings]
    signed = [w - (1 << 64) if w >> 63 else w for w in words]
    s = Samples(torch.tensor(signed, dtype=torch.int64), torch.zeros(5, dtype=torch.float64), 5, 0, 0.5, 5, 64)
    assert s.bitstrings() == strings
    short = Samples(torch.tensor([0b101, 0b010], dtype=torch.int64), torch.zeros(2, dtype=torch.float64), 2, 0, 0.5, 2, 3)
    assert short.bitstrings() == ["101", "010"]
