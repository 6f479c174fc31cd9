"""Sampling throughput (tnc_b200.Sampler, tncb_plan_sample) against the host loop it replaces.

Workloads: a 20-qubit, 10-round random circuit (seed 1) with k = 0, 4, 8 open qubits (0, 5, 10, 15 ... spread over the
register), and bench.py's 36-qubit circuit (random_circuit_builder(36, 10, 0.5, 0.5), seed 1) with qubits 0-3 open.
Per workload one JSON line:
  device:  samples/s and candidates/s of Sampler.sample (median of the repeats, host clock around calls that end in a
           device synchronise), with m = 1.01 x the max_ratio of a pilot call at m = 1;
           36 qubits: 16 samples, one timed call;
  split:   device time of the kernels of one call of up to 64 samples, from a torch.profiler run of its own: the
           sampling kernels (sample_candidates / sample_select / sample_compact) against everything else (leaf staging +
           contraction), with the call's passes and the host-to-device / device-to-host copies the trace lists;
  host:    the same candidates through the loop a user writes without Sampler (numpy Philox prefixes, host networks,
           stage_slices, run_batch, download, accept / pick on the host), samples/s; 36 qubits: not measured.
The first line holds the card's name and power limit (nvidia-smi query, same process).

usage: python tools/bench_sample.py [--samples 1000] [--repeats 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the record says so instead of guessing
        return {"gpu": None, "power_limit": None, "nvidia_smi_error": str(e)}


def timed(fn, repeats):
    import torch
    out, ts = None, []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, statistics.median(ts)


def split(fn):
    """device microseconds of the sampling kernels and of the rest, and the copies, from one profiled call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    own = rest = 0.0
    h2d = d2h = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        if "Memcpy HtoD" in name:
            h2d += 1
        elif "Memcpy DtoH" in name:
            d2h += 1
        elif "sample_" in name:
            own += e.device_time
        elif "Memcpy" not in name and "Memset" not in name:
            rest += e.device_time
    return {"sampling_kernels_us": own, "contraction_us": rest, "h2d_copies": h2d, "d2h_copies": d2h}


def host_loop(c, sampler, m, seed, count, batch):
    """Sampler's candidates through the host: prefixes from numpy's Philox, one host network per candidate, stage_slices
    + run_batch, download, accept and pick on the host.  Returns the samples (host words)."""
    n, k = c.num_qubits(), len(sampler.open_qubits)
    plan = sampler.plan
    words = []
    for start in range(0, count, batch):
        nets, draws = [], []
        for i in range(start, min(count, start + batch)):
            g = np.random.Philox(key=np.array([seed, 0], dtype=np.uint64), counter=(i - 1) % (1 << 256))
            w = [int(x) for x in g.random_raw(4)]
            closed = {q: (w[0] >> j) & 1 for j, q in enumerate(sampler.closed_qubits)}
            st = "".join("*" if q in sampler.open_qubits else str(closed[q]) for q in range(n))
            nets.append(c.into_amplitude_network(st)[0])
            draws.append((closed, (w[1] >> 11) * 2.0 ** -53, (w[2] >> 11) * 2.0 ** -53))
        plan.stage_slices(nets)
        _, rows = plan.run_batch(0, len(nets))
        amps = rows.to_numpy().reshape(len(nets), -1)
        for (closed, u, v), a in zip(draws, amps):
            p = a.real * a.real + a.imag * a.imag
            cdf = np.cumsum(p)
            if u < cdf[-1] * 2.0 ** (n - k) / m:
                y = int(np.argmax(cdf > v * cdf[-1]))
                word = sum(b << q for q, b in closed.items())
                word |= sum(((y >> (k - 1 - r)) & 1) << q for r, q in enumerate(sampler.result_qubits))
                words.append(word)
    return words


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sample.jsonl"))
    a = ap.parse_args()
    import torch
    import tnc_b200 as tb
    from tnc_b200.builders.random_circuit import random_circuit_builder
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py measures on a GPU; none is visible")
    ctx = tb.Context(0)
    lines = [dict(card(), tool="bench_sample.py")]
    work = [("amp20", 20, [q for q in range(0, 20, 20 // k)][:k] if k else [], a.samples) for k in (0, 4, 8)]
    work.append(("bench36", 36, [0, 1, 2, 3], 16))
    for name, n, opened, S in work:
        c = random_circuit_builder(n, 10, 0.5, 0.5, np.random.default_rng(1))
        t0 = time.perf_counter()
        s = tb.Sampler(c, opened, ctx=ctx)
        setup = time.perf_counter() - t0
        k = len(opened)
        pilot = s.sample(64, 1.0, seed=99, max_candidates=2048 if n < 36 else 16)   # m = 1: max_ratio = max q 2^(n-k)
        m = 1.01 * pilot.max_ratio
        s.sample(min(S, 4), m, seed=2)                  # warm-up of every shape the timed calls use
        out, sec = timed(lambda: s.sample(S, m, seed=1), a.repeats if n < 36 else 1)
        info = s.plan.info()
        rec = {"workload": name, "qubits": n, "open": opened, "flops_per_candidate": info["flops"], "m": m,
               "samples": int(out.bits.numel()), "candidates": out.candidates, "passes": out.passes,
               "clipped": out.clipped, "max_ratio": out.max_ratio, "sampler_setup_s": setup, "call_s": sec,
               "samples_per_s": out.bits.numel() / sec, "candidates_per_s": out.candidates / sec}
        small = s.sample(min(S, 64), m, seed=3)
        rec["split_call"] = {"samples": int(small.bits.numel()), "candidates": small.candidates, "passes": small.passes}
        rec["split_call"].update(split(lambda: s.sample(min(S, 64), m, seed=3)))
        if n < 36:       # the host loop over the first candidates of the timed call
            count = min(out.candidates, 2048)
            words, hsec = timed(lambda: host_loop(c, s, m, 1, count, 1024), 1)
            dev = [int(w) & ((1 << 64) - 1) for w in out.bits.cpu().tolist()]
            rec.update({"host_loop_candidates": count, "host_loop_s": hsec, "host_loop_samples_per_s": len(words) / hsec,
                        "host_loop_candidates_per_s": count / hsec, "host_loop_same_samples": words == dev[:len(words)]})
        else:
            rec.update({"host_loop_s": "not measured", "host_loop_samples_per_s": "not measured"})
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del s
    with open(a.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
