"""Sampling sliced circuits (Sampler(..., sliced_legs=...), tncb_plan_sample_slices) on one GPU.

Workloads, one JSON line each:
  d12:    Sycamore-53 depth 12 (bench.py's config 5): the committed tree (bench_inputs/sycamore53_d12.json) made open by
          open_path for qubits 2, 8, 12, 13, 16, 18, 22, 29, 32, 35, its 6 sliced legs (64 slices), --d12-samples
          samples.  s per candidate and per sample, next to one amplitude of the closed tree (SlicedPlan.run, 64 slices)
          timed on the same card;
  d10:    Sycamore-53 depth 10: open_path of the committed d10 tree with the same 10 open qubits, 8 samples, sliced on
          the first 3 legs find_slices picks that are neither open nor on a bra (8 slices), against the unsliced Sampler
          on the same open path;
  amp20:  tools/bench_sample.py's 20-qubit circuit with k = 4 (qubits 0, 5, 10, 15), 2 sliced legs against unsliced;
  split:  amp20 sliced, a torch.profiler run of its own: the accumulate kernel's device time against the rest.
m is 1.05 x the max_ratio of a pilot call at m = 1.  Every line reports the clipped count, passes, and whether a workspace
copy fitted beside the plan (torch.cuda.mem_get_info before the call against peak_bytes + 1 GiB + the int8 engine's
12 GiB).  Times: host clock around calls that end in a device synchronise.  The first line holds the card's name and
power limit (nvidia-smi query, same process).

usage: python tools/bench_sample_sliced.py [--d12-samples 8] [--skip-d12] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sample import card, timed  # noqa: E402

OPEN10 = [2, 8, 12, 13, 16, 18, 22, 29, 32, 35]
KEEP = (1 << 30) + (12 << 30)      # what a workspace copy must leave free (include/tncb.h, tncb_plan_run_batch)


def tree(name):
    from tnc_b200.contractionpath import ContractionPath
    with open(os.path.join(ROOT, "bench_inputs", name)) as f:
        d = json.load(f)
    return ContractionPath.simple([tuple(x) for x in d["toplevel"]]), d.get("sliced_legs", [])


def measure(s, samples, label):
    """pilot, then one timed call of `samples` samples; the record of one sampler"""
    import torch
    pilot = s.sample(1, 1.0, seed=99, max_candidates=2 if s.n_qubits > 36 else 256)
    m = 1.05 * pilot.max_ratio
    free, _ = torch.cuda.mem_get_info()
    info = s.plan.info()
    out, sec = timed(lambda: s.sample(samples, m, seed=1), 1)
    return {"workload": label, "open": s.open_qubits, "slices": s.n_slices, "flops_per_slice": info["flops"],
            "peak_bytes": info["peak_bytes"], "copy_fits_beside_plan": free > info["peak_bytes"] + KEEP,
            "pilot_candidates": pilot.candidates, "pilot_max_ratio": pilot.max_ratio, "m": m,
            "samples": int(out.bits.numel()), "candidates": out.candidates, "passes": out.passes, "clipped": out.clipped,
            "max_ratio": out.max_ratio, "call_s": sec, "s_per_candidate": sec / max(out.candidates, 1),
            "s_per_sample": sec / max(int(out.bits.numel()), 1), "samples_per_s": out.bits.numel() / sec}


def split(fn):
    """device microseconds of the accumulate kernel, the other sampling kernels and the rest, from one profiled call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    acc = own = rest = 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or "Memcpy" in e.name or "Memset" in e.name:
            continue
        if "sample_accumulate" in e.name:
            acc += e.device_time
        elif "sample_" in e.name:
            own += e.device_time
        else:
            rest += e.device_time
    return {"accumulate_us": acc, "other_sampling_kernels_us": own, "contraction_us": rest}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d12-samples", type=int, default=8)
    ap.add_argument("--skip-d12", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sample_sliced.jsonl"))
    a = ap.parse_args()
    import torch
    import tnc_b200 as tb
    from tnc_b200.builders import sycamore_circuit
    from tnc_b200.builders.random_circuit import random_circuit_builder
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    from tnc_b200.sampling import open_path
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample_sliced.py measures on a GPU; none is visible")
    ctx = tb.Context(0)
    lines = [dict(card(), tool="bench_sample_sliced.py")]

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    # amp20: launch-bound, k = 4, 2 sliced legs against unsliced
    c = random_circuit_builder(20, 10, 0.5, 0.5, np.random.default_rng(1))
    opened = [0, 5, 10, 15]
    tn, _ = c.into_amplitude_network("".join("*" if q in opened else "0" for q in range(20)))
    path = open_path(c, _closed_path(c), opened)
    legs = [l for l in find_slices(tn, path, min_slices=16) if l not in c.open_edges][:2]
    for sl in (None, legs):
        s = tb.Sampler(c, opened, path=path, ctx=ctx, sliced_legs=sl)
        s.sample(16, 2.0, seed=2)                            # warm-up
        emit(dict(measure(s, 1000, "amp20" + (" sliced" if sl else "")), sliced_legs=sl))
        if sl:
            emit(dict(workload="amp20 sliced split", **split(lambda: s.sample(64, 2.0, seed=3))))
        del s
    # d10: 8 slices by find_slices against unsliced on the same open path
    c = sycamore_circuit(53, 10, np.random.default_rng(1))
    closed10, _ = tree("sycamore53_d10.json")
    path = open_path(c, closed10, OPEN10)
    tn, _ = c.into_amplitude_network("".join("*" if q in OPEN10 else "0" for q in range(53)))
    legs = [l for l in find_slices(tn, path, min_slices=64) if l not in c.open_edges][:3]
    for sl in (None, legs):
        s = tb.Sampler(c, OPEN10, path=path, ctx=ctx, sliced_legs=sl)
        emit(dict(measure(s, 8, "d10" + (" sliced" if sl else "")), sliced_legs=sl))
        del s
        torch.cuda.synchronize()
    if not a.skip_d12:
        c = sycamore_circuit(53, 12, np.random.default_rng(1))
        closed12, legs = tree("sycamore53_d12.json")
        tn0, _ = c.into_amplitude_network("0" * 53)
        amp = SlicedPlan(tn0, closed12, legs, ctx=ctx)
        amp.run()                                            # warm-up
        _, amp_s = timed(amp.run, 1)
        del amp
        s = tb.Sampler(c, OPEN10, path=open_path(c, closed12, OPEN10), ctx=ctx, sliced_legs=legs)
        emit(dict(measure(s, a.d12_samples, "d12"), sliced_legs=legs, closed_amplitude_s=amp_s))
        del s
    with open(a.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


def _closed_path(c):
    from tnc_b200.contractionpath.paths import Cotengrust
    tn, _ = c.into_amplitude_network("0" * c.num_qubits())
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


if __name__ == "__main__":
    main()
