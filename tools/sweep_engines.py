"""DMMA (K1) vs the int8 tensor-core engines (K1': modular/CRT with several modulus counts, legacy digit slicing) over GEMM
shapes: device time per pair on the same box, error against the DMMA result.
usage: python tools/sweep_engines.py [MxNxK ...]"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import tnc_b200 as tb

ctx = tb.Context(0)
stream = torch.cuda.ExternalStream(ctx.stream, device=0)
shapes = [(256, 256, 256), (512, 512, 512), (1024, 1024, 1024), (2048, 2048, 2048), (4096, 4096, 4096), (1024, 1024, 4096), (4096, 4096, 512),
          (4096, 4096, 256), (2048, 512, 2048), (512, 4096, 4096), (8192, 8192, 1024), (16384, 8192, 4096), (65536, 2048, 512), (256, 128, 262144)]
if len(sys.argv) > 1:
    shapes = [tuple(int(x) for x in s.split("x")) for s in sys.argv[1:]]
rng = np.random.default_rng(0)
ctx.set_tcgen05_threshold(1, 128)


def timed(reps=5):
    for _ in range(2):
        tb.contract_pair_into(ctx, [0, 1], a, [2, 0], b, c)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        tb.contract_pair_into(ctx, [0, 1], a, [2, 0], b, c)
    e1.record(stream); ctx.synchronize(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


for (M, N, K) in shapes:
    a = tb.DeviceTensor.from_numpy(ctx, (rng.standard_normal((K, M)) + 1j * rng.standard_normal((K, M))))
    b = tb.DeviceTensor.from_numpy(ctx, (rng.standard_normal((N, K)) + 1j * rng.standard_normal((N, K))))
    c = tb.DeviceTensor.empty(ctx, (N, M))
    out = {"M": M, "N": N, "K": K}
    small = M * N <= 2048 * 2048
    ctx.set_tcgen05_slices(0)
    ms = timed()
    ref = c.to_numpy() if small else None
    out["dmma_ms"] = round(ms, 4); out["dmma_tf"] = round(8.0 * M * N * K / ms * 1e-9, 1)
    ctx.set_tcgen05_slices(8)
    ctx.time_gemm(True)
    for nm, pr in ((0, 4), (0, 3), (14, 0), (12, 0)):
        ctx.set_tcgen05_moduli(nm); ctx.set_tcgen05_products(pr)
        ms = timed()
        info = ctx.last_tcgen05_info()
        tag = f"crt{info['n_moduli']}" + (f"p{pr}" if pr else "")
        out[tag + "_ms"] = round(ms, 4); out[tag + "_tf"] = round(8.0 * M * N * K / ms * 1e-9, 1)
        out[tag + "_gemm_ms"] = round(ctx.last_gemm_ms(), 4)
        if small:
            out[tag + "_err"] = float(np.abs(c.to_numpy() - ref).max() / np.abs(ref).max())
    ctx.set_tcgen05_moduli(0); ctx.set_tcgen05_products(0)
    if min(M, N, K) >= 256:
        ctx.set_tcgen05_engine(1)
        ms = timed()
        out["slice8_ms"] = round(ms, 4); out["slice8_tf"] = round(8.0 * M * N * K / ms * 1e-9, 1)
        if small:
            out["slice8_err"] = float(np.abs(c.to_numpy() - ref).max() / np.abs(ref).max())
        ctx.set_tcgen05_engine(0)
    ctx.time_gemm(False)
    print(json.dumps(out), flush=True)
    a.free(); b.free(); c.free()
