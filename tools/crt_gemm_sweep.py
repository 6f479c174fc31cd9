"""Kernel time of crt_gemm_kernel alone (CUDA events around each launch, tncb_ctx_time_gemm accumulate mode) at the six
int8 pairs of the benchmark network, for ring variants of the GEMM's stage ring; with --passes, the time of every kernel
of an int8 pair instead.

The ring (slots x K bytes per slot, one configuration per product form) is a compile-time constant of csrc/crt.cu.  Each
variant is a separate copy of the library: crt.cu compiled with -D overrides of CRT_RING3_* / CRT_RING4_*, linked with the
other objects of the tree's own build (run `python __graft_entry__.py` first), under build/crt_sweep/<variant>/.  Every
variant runs in a child process of its own.  `--lib NAME=PATH` adds an already built libtncb200.so (another revision of
the library, same C ABI) to the comparison.

The pairs use the exact M, N and K of the network; the engine picks products, moduli, K chunks and panels for them as it
does inside the network (default context).  Per pair and variant one JSON line: GEMM-kernel ms per call, int8 ops per
call, the rate, and the SM clock sampled by nvidia-smi during the timed window.  The output starts with the card's name,
power limit and maximum SM clock, and the tools/i8_peak lines (what the tensor pipe sustains on this card).

--passes times each kernel of the pair (row maxima and residues of Bt and At, GEMM, reconstruction) with torch.profiler
(CUDA activities, a run of its own, no GEMM events) and prints per kernel its HBM bytes from the shape model below, the
rate and the fraction of the H100 SXM data sheet's 3.35 TB/s.  Only the libraries given with --lib run (the tree's own
build when there is none); no ring variant is built.

usage: python tools/crt_gemm_sweep.py [--variant NAME=S3xBK3,S4xBK4 ...] [--lib NAME=PATH ...] [--build-only] [--passes]
                                      [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (step in the greedy path, M, N, K) of the benchmark network's int8 pairs: random_circuit(36, 10, 0.5, 0.5, seed 1)
PAIRS = [(484, 65536, 4096, 2048), (482, 16384, 4096, 2048), (483, 65536, 2048, 512),
         (479, 16384, 2048, 1024), (481, 32768, 1024, 512), (478, 32768, 512, 512)]
# three-product ring x four-product ring, "stages x K bytes per stage"
VARIANTS = {
    "r3x128_2x128": "3x128,2x128",
    "r2x128_2x128": "2x128,2x128",
    "r4x128_5x64": "4x128,5x64",
    "r8x64_4x64": "8x64,4x64",
    "r9x64_3x64": "9x64,3x64",
}
SWEEP_DIR = os.path.join(ROOT, "build", "crt_sweep")
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def pass_bytes(M, N, K, products, nmod, nkc):
    """Compulsory HBM bytes per kernel and call (all panels): operands are complex128 (16 B), planes and residues one byte.
    rowmax reads its operand; residue reads it and writes NPL planes per modulus (three products: 3 per side, four: 2 for
    Bt and 3 for At); the GEMM reads every plane once and writes the residues; the reconstruction reads the residues
    (three or two planes per modulus and K chunk) and writes complex128 C."""
    npb, npr = (3, 3) if products == 3 else (2, 2)
    planes_b, planes_a = nmod * npb * N * K, nmod * 3 * M * K
    residues = nmod * nkc * npr * N * M
    return {"rowmax_bt": 16 * N * K, "rowmax_at": 16 * M * K,
            "residue_bt": 16 * N * K + planes_b, "residue_at": 16 * M * K + planes_a,
            "gemm": planes_b + planes_a + residues, "reconstruct": residues + 16 * N * M}


def pass_of(kernel, following):
    """the pass a kernel name belongs to; a row-max kernel takes its side from the residue kernel that follows it"""
    if "crt_residue_kernel<2" in kernel:
        return "residue_bt"
    if "crt_residue_kernel<3" in kernel:
        return "residue_at"
    if "crt_rowmax_kernel" in kernel:
        return None if following is None else "rowmax_" + pass_of(following, None).split("_")[1]
    if "crt_gemm_kernel" in kernel:
        return "gemm"
    if "crt_reconstruct_kernel" in kernel:
        return "reconstruct"
    return None


def defines(spec):
    (s3, b3), (s4, b4) = (tuple(int(v) for v in f.split("x")) for f in spec.split(","))
    return [f"-DCRT_RING3_STAGES={s3}", f"-DCRT_RING3_BK={b3}", f"-DCRT_RING4_STAGES={s4}", f"-DCRT_RING4_BK={b4}"]


def build_variants(variants):
    """crt.cu with the variant's -D flags + the tree's other objects -> build/crt_sweep/<name>/libtncb200.so"""
    import __graft_entry__ as ge
    deps = [os.path.join(ge.CSRC, f) for f in ("crt.cu", "sm90.h", "internal.h")]
    others = [os.path.join(ge.OBJDIR, s + ".o") for s in ge.SOURCES if s != "crt.cu"]
    missing = [o for o in others if not os.path.exists(o)]
    if missing:
        raise SystemExit(f"{missing[0]} is missing: build the library first (python __graft_entry__.py)")
    procs, libs = [], {}
    for name, spec in variants.items():
        d = os.path.join(SWEEP_DIR, name)
        os.makedirs(d, exist_ok=True)
        obj, lib = os.path.join(d, "crt.cu.o"), os.path.join(d, "libtncb200.so")
        libs[name] = lib
        stamp = os.path.join(d, "defines.txt")
        same = os.path.exists(stamp) and open(stamp).read() == spec
        if same and os.path.exists(lib) and all(os.path.getmtime(lib) > os.path.getmtime(x) for x in deps + others):
            continue
        cmd = [ge._nvcc(), *ge.NVCC_FLAGS, *defines(spec), "-c", os.path.join(ge.CSRC, "crt.cu"), "-o", obj]
        procs.append((name, spec, obj, lib, stamp, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for name, spec, obj, lib, stamp, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise SystemExit(f"nvcc failed on variant {name}:\n{out.decode()}")
        r = subprocess.run([ge._nvcc(), "-shared", "-o", lib, obj, *others, "-cudart", "static", "-ldl", "-lpthread", "-lz"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise SystemExit(f"link failed on variant {name}:\n{r.stdout.decode()}")
        with open(stamp, "w") as f:
            f.write(spec)
    return libs


class _DevView:
    """__cuda_array_interface__ of a DeviceTensor's complex128 buffer as float64 [..., 2], so torch can fill it"""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape) + (2,), "typestr": "<f8", "data": (ptr, False),
                                         "version": 3, "strides": None}


class ClockSampler:
    """nvidia-smi's SM clock every 50 ms while the `with` block runs"""

    def __enter__(self):
        self.p = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "50"],
                                  stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        time.sleep(0.3)   # nvidia-smi's own start-up
        return self

    def __exit__(self, *exc):
        self.p.terminate()
        out, _ = self.p.communicate()
        self.mhz = [int(x) for x in out.split() if x.strip().isdigit()]
        return False


def profile_passes(ctx, tb, a, b, c, reps):
    """device ms per call of each pass, from one torch.profiler run of `reps` calls; nkc from the reconstruction's name"""
    import tempfile
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            tb.contract_pair_into(ctx, [0, 1], a, [2, 0], b, c)
        ctx.synchronize()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    us, count, one_chunk = {}, {}, None
    for i, e in enumerate(kernels):
        nxt = kernels[i + 1]["name"] if i + 1 < len(kernels) else None
        p = pass_of(e["name"], nxt)
        if p is None:
            continue
        if p == "reconstruct":
            one_chunk = "crt_reconstruct_kernel<true" in e["name"]
        us[p] = us.get(p, 0.0) + e["dur"]
        count[p] = count.get(p, 0) + 1
    return {p: v / 1e3 / reps for p, v in us.items()}, {p: v // reps for p, v in count.items()}, one_chunk


def child(name, lib_path, min_window_s, passes=False):
    import torch
    import tnc_b200 as tb
    import tnc_b200._lib as tl
    tl.LIB_PATH = lib_path   # before the first lib() call: this process runs this variant only
    ctx = tb.Context(0)
    assert tl.lib()._name == lib_path, tl.lib()._name
    ctx.set_tcgen05_slices(8)
    ctx.set_tcgen05_threshold(1, 128)
    gen = torch.Generator(device="cuda")
    for step, M, N, K in PAIRS:
        a = tb.DeviceTensor.empty(ctx, (K, M))
        b = tb.DeviceTensor.empty(ctx, (N, K))
        c = tb.DeviceTensor.empty(ctx, (N, M))
        gen.manual_seed(step)
        for t, shape in ((a, (K, M)), (b, (N, K))):
            torch.as_tensor(_DevView(t.device_ptr(), shape), device="cuda").normal_(generator=gen)
        torch.cuda.synchronize()
        if passes:
            for _ in range(2):   # warm-up: module load, arena growth
                tb.contract_pair_into(ctx, [0, 1], a, [2, 0], b, c)
            ctx.synchronize()
            reps = 5
            with ClockSampler() as clk:
                ms, launches, one_chunk = profile_passes(ctx, tb, a, b, c, reps)
            info = ctx.last_tcgen05_info()
            assert one_chunk, "the byte model below takes one K chunk"
            model = pass_bytes(M, N, K, info["products"], info["n_moduli"], 1)
            rec = {"variant": name, "step": step, "M": M, "N": N, "K": K, "products": info["products"],
                   "n_moduli": info["n_moduli"], "k_chunks": 1, "reps": reps,
                   "sm_clock_mhz_median": statistics.median(clk.mhz) if clk.mhz else None,
                   "sm_clock_mhz_min": min(clk.mhz) if clk.mhz else None, "passes": {}}
            for p, nbytes in model.items():
                rate = nbytes / (ms[p] * 1e-3)
                rec["passes"][p] = {"ms": round(ms[p], 4), "launches": launches[p], "gb": round(nbytes / 1e9, 3),
                                    "gb_per_s": round(rate / 1e9, 1), "of_hbm_peak": round(rate / HBM_BYTES_PER_S, 3)}
            rec["total_ms"] = round(sum(ms[p] for p in model), 4)
            print(json.dumps(rec), flush=True)
            for t in (a, b, c):
                t.free()
            continue
        ctx.time_gemm(2)
        t0 = time.perf_counter()
        for _ in range(2):   # warm-up: module load, arena growth
            tb.contract_pair_into(ctx, [0, 1], a, [2, 0], b, c)
        ctx.synchronize()
        per_call = (time.perf_counter() - t0) / 2
        ctx.gemm_totals()   # discard the warm-up launches
        reps = max(3, min(50, int(min_window_s / max(per_call, 1e-4)) + 1))
        with ClockSampler() as clk:
            for _ in range(reps):
                tb.contract_pair_into(ctx, [0, 1], a, [2, 0], b, c)
            tot = ctx.gemm_totals()
        info = ctx.last_tcgen05_info()
        ctx.time_gemm(0)
        assert ctx.engine_counts()["k1_tcgen05"] > 0, "the pair did not take the int8 engine"
        ms, ops = tot["ms"] / reps, tot["int8_ops"] / reps
        rec = {"variant": name, "step": step, "M": M, "N": N, "K": K,
               "products": info["products"], "n_moduli": info["n_moduli"], "gemm_launches_per_call": tot["launches"] // reps,
               "reps": reps, "gemm_ms": round(ms, 4), "int8_ops": ops, "pops": round(ops / ms * 1e-12, 4),
               "sm_clock_mhz_median": statistics.median(clk.mhz) if clk.mhz else None,
               "sm_clock_mhz_min": min(clk.mhz) if clk.mhz else None}
        print(json.dumps(rec), flush=True)
        for t in (a, b, c):
            t.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", action="append", default=[], metavar="NAME=S3xBK3,S4xBK4",
                    help="ring variant (default: the built-in list)")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="an already built libtncb200.so")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--passes", action="store_true", help="per-kernel times and HBM rates of every pass (--lib builds only)")
    ap.add_argument("--window", type=float, default=0.4, help="seconds of GEMM calls per pair and variant (at least 3 calls)")
    ap.add_argument("--out", default=None, help="also write the records to this file")
    ap.add_argument("--child", nargs=2, metavar=("NAME", "LIB"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a.child[0], a.child[1], a.window, a.passes)
    variants = dict(v.split("=", 1) for v in a.variant) if a.variant else dict(VARIANTS)
    libs = {k: os.path.abspath(v) for k, v in (x.split("=", 1) for x in a.lib)}
    if a.passes:
        variants = {}
        if not libs:
            import tnc_b200._lib as tl
            libs["tree"] = tl.LIB_PATH
    libs.update(build_variants(variants))
    if a.build_only:
        return
    lines = [subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                            stdout=subprocess.PIPE, text=True, check=True).stdout.strip()]
    peak = subprocess.run([os.path.join(ROOT, "tools", "i8_peak")], stdout=subprocess.PIPE, text=True, check=True).stdout
    lines.append(json.dumps({"i8_peak": peak.strip().splitlines()}))
    for ln in lines:
        print(ln, flush=True)
    for name, lib in libs.items():
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--window", str(a.window), "--child", name, lib]
                           + (["--passes"] if a.passes else []), stdout=subprocess.PIPE, text=True)
        for ln in r.stdout.strip().splitlines():
            rec = json.loads(ln)
            rec["ring"] = variants.get(name, "library as built")
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
        if r.returncode != 0:
            raise SystemExit(f"variant {name} failed with exit code {r.returncode}")
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
