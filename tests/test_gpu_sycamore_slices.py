"""BASELINE config 5 -- the Sycamore-53 depth-12 amplitude as 64 slices of a committed path -- checked pair by pair.

bench.py times this object through SlicedPlan.  One slice of either committed tree (bench_inputs/sycamore53_d12.json and
its alternative, which slices other legs) runs ~1050 pairs, among them shapes that no other test reaches:

  * K2 with a 2^26-row big side (30 legs, 16 GiB in and 16 GiB out), NS = 16, K = 16: ~62 grid-stride trips per thread;
  * K1 DMMA with 32x64 tiles at M = 2^25, N = 32, K = 32 and with 64x32 tiles at M = 16, N = 2^24, K = 64;
  * a 128 x 128 x 2^23 pair (alternative tree) that the int8 engine refuses (its K chunks would exceed CRT_KCHUNK_MAX),
    so launch_k1 falls back to DMMA split-K.

1. Inventory (no GPU): both trees replayed on metadata, every step classified by tncb_pair_kernel_class.
2. Slice 0 step by step: every pair through contract_pair_into, its engine counter and arena balance asserted, every
   output entry compared with four real FP64 torch matmuls on the GEMM view, and sampled entries -- edges, tile edges,
   K2 grid-stride seams -- with a long-double host sum.  Cases: the main tree with the circuit's gates, and the
   alternative tree with seeded Haar-random unitaries in place of every gate (no all-real blocks, magnitudes kept in
   range by unitarity).
3. SlicedPlan.run_slices(0, 64), the executor the benchmark times, gives the step-by-step scalar bit for bit.
4. The full 64-slice amplitude: both trees agree, and equal the committed value.

The alternative tree's level-ordered static layout needs 64.1 GiB, above the default cap of 0.62 x device memory
(network.cpp: plan_static_layout), so without a raised cap tncb_plan_stage_slices refuses it; its plans here are created
with TNCB_PLAN_WS_GB raised to 68."""
import functools
import json
import os
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TREES = {"main": "sycamore53_d12.json", "alt": "sycamore53_d12_alt.json"}
# <0^53| C |0^53> of sycamore_circuit(53, 12, default_rng(1)); bench.py's CONFIG5_AMPLITUDE (the config-5 regression value)
CONFIG5_AMPLITUDE = complex(-6.148484459425177e-09, -5.130555022162778e-09)
U = 2.0 ** -53
PLAN_WS_GB = {"alt": "68"}   # static workspace cap for SlicedPlan (see above); the default serves the main tree
CHECK_BYTES = 8 << 30        # the checker's own device temporaries per step
TMP_PER_ELEM = 64            # bytes of checker temporaries per gathered or output element (indices, re/im, |.|, sums)
DEVICE = "cuda"


@functools.lru_cache(maxsize=None)
def network():
    from tnc_b200.builders import sycamore_circuit
    return sycamore_circuit(53, 12, np.random.default_rng(1)).into_amplitude_network("0" * 53)[0]


def tree(name):
    from tnc_b200.contractionpath import ContractionPath
    with open(os.path.join(ROOT, "bench_inputs", TREES[name])) as f:
        d = json.load(f)
    return ContractionPath.simple([tuple(x) for x in d["toplevel"]]), list(d["sliced_legs"])


def haar_network(seed):
    """The network with every gate leaf replaced by a Haar-random unitary of the same arity, [old..., new...] layout"""
    from tnc_b200.tensornetwork import Tensor, TensorData
    rng = np.random.default_rng(seed)
    leaves = []
    for t in network().tensors:
        if t.tensordata.kind == "gate":
            d = 2 ** (len(t.legs) // 2)
            q, r = np.linalg.qr((rng.standard_normal((d, d)) + 1j * rng.standard_normal((d, d))) / np.sqrt(2))
            u = q * (np.diag(r) / np.abs(np.diag(r)))
            t = Tensor(t.legs, t.bond_dims, tensordata=TensorData.Matrix(u.reshape(t.bond_dims)))
        leaves.append(t)
    return Tensor.new_composite(leaves)


def pair_mnk(built_lib, al, ad, bl, bd):
    import ctypes as C
    from tnc_b200._lib import check, u64_array
    m, n, k = C.c_uint64(), C.c_uint64(), C.c_uint64()
    check(built_lib.tncb_pair_out_legs(len(al), u64_array(al), u64_array(ad), len(bl), u64_array(bl), u64_array(bd),
                                       None, None, None, C.byref(m), C.byref(n), C.byref(k)))
    return m.value, n.value, k.value


def replay(built_lib, name):
    """(a legs, a dims, b legs, b dims, kernel class, M, N, K) of every step of one slice of a tree (sliced legs removed)"""
    from tnc_b200._lib import u64_array
    path, sliced = tree(name)
    ts = [[(l, d) for l, d in t.edges() if l not in sliced] for t in network().tensors]
    out = []
    for i, j in path.toplevel:
        al, ad = [l for l, _ in ts[i]], [d for _, d in ts[i]]
        bl, bd = [l for l, _ in ts[j]], [d for _, d in ts[j]]
        cls = built_lib.tncb_pair_kernel_class(len(al), u64_array(al), u64_array(ad), len(bl), u64_array(bl), u64_array(bd))
        out.append((al, ad, bl, bd, cls) + pair_mnk(built_lib, al, ad, bl, bd))
        ts[i] = [e for e in ts[j] if e[0] not in al] + [e for e in ts[i] if e[0] not in bl]
        ts[j] = None
    return out


def shape_kind(cls, M, N, K):
    """the large shapes only the config-5 slices reach (None for every other step)"""
    if cls == 2 and max(M, N) == 2 ** 26 and min(M, N) == 16 and K == 16:
        return "k2_2^26"
    if cls == 1 and (M, N, K) == (2 ** 25, 32, 32):
        return "k1_32x64_2^25"
    if cls == 1 and (M, N, K) == (16, 2 ** 24, 64):
        return "k1_64x32_2^24"
    if cls == 1 and (M, N, K) == (128, 128, 2 ** 23):
        return "k1_128x128x2^23"
    return None


# ================================================================================================================
# 1. inventory
# ================================================================================================================
INVENTORY = {
    "main": {"classes": {0: 1014, 1: 20, 2: 18}, "k2_2^26": 7, "k1_32x64_2^25": 1, "k1_64x32_2^24": 1, "k1_128x128x2^23": 0},
    "alt": {"classes": {0: 1015, 1: 23, 2: 14}, "k2_2^26": 3, "k1_32x64_2^25": 2, "k1_64x32_2^24": 0, "k1_128x128x2^23": 1},
}


@pytest.mark.parametrize("name", ["main", "alt"])
def test_inventory(built_lib, name):
    """Step classes and the large shapes of one slice, as the library classifies them."""
    steps = replay(built_lib, name)
    assert len(steps) == 1052
    classes = {c: sum(1 for s in steps if s[4] == c) for c in (0, 1, 2)}
    assert classes == INVENTORY[name]["classes"]
    kinds = [shape_kind(*s[4:]) for s in steps]
    for kind in ("k2_2^26", "k1_32x64_2^25", "k1_64x32_2^24", "k1_128x128x2^23"):
        assert kinds.count(kind) == INVENTORY[name][kind], kind
    for s, kind in zip(steps, kinds):
        al, ad, bl, bd, cls, M, N, K = s
        if kind == "k2_2^26":      # the big operand: 30 legs (16 GiB), and so is the output
            assert max(len(al), len(bl)) == 30 and 16 * M * N == 16 << 30
        if kind == "k1_128x128x2^23":
            assert len(al) == len(bl) == 30     # A and B are 16 GiB each


# ================================================================================================================
# 2. + 3. slice 0 step by step, then the sliced plan
# ================================================================================================================
def mixed_radix(dims, strides):
    """offsets, in an operand with the given strides, of every index of the row-major box over dims"""
    off = np.zeros(1, dtype=np.int64)
    for d, s in zip(dims, strides):
        off = (off[:, None] + np.arange(d, dtype=np.int64) * int(s)).reshape(-1)
    return off


def row_major_strides(dims):
    s, out = 1, []
    for d in reversed(dims):
        out.append(s)
        s *= d
    return out[::-1]


def gemm_view(al, ad, bl, bd):
    """offAm, offBn, offAk, offBk of C[n, m] = sum_k Bt[n, k] At[k, m] with C's legs (b \\ a) ++ (a \\ b) and the shared
    legs in a's order"""
    sa, sb = dict(zip(al, row_major_strides(ad))), dict(zip(bl, row_major_strides(bd)))
    da, db = dict(zip(al, ad)), dict(zip(bl, bd))
    m = [l for l in al if l not in sb]
    n = [l for l in bl if l not in sa]
    k = [l for l in al if l in sb]
    return (mixed_radix([da[l] for l in m], [sa[l] for l in m]), mixed_radix([db[l] for l in n], [sb[l] for l in n]),
            mixed_radix([da[l] for l in k], [sa[l] for l in k]), mixed_radix([da[l] for l in k], [sb[l] for l in k]))


class _Cai:
    """__cuda_array_interface__ of a library tensor as float64 [elements, 2] (no copy)"""

    def __init__(self, dt):
        elems = int(np.prod(dt.shape, dtype=np.int64))
        self.__cuda_array_interface__ = {"shape": (elems, 2), "typestr": "<f8", "data": (dt.device_ptr(), False),
                                         "version": 3, "strides": None}


def as_complex(torch, dt):
    return torch.view_as_complex(torch.as_tensor(_Cai(dt), device="cuda"))


def arena_bytes(elems):
    """bytes the arena books for a tensor (runtime.cu: at least 16 B, 256-byte granularity)"""
    b = max(16 * elems, 16)
    return (max(b, 256) + 255) // 256 * 256


def edges(X):
    return sorted({0, X - 1} | {e for e in (31, 32, 63, 64, 127, 128) if e < X})


def k2_seams(big, sm_count):
    """x = j * stride - 1 and j * stride of the K2 grid-stride loop (launch_k2: min(ceil(BIG/256), 32 SMs) blocks of 256)"""
    stride = 256 * min((big + 255) // 256, 32 * sm_count)
    return [x for j in range(1, big // stride + 1) for x in (j * stride - 1, j * stride) if x < big]


def check_step(torch, step, da, db, dc, view, cls, ks, sm_count, rng):
    """(entries sampled, failures) of one step.  A failure comes back as text: an exception raised where torch views of
    library memory are arguments would have pytest print those views after the context that owns the memory is closed."""
    try:
        return _check_step(torch, step, as_complex(torch, da), as_complex(torch, db), as_complex(torch, dc), view, cls,
                           ks, sm_count, rng), []
    except Exception as e:
        return 0, [f"{type(e).__name__}: {e}"]


def _check_step(torch, step, A, B, C, view, cls, ks, sm_count, rng):
    """Every entry against four FP64 matmuls on the device; sampled entries against a long-double host sum."""
    offAm, offBn, offAk, offBk = view
    M, N, K = len(offAm), len(offBn), len(offAk)
    dev = lambda x: torch.from_numpy(x).to(DEVICE)
    dAm, dBn, dAk, dBk = dev(offAm), dev(offBn), dev(offAk), dev(offBk)
    gather = lambda X, rows, cols: X[rows[:, None] + cols[None, :]]
    Cv = torch.view_as_real(C).view(N, M, 2)
    budget = CHECK_BYTES - 8 * (M + N + 2 * K)
    fixed = {"M": N * K, "N": K * M, "K": N * M}
    unit = {"M": K + N, "N": K + M, "K": N + M}
    axis = max(("M", M), ("N", N), ("K", K), key=lambda t: t[1])[0]
    chunk = max(1, (budget // TMP_PER_ELEM - fixed[axis]) // unit[axis])
    assert TMP_PER_ELEM * (fixed[axis] + unit[axis]) <= budget, (step, M, N, K)

    def four(Bt, At):
        br, bi, ar, ai = Bt.real, Bt.imag, At.real, At.imag
        return br @ ar - bi @ ai, br @ ai + bi @ ar, Bt.abs() @ At.abs()

    def compare(got, cr, ci, p, n_kchunks, where):
        tol = (4 * K + 1100) * U * p + n_kchunks * 2.0 ** -52 * p
        bad = ~((got[..., 0] - cr).abs() <= tol) | ~((got[..., 1] - ci).abs() <= tol)
        nbad = int(bad.sum())
        assert nbad == 0, f"step {step} ({M}x{N}x{K}, class {cls}) {where}: {nbad} entries outside the bound"

    if axis == "K":          # partial sums over K chunks: one more rounding of P's size per chunk
        cr = ci = p = None
        n_kc = 0
        for k0 in range(0, K, chunk):
            k1 = min(K, k0 + chunk)
            r = four(gather(B, dBn, dBk[k0:k1]), gather(A, dAk[k0:k1], dAm))
            cr, ci, p = r if cr is None else (cr + r[0], ci + r[1], p + r[2])
            del r
            n_kc += 1
        compare(Cv, cr, ci, p, n_kc, "all")
        del cr, ci, p
    elif axis == "M":
        Bt = gather(B, dBn, dBk)
        for m0 in range(0, M, chunk):
            m1 = min(M, m0 + chunk)
            compare(Cv[:, m0:m1], *four(Bt, gather(A, dAk, dAm[m0:m1])), 1, f"columns {m0}..{m1}")
        del Bt
    else:
        At = gather(A, dAk, dAm)
        for n0 in range(0, N, chunk):
            n1 = min(N, n0 + chunk)
            compare(Cv[n0:n1], *four(gather(B, dBn[n0:n1], dBk), At), 1, f"rows {n0}..{n1}")
        del At

    # ---- sampled entries in long double ----
    ms, ns = edges(M), edges(N)
    if cls == 2:           # K2: x runs over the big free side
        if M >= N:
            ms = sorted(set(ms) | set(k2_seams(M, sm_count)))
        else:
            ns = sorted(set(ns) | set(k2_seams(N, sm_count)))
    while len(ms) * len(ns) < min(16, M * N):
        if len(ms) < M:
            ms = sorted(set(ms) | {int(rng.integers(M))})
        if len(ns) < N:
            ns = sorted(set(ns) | {int(rng.integers(N))})
    tms, tns = torch.tensor(ms, device=DEVICE), torch.tensor(ns, device=DEVICE)
    ref = np.zeros((len(ns), len(ms)), np.clongdouble)
    pl = np.zeros((len(ns), len(ms)), np.longdouble)
    kc = max(1, (1 << 22) // (len(ms) + len(ns)))
    for k0 in range(0, K, kc):
        bt = gather(B, dBn[tns], dBk[k0:k0 + kc]).cpu().numpy().astype(np.clongdouble)
        at = gather(A, dAk[k0:k0 + kc], dAm[tms]).cpu().numpy().astype(np.clongdouble)
        ref += bt @ at
        pl += np.abs(bt) @ np.abs(at)
    got = Cv[tns[:, None], tms[None, :]].cpu().numpy().astype(np.longdouble)
    tol = (2 * K + ks + 8) * U * pl
    ok = (np.abs(got[..., 0] - ref.real) <= tol) & (np.abs(got[..., 1] - ref.imag) <= tol)
    assert ok.all(), f"step {step} ({M}x{N}x{K}, class {cls}): sampled entries {np.argwhere(~ok)[:8].tolist()} outside the bound"
    return len(ms) * len(ns)


CASES = {"main_gates": ("main", None), "alt_haar": ("alt", 20261015)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_slice0_step_by_step(ctx, built_lib, monkeypatch, case):
    """Slice 0 of a config-5 tree, pair by pair, against FP64 and long-double references; then the sliced plan."""
    import torch
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedNetwork, SlicedPlan, _leaf_array
    name, seed = CASES[case]
    tn = network() if seed is None else haar_network(seed)
    path, sliced = tree(name)
    steps = replay(built_lib, name)
    ctx.trim()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(7)
    t0 = time.perf_counter()

    sn = SlicedNetwork(tn, sliced)
    net = sn.slice(sn.assignments[0])
    sctx = tb.Context(0)
    min_free = torch.cuda.mem_get_info()[0]
    try:
        with torch.cuda.stream(torch.cuda.ExternalStream(sctx.stream)):
            ts = [(list(t.legs), list(t.bond_dims), tb.DeviceTensor.from_numpy(sctx, _leaf_array(t))) for t in net.tensors]
            kinds_seen, sampled, arena_peak = [], 0, 0
            for step, ((i, j), (al, ad, bl, bd, cls, M, N, K)) in enumerate(zip(path.toplevel, steps)):
                (al2, ad2, da), (bl2, bd2, db) = ts[i], ts[j]
                assert (al2, bl2) == (al, bl)
                out_legs = [l for l in bl if l not in al] + [l for l in al if l not in bl]
                out_dims = [d for l, d in zip(bl, bd) if l not in al] + [d for l, d in zip(al, ad) if l not in bl]
                live0 = sctx.stats()["arena_live_bytes"]
                dc = tb.DeviceTensor.empty(sctx, out_dims)
                sctx.reset_stats()
                tb.contract_pair_into(sctx, al, da, bl, db, dc)
                cnt = sctx.engine_counts()
                arena_peak = max(arena_peak, sctx.stats()["arena_peak_bytes"])
                want = {0: ("k0", "k0_splitk"), 1: ("k1_dmma", "k1_dmma_splitk"), 2: ("k2",)}[cls]
                assert sum(cnt[c] for c in want) == 1 and sum(cnt.values()) == 1, (step, cls, cnt)
                kind = shape_kind(cls, M, N, K)
                if kind == "k1_128x128x2^23":     # the int8 engine refused (K too long): DMMA split-K, nothing leaked
                    assert cnt["k1_dmma_splitk"] == 1 and cnt["k1_tcgen05"] == 0, cnt
                if kind:
                    kinds_seen.append(kind)
                split = cnt["k0_splitk"] + cnt["k1_dmma_splitk"] > 0
                # upper bound on the K ranges of either split-K form (k0_config: <= 1024 and <= K/32; K1: <= K/128)
                ks = min(1024, max(1, K // 32)) if split else 1
                n, errors = check_step(torch, step, da, db, dc, gemm_view(al, ad, bl, bd), cls, ks, sm_count, rng)
                assert not errors, errors
                sampled += n
                if M * N * 16 >= 1 << 30 or M * K * 16 >= 1 << 30 or N * K * 16 >= 1 << 30:
                    min_free = min(min_free, torch.cuda.mem_get_info()[0])
                    torch.cuda.empty_cache()
                na, nb = int(np.prod(ad, dtype=np.int64)), int(np.prod(bd, dtype=np.int64))
                da.free(); db.free()
                sctx.synchronize()
                assert sctx.stats()["arena_live_bytes"] == live0 + arena_bytes(int(np.prod(out_dims, dtype=np.int64))) \
                    - arena_bytes(na) - arena_bytes(nb), step
                ts[i], ts[j] = (out_legs, out_dims, dc), None
            last = path.toplevel[-1][0]
            assert ts[last][0] == []
            amp_steps = complex(ts[last][2].to_numpy())
            ts[last][2].free()
        tr = sctx.trim()
    finally:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()     # (cached blocks were used on the context's stream)
        sctx.close()
    wall = time.perf_counter() - t0
    total = torch.cuda.get_device_properties(0).total_memory
    print(f"\n[{case}] {len(steps)} steps, {sampled} long-double samples, {wall:.1f} s; torch max_memory_allocated "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB, arena peak live {arena_peak / 2**30:.2f} GiB, arena reserved "
          f"{(tr['freed_bytes'] + tr['reserved_bytes']) / 2**30:.2f} GiB, device in use at most {(total - min_free) / 2**30:.2f} GiB")
    expect = {k: INVENTORY[name][k] for k in ("k2_2^26", "k1_32x64_2^25", "k1_64x32_2^24", "k1_128x128x2^23")}
    assert {k: kinds_seen.count(k) for k in expect} == expect
    assert amp_steps != 0

    # ---- 3. the executor the benchmark times, in a fresh context: slice 0 alone, bit for bit ----
    if name in PLAN_WS_GB:
        monkeypatch.setenv("TNCB_PLAN_WS_GB", PLAN_WS_GB[name])
    pctx = tb.Context(0)
    try:
        sp = SlicedPlan(tn, path, sliced, ctx=pctx)
        assert sp.n_slices == 64
        res = sp.plan.run_slices(0, 64)
        amp_plan = complex(res.to_numpy())
        del res, sp
    finally:
        pctx.close()
    assert np.array([amp_plan]).view(np.float64).tobytes() == np.array([amp_steps]).view(np.float64).tobytes(), \
        (amp_plan, amp_steps)


# ================================================================================================================
# 4. the whole amplitude
# ================================================================================================================
@pytest.mark.gpu
def test_config5_amplitude(ctx, monkeypatch):
    """All 64 slices through SlicedPlan.run(), both trees: they agree with each other and with the committed value."""
    import torch
    from tnc_b200.contractionpath.slicing import SlicedPlan
    ctx.trim()
    torch.cuda.empty_cache()
    amps = {}
    for name in TREES:
        path, sliced = tree(name)
        if name in PLAN_WS_GB:
            monkeypatch.setenv("TNCB_PLAN_WS_GB", PLAN_WS_GB[name])
        sp = SlicedPlan(network(), path, sliced, ctx=ctx)
        amps[name] = complex(sp.run().to_numpy())
        del sp
        monkeypatch.delenv("TNCB_PLAN_WS_GB", raising=False)
        ctx.trim()
    rel = lambda x, y: abs(x - y) / abs(y)
    assert rel(amps["alt"], amps["main"]) <= 1e-12, amps
    assert rel(amps["main"], CONFIG5_AMPLITUDE) <= 1e-12, amps
    assert rel(amps["alt"], CONFIG5_AMPLITUDE) <= 1e-12, amps
