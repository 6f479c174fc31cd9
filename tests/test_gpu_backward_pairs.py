"""Reverse-mode gradients element by element at the sizes the product exists for.

The gradient tests of smaller networks compare every G_l with a torch replay; at benchmark scale the suite otherwise
checks gradients through aggregates only (multilinearity, int8 engine against DMMA), which cannot see a leg-order error in
a symmetric leaf (sx, sz, fsim(0.3, 0.2)) or an error confined to small entries.  This file checks every backward pair
of those networks element by element.

1. Inventory (no GPU).  A restatement of network.cpp: build_backward with every leaf requested: walk the forward steps
   from the root; for each, the pair (adjoint C-bar, other operand) of operand a, then of operand b; the adjoint's legs
   are (other \\ C-bar) ++ (C-bar \\ other).  Pinned to the library: pair count and flops (same summation order) equal
   tncb_plan_info of a host-only gradient plan of bench.py's network and of a sliced gradient plan of the Sycamore-53
   depth-12 main tree on its 6 committed legs plus 1088, 155, 515 (one slice's structure).  Then the class counts by
   tncb_pair_kernel_class and the long-K shapes only the backward pass reaches: int8-engine pairs with K = 65536 (two K
   chunks of CRT_KCHUNK_MAX, 16 moduli) and K = 16384 on bench.py's network, DMMA split-K at 16 x 16 x 2^23 and K0 split-K
   at 16 x 8 x 2^23 in the slice.
2. Every backward pair of both inventories through tncb_contract_pair_into on random operands with a per-row exponent
   spread (test_gpu_engine_matrix.operand), in a fresh context with the default int8 settings, which plans the pair with
   the same plan_pair as the gradient plan and so takes the same engine.  Per pair: the engine counter; every output entry
   against four real FP64 torch matmuls on the GEMM view, their own rounding counted in; sampled entries -- first and last
   rows and columns, tile edges 63/64 and 127/128, K2 grid-stride seams -- against a long-double host sum.  Bounds:
     FP64 K0 / K1 / K2:  (2K + ksplit + 8) 2^-53 sum_k |b||a|
     int8 engine:        tcgen05_bound(K)["bound"] max|b[n,:]| max|a[m,:]|
   A K-range seam (the int8 K-chunk boundary 32767/32768, the K0 kchunk and K1 chunks_per_split boundaries) is not an
   output index: a term dropped, doubled or mis-addressed there moves every output entry by one term |b[n,k] a[k,m]|, which
   even at K = 2^23 is 2^5 times the FP64 bound of the entry (2^24 u sum_k, sum_k ~ K |term|) and far above the int8 one
   (K 2^-49 max|b| max|a| at K <= 65536), so the every-entry comparison covers the seams; the inventory asserts that the
   pairs have them.  Pairs whose legs, dims and operand roles agree after relabelling are checked once: 553 of bench.py's
   976 backward pairs and 595 of the slice's 2104 are distinct.
3. bench.py's whole gradient block, every leaf, seed 1 and a random complex seed, from NetworkPlan.for_gradients against
   an independent host replay of the same path with a hand-written reverse pass, element by element in per-leaf
   normwise units; plus the checks that this comparator rejects a transposed sx adjoint, which multilinearity accepts.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: bench.py's 553 distinct pairs (523 K0, 1 K0 split-K,
4 DMMA, 10 DMMA split-K, 14 int8 engine, 1 K2) in 167 s, torch max_memory_allocated 6.0 GiB, arena peak 15.5 GiB; the
slice's 595 (524 K0, 6 K0 split-K, 16 DMMA, 29 DMMA split-K, 20 K2) in 266 s, 4.5 GiB and 4.0 GiB; the whole gradient block
in 46 s, with its reference replay on the host.

Not covered here: Hessian-vector plans, whose pairs have the shapes of the forward and backward pairs (a tangent pair
copies its forward step's PairPlan, a backward-tangent pair its backward pair's); test_gpu_hvp_bench.py asserts that and
checks bench.py's whole Ġ block element by element.  Whole gradients of Sycamore slices: an autograd replay of a slice
with 2^27-element intermediates does not fit in host memory, but the hand-written reference_gradient below does (its
forward intermediates total 26.6 GB against 9.9 GB for bench.py's network; one slice took 64 s at a peak RSS of 29.2 GiB
on 8 CPU cores), and test_gpu_vjp_sliced_bench.py checks two slices of the 512-slice gradient with it."""
import ctypes as C
import functools
import os
import sys
import time

import numpy as np
import pytest

from test_gpu_engine_matrix import View, int8_route, k1_config, k1_ksplit, operand
from test_gpu_sycamore_slices import CHECK_BYTES, TMP_PER_ELEM, as_complex, check_step, edges, gemm_view, network, tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -53
D12_LEGS = [157, 1115, 231, 606, 1084, 986, 1088, 155, 515]     # the committed 6 + three more: 512 slices, 28.3 GB each
CRT_KCHUNK_MAX = 32768                                          # crt.cu: longest K chunk of the int8 engine
CRT_MAX_CHUNKS = 32                                             # crt.cu: the reconstruction sums at most 32 chunks


# ================================================================================================================
# 1. inventory
# ================================================================================================================
def _lib():
    from tnc_b200._lib import lib
    return lib()


def out_legs(al, ad, bl, bd):
    """legs and dims of contract(a, b): (b \\ a) ++ (a \\ b)"""
    return ([l for l in bl if l not in al] + [l for l in al if l not in bl],
            [d for l, d in zip(bl, bd) if l not in al] + [d for l, d in zip(al, ad) if l not in bl])


def mnk(al, ad, bl, bd):
    M = int(np.prod([d for l, d in zip(al, ad) if l not in bl], dtype=np.int64))
    N = int(np.prod([d for l, d in zip(bl, bd) if l not in al], dtype=np.int64))
    K = int(np.prod([d for l, d in zip(al, ad) if l in bl], dtype=np.int64))
    return M, N, K


def forward_steps(tensors, path, sliced=()):
    """(slot of a, slot of b, a legs, a dims, b legs, b dims) of every step of a replace-left path, sliced legs removed;
    a slot is ("leaf", i) or ("step", q)"""
    ts = [([l for l in t.legs if l not in sliced], [d for l, d in zip(t.legs, t.bond_dims) if l not in sliced])
          for t in tensors]
    slot = [("leaf", i) for i in range(len(ts))]
    steps = []
    for q, (i, j) in enumerate(path.toplevel):
        (al, ad), (bl, bd) = ts[i], ts[j]
        steps.append((slot[i], slot[j], al, ad, bl, bd))
        ts[i], ts[j] = out_legs(al, ad, bl, bd), None
        slot[i], slot[j] = ("step", q), None
    return steps


def backward_pairs(steps):
    """(C-bar legs, C-bar dims, other legs, other dims) of every backward pair, every leaf requested, in build_backward's
    order; the root's adjoint is the seed, with the result's legs"""
    adj = {("step", len(steps) - 1): out_legs(*steps[-1][2:])}
    pairs = []
    for q in range(len(steps) - 1, -1, -1):
        a, b, al, ad, bl, bd = steps[q]
        gl, gd = adj.pop(("step", q))
        for x, (ol, od) in ((a, (bl, bd)), (b, (al, ad))):
            pairs.append((gl, gd, ol, od))
            adj[x] = out_legs(gl, gd, ol, od)
    return pairs


def kernel_class(al, ad, bl, bd):
    from tnc_b200._lib import u64_array
    return _lib().tncb_pair_kernel_class(len(al), u64_array(al), u64_array(ad), len(bl), u64_array(bl), u64_array(bd))


def plan_info(h):
    n, k, pk = C.c_uint64(), C.c_uint64(), C.c_uint64()
    fl, by = C.c_double(), C.c_double()
    assert _lib().tncb_plan_info(h, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)) == 0
    return n.value, fl.value


def host_plan(tn, path, sliced=None):
    """a gradient plan of every leaf compiled without a device (sliced: tncb_plan_create_vjp_sliced)"""
    from tnc_b200._lib import u64_array
    from tnc_b200.tensornetwork.contraction import _Marshal
    m = _Marshal()
    ct, cp = m.tn(tn), m.path(path)
    h = C.c_void_p()
    if sliced is None:
        rc = _lib().tncb_plan_create_vjp(None, C.byref(ct), C.byref(cp), None, C.byref(h))
    else:
        rc = _lib().tncb_plan_create_vjp_sliced(None, C.byref(ct), C.byref(cp), len(sliced), u64_array(sliced), None,
                                                 C.byref(h))
    assert rc == 0, _lib().tncb_last_error()
    return h


@functools.lru_cache(maxsize=None)
def bench_net():
    sys.path.insert(0, ROOT)
    import bench
    tn = bench.build_network()
    return tn, bench.greedy_path(tn)


@functools.lru_cache(maxsize=None)
def inventory(name):
    """(forward steps, backward pairs with their kernel class and M, N, K) of bench.py's network or of one slice of the
    Sycamore-53 depth-12 main tree on D12_LEGS"""
    if name == "bench":
        tn, path = bench_net()
        steps = forward_steps(tn.tensors, path)
    else:
        path, _ = tree("main")
        steps = forward_steps(network().tensors, path, D12_LEGS)
    pairs = [p + (kernel_class(*p),) + mnk(*p) for p in backward_pairs(steps)]
    return steps, pairs


def canonical(gl, gd, ol, od):
    """the pair with its legs renumbered by first appearance: pairs with equal keys run the same GEMM view"""
    ren = {}
    for l in list(gl) + list(ol):
        ren.setdefault(l, len(ren))
    return tuple(ren[l] for l in gl), tuple(gd), tuple(ren[l] for l in ol), tuple(od)


def distinct(pairs):
    seen, out = set(), []
    for p in pairs:
        key = canonical(*p[:4])
        if key not in seen:
            seen.add(key)
            out.append(p)
    return out


# ---- the engine each pair takes, mirrored --------------------------------------------------------------------------
SM_COUNT = 132      # H100 SXM; the GPU tests pass the device's own count


def k0_split(M, N, K, sms):
    """kernels.cu: k0_config -> (ksplit, kchunk)"""
    MN, target, G = M * N, sms * 1024, 1
    while G < 32 and MN * G < target and G * 2 <= K:
        G *= 2
    ks, per_lane = 1, K // G
    if MN * G < target and per_lane > 64:
        ks = max(1, min(min(target // max(1, MN * G), per_lane // 32), 1024))
    kchunk = -(-K // ks)
    return -(-K // kchunk), kchunk


def int8_chunks(K):
    """K chunks of the int8 engine at least (crt.cu: launch_k1_crt, before the split for too few tiles); 0 = refused"""
    n = -(-K // CRT_KCHUNK_MAX)
    return n if n <= CRT_MAX_CHUNKS else 0


def engine(cls, M, N, K, sms=SM_COUNT):
    """(engine counter, K ranges) the default context gives one pair"""
    if cls == 2:
        return "k2", 1
    if cls == 0:
        ks, _ = k0_split(M, N, K, sms)
        return ("k0_splitk" if ks > 1 else "k0"), ks
    if int8_route(M, N, K) and int8_chunks(K):
        return "k1_tcgen05", int8_chunks(K)
    ks = k1_ksplit(k1_config(M, N), M, N, K, sms)
    return ("k1_dmma_splitk" if ks > 1 else "k1_dmma"), ks


BENCH_TOTAL = (1464, 20067874631496.0)
SLICE_TOTAL = (3156, 742871630832.0)
INVENTORY = {
    "bench": {"classes": {0: 946, 1: 28, 2: 2}, "distinct": 553},
    "slice": {"classes": {0: 2039, 1: 45, 2: 20}, "distinct": 595},
}


def test_inventory_matches_the_library(built_lib):
    """The restated backward schedule has the library's pair count and flops, bit for bit (forward steps first, then the
    backward pairs, both in the library's order)."""
    for name, total in (("bench", BENCH_TOTAL), ("slice", SLICE_TOTAL)):
        steps, pairs = inventory(name)
        flops = 0.0
        for s in steps:
            M, N, K = mnk(*s[2:])
            flops += 8.0 * M * N * K
        for *_, M, N, K in pairs:
            flops += 8.0 * M * N * K
        if name == "bench":
            h = host_plan(*bench_net())
        else:
            path, _ = tree("main")
            h = host_plan(network(), path, D12_LEGS)
        try:
            got = plan_info(h)
        finally:
            _lib().tncb_plan_destroy(h)
        assert got == total, (name, got)
        assert (len(steps) + len(pairs), flops) == total, name
        assert len(pairs) == 2 * len(steps)               # every leaf requested: two backward pairs per forward step


def test_inventory_long_k_shapes(built_lib):
    """Class counts, distinct pairs, and the long-K backward shapes no forward pair reaches."""
    for name in ("bench", "slice"):
        _, pairs = inventory(name)
        classes = {c: sum(1 for p in pairs if p[4] == c) for c in (0, 1, 2)}
        assert classes == INVENTORY[name]["classes"], (name, classes)
        assert len(distinct(pairs)) == INVENTORY[name]["distinct"], name
    # bench.py's network: int8-engine pairs with two K chunks (K = 65536, 16 moduli) and with K = 16384
    import tnc_b200 as tb
    _, pairs = inventory("bench")
    eng = [(engine(*p[4:]), p[5:]) for p in pairs]
    int8 = [mnk_ for (e, _), mnk_ in eng if e == "k1_tcgen05"]
    assert sorted({K for *_, K in int8 if K > CRT_KCHUNK_MAX}) == [65536]
    assert sorted({(M, N) for M, N, K in int8 if K == 65536}) == [(256, 128), (2048, 512), (4096, 2048)]
    assert sum(K > CRT_KCHUNK_MAX for *_, K in int8) == 3
    assert sum(K == 16384 for *_, K in int8) == 2
    assert int8_chunks(65536) == 2 and tb.tcgen05_bound(65536)["n_moduli"] == 16
    fwd = [mnk(*s[2:]) for s in inventory("bench")[0]]
    assert max(K for M, N, K in fwd if int8_route(M, N, K)) <= 2048          # the forward int8 pairs: one K chunk
    # the slice: DMMA split-K at 16 x 16 x 2^23 and K0 split-K at 16 x 8 x 2^23; no int8 pair
    _, pairs = inventory("slice")
    long_k = sorted({(engine(*p[4:])[0], *p[5:]) for p in pairs if p[7] >= 1 << 23})
    assert long_k == [("k0_splitk", 16, 8, 1 << 23), ("k1_dmma_splitk", 16, 16, 1 << 23)], long_k
    assert not any(engine(*p[4:])[0] == "k1_tcgen05" for p in pairs)
    assert sum(p[4] == 1 and p[7] >= 1 << 23 for p in pairs) == 7
    assert sum(p[4] == 0 and p[7] >= 1 << 23 for p in pairs) == 1
    # their K ranges on 132 SMs: 33 for K0, 264 for DMMA
    assert k0_split(16, 8, 1 << 23, SM_COUNT)[0] == 33
    assert k1_ksplit(k1_config(16, 16), 16, 16, 1 << 23, SM_COUNT) == 264


# ================================================================================================================
# 2. every backward pair against FP64 and long-double references
# ================================================================================================================
def check_int8_step(torch, da, db, dc, view, v, rng):
    """The int8 bound on every entry against four FP64 matmuls on the device (plus their own rounding), and on sampled
    entries against a long-double host sum; v: a View of the host operands (row maxima).  Failures come back as text (see
    test_gpu_sycamore_slices.check_step)."""
    try:
        return _check_int8_step(torch, as_complex(torch, da), as_complex(torch, db), as_complex(torch, dc), view, v, rng), []
    except Exception as e:
        return 0, [f"{type(e).__name__}: {e}"]


def _check_int8_step(torch, A, B, C, view, v, rng):
    import tnc_b200 as tb
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to("cuda")
    dAm, dBn, dAk, dBk = (dev(x) for x in view)
    M, N, K = len(dAm), len(dBn), len(dAk)
    unit = tb.tcgen05_bound(K)["bound"]
    mb, ma = dev(v.row_max_b()), dev(v.row_max_a())
    Cv = torch.view_as_real(C).view(N, M, 2)
    gather = lambda X, rows, cols: X[rows[:, None] + cols[None, :]]
    # column chunks whose running sums take at most half of CHECK_BYTES, K chunks within them the other half
    mc = max(1, min(M, (CHECK_BYTES // 2) // (48 * N)))
    n_kc = 0
    for m0 in range(0, M, mc):
        m1 = min(M, m0 + mc)
        kc = max(1, (CHECK_BYTES // 2) // (TMP_PER_ELEM * (N + m1 - m0)))
        cr = ci = p = None
        n_kc = 0
        for k0 in range(0, K, kc):
            Bt, At = gather(B, dBn, dBk[k0:k0 + kc]), gather(A, dAk[k0:k0 + kc], dAm[m0:m1])
            r = (Bt.real @ At.real - Bt.imag @ At.imag, Bt.real @ At.imag + Bt.imag @ At.real, Bt.abs() @ At.abs())
            del Bt, At
            cr, ci, p = r if cr is None else (cr + r[0], ci + r[1], p + r[2])
            del r
            n_kc += 1
        tol = unit * mb[:, None] * ma[None, m0:m1] + ((2 * K + 8) * U + n_kc * 2.0 ** -52) * p
        got = Cv[:, m0:m1]
        nbad = int((~((got[..., 0] - cr).abs() <= tol) | ~((got[..., 1] - ci).abs() <= tol)).sum())
        assert nbad == 0, f"{M}x{N}x{K} int8, columns {m0}..{m1}: {nbad} entries outside the bound"
    del cr, ci, p, tol
    ms, ns = edges(M), edges(N)
    ms = sorted(set(ms) | {int(x) for x in rng.integers(M, size=8)})
    ns = sorted(set(ns) | {int(x) for x in rng.integers(N, size=8)})
    tms, tns = torch.tensor(ms, device="cuda"), torch.tensor(ns, device="cuda")
    ref = np.zeros((len(ns), len(ms)), np.clongdouble)
    kc = max(1, (1 << 22) // (len(ms) + len(ns)))
    for k0 in range(0, K, kc):
        bt = gather(B, dBn[tns], dBk[k0:k0 + kc]).cpu().numpy().astype(np.clongdouble)
        at = gather(A, dAk[k0:k0 + kc], dAm[tms]).cpu().numpy().astype(np.clongdouble)
        ref += bt @ at
    got = Cv[tns[:, None], tms[None, :]].cpu().numpy().astype(np.longdouble)
    allowed = unit * (v.row_max_b()[ns][:, None] * v.row_max_a()[ms][None, :]).astype(np.longdouble)
    ok = (np.abs(got[..., 0] - ref.real) <= allowed) & (np.abs(got[..., 1] - ref.imag) <= allowed)
    assert ok.all(), f"{M}x{N}x{K} int8: sampled entries {np.argwhere(~ok)[:8].tolist()} outside the bound"
    return len(ms) * len(ns)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench", "slice"])
def test_every_backward_pair(built_lib, name):
    """Every distinct backward pair of bench.py's network (every leaf requested) or of one Sycamore-53 depth-12 slice on
    D12_LEGS, on random operands, through contract_pair_into in a fresh context.  Each pair's engine is asserted, every
    entry is checked in units of its engine's bound, and edges-included samples against long double; the arena's live
    bytes return to their value before each pair."""
    import torch
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    _, pairs = inventory(name)
    todo = distinct(pairs)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng({"bench": 31, "slice": 32}[name])
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    seen, sampled, arena_peak = {}, 0, 0
    ctx = tb.Context(0)
    try:
        with torch.cuda.stream(torch.cuda.ExternalStream(ctx.stream)):
            for idx, (gl, gd, ol, od, cls, M, N, K) in enumerate(todo):
                a = operand(rng, gd, [i for i, l in enumerate(gl) if l not in ol])
                b = operand(rng, od, [i for i, l in enumerate(ol) if l not in gl])
                ctx.synchronize()
                live0 = ctx.stats()["arena_live_bytes"]
                da, db = DeviceTensor.from_numpy(ctx, a), DeviceTensor.from_numpy(ctx, b)
                dc = DeviceTensor.empty(ctx, out_legs(gl, gd, ol, od)[1])
                ctx.reset_stats()
                tb.contract_pair_into(ctx, gl, da, ol, db, dc)
                cnt = ctx.engine_counts()
                arena_peak = max(arena_peak, ctx.stats()["arena_peak_bytes"])
                want, ks = engine(cls, M, N, K, sms)
                where = (name, idx, cls, M, N, K)
                assert cnt[want] == 1 and sum(cnt.values()) == 1, (where, want, cnt)
                seen[want] = seen.get(want, 0) + 1
                view = gemm_view(gl, gd, ol, od)
                if want == "k1_tcgen05":
                    assert ctx.last_tcgen05_info()["n_moduli"] == tb.tcgen05_bound(K)["n_moduli"], where
                    n, errors = check_int8_step(torch, da, db, dc, view, View(gl, a, ol, b), rng)
                else:
                    n, errors = check_step(torch, idx, da, db, dc, view, cls, ks, sms, rng)
                assert not errors, (where, errors)
                sampled += n
                da.free(); db.free(); dc.free()
                ctx.synchronize()
                assert ctx.stats()["arena_live_bytes"] == live0, where          # the engine's workspace went back
                del a, b, view
                if max(M * N, M * K, N * K) >= 1 << 24:
                    ctx.synchronize()
                    torch.cuda.empty_cache()
    finally:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        ctx.close()
    print(f"\n[{name}] {len(todo)} distinct of {len(pairs)} backward pairs, engines {seen}, {sampled} long-double samples, "
          f"{time.perf_counter() - t0:.1f} s; torch max_memory_allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB, "
          f"arena peak {arena_peak / 2**30:.2f} GiB")
    assert sum(seen.values()) == len(todo)
    if name == "bench":
        assert seen.get("k1_tcgen05", 0) >= 10, seen



# ================================================================================================================
# 3. bench.py's whole gradient block against an independent replay
# ================================================================================================================
def fused_permute(x, legs, order):
    """x (legs `legs`) with its legs in `order`, contiguous.  Runs of legs adjacent in both orders move as one axis, so a
    tensor of 28 legs of dimension 2 is permuted on a handful of axes."""
    pos = {l: i for i, l in enumerate(legs)}
    groups = []
    for l in order:
        if groups and pos[l] == pos[groups[-1][-1]] + 1:
            groups[-1].append(l)
        else:
            groups.append([l])
    src = sorted(range(len(groups)), key=lambda g: pos[groups[g][0]])
    dims = [int(np.prod([x.shape[pos[l]] for l in groups[g]], dtype=np.int64)) for g in src]
    y = x.reshape(dims).permute([src.index(g) for g in range(len(groups))])
    return y.contiguous().reshape([int(x.shape[pos[l]]) for l in order])


def tcontract(al, A, bl, B):
    """(legs, C) of contract(A, B) with torch: transpose, reshape, one GEMM; C's legs (b \\ a) ++ (a \\ b)"""
    shared = [l for l in al if l in bl]
    am = [l for l in al if l not in bl]
    bn = [l for l in bl if l not in al]
    dim = dict(zip(al, A.shape)) | dict(zip(bl, B.shape))
    size = lambda ls: int(np.prod([dim[l] for l in ls], dtype=np.int64))
    At = fused_permute(A, al, shared + am).reshape(size(shared), size(am))
    Bt = fused_permute(B, bl, bn + shared).reshape(size(bn), size(shared))
    return bn + am, (Bt @ At).reshape([int(dim[l]) for l in bn + am])


def reference_gradient(tensors, path, xs, seed):
    """(R, {leaf: G}) of a flat network along a replace-left path, by hand in torch: the forward steps keep their
    outputs, then the steps are walked from the root and each operand's adjoint is contract(adjoint of the output, the
    other operand) -- the chain rule of a multilinear contraction, G_l[e] = sum_r seed[r] dR[r]/dX_l[e], no conjugation.
    A leaf's adjoint is permuted into the leaf's own leg order."""
    steps = forward_steps(tensors, path)
    val = {("leaf", i): (list(t.legs), x) for i, (t, x) in enumerate(zip(tensors, xs))}
    for q, (a, b, *_) in enumerate(steps):
        val[("step", q)] = tcontract(*val[a], *val[b])
    root = ("step", len(steps) - 1)
    legs, R = val[root]
    adj = {root: (legs, seed.reshape(R.shape))}
    grads = {}
    for q in range(len(steps) - 1, -1, -1):
        a, b, *_ = steps[q]
        gl, g = adj.pop(("step", q))
        for x, other in ((a, b), (b, a)):
            xl, xbar = tcontract(gl, g, *val[other])
            if x[0] == "leaf":
                grads[x[1]] = fused_permute(xbar, xl, val[x][0])
            else:
                adj[x] = (xl, xbar)
        del g, xbar
        val.pop(a), val.pop(b)
        if q == len(steps) - 1:
            val.pop(root)
    return R, grads


TAU = 1e-10


def outside(G, ref, tau=TAU):
    """leaves l with an element outside |G_l - ref_l| <= tau max_e |ref_l|"""
    return [l for l in sorted(ref) if not np.all(np.abs(G[l] - ref[l]) <= tau * np.abs(ref[l]).max())]


def worst(G, ref):
    return max(float(np.abs(G[l] - ref[l]).max() / np.abs(ref[l]).max()) for l in ref)


@pytest.mark.gpu
def test_bench_gradient_block(built_lib):
    """bench.py's gradient block, all 489 leaves, from NetworkPlan.for_gradients (stage, run, vjp; the int8 engine as
    bench.py runs it) with seed 1 and with a random complex seed, element by element against an independent reference.

    Reference: reference_gradient, a complex128 TTGT replay of the same path with torch on the host (one GEMM per step),
    forward and then by hand backward; no code of this library.  The random seed's reference is S times seed 1's (G is
    linear in S).  The replay runs on the host: on the device, torch's replay of this path did not finish within seven
    minutes on an H100, while on the host it takes about 35 s; it holds the forward intermediates, 9.9 GB by their
    shapes.  On an H100 80GB HBM3 (700 W) with 16 host CPUs the whole test took 46 s.

    What this reaches that the pair tests do not: the plan's static layout, its level order and slot reuse, the seed, and
    grad_gather_kernel's permutation into each leaf's leg order.

    Units: max_e |G_ref_l| per leaf.  The sum of |terms| of an element (the same replay on |X_l|) is no usable scale
    here: a random circuit's amplitude cancels over 2^36 paths, and sum |terms| exceeds |G_l[e]| by 10^21 and more, so a
    comparator in those units accepts a transposed adjoint.  tau: every pair's bound is normwise (int8: K 2^-49
    max|b| max|a| per entry, FP64 pairs far tighter), a gradient element passes through at most 18 forward pairs (the
    tree's depth) and as many backward ones, and to first order their normwise relative errors add:
    36 * 2^-49 * kappa, where kappa = K max|b| max|a| / max|C| measures a pair's cancellation.  That stays below tau
    for kappa up to 1.5e3; the measured worst is 8.2e-14, and
    tau = 1e-10 keeps the checks below meaningful: a transposed leaf and a 1e-8 relative change of one element both lie
    far outside it.

    Then, on the downloaded arrays only: the comparator rejects G with one sx leaf's adjoint transposed, and with one
    element off by 1e-8 relative, while multilinearity (sum_e G_l[e] X_l[e] = R) accepts the transposed copy -- the blind
    spot of the multilinearity tests."""
    import torch
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from test_gpu_vjp import leaf_array
    tn, path = bench_net()
    lv = leaves(tn)
    assert len(lv) == len(tn.tensors) == 489
    xs = [leaf_array(l) for l in lv]
    steps, _ = inventory("bench")
    depth = {}
    for q, (a, b, *_) in enumerate(steps):
        depth[("step", q)] = max(depth.get(a, 0), depth.get(b, 0)) + 1
    assert max(depth.values()) == 18
    assert 2 * 18 * 16 * 2.0 ** -49 <= TAU / 50
    rng = np.random.default_rng(41)
    seeds = [None, np.array(complex(rng.standard_normal(), rng.standard_normal()))]
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    try:
        plan = NetworkPlan.for_gradients(tn, path, ctx=ctx)
        plan.stage(tn)
        got = []
        for s in seeds:
            R = plan.run().to_numpy()
            ctx.reset_stats()
            got.append(plan.vjp(s))
            assert ctx.engine_counts()["k1_tcgen05"] >= 1
        ctx._l.tncb_plan_destroy(plan.handle)           # its 15.24 GB workspace makes room for the reference
        plan.handle = None
        ctx.trim()
    finally:
        ctx.close()
    t_plan = time.perf_counter() - t0
    print(f"\n[bench gradient block] plan, two run + vjp: {t_plan:.1f} s", flush=True)
    # the reference, on the host: seed 1, then the random seed by linearity
    with torch.no_grad():
        R_ref, g = reference_gradient(tn.tensors, path, [torch.from_numpy(x) for x in xs],
                                      torch.tensor(1.0 + 0j, dtype=torch.complex128))
        ref1 = {l: v.numpy() for l, v in g.items()}
        R_ref = complex(R_ref.item())
        del g
    ref = [ref1 if s is None else {l: complex(s) * v for l, v in ref1.items()} for s in seeds]
    wall = time.perf_counter() - t0
    assert abs(complex(R) - R_ref) <= 1e-10 * abs(R_ref)
    print(f"[bench gradient block] {wall:.1f} s; worst |G_l - ref_l| / max|ref_l| "
          f"{max(worst(G, rf) for G, rf in zip(got, ref)):.2e}")
    for G, rf in zip(got, ref):
        assert sorted(G) == list(range(len(lv))) == sorted(rf)
        assert all(G[l].shape == rf[l].shape for l in rf)
        bad = outside(G, rf)
        assert not bad, (bad[:8], worst(G, rf))

    # the comparator sees what multilinearity cannot: one sx leaf's adjoint transposed ...
    G, rf = got[0], ref[0]
    sx = next(l for l, t in enumerate(lv) if t.tensordata.kind == "gate" and t.tensordata.gate[0] == "sx"
              and np.abs(G[l] - G[l].T).max() > 1e-3 * np.abs(G[l]).max())
    assert np.array_equal(xs[sx], xs[sx].T)
    bad = dict(G)
    bad[sx] = G[sx].T.copy()
    assert outside(bad, rf) == [sx]
    r = complex(R)
    for g in (G[sx], bad[sx]):                   # ... which sum_e G X = R accepts either way
        assert abs(complex(np.sum(g * xs[sx])) - r) <= 1e-9 * float(np.sum(np.abs(g) * np.abs(xs[sx])))
    # ... and one element off by 1e-8 relative: the largest element of an fsim leaf's adjoint
    l = next(l for l, t in enumerate(lv) if t.tensordata.kind == "gate" and t.tensordata.gate[0] == "fsim")
    e = int(np.argmax(np.abs(G[l])))
    off = dict(G)
    off[l] = G[l].copy()
    off[l].flat[e] *= 1 + 1e-8
    assert outside(off, rf) == [l]
