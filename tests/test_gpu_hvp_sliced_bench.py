"""Sliced tangents and Hessian-vector products element by element at the sizes the feature exists for.

test_gpu_hvp_sliced.py checks R, Ṙ, G and Ġ of small networks against torch.func; at benchmark scale it checks bench.py's
network with 2 sliced legs against the unsliced Hessian-vector plan in one global scale (1e-9 x the largest entry over
all 489 leaves), which a wrong small leaf passes, and so does a wrong seed-tangent term (Ṡ·G1 is small next to the
largest S·H entry).  The 1- and 3-leg slicings and the 1024-slice Sycamore-53 depth-12 Hessian-vector slicing never run
on a device there.  Nor does any test compare a partial range (rank, world) with a reference for exactly its slices: a
slice-numbering error shared by the leaf extract, the tangent extract and the Ġ accumulate of run_sliced still maps
slices one to one, so every full-range sum stays right.  Nor is per-slice state checked at scale: the tangents
re-extracted every slice (the layout releases tangent slots), the seed tangent written per slice into memory the forward
levels freed (a memset when Ṡ is NULL), a call with only Ġ requested (the backward levels with only the Ġ accumulate),
and a carrier leaf (one with a sliced leg) left out of wrt, which keeps its extract item but gets no tangent or
accumulate item.  This file closes those gaps.

The reference uses no code of the library: leaves materialised by the oracle (test_gpu_vjp.leaf_array), slice q of the
leaves and of their tangents cut by numpy indexing (test_gpu_vjp_sliced_bench.cut, q's digits row-major over the sliced
legs, last leg fastest), each slice replayed forward-over-reverse by test_gpu_hvp_bench.reference_hvp with seed 1 and
Ṡ = 0 (R_q, Ṙ_q, G1_q, H_q), G1_q and H_q placed back into the full leaf shapes and folded in q order.  The result is a
scalar, so for any seed S and seed tangent Ṡ: G = S·ΣG1_q and Ġ = Ṡ·ΣG1_q + S·ΣH_q.

T, the tangent set on bench.py's network: test_gpu_hvp_bench.Q (the first 245 leaves in circuit order) without the
carriers 113 and 161.  It keeps the carriers 110, 114, 116 and 131, so at 2 legs wrt = T leaves the carriers 113 and
161 unrequested; tangents are random complex on T, zero elsewhere, and one unsliced replay serves the every-leaf plans
and the plans with wrt = T.

1. Host only.  T's membership and carriers; the 20 carriers of D12_HVP_LEGS on the depth-12 main tree, one sliced leg
   each, the same legs in the Haar-random network; the depth-12 tangent cluster D12_CLUSTER (the first 500 leaves in
   circuit order: the carriers up to leaf 488 in, the nine from 503 on out).  And the sliced reference itself: on a
   12-qubit network at 2 and 3 sliced legs with tangents on half of the leaves, the fold of every slice's embedded
   reference_hvp equals torch.func (test_gpu_hvp.reference_hvp) of the unsliced network.
2. bench.py's network (the int8 engine as bench.py runs it) at 1, 2 and 3 sliced legs, every leaf, seed cases (1, Ṡ
   NULL) and (random S, random Ṡ): all 489 full-shape G_l and Ġ_l against the unsliced host reference in per-leaf units,
   R and Ṙ, R bit for bit against run; SlicedPlan.for_tangents on the same legs.  At 2 legs wrt = T and a call with
   only Ġ requested.  At 3 legs the single slices q = 1 (digits 0,0,1) and q = 4 (1,0,0) and the range rank = 1,
   world = 3 (slices 1, 4, 7) against host replays of exactly those slices, with exact zeros outside their sub-blocks;
   every call bit for bit against a fold of a plain Hessian-vector (and tangent) plan over the host-sliced networks,
   engine counters included.  On the downloaded arrays: a Ġ whose slices are numbered first leg fastest passes the full
   range and fails q = 1, and a Ġ whose seed-tangent term reaches only the first slice fails the full range.
3. The Sycamore-53 depth-12 main tree on D12_HVP_LEGS (1024 slices) with Haar-random unitaries in place of the gates
   (the circuit's own gates give slices of exact-zero amplitude, which would hide addressing errors): the range rank = 1,
   world = 3 (341 slices, every digit of every leg, up to slice 1021) and the single slices q = 1 and q = 601, seed 1
   and a random Ṡ, leaf by leaf and bit for bit against the fold in q order of one plain Hessian-vector plan over the
   host-sliced networks, engine counters equal; the sliced tangent plan on the range likewise, and its Ṙ bit for bit
   against the Hessian-vector plan's (no pair of these slices runs on the int8 engine); slice 601 against a host replay.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, with 16 host CPUs (errors in units of each leaf's largest
reference entry), the GPU tests 465-496 s in all over two runs:
- the unsliced host reference of bench.py's network with tangents on T, once per module: 105-116 s, peak RSS 38.4 GiB;
- bench.py's network at 1, 2, 3 sliced legs: 3.0-4.7 s on the device each, arena peaks 26.9, 14.4 and 8.1 GiB, worst
  errors 8.3e-14, 9.8e-14, 1.1e-13 (G) and 2.4e-13, 2.3e-13, 4.3e-13 (Ġ), Ṙ of the tangent plans within 1.3e-13;
- the 3-leg ranges: 9.2-9.4 s on the device, 53-67 s for the host replays of slices 1, 4 and 7, worst errors (G, Ġ)
  1.9e-14, 2.8e-14 (q = 1), 6.2e-14, 1.4e-13 (q = 4) and 3.2e-14, 2.7e-14 (1, 4, 7); the digit-reversed Ġ fails q = 1
  on all 489 leaves, the Ġ with the seed tangent in the first slice only fails the full range on all 489;
- the 341 depth-12 slices: 277-282 s.  The sliced hvp takes 78 s, the plain hvp loop 94 s, the sliced jvp 20 s, the
  plain jvp loop 30-32 s; the arena peaks at 30.8 GiB; the host replay of slice 601 with D12_CLUSTER's tangents takes
  54-59 s (139 s on 8 host CPUs, at a peak RSS of 29.4 GiB), worst errors 1.4e-14 (G) and 2.8e-14 (Ġ)."""
import time

import numpy as np
import pytest

from test_gpu_backward_pairs import TAU, bench_net, outside, worst
from test_gpu_hvp import crandn
from test_gpu_hvp_bench import Q, reference_hvp
from test_gpu_sycamore_slices import haar_network, network, tree
from test_gpu_vjp import leaf_array
from test_gpu_vjp_sliced_bench import (BENCH_CARRIERS, BENCH_LEGS, HAAR_SEED, cut, destroy, digits, embed, fold, index,
                                       matrix_net, peak_rss_gib, random_seed, summed, zeros_outside)
from test_hvp_sliced_host import D12_HVP_LEGS

T = [l for l in Q if l not in (113, 161)]
D12_CARRIERS = [131, 133, 191, 192, 195, 204, 344, 359, 416, 429, 488, 503, 784, 805, 860, 862, 877, 881, 889, 935]
D12_CLUSTER = list(range(500))


# ================================================================================================================
# the reference: slices of leaves and tangents cut, results embedded by numpy indexing
# ================================================================================================================
def cut_tangents(tensors, tans, val):
    """{leaf: slice `val`'s sub-block of its tangent}"""
    return {l: np.ascontiguousarray(t[index(tensors[l].legs, val)]) for l, t in tans.items()}


def slice_reference(tensors, path, xs, tans, legs, q):
    """(R_q, Ṙ_q, {leaf: G1_q}, {leaf: H_q}) of slice q for seed 1 and Ṡ = 0, by reference_hvp on the host; G1_q and
    H_q embedded into the full leaf shapes"""
    import torch
    ts, arrs, val = cut(tensors, xs, legs, q)
    with torch.no_grad():
        R, Rd, g1, h = reference_hvp(ts, path, [torch.from_numpy(a) for a in arrs],
                                     {l: torch.from_numpy(t) for l, t in cut_tangents(tensors, tans, val).items()})
        out = (complex(R.item()), complex(Rd.item()), embed(tensors, {l: v.numpy() for l, v in g1.items()}, val),
               embed(tensors, {l: v.numpy() for l, v in h.items()}, val))
        del g1, h
    return out


def sliced_reference(tensors, path, xs, tans, legs, qs):
    """(ΣR_q, ΣṘ_q, {leaf: ΣG1_q}, {leaf: ΣH_q}) over the slices qs, folded in q order"""
    R, Rd, G1, H = 0j, 0j, None, None
    for q in qs:
        r, rd, g1, h = slice_reference(tensors, path, xs, tans, legs, q)
        R, Rd = R + r, Rd + rd
        G1, H = fold(G1, g1), fold(H, h)
    return R, Rd, G1, H


def seeded(ref, S, Sd, sel=None):
    """({leaf: G}, {leaf: Ġ}) of seed S and seed tangent Ṡ (None: 1 and 0) from a reference's G1 and H, for the leaves
    sel (None: all): G = S·G1, Ġ = Ṡ·G1 + S·H"""
    _, _, g1, h = ref
    s = 1.0 if S is None else complex(S)
    sd = 0.0 if Sd is None else complex(Sd)
    sel = sorted(g1) if sel is None else sel
    return {l: s * g1[l] for l in sel}, {l: sd * g1[l] + s * h[l] for l in sel}


def unpack(flat, offs, shapes):
    """{leaf: its block of a downloaded grad / grad-tangent block at grad_offsets()}"""
    return {i: flat[o:o + int(np.prod(s, dtype=np.int64))].reshape(s) for i, (o, s) in enumerate(zip(offs, shapes))
            if o >= 0}


def bench_tangents(xs):
    rng = np.random.default_rng(81)
    return {i: crandn(rng, xs[i].shape) for i in T}


# ================================================================================================================
# 1. host only
# ================================================================================================================
def test_tangent_set(built_lib):
    """T = Q without 113 and 161: 243 leaves, the first 245 in circuit order but two; it keeps the carriers 110, 114
    (legs 149, 156) and 116, 131 (leg 160) and leaves out 113 and 161, so every slicing has carriers with a tangent and
    carriers without one, and at 2 legs wrt = T leaves 113 and 161 unrequested."""
    tn, _ = bench_net()
    assert Q == list(range(245)) and len(T) == 243 and 113 not in T and 161 not in T
    assert sorted(c for c in BENCH_CARRIERS if c in T) == [110, 114, 116, 131]
    assert sorted(c for c in BENCH_CARRIERS if c not in T) == [113, 161]
    for n, legs in BENCH_LEGS.items():
        car = {i for i, t in enumerate(tn.tensors) if any(l in legs for l in t.legs)}
        assert car & set(T) and car - set(T), n
    car2 = {i for i, t in enumerate(tn.tensors) if any(l in BENCH_LEGS[2] for l in t.legs)}
    assert car2 - set(T) == {113, 161} and car2 & set(T) == {110, 114}


def test_d12_hvp_carriers(built_lib):
    """On the Sycamore-53 depth-12 main tree, the legs of D12_HVP_LEGS are carried by the 20 leaves D12_CARRIERS, one
    sliced leg each and each leg by two of them; the Haar-random network has the same legs.  D12_CLUSTER holds the
    carriers up to leaf 488 and leaves the nine from 503 on out."""
    tn = network()
    car = {i: [l for l in t.legs if l in D12_HVP_LEGS] for i, t in enumerate(tn.tensors)}
    car = {i: v for i, v in car.items() if v}
    assert sorted(car) == D12_CARRIERS
    assert all(len(v) == 1 for v in car.values())
    assert sorted(v[0] for v in car.values()) == sorted(D12_HVP_LEGS * 2)
    hn = haar_network(HAAR_SEED)
    assert [list(t.legs) for t in hn.tensors] == [list(t.legs) for t in tn.tensors]
    assert all(t.tensordata.kind == "matrix" for t in hn.tensors if len(t.legs) > 1)
    inside = [c for c in D12_CARRIERS if c in D12_CLUSTER]
    assert inside == D12_CARRIERS[:11] and inside[-1] == 488
    assert [c for c in D12_CARRIERS if c not in D12_CLUSTER] == D12_CARRIERS[11:]
    assert D12_CLUSTER == list(range(len(D12_CLUSTER))) and len(D12_CLUSTER) < len(tn.tensors)


@pytest.mark.parametrize("n_legs", [2, 3])
def test_sliced_reference_against_torch_func(built_lib, n_legs):
    """The fold over every slice of the embedded per-slice reference_hvp equals torch.func.jvp of torch.func.vjp of the
    unsliced TTGT replay (test_gpu_hvp.reference_hvp) for a random S and Ṡ, tangents on the first half of the leaves:
    Ṙ, every G_l = S·ΣG1_q and Ġ_l = Ṡ·ΣG1_q + S·ΣH_q (test_gpu_hvp.close), and ΣR_q against the replay.  The
    reference of sections 2 and 3 cuts leaves and tangents, replays and embeds slices right."""
    import torch
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    from test_gpu_hvp import amplitude_net, close, greedy, reference_hvp as torch_hvp, replay
    tn = amplitude_net(12, 6, 5)
    path = greedy(tn)
    assert list(leaves(tn)) == list(tn.tensors) and not path.nested
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert len(legs) == n_legs
    xs = [leaf_array(t) for t in tn.tensors]
    rng = np.random.default_rng(70 + n_legs)
    half = range(len(xs) // 2)
    tans = {i: crandn(rng, xs[i].shape) for i in half}
    car = [i for i, t in enumerate(tn.tensors) if any(l in legs for l in t.legs)]
    assert any(i in tans for i in car) and any(i not in tans for i in car)
    S, Sd = crandn(rng, ()), crandn(rng, ())
    ref = sliced_reference(tn.tensors, path, xs, tans, legs, range(2 ** n_legs))
    G, Gd = seeded(ref, S, Sd)
    every = list(range(len(xs)))
    Rd_t, G_t, Gd_t, sRd, sGd = torch_hvp(tn, path, xs, [tans.get(i, np.zeros_like(x)) for i, x in enumerate(xs)],
                                           S, Sd, every)
    R_t = complex(replay(tn, path, [torch.from_numpy(x) for x in xs])[1])
    assert abs(ref[0] - R_t) <= 1e-12 * abs(R_t)
    assert close(np.asarray(ref[1]), Rd_t, sRd), (ref[1], Rd_t)
    assert sorted(G) == sorted(Gd) == every
    for l in every:
        assert G[l].shape == Gd[l].shape == xs[l].shape, l
        assert np.abs(G[l] - G_t[l]).max() <= 1e-12 * np.abs(G_t[l]).max(), (l, np.abs(G[l] - G_t[l]).max())
        assert close(Gd[l], Gd_t[l], sGd[l]), (l, np.abs(Gd[l] - Gd_t[l]).max())


# ================================================================================================================
# 2. bench.py's network
# ================================================================================================================
@pytest.fixture(scope="module")
def bench_ref(built_lib):
    """(leaf arrays, tangents on T, (R, Ṙ, {leaf: G1}, {leaf: H})) of bench.py's UNSLICED network for seed 1 and Ṡ = 0,
    by reference_hvp on the host"""
    import torch
    tn, path = bench_net()
    xs = [leaf_array(t) for t in tn.tensors]
    tans = bench_tangents(xs)
    t0 = time.perf_counter()
    with torch.no_grad():
        R, Rd, g1, h = reference_hvp(tn.tensors, path, [torch.from_numpy(x) for x in xs],
                                     {i: torch.from_numpy(t) for i, t in tans.items()})
        ref = (complex(R.item()), complex(Rd.item()), {l: v.numpy() for l, v in g1.items()},
               {l: v.numpy() for l, v in h.items()})
        del g1, h
    print(f"\n[bench reference] unsliced replay {time.perf_counter() - t0:.1f} s, peak RSS {peak_rss_gib():.1f} GiB",
          flush=True)
    assert all(np.abs(ref[3][l]).max() > 0 for l in ref[3])         # every leaf's Ġ has a Hessian term
    return xs, tans, ref


def check_call(out, ref, S, Sd, sel):
    """R, Ṙ, G and Ġ of one hvp call against a reference, per-leaf units for G and Ġ; (worst G, worst Ġ)"""
    val, tan, G, Gd = out
    G_ref, Gd_ref = seeded(ref, S, Sd, sel)
    assert abs(complex(val) - ref[0]) <= TAU * abs(ref[0]), (complex(val), ref[0])
    assert abs(complex(tan) - ref[1]) <= TAU * abs(ref[1]), (complex(tan), ref[1])
    assert sorted(G) == sorted(Gd) == sel
    bad = outside(G, G_ref)
    assert not bad, ("G", bad[:8], worst(G, G_ref))
    bad = outside(Gd, Gd_ref)
    assert not bad, ("Ġ", bad[:8], worst(Gd, Gd_ref))
    return worst(G, G_ref), worst(Gd, Gd_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("n_legs", [1, 2, 3])
def test_bench_sliced_hvp(built_lib, bench_ref, n_legs):
    """bench.py's network sliced on 1, 2 or 3 legs (SlicedPlan.for_hvp, stage, hvp; the int8 engine as bench.py runs
    it), every leaf, tangents on T, seed cases (1, Ṡ NULL: the seed tangent memset) and (random S, random Ṡ): all 489
    full-shape G_l and Ġ_l against the unsliced host reference in units of max_e |ref_l| per leaf, tau = TAU (the
    argument of test_gpu_hvp_bench.test_bench_hvp_block); R and Ṙ within TAU, R bit for bit against run;
    k1_tcgen05 advanced in every call.  SlicedPlan.for_tangents on the same legs and tangents: Ṙ against the reference,
    its value bit for bit against run.  At 2 legs also: wrt = T (the carriers 113 and 161 unrequested: extracted, no
    tangent or accumulate item), G's and Ġ's keys exactly T; and outputs = (False, False, False, True), Ġ bit for bit
    the full call's.  One plan on the device at a time."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan
    tn, path = bench_net()
    xs, tans, ref = bench_ref
    legs = BENCH_LEGS[n_legs]
    full = matrix_net(tn.tensors, xs)
    rng = np.random.default_rng(91 + n_legs)
    S, Sd = random_seed(rng), random_seed(rng)
    every = list(range(len(xs)))
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    calls, peak = [], 0

    def call(fn):
        nonlocal peak
        ctx.synchronize()
        ctx.reset_stats()
        out = fn()
        ctx.synchronize()
        peak = max(peak, ctx.stats()["arena_peak_bytes"])
        return out, ctx.engine_counts()

    try:
        plans = [None] + ([T] if n_legs == 2 else [])
        for wrt in plans:                              # one plan on the device at a time
            sp = SlicedPlan.for_hvp(full, path, legs, wrt=wrt, ctx=ctx)
            sp.stage(full)
            assert sp.n_slices == 2 ** n_legs
            run = sp.run().to_numpy()
            for s, sd in ([(None, None)] if wrt is None else []) + [(S, Sd)]:
                out, ec = call(lambda: sp.hvp(tans, s, sd))
                calls.append((wrt, s, sd, out, ec, run))
            if n_legs == 2 and wrt is None:
                blocks, ec_only = call(lambda: sp.hvp_blocks(tans, S, Sd, outputs=(False, False, False, True)))
                assert blocks[:3] == [None, None, None]
                only = unpack(blocks[3].to_numpy(), sp.grad_offsets(), sp.plan.leaf_shapes)
                blocks[3].free()
            destroy(ctx, sp.plan)
        tp = SlicedPlan.for_tangents(full, path, legs, ctx=ctx)
        tp.stage(full)
        t_run = tp.run().to_numpy()
        (t_val, t_tan), t_ec = call(lambda: tp.jvp(tans))
        t_val = t_val.to_numpy()
        destroy(ctx, tp.plan)
    finally:
        ctx.close()
    t_dev = time.perf_counter() - t0
    errs = []
    for wrt, s, sd, out, ec, run in calls:
        assert ec["k1_tcgen05"] >= 1, (wrt is None, s is None, ec)
        assert out[0].tobytes() == run.tobytes()
        errs.append(check_call(out, ref, s, sd, every if wrt is None else T))
    if n_legs == 2:
        full_gd = calls[1][3][3]
        assert sorted(only) == every
        same = [l for l in every if only[l].tobytes() != full_gd[l].tobytes()]
        assert not same, same[:8]
        print(f"\n[bench sliced hvp, 2 legs] Ġ alone: bit for bit the full call's, engines {ec_only}", flush=True)
    assert t_ec["k1_tcgen05"] >= 1, t_ec
    assert t_val.tobytes() == t_run.tobytes() == calls[0][5].tobytes()
    assert abs(complex(t_tan) - ref[1]) <= TAU * abs(ref[1]), (complex(t_tan), ref[1])
    print(f"\n[bench sliced hvp, {n_legs} legs] device {t_dev:.1f} s, arena peak {peak / 2**30:.2f} GiB; worst per-leaf "
          f"error G {max(e[0] for e in errs):.2e}, Ġ {max(e[1] for e in errs):.2e}; Ṙ of the tangent plan "
          f"{abs(complex(t_tan) - ref[1]) / abs(ref[1]):.2e}; engines {calls[0][4]}, tangent plan {t_ec}", flush=True)


@pytest.mark.gpu
def test_bench_three_legs_ranges(built_lib, bench_ref):
    """bench.py's network on 3 sliced legs (8 slices), every leaf, tangents on T, seed S and seed tangent Ṡ:

    - single slices q = 1 (digits 0,0,1) and q = 4 (1,0,0) and the range rank = 1, world = 3 (slices 1, 4, 7), each
      against the fold of host replays of exactly those slices (R, Ṙ, and G, Ġ in per-leaf units, TAU), with every
      entry of a carrier's G and Ġ outside the covered sub-blocks exactly 0, and the value bit for bit against
      run(rank, world);
    - every call -- the full range with (1, Ṡ NULL) and with (S, Ṡ), every single slice, the range 1, 4, 7 -- bit for
      bit (==) against the fold in q order of a plain NetworkPlan.for_hvp staged with each host-sliced network and its
      cut tangents, with equal summed engine counters; the sliced tangent plan's calls likewise against a plain
      NetworkPlan.for_tangents;
    - on the downloaded arrays: a Ġ whose slices are numbered first leg fastest passes the full-range comparison and
      fails the q = 1 one; a Ġ whose seed-tangent term reaches only the first slice of the range (per slice, by
      linearity, Ġ_q(Ṡ = 0) = Ġ_q - (Ṡ/S)·G_q) fails the full-range one."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = bench_net()
    xs, tans, ref_full = bench_ref
    legs, n = BENCH_LEGS[3], 8
    rng = np.random.default_rng(61)
    S, Sd = random_seed(rng), random_seed(rng)
    s, sd = complex(S), complex(Sd)
    full = matrix_net(tn.tensors, xs)
    ranges = {"full": (0, 1), **{f"q={q}": (q, n) for q in range(n)}, "rank 1 of 3": (1, 3)}
    members = {k: list(range(r, n, w)) for k, (r, w) in ranges.items()}
    assert members["q=1"] == [1] and members["rank 1 of 3"] == [1, 4, 7]
    assert digits(1, [2, 2, 2]) == (0, 0, 1) and digits(4, [2, 2, 2]) == (1, 0, 0)
    every = list(range(len(xs)))
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    got, got_t, peak = {}, {}, 0

    def counted(fn):
        nonlocal peak
        ctx.synchronize()
        ctx.reset_stats()
        out = fn()
        ctx.synchronize()
        peak = max(peak, ctx.stats()["arena_peak_bytes"])
        return out, ctx.engine_counts()

    try:
        sp = SlicedPlan.for_hvp(full, path, legs, ctx=ctx)
        sp.stage(full)
        for key, (a, b) in [("full/1", (None, None))] + [(k, (S, Sd)) for k in ranges]:
            r, w = ranges[key.split("/")[0]]
            out, ec = counted(lambda: sp.hvp(tans, a, b, rank=r, world=w, allreduce=False))
            got[key] = (out, ec, sp.run(r, w, allreduce=False).to_numpy())
            assert ec["k1_tcgen05"] >= 1, (key, ec)
        destroy(ctx, sp.plan)
        tp = SlicedPlan.for_tangents(full, path, legs, ctx=ctx)
        tp.stage(full)
        for key, (r, w) in ranges.items():
            (v, t), ec = counted(lambda: tp.jvp(tans, rank=r, world=w, allreduce=False))
            got_t[key] = (v.to_numpy(), t, ec, tp.run(r, w, allreduce=False).to_numpy())
        destroy(ctx, tp.plan)
        # one plain plan of each kind, every host-sliced network and its cut tangents staged in turn
        nets = [cut(tn.tensors, xs, legs, q) for q in range(n)]
        cuts = [cut_tangents(tn.tensors, tans, val) for _, _, val in nets]
        per, per_t = {}, {}
        plain = NetworkPlan.for_hvp(matrix_net(*nets[0][:2]), path, ctx=ctx)
        for q, (ts, arrs, val) in enumerate(nets):
            plain.stage(matrix_net(ts, arrs))
            for one, (a, b) in ((True, (None, None)), (False, (S, Sd))):
                (v, t, g, gd), ec = counted(lambda: plain.hvp(cuts[q], a, b))
                per[q, one] = (v, t, embed(tn.tensors, g, val), embed(tn.tensors, gd, val), ec)
        destroy(ctx, plain)
        plain = NetworkPlan.for_tangents(matrix_net(*nets[0][:2]), path, ctx=ctx)
        for q, (ts, arrs, val) in enumerate(nets):
            plain.stage(matrix_net(ts, arrs))
            (v, t), ec = counted(lambda: plain.jvp(cuts[q]))
            per_t[q] = (v.to_numpy(), t, ec)
        destroy(ctx, plain)
    finally:
        ctx.close()
    t_dev = time.perf_counter() - t0

    def left_fold(xs_):
        return sum(xs_[1:], xs_[0].copy())

    # bit for bit against the plain plans' folds, engine counters summed over the slices
    for key, ((val, tan, G, Gd), ec, run) in got.items():
        one = key == "full/1"
        qs = members[key.split("/")[0]]
        assert val.tobytes() == run.tobytes(), key
        assert val == left_fold([per[q, one][0] for q in qs]), key
        assert tan == left_fold([per[q, one][1] for q in qs]), key
        for k, out in ((2, G), (3, Gd)):
            acc = None
            for q in qs:
                acc = fold(acc, per[q, one][k])
            assert sorted(out) == sorted(acc) == every, key
            same = [l for l in every if not np.array_equal(out[l], acc[l])]
            assert not same, (key, k, same[:8])
        assert ec == summed([per[q, one][4] for q in qs]), (key, ec)
    for key, (val, tan, ec, run) in got_t.items():
        qs = members[key]
        assert val.tobytes() == run.tobytes(), key
        assert val == left_fold([per_t[q][0] for q in qs]), key
        assert tan == left_fold([per_t[q][1] for q in qs]), key
        assert ec == summed([per_t[q][2] for q in qs]), (key, ec)
    print(f"\n[bench sliced hvp, 3 legs, ranges] device {t_dev:.1f} s, arena peak {peak / 2**30:.2f} GiB; "
          f"{len(got)} Hessian-vector and {len(got_t)} tangent calls bit for bit against the plain plans' folds",
          flush=True)

    # single slices and the range 1, 4, 7 against host replays of those slices
    t1 = time.perf_counter()
    host = {q: slice_reference(tn.tensors, path, xs, tans, legs, q) for q in (1, 4, 7)}
    t_ref = time.perf_counter() - t1
    errs = {}
    for key in ("q=1", "q=4", "rank 1 of 3"):
        qs = members[key]
        g1 = h = None
        for q in qs:
            g1, h = fold(g1, host[q][2]), fold(h, host[q][3])
        ref = (sum(host[q][0] for q in qs), sum(host[q][1] for q in qs), g1, h)
        out = got[key][0]
        errs[key] = check_call(out, ref, S, Sd, every)
        assert abs(complex(got_t[key][1]) - ref[1]) <= TAU * abs(ref[1]), key
        assert zeros_outside(tn.tensors, out[2], legs, qs) == [], key
        assert zeros_outside(tn.tensors, out[3], legs, qs) == [], key
    print(f"[bench sliced hvp, 3 legs, ranges] host replays of slices 1, 4, 7 {t_ref:.1f} s, peak RSS "
          f"{peak_rss_gib():.1f} GiB; worst per-leaf error (G, Ġ) "
          + ", ".join(f"{k} {g:.2e} {gd:.2e}" for k, (g, gd) in errs.items()), flush=True)

    # the comparator, 1: slices numbered first leg fastest.  Call q then computes and accumulates slice rev(q).
    rev = lambda q: int(np.ravel_multi_index(digits(q, [2, 2, 2])[::-1], [2, 2, 2]))
    assert [rev(q) for q in range(n)] == [0, 4, 2, 6, 1, 5, 3, 7]
    wrong = None
    for q in range(n):
        wrong = fold(wrong, per[rev(q), False][3])
    _, full_ref = seeded(ref_full, S, Sd)
    assert outside(got["full"][0][3], full_ref) == []
    assert outside(wrong, full_ref) == []                    # the full range cannot see the numbering
    _, one_ref = seeded(host[1], S, Sd)
    assert outside(per[1, False][3], one_ref) == []
    rejected = outside(per[rev(1), False][3], one_ref)        # q = 1 can
    assert rejected, "the q = 1 comparison accepts slices numbered first leg fastest"
    # the comparator, 2: the seed-tangent term only in the first slice of the range
    wrong = None
    for q in range(n):
        _, _, g, gd, _ = per[q, False]
        wrong = fold(wrong, gd if q == 0 else {l: gd[l] - (sd / s) * g[l] for l in gd})
    missed = outside(wrong, full_ref)
    assert missed, "the full-range comparison accepts a seed tangent that reaches only the first slice"
    print(f"[bench sliced hvp, 3 legs, ranges] digit-reversed numbering: full range accepted, q = 1 rejected on "
          f"{len(rejected)} of {len(xs)} leaves; seed tangent in the first slice only: full range rejected on "
          f"{len(missed)} of {len(xs)} leaves", flush=True)


# ================================================================================================================
# 3. Sycamore-53 depth-12, 1024 slices
# ================================================================================================================
@pytest.mark.gpu
def test_sycamore_d12_hvp_slices(built_lib):
    """The Sycamore-53 depth-12 main tree on D12_HVP_LEGS (1024 slices, 33.0 GB workspace per slice) with Haar-random
    unitaries for the gates, tangents on D12_CLUSTER, seed 1 and a random Ṡ, one plan on the device at a time:

    1. SlicedPlan.for_hvp, stage: the range rank = 1, world = 3 (slices 1, 4, ..., 1021: 341 slices; 3 is coprime to
       every radix, so every digit of every leg occurs) and the single slices q = 1 and q = 601 (digits of mixed
       value), downloaded; SlicedPlan.for_tangents on the same range.
    2. One NetworkPlan.for_hvp and one NetworkPlan.for_tangents of the host-sliced network, staged with each host-sliced
       network of the range in turn with its cut tangents: R, Ṙ, G and Ġ folded in q order from zeros.  Every call
       equals its fold bit for bit, leaf by leaf, with equal engine counters.  The sliced tangent plan's Ṙ equals the
       Hessian-vector plan's bit for bit: no pair of these slices runs on the int8 engine (k1_tcgen05 = 0 in both), so
       the forward and tangent pairs of the two plans run the same FP64 kernels.
    3. Slice 601 against a host reference_hvp replay: per-leaf units, tau = TAU; exact zeros outside its sub-blocks of
       the carriers; R and Ṙ against the replay's."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    path, _ = tree("main")
    hn = haar_network(HAAR_SEED)
    tensors = list(hn.tensors)
    xs = [leaf_array(t) for t in tensors]
    full = matrix_net(tensors, xs)
    rng = np.random.default_rng(101)
    tans = {i: crandn(rng, xs[i].shape) for i in D12_CLUSTER}
    Sd = random_seed(rng)
    n = 1024
    qs = list(range(1, n, 3))
    assert len(qs) == 341 and qs[-1] == 1021 and 601 in qs
    singles = (1, 601)
    dims = [2] * len(D12_HVP_LEGS)
    assert digits(601, dims) == (1, 0, 0, 1, 0, 1, 1, 0, 0, 1)
    every = list(range(len(tensors)))
    times, peak = {}, 0
    t0 = time.perf_counter()
    ctx = tb.Context(0)

    def counted(fn):
        nonlocal peak
        ctx.synchronize()
        ctx.reset_stats()
        out = fn()
        ctx.synchronize()
        peak = max(peak, ctx.stats()["arena_peak_bytes"])
        return out, ctx.engine_counts()

    try:
        sp = SlicedPlan.for_hvp(full, path, D12_HVP_LEGS, ctx=ctx)
        sp.stage(full)
        assert sp.n_slices == n
        t1 = time.perf_counter()
        rng_out, ec_rng = counted(lambda: sp.hvp(tans, None, Sd, rank=1, world=3, allreduce=False))
        times["sliced hvp, 341 slices"] = time.perf_counter() - t1
        one = {q: counted(lambda: sp.hvp(tans, None, Sd, rank=q, world=n, allreduce=False)) for q in singles}
        destroy(ctx, sp.plan)
        tp = SlicedPlan.for_tangents(full, path, D12_HVP_LEGS, ctx=ctx)
        tp.stage(full)
        t1 = time.perf_counter()
        (tv, tt), ec_t = counted(lambda: tp.jvp(tans, rank=1, world=3, allreduce=False))
        tv = tv.to_numpy()
        times["sliced jvp, 341 slices"] = time.perf_counter() - t1
        destroy(ctx, tp.plan)
        # the plain plans over the host-sliced networks of the range
        ts0, arrs0, _ = cut(tensors, xs, D12_HVP_LEGS, qs[0])
        t1 = time.perf_counter()
        plain = NetworkPlan.for_hvp(matrix_net(ts0, arrs0), path, ctx=ctx)
        acc, counts, per = [None, None, None, None], [], {}
        for q in qs:
            ts, arrs, vq = cut(tensors, xs, D12_HVP_LEGS, q)
            plain.stage(matrix_net(ts, arrs))
            (v, t, g, gd), ec = counted(lambda: plain.hvp(cut_tangents(tensors, tans, vq), None, Sd))
            counts.append(ec)
            g, gd = embed(tensors, g, vq), embed(tensors, gd, vq)
            acc[0] = v.copy() if acc[0] is None else acc[0] + v
            acc[1] = t.copy() if acc[1] is None else acc[1] + t
            acc[2], acc[3] = fold(acc[2], g), fold(acc[3], gd)
            if q in singles:
                per[q] = (v, t, g, gd, ec)
        destroy(ctx, plain)
        times["plain hvp loop, 341 slices"] = time.perf_counter() - t1
        t1 = time.perf_counter()
        plain = NetworkPlan.for_tangents(matrix_net(ts0, arrs0), path, ctx=ctx)
        tacc, tcounts = [None, None], []
        for q in qs:
            ts, arrs, vq = cut(tensors, xs, D12_HVP_LEGS, q)
            plain.stage(matrix_net(ts, arrs))
            (v, t), ec = counted(lambda: plain.jvp(cut_tangents(tensors, tans, vq)))
            v = v.to_numpy()
            tcounts.append(ec)
            tacc = [v.copy(), t.copy()] if tacc[0] is None else [tacc[0] + v, tacc[1] + t]
        destroy(ctx, plain)
        times["plain jvp loop, 341 slices"] = time.perf_counter() - t1
    finally:
        ctx.close()
    print(f"\n[d12 sliced hvp] " + ", ".join(f"{k} {v:.1f} s" for k, v in times.items())
          + f"; arena peak {peak / 2**30:.2f} GiB; engines of the range: hvp {ec_rng}, jvp {ec_t}", flush=True)

    def same_as(out, ref, what):
        val, tan, G, Gd = out
        assert val.tobytes() == ref[0].tobytes() and tan.tobytes() == ref[1].tobytes(), what
        for k, got in ((2, G), (3, Gd)):
            assert sorted(got) == sorted(ref[k]) == every, what
            diff = [l for l in every if not np.array_equal(got[l], ref[k][l])]
            assert not diff, (what, k, diff[:8])

    same_as(rng_out, acc, "range 1 of 3")
    assert ec_rng == summed(counts), (ec_rng, summed(counts))
    for q in singles:
        same_as(one[q][0], per[q], f"q={q}")
        assert one[q][1] == per[q][4], (q, one[q][1], per[q][4])
    assert tv.tobytes() == tacc[0].tobytes() and tt.tobytes() == tacc[1].tobytes()
    assert ec_t == summed(tcounts), (ec_t, summed(tcounts))
    assert ec_rng["k1_tcgen05"] == 0 and ec_t["k1_tcgen05"] == 0, (ec_rng, ec_t)
    assert tt.tobytes() == rng_out[1].tobytes()
    assert tv.tobytes() == rng_out[0].tobytes()
    print(f"[d12 sliced hvp] 341 of 1024 slices bit for bit through the folds; single slices {singles} bit for bit; "
          f"the tangent plan's Ṙ equals the Hessian-vector plan's", flush=True)
    del acc
    # slice 601 against a host replay
    t1 = time.perf_counter()
    ref = slice_reference(tensors, path, xs, tans, D12_HVP_LEGS, 601)
    times["host replay q=601"] = time.perf_counter() - t1
    assert ref[0] != 0 and ref[1] != 0 and all(np.abs(ref[2][l]).max() > 0 for l in ref[2])
    out = one[601][0]
    g_err, gd_err = check_call(out, ref, None, Sd, every)
    assert zeros_outside(tensors, out[2], D12_HVP_LEGS, [601]) == []
    assert zeros_outside(tensors, out[3], D12_HVP_LEGS, [601]) == []
    print(f"[d12 sliced hvp] host replay of q=601 {times['host replay q=601']:.1f} s, peak RSS {peak_rss_gib():.1f} GiB; "
          f"worst per-leaf error G {g_err:.2e}, Ġ {gd_err:.2e}; total {time.perf_counter() - t0:.1f} s", flush=True)
