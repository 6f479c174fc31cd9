"""Sliced gradients element by element at the sizes the feature exists for.

test_gpu_vjp_sliced.py checks every G_l of small networks against torch autograd; at benchmark scale it checks bench.py's
network with 2 sliced legs against the unsliced gradient plan in one global scale (1e-9 x the largest entry over all 489
leaves), which a wrong small leaf passes, and nothing runs the 512-slice Sycamore-53 depth-12 gradient the feature was built
for.  Nor does any test compare a partial range (rank, world) with a reference for exactly its slices: a slice-numbering
error shared by slice_extract_kernel and grad_accumulate_kernel still maps slices one to one, so every full-range sum
stays right.  Nor does a single-slice call see a constant leaf (no sliced leg; copied into the workspace once per call by
run_sliced) clobbered by a later slice.  This file closes those gaps.

The reference uses no code of the library: leaves materialised by the oracle (test_gpu_vjp.leaf_array), slice q cut by
numpy indexing (arr[digit if sliced else :]) with q's digits row-major over the sliced legs, last leg fastest (the
documented order of slice_assignments), each slice replayed by test_gpu_backward_pairs.reference_gradient, and its
gradient placed back into the full leaf shape with the same indexing.

1. Host only.  The inputs are pinned: find_slices on bench.py's network gives [149], [149, 156], [149, 156, 160] for
   2, 4, 8 slices, carried by fsim leaves 110 and 113 (leg 149), 114 and 161 (156), 116 (160) at positions 1, 2 or 3,
   and by the sx leaf 131 (160) at position 0; on the depth-12 main tree 18 leaves carry one leg of D12_LEGS each and
   none carries two.  A leaf with several sliced legs stays covered only by the small
   test_gpu_vjp_sliced.test_every_leg_of_a_leaf_sliced.  And the sliced reference itself: on a 12-qubit network at 2 and
   3 sliced legs, the fold of every slice's embedded reference_gradient equals torch autograd of the unsliced replay.
2. bench.py's network (the int8 engine in every slice), 1, 2 and 3 sliced legs, every leaf, seed 1 and a random complex
   seed: all 489 full-shape G_l against the unsliced host reference in per-leaf units, the value against it and bit for
   bit against run_slices.  At 2 legs a wrt subset.  At 3 legs the single slices q = 1 (digits 0,0,1) and q = 4 (1,0,0)
   and the range rank = 1, world = 3 (slices 1, 4, 7) against host replays of exactly those slices, with exact zeros
   outside their sub-blocks; and every call bit for bit against a fold of a plain gradient plan over the host-sliced
   networks, engine counters included (the int8 engine falls back to DMMA when free memory is short, so equal counters
   are part of the claim).  The comparator accepts a gradient whose slices are numbered first leg fastest on the full
   range and rejects it on q = 1: why the partial ranges are here.
3. The Sycamore-53 depth-12 main tree on D12_LEGS, 512 slices, with Haar-random unitaries in place of the gates (the
   circuit's own gates give slices whose amplitude is exactly 0, which would hide addressing errors; the circuit's value
   is anchored to CONFIG5_AMPLITUDE by test_gpu_sycamore_slices).  The full 512-slice gradient equals, leaf by leaf and
   bit for bit, the fold in q order of a plain gradient plan over all 512 host-sliced networks: extract, accumulate and
   the constant-leaf copy are right for every slice.  Slices 0 and 300 against host replays: the schedule they share is
   right element by element.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, with 16 host CPUs (errors in units of each leaf's largest
reference entry):
- the unsliced host reference of bench.py's network, once per module: 38-40 s, peak RSS 23.4 GiB;
- bench.py's network at 1, 2, 3 sliced legs: about 1 s each, arena peaks 16.8, 8.9 and 5.0 GiB, worst errors 7.8e-14,
  9.8e-14 and 1.1e-13;
- the 3-leg ranges: 24 s (3 s on the device, 21 s for the host replays of slices 1, 4 and 7), worst errors 1.9e-14
  (q = 1), 6.2e-14 (q = 4) and 3.2e-14 (1, 4, 7); the digit-reversed gradient fails q = 1 on all 489 leaves;
- the 512 Haar slices: 245-250 s.  The sliced vjp takes 63 s, the plain loop 80 s (0.16 s per slice), each host replay
  of slice 0 or 300 43-51 s at a peak RSS of 34 GiB; the arena peaks at 26.4 GiB; all 512 slices equal bit for bit;
  worst errors 1.5e-14 (q = 0) and 2.1e-14 (q = 300)."""
import resource
import time

import numpy as np
import pytest

from test_gpu_backward_pairs import D12_LEGS, TAU, bench_net, outside, reference_gradient, worst
from test_gpu_sycamore_slices import haar_network, network, tree
from test_gpu_vjp import leaf_array

BENCH_LEGS = {1: [149], 2: [149, 156], 3: [149, 156, 160]}
BENCH_CARRIERS = {110: (149, 3), 113: (149, 1), 114: (156, 2), 161: (156, 1), 116: (160, 2), 131: (160, 0)}
HAAR_SEED = 20261016
ENGINES = ["k0", "k0_splitk", "k1_dmma", "k1_dmma_splitk", "k1_tcgen05", "k2", "permute", "reserved"]


# ================================================================================================================
# the reference: slices cut and gradients embedded by numpy indexing
# ================================================================================================================
def digits(q, dims):
    """slice q's digit vector: row-major over the sliced legs, last leg fastest"""
    return tuple(int(d) for d in np.unravel_index(q, dims))


def index(leaf_legs, val):
    """the numpy index of a slice's sub-block of a full leaf: the digit on a sliced leg, everything on the others"""
    return tuple(val[l] if l in val else slice(None) for l in leaf_legs)


def cut(tensors, xs, legs, q):
    """(leaf Tensors with the sliced legs removed, their arrays, {leg: digit}) of slice q"""
    from tnc_b200.tensornetwork import Tensor
    dim = {l: int(d) for t in tensors for l, d in zip(t.legs, t.bond_dims)}
    val = dict(zip(legs, digits(q, [dim[l] for l in legs])))
    ts, arrs = [], []
    for t, x in zip(tensors, xs):
        keep = [(l, int(d)) for l, d in zip(t.legs, t.bond_dims) if l not in val]
        ts.append(Tensor([l for l, _ in keep], [d for _, d in keep]))
        arrs.append(np.ascontiguousarray(x[index(t.legs, val)]))
    return ts, arrs, val


def matrix_net(ts, arrs):
    """a flat network of Matrix leaves with these legs and payloads"""
    from tnc_b200.tensornetwork import Tensor, TensorData
    return Tensor.new_composite([Tensor(list(t.legs), list(t.bond_dims), tensordata=TensorData.Matrix(a))
                                 for t, a in zip(ts, arrs)])


def embed(tensors, g, val):
    """{leaf: full-shape array} with slice `val`'s gradient g in its sub-block and zeros elsewhere"""
    out = {}
    for l, v in g.items():
        t = tensors[l]
        full = np.zeros([int(d) for d in t.bond_dims], np.complex128)
        full[index(t.legs, val)] = v
        out[l] = full
    return out


def fold(acc, g):
    """acc + g leaf by leaf (acc None: zeros), in place"""
    if acc is None:
        return {l: np.zeros_like(v) + v for l, v in g.items()}
    for l, v in g.items():
        acc[l] += v
    return acc


def sliced_reference(tensors, path, xs, legs, qs):
    """(sum of R, {leaf: sum of embedded G}) over the slices qs in q order, seed 1, each slice replayed on the host"""
    import torch
    R, acc = 0j, None
    for q in qs:
        ts, arrs, val = cut(tensors, xs, legs, q)
        with torch.no_grad():
            r, g = reference_gradient(ts, path, [torch.from_numpy(a) for a in arrs],
                                      torch.tensor(1.0 + 0j, dtype=torch.complex128))
            g = {l: v.numpy() for l, v in g.items()}
        R += complex(r.item())
        acc = fold(acc, embed(tensors, g, val))
        del g
    return R, acc


def zeros_outside(tensors, G, legs, qs):
    """carrier leaves l (a sliced leg among their legs) with a nonzero entry outside the sub-blocks of the slices qs"""
    dim = {l: int(d) for t in tensors for l, d in zip(t.legs, t.bond_dims)}
    bad = []
    for l in sorted(G):
        t = tensors[l]
        if not any(x in legs for x in t.legs):
            continue
        mask = np.ones(G[l].shape, bool)
        for q in qs:
            mask[index(t.legs, dict(zip(legs, digits(q, [dim[x] for x in legs]))))] = False
        if np.any(G[l][mask] != 0):
            bad.append(l)
    return bad


def peak_rss_gib():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20


def summed(counts):
    return {k: sum(c[k] for c in counts) for k in ENGINES}


def destroy(ctx, plan):
    """give a plan's workspace back now (NetworkPlan; a SlicedPlan's is .plan)"""
    ctx._l.tncb_plan_destroy(plan.handle)
    plan.handle = None
    ctx.trim()


# ================================================================================================================
# 1. host only
# ================================================================================================================
def test_bench_sliced_legs_and_carriers(built_lib):
    """find_slices on bench.py's network for 2, 4, 8 slices, and the leaves that carry those legs: fsim leaves with the
    sliced leg at positions 1, 2 or 3 and one sx leaf with it at position 0."""
    from tnc_b200.contractionpath.slicing import find_slices
    tn, path = bench_net()
    assert len(tn.tensors) == 489 and not path.nested
    for n, legs in BENCH_LEGS.items():
        assert find_slices(tn, path, min_slices=2 ** n) == legs, n
        car = {i: t for i, t in enumerate(tn.tensors) if any(l in legs for l in t.legs)}
        assert sorted(car) == sorted(i for i, (l, _) in BENCH_CARRIERS.items() if l in legs), n
    for i, (leg, pos) in BENCH_CARRIERS.items():
        t = tn.tensors[i]
        assert t.tensordata.kind == "gate" and t.tensordata.gate[0] == ("sx" if i == 131 else "fsim"), i
        assert list(t.legs).index(leg) == pos and [l for l in t.legs if l in BENCH_LEGS[3]] == [leg], i
        assert t.bond_dims[pos] == 2


def test_d12_carriers(built_lib):
    """On the Sycamore-53 depth-12 main tree, each leg of D12_LEGS is carried by two leaves and no leaf carries two:
    18 carriers, the same set in the Haar-random network.  A leaf with several sliced legs is checked only by
    test_gpu_vjp_sliced.test_every_leg_of_a_leaf_sliced, on a 12-qubit network."""
    tn = network()
    car = {i: [l for l in t.legs if l in D12_LEGS] for i, t in enumerate(tn.tensors)}
    car = {i: v for i, v in car.items() if v}
    assert len(car) == 18 and all(len(v) == 1 for v in car.values())
    assert sorted(v[0] for v in car.values()) == sorted(D12_LEGS * 2)
    hn = haar_network(HAAR_SEED)
    assert [list(t.legs) for t in hn.tensors] == [list(t.legs) for t in tn.tensors]
    assert all(t.tensordata.kind == "matrix" for t in hn.tensors if len(t.legs) > 1)


@pytest.mark.parametrize("n_legs", [2, 3])
def test_sliced_reference_against_autograd(built_lib, n_legs):
    """The fold over every slice of the embedded per-slice reference_gradient equals torch autograd of the unsliced TTGT
    replay (test_gpu_vjp_sliced.reference_grads), within 1e-12 of each leaf's largest entry, and the summed R equals the
    replay's: the reference of sections 2 and 3 cuts, replays and embeds slices right."""
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    from test_gpu_vjp_sliced import amplitude_net, greedy, reference_grads
    tn = amplitude_net(12, 6, 5)
    path = greedy(tn)
    assert list(leaves(tn)) == list(tn.tensors) and not path.nested
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    assert len(legs) == n_legs
    xs = [leaf_array(t) for t in tn.tensors]
    R, G = sliced_reference(tn.tensors, path, xs, legs, range(2 ** n_legs))
    _, R_t, G_t = reference_grads(tn, path)
    assert abs(R - complex(R_t)) <= 1e-12 * abs(complex(R_t))
    assert sorted(G) == list(range(len(xs)))
    for l in G:
        assert G[l].shape == G_t[l].shape == xs[l].shape, l
        assert np.abs(G[l] - G_t[l]).max() <= 1e-12 * np.abs(G_t[l]).max(), (l, np.abs(G[l] - G_t[l]).max())
    assert any(any(x in legs for x in t.legs) for t in tn.tensors)


# ================================================================================================================
# 2. bench.py's network
# ================================================================================================================
@pytest.fixture(scope="module")
def bench_ref(built_lib):
    """(leaf arrays, R, {leaf: G}) of bench.py's UNSLICED network for seed 1, by reference_gradient on the host"""
    import torch
    tn, path = bench_net()
    xs = [leaf_array(t) for t in tn.tensors]
    t0 = time.perf_counter()
    with torch.no_grad():
        R, g = reference_gradient(tn.tensors, path, [torch.from_numpy(x) for x in xs],
                                  torch.tensor(1.0 + 0j, dtype=torch.complex128))
        ref = {l: v.numpy() for l, v in g.items()}
        R = complex(R.item())
        del g
    print(f"\n[bench reference] unsliced replay {time.perf_counter() - t0:.1f} s, peak RSS {peak_rss_gib():.1f} GiB",
          flush=True)
    return xs, R, ref


def random_seed(rng):
    return np.asarray(complex(rng.standard_normal(), rng.standard_normal()))


@pytest.mark.gpu
@pytest.mark.parametrize("n_legs", [1, 2, 3])
def test_bench_sliced_gradient(built_lib, bench_ref, n_legs):
    """bench.py's network sliced on 1, 2 or 3 legs (SlicedPlan.for_gradients, stage, vjp; the int8 engine as bench.py
    runs it), every leaf, seed 1 and a random complex seed S: all 489 full-shape G_l against the unsliced host reference
    (S times seed 1's) in units of max_e |ref_l| per leaf, tau = TAU (the argument of
    test_gpu_backward_pairs.test_bench_gradient_block: every pair's bound is normwise, the depth 18); the value against
    R and bit for bit against run_slices; k1_tcgen05 advanced in every call.  At 2 legs also wrt = the four carriers plus
    every fifth other leaf: G's keys are that subset and each G_l matches."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan
    tn, path = bench_net()
    xs, R1, ref1 = bench_ref
    legs = BENCH_LEGS[n_legs]
    full = matrix_net(tn.tensors, xs)
    seeds = [None, random_seed(np.random.default_rng(51 + n_legs))]
    plans = [(None, seeds)]
    if n_legs == 2:
        carriers = sorted(i for i, (l, _) in BENCH_CARRIERS.items() if l in legs)
        assert carriers == [110, 113, 114, 161]
        plans.append((sorted(carriers + [l for l in range(len(xs)) if l not in carriers][::5]), seeds[1:]))
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    calls, peak = [], 0
    try:
        for wrt, ss in plans:                        # one plan on the device at a time
            sp = SlicedPlan.for_gradients(full, path, legs, wrt=wrt, ctx=ctx)
            sp.stage(full)
            assert sp.n_slices == 2 ** n_legs
            run = sp.run().to_numpy()
            for s in ss:
                ctx.synchronize()
                ctx.reset_stats()
                val, G = sp.vjp(s)
                ctx.synchronize()
                calls.append((wrt, s, val.to_numpy(), G, ctx.engine_counts(), run))
                peak = max(peak, ctx.stats()["arena_peak_bytes"])
            destroy(ctx, sp.plan)
    finally:
        ctx.close()
    errs = []
    for w, s, val, G, ec, run in calls:
        scale = 1.0 if s is None else complex(s)
        sel = list(range(len(xs))) if w is None else w
        ref = {l: scale * ref1[l] for l in sel}
        assert ec["k1_tcgen05"] >= 1, ec
        assert val.tobytes() == run.tobytes()
        assert abs(complex(val) - R1) <= TAU * abs(R1)
        assert sorted(G) == sel
        assert all(G[l].shape == xs[l].shape for l in sel)
        bad = outside(G, ref)
        assert not bad, (w is not None, bad[:8], worst(G, ref))
        errs.append(worst(G, ref))
    print(f"\n[bench sliced, {n_legs} legs] {time.perf_counter() - t0:.1f} s, arena peak {peak / 2**30:.2f} GiB, "
          f"worst |G_l - ref_l| / max|ref_l| {max(errs):.2e}, engines {calls[0][4]}", flush=True)


@pytest.mark.gpu
def test_bench_three_legs_ranges(built_lib, bench_ref):
    """bench.py's network on 3 sliced legs (8 slices), seed S:

    - single slices q = 1 (digits 0,0,1) and q = 4 (1,0,0) and the range rank = 1, world = 3 (slices 1, 4, 7), each
      against the fold of host replays of exactly those host-sliced networks (per-leaf units, TAU), with every entry of a
      carrier leaf outside the covered sub-blocks exactly 0, and the value bit for bit against run(rank, world);
    - every call -- the full range with seed 1 and with S, every single slice, the range 1, 4, 7 -- bit for bit (==)
      against the fold in q order of a plain NetworkPlan.for_gradients over the host-sliced networks of its slices, with
      equal engine counters per slice;
    - on the downloaded arrays: a gradient whose slices are numbered first leg fastest (slice q computed and accumulated
      at the digit-reversed slice, the same error in extract and accumulate) passes the full-range comparison and fails
      the q = 1 one."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = bench_net()
    xs, R1, ref1 = bench_ref
    legs, n = BENCH_LEGS[3], 8
    S = random_seed(np.random.default_rng(61))
    s = complex(S)
    full = matrix_net(tn.tensors, xs)
    ranges = {"full": (0, 1), **{f"q={q}": (q, n) for q in range(n)}, "rank 1 of 3": (1, 3)}
    members = {k: list(range(r, n, w)) for k, (r, w) in ranges.items()}
    assert members["q=1"] == [1] and members["rank 1 of 3"] == [1, 4, 7]
    assert digits(1, [2, 2, 2]) == (0, 0, 1) and digits(4, [2, 2, 2]) == (1, 0, 0)
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    got, peak = {}, 0
    try:
        sp = SlicedPlan.for_gradients(full, path, legs, ctx=ctx)
        sp.stage(full)
        for key, seed in [("full/1", None)] + [(k, S) for k in ranges]:
            r, w = ranges[key.split("/")[0]]
            ctx.synchronize()
            ctx.reset_stats()
            val, G = sp.vjp(seed, rank=r, world=w, allreduce=False)
            ctx.synchronize()
            ec = ctx.engine_counts()
            peak = max(peak, ctx.stats()["arena_peak_bytes"])
            got[key] = (val.to_numpy(), G, ec, sp.run(r, w, allreduce=False).to_numpy())
            assert ec["k1_tcgen05"] >= 1, (key, ec)
        destroy(ctx, sp.plan)
        # one plain gradient plan, every slice staged in turn: run + vjp with seed 1 and with S
        nets = [cut(tn.tensors, xs, legs, q) for q in range(n)]
        plain = NetworkPlan.for_gradients(matrix_net(*nets[0][:2]), path, ctx=ctx)
        per = {}
        for q, (ts, arrs, val) in enumerate(nets):
            plain.stage(matrix_net(ts, arrs))
            for seed in (None, S):
                ctx.synchronize()
                ctx.reset_stats()
                r = plain.run().to_numpy()
                g = plain.vjp(seed)
                ctx.synchronize()
                per[q, seed is None] = (r, embed(tn.tensors, g, val), ctx.engine_counts())
                peak = max(peak, ctx.stats()["arena_peak_bytes"])
        destroy(ctx, plain)
    finally:
        ctx.close()
    t_dev = time.perf_counter() - t0
    # bit for bit against the plain plan's fold, engine counters per slice
    for key, (val, G, ec, run) in got.items():
        one = key == "full/1"
        qs = members[key.split("/")[0]]
        assert val.tobytes() == run.tobytes(), key
        r_fold = sum((per[q, one][0] for q in qs[1:]), per[qs[0], one][0].copy())
        G_fold = None
        for q in qs:
            G_fold = fold(G_fold, per[q, one][1])
        assert val == r_fold, key
        assert sorted(G) == sorted(G_fold) == list(range(len(xs))), key
        same = [l for l in G if not np.array_equal(G[l], G_fold[l])]
        assert not same, (key, same[:8])
        assert ec == summed([per[q, one][2] for q in qs]), (key, ec)
    # single slices and the range 1, 4, 7 against host replays of those slices
    t1 = time.perf_counter()
    host = {}
    for q in (1, 4, 7):
        host[q] = sliced_reference(tn.tensors, path, xs, legs, [q])
    t_ref = time.perf_counter() - t1
    errs = {}
    for key in ("q=1", "q=4", "rank 1 of 3"):
        qs = members[key]
        R = sum(host[q][0] for q in qs)
        ref = None
        for q in qs:
            ref = fold(ref, host[q][1])
        ref = {l: s * v for l, v in ref.items()}
        val, G, _, _ = got[key]
        assert abs(complex(val) - R) <= TAU * abs(R), key          # the value does not depend on the seed
        bad = outside(G, ref)
        assert not bad, (key, bad[:8], worst(G, ref))
        assert zeros_outside(tn.tensors, G, legs, qs) == [], key
        errs[key] = worst(G, ref)
    print(f"\n[bench sliced, 3 legs, ranges] device {t_dev:.1f} s, host replays of slices 1, 4, 7 {t_ref:.1f} s, "
          f"arena peak {peak / 2**30:.2f} GiB, peak RSS {peak_rss_gib():.1f} GiB; worst per-leaf error "
          + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()), flush=True)

    # the comparator: slices numbered first leg fastest.  Call q then computes and accumulates slice rev(q).
    rev = lambda q: int(np.ravel_multi_index(digits(q, [2, 2, 2])[::-1], [2, 2, 2]))
    assert [rev(q) for q in range(n)] == [0, 4, 2, 6, 1, 5, 3, 7]
    wrong = None
    for q in range(n):
        wrong = fold(wrong, per[rev(q), False][1])
    full_ref = {l: s * v for l, v in ref1.items()}
    assert outside(got["full"][1], full_ref) == []
    assert outside(wrong, full_ref) == []                    # the full range cannot see the numbering
    one_ref = {l: s * v for l, v in host[1][1].items()}
    assert outside(per[1, False][1], one_ref) == []
    rejected = outside(per[rev(1), False][1], one_ref)        # q = 1 can
    assert rejected, "the q = 1 comparison accepts slices numbered first leg fastest"
    print(f"[bench sliced, 3 legs, ranges] digit-reversed numbering: full range accepted, q = 1 rejected on "
          f"{len(rejected)} of {len(xs)} leaves", flush=True)


# ================================================================================================================
# 3. Sycamore-53 depth-12, 512 slices
# ================================================================================================================
@pytest.mark.gpu
def test_sycamore_d12_all_slices(built_lib):
    """The Sycamore-53 depth-12 main tree on D12_LEGS (512 slices, 28.3 GB workspace per slice) with Haar-random
    unitaries for the gates, seed 1, one plan on the device at a time:

    1. SlicedPlan.for_gradients, stage: the full vjp (its value bit for bit against run) and the single-slice ranges
       q = 0 and q = 300, downloaded; the plan destroyed.
    2. One NetworkPlan.for_gradients of the host-sliced slice-0 network; for q = 0..511: stage the host-sliced network q,
       run, vjp, embed, fold in q order from zeros.  The full sliced G equals that fold bit for bit, leaf by leaf; each
       single-slice range equals its embedded slice; the engine counters equal per slice.  A slice compiles exactly as
       the host-sliced network does (tncb_plan_create_vjp_sliced) and the device adds in q order from zero, so bit
       identity is the expected result.
    3. The plan destroyed, q = 0 and q = 300 against host reference_gradient replays of those slices: per-leaf units,
       tau = TAU; exact zeros outside each slice's sub-blocks of the carriers; the value against the replay's.  Every
       pair of a slice is FP64 (no int8 pair: test_gpu_backward_pairs' inventory), so TAU is far above what depth 56
       and K up to 2^23 in split-K chunks give."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan
    from tnc_b200.tensornetwork import NetworkPlan
    path, _ = tree("main")
    hn = haar_network(HAAR_SEED)
    tensors = list(hn.tensors)
    xs = [leaf_array(t) for t in tensors]
    full = matrix_net(tensors, xs)
    n = 512
    singles = (0, 300)
    times = {}
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    peak = 0
    try:
        sp = SlicedPlan.for_gradients(full, path, D12_LEGS, ctx=ctx)
        sp.stage(full)
        assert sp.n_slices == n
        ctx.synchronize()
        ctx.reset_stats()
        val, G = sp.vjp()
        val = val.to_numpy()
        ec_full = ctx.engine_counts()
        times["vjp, 512 slices"] = time.perf_counter() - t0
        run = sp.run().to_numpy()
        assert val.tobytes() == run.tobytes()
        one = {}
        for q in singles:
            ctx.synchronize()
            ctx.reset_stats()
            v, g = sp.vjp(rank=q, world=n, allreduce=False)
            ctx.synchronize()
            one[q] = (v.to_numpy(), g, ctx.engine_counts())
        peak = max(peak, ctx.stats()["arena_peak_bytes"])
        destroy(ctx, sp.plan)
        times["sliced plan"] = time.perf_counter() - t0
        # 2. the plain plan over every host-sliced network
        t1 = time.perf_counter()
        ts0, arrs0, _ = cut(tensors, xs, D12_LEGS, 0)
        plain = NetworkPlan.for_gradients(matrix_net(ts0, arrs0), path, ctx=ctx)
        acc, r_acc, counts, per = None, None, [], {}
        for q in range(n):
            ts, arrs, vq = cut(tensors, xs, D12_LEGS, q)
            plain.stage(matrix_net(ts, arrs))
            ctx.synchronize()
            ctx.reset_stats()
            r = plain.run().to_numpy()
            e = embed(tensors, plain.vjp(), vq)
            ctx.synchronize()
            counts.append(ctx.engine_counts())
            peak = max(peak, ctx.stats()["arena_peak_bytes"])
            r_acc = r.copy() if r_acc is None else r_acc + r
            acc = fold(acc, e)
            if q in singles:
                per[q] = (r, e)
        destroy(ctx, plain)
        times["plain loop, 512 slices"] = time.perf_counter() - t1
    finally:
        ctx.close()
    print(f"\n[d12 sliced] " + ", ".join(f"{k} {v:.1f} s" for k, v in times.items())
          + f"; arena peak {peak / 2**30:.2f} GiB; engines per call {ec_full}", flush=True)
    assert val == r_acc
    assert sorted(G) == sorted(acc) == list(range(len(tensors)))
    same = [l for l in G if not np.array_equal(G[l], acc[l])]
    assert not same, same[:8]
    assert ec_full == summed(counts), (ec_full, summed(counts))
    for q in singles:
        v, g, ec = one[q]
        assert v == per[q][0], q
        assert sorted(g) == sorted(per[q][1])
        assert not [l for l in g if not np.array_equal(g[l], per[q][1][l])], q
        assert ec == counts[q], (q, ec, counts[q])
    print(f"[d12 sliced] 512 of 512 slices compared bit for bit through the fold; single slices {singles} bit for bit",
          flush=True)
    del G, acc
    # 3. slices 0 and 300 against host replays
    errs = {}
    for q in singles:
        t1 = time.perf_counter()
        R, ref = sliced_reference(tensors, path, xs, D12_LEGS, [q])
        times[f"host replay q={q}"] = time.perf_counter() - t1
        v, g, _ = one[q]
        assert R != 0 and all(np.abs(ref[l]).max() > 0 for l in ref), q       # no slice of exact zeros
        assert abs(complex(v) - R) <= TAU * abs(R), (q, complex(v), R)
        bad = outside(g, ref)
        assert not bad, (q, bad[:8], worst(g, ref))
        assert zeros_outside(tensors, g, D12_LEGS, [q]) == [], q
        errs[q] = worst(g, ref)
        del ref
    print(f"[d12 sliced] " + ", ".join(f"{k} {v:.1f} s" for k, v in times.items() if k.startswith("host"))
          + f", peak RSS {peak_rss_gib():.1f} GiB; worst per-leaf error "
          + ", ".join(f"q={q} {e:.2e}" for q, e in errs.items())
          + f"; total {time.perf_counter() - t0:.1f} s", flush=True)
