"""Hessian-vector products element by element at the size the feature exists for.

test_gpu_hvp.py checks every Ġ_l of small networks against torch.func; on bench.py's network it checks aggregates only
(Euler's identity with Ẋ = X, Hessian symmetry, a zero seed tangent), which never see the seed tangent's term, a wrt
subset (one-sided tangent pairs, backward pairs with no tangent on the other operand), a liveness or slot-reuse error in
the static layout that hits a few leaves, or an error confined to small entries.  This file closes that gap.

1. The schedule (no GPU).  hvp_pairs restates network.cpp: the forward steps; build_tangent (per forward step, one
   tangent pair per operand whose subtree holds a requested leaf, on the step's own PairPlan); build_backward (as
   test_gpu_backward_pairs.backward_pairs, restricted to subtrees that hold a requested leaf); build_backward_tangent (per
   backward pair x̄ = C̄·O, the pair dC̄·O -- the seed always has a tangent slot -- then C̄·dO when O has a tangent).  Its
   pair count and flops (same summation order) equal tncb_plan_info of host-only Hessian-vector plans of bench.py's
   network with every leaf requested (4392 = 9 x 488 pairs) and with wrt = Q.  Every tangent pair's canonical key is a
   forward pair's and every backward-tangent pair's is a backward pair's (of the every-leaf gradient schedule), so the
   element-wise checks of every backward pair in test_gpu_backward_pairs.py cover every pair shape of a Hessian-vector
   plan.  For Q the three kinds of forward step (two-sided, one-sided, no tangent) and both kinds of backward pair (O with
   and without a tangent) occur, and the int8 engine takes pairs in each of the four roles.
2. bench.py's whole Ġ block (GPU) against reference_hvp, a forward-over-reverse replay of the same path by hand in
   complex128 torch on the host, with seed 1, zero seed tangent and random complex tangents on Q; by linearity in the
   seed, G = S·G1 and Ġ = Ṡ·G1 + S·H(Ẋ).  Two plans, one at a time, each destroyed before the replay runs: every leaf
   requested with tangents zero outside Q (Ġ_l of all 489 leaves, G_l, Ṙ, R), and wrt = Q.
3. reference_hvp against torch.func.jvp of torch.func.vjp of the TTGT replay on a 12-qubit network (no GPU): the bench
   check is only as good as its reference.

Q: the first 245 leaves in circuit order (the 36 input kets and the gates of the first rounds), a cluster rather than a
scatter, so that subtrees of late gates alone have no tangent.  Along bench.py's greedy path that gives 244 two-sided, 47
one-sided and 197 forward steps without a tangent; 2581 pairs, 55 of them on the int8 engine (6 forward, 11 tangent, 13
backward, 25 backward-tangent).

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, with 16 host CPUs: the whole-block test takes 102 s, of
which the host replay takes 92 s at a peak RSS of 38.6 GiB (forward values and forward tangents, 9.9 and 9.7 GB by their
shapes, plus the GEMM temporaries; on 8 host CPUs 156 s and 35 GiB); the library's arena peaks at 43.4 GiB.  The worst
error over both plans is 4.6e-14 of each leaf's largest entry for Ġ and 8.0e-14 for G."""
import collections
import resource
import time

import numpy as np
import pytest

from test_gpu_backward_pairs import (TAU, bench_net, canonical, engine, forward_steps, fused_permute, inventory,
                                     kernel_class, mnk, out_legs, outside, tcontract, worst)

Q = list(range(245))
ROLES = ("forward", "tangent", "backward", "backward-tangent")
ENGINES = ["k0", "k0_splitk", "k1_dmma", "k1_dmma_splitk", "k1_tcgen05", "k2", "permute", "reserved"]


# ================================================================================================================
# 1. the schedule
# ================================================================================================================
def requested(steps, wrt):
    """the forward slots whose subtree holds a leaf of wrt: the slots that get a tangent and an adjoint"""
    want = {("leaf", i) for i in wrt}
    for q, (a, b, *_) in enumerate(steps):
        if a in want or b in want:
            want.add(("step", q))
    return want


def hvp_pairs(steps, wrt):
    """(role, (a legs, a dims, b legs, b dims)) of every pair of a Hessian-vector plan with the leaves wrt requested, in
    network.cpp's order: forward steps, build_tangent, build_backward, build_backward_tangent.  A tangent slot has its
    primal slot's legs, so a tangent pair has its forward step's operands and a backward-tangent pair its backward pair's."""
    want = requested(steps, wrt)
    pairs = [("forward", tuple(s[2:])) for s in steps]
    pairs += [("tangent", tuple(s[2:])) for s in steps for x in s[:2] if x in want]
    adj = {("step", len(steps) - 1): out_legs(*steps[-1][2:])}
    backward = []                                   # (C-bar legs, C-bar dims, O legs, O dims), O's slot
    for q in range(len(steps) - 1, -1, -1):
        a, b, al, ad, bl, bd = steps[q]
        if ("step", q) not in want:
            continue
        gl, gd = adj.pop(("step", q))
        for x, o, (ol, od) in ((a, b, (bl, bd)), (b, a, (al, ad))):
            if x in want:
                backward.append(((gl, gd, ol, od), o))
                adj[x] = out_legs(gl, gd, ol, od)
    pairs += [("backward", p) for p, _ in backward]
    for p, o in backward:
        pairs.append(("backward-tangent", p))       # dC̄·O
        if o in want:
            pairs.append(("backward-tangent", p))   # C̄·dO
    return pairs


def totals(pairs):
    flops = 0.0
    for _, p in pairs:
        M, N, K = mnk(*p)
        flops += 8.0 * M * N * K
    return len(pairs), flops


def predicted_engines(pairs, sms):
    """the engine counters of one hvp call: every pair counted once, on the engine the default context gives it"""
    cls = {}
    counts = dict.fromkeys(ENGINES, 0)
    for _, p in pairs:
        key = canonical(*p)
        if key not in cls:
            cls[key] = kernel_class(*p)
        counts[engine(cls[key], *mnk(*p), sms)[0]] += 1
    return counts


def library_totals(tn, path, wrt):
    from test_hvp_host import Plan
    info = Plan(tn, path, wrt).info()
    return info["pairs"], info["flops"]


def test_schedule_matches_the_library(built_lib):
    """Pair count and flops of the restated schedule equal tncb_plan_info, with every leaf requested and with wrt = Q."""
    tn, path = bench_net()
    steps = forward_steps(tn.tensors, path)
    every = list(range(len(tn.tensors)))
    pairs = hvp_pairs(steps, every)
    assert totals(pairs) == library_totals(tn, path, None) == (4392, 60203623894488.0)
    assert len(pairs) == 9 * len(steps) == 9 * 488
    assert collections.Counter(r for r, _ in pairs) == {"forward": 488, "tangent": 976, "backward": 976,
                                                        "backward-tangent": 1952}
    sub = hvp_pairs(steps, Q)
    assert totals(sub) == library_totals(tn, path, Q)
    assert collections.Counter(r for r, _ in sub) == {"forward": 488, "tangent": 535, "backward": 535,
                                                      "backward-tangent": 1023}


def test_schedule_adds_no_pair_shapes(built_lib):
    """Tangent pairs have forward pairs' canonical keys and backward-tangent pairs have backward pairs' keys (of the
    every-leaf gradient schedule that test_gpu_backward_pairs checks pair by pair), with every leaf and with wrt = Q."""
    tn, path = bench_net()
    steps, bw = inventory("bench")
    fwd_keys = {canonical(*s[2:]) for s in steps}
    bw_keys = {canonical(*p[:4]) for p in bw}
    for wrt in (range(len(tn.tensors)), Q):
        pairs = hvp_pairs(steps, wrt)
        keys = {r: {canonical(*p) for role, p in pairs if role == r} for r in ROLES}
        assert keys["forward"] == fwd_keys
        assert keys["tangent"] <= fwd_keys
        assert keys["backward"] <= bw_keys
        assert keys["backward-tangent"] <= bw_keys
        assert keys["backward-tangent"] == keys["backward"]


def test_subset_reaches_every_kind(built_lib):
    """wrt = Q: forward steps with a tangent on both sides, on one side and on neither; backward pairs whose other
    operand has a tangent and ones whose has none; int8-engine pairs in each of the four roles."""
    tn, path = bench_net()
    steps = forward_steps(tn.tensors, path)
    want = requested(steps, Q)
    sides = collections.Counter((a in want) + (b in want) for a, b, *_ in steps)
    assert sides == {2: 244, 1: 47, 0: 197}, sides
    pairs = hvp_pairs(steps, Q)
    n = collections.Counter(r for r, _ in pairs)
    assert n["tangent"] == sides[1] + 2 * sides[2]
    assert n["backward"] == n["tangent"]
    with_do = n["backward-tangent"] - n["backward"]           # backward pairs whose O has a tangent
    assert 0 < with_do < n["backward"], (with_do, n)
    int8 = collections.Counter(r for r, p in pairs if engine(kernel_class(*p), *mnk(*p))[0] == "k1_tcgen05")
    assert int8 == {"forward": 6, "tangent": 11, "backward": 13, "backward-tangent": 25}, int8


# ================================================================================================================
# 2. bench.py's whole Ġ block against a forward-over-reverse replay
# ================================================================================================================
def _add(x, y):
    """x + y with None for zero; x, when there is one, is a fresh term and takes the sum in place"""
    return y if x is None else x if y is None else x.add_(y)


def reference_hvp(tensors, path, xs, ts):
    """(R, Ṙ, {leaf: G1}, {leaf: H}) of a flat network along a replace-left path for seed 1 and zero seed tangent, by hand
    in torch: reference_gradient (test_gpu_backward_pairs) differentiated by the product rule.  Forward: C = A·B and
    dC = dA·B + A·dB; backward: x̄ = C̄·O and dx̄ = dC̄·O + C̄·dO; G1_l and H_l = d(G1_l)[Ẋ] in leaf l's own leg order.
    ts: {leaf: tangent}, the others zero; a zero tangent is None throughout and costs nothing."""
    import torch
    steps = forward_steps(tensors, path)
    val = {("leaf", i): (list(t.legs), x) for i, (t, x) in enumerate(zip(tensors, xs))}
    tan = {("leaf", i): t for i, t in ts.items()}
    for q, (a, b, *_) in enumerate(steps):
        (al, A), (bl, B) = val[a], val[b]
        val[("step", q)] = tcontract(al, A, bl, B)
        dc = None
        if a in tan:
            dc = tcontract(al, tan[a], bl, B)[1]
        if b in tan:
            dc = _add(dc, tcontract(al, A, bl, tan[b])[1])
        if dc is not None:
            tan[("step", q)] = dc
    root = ("step", len(steps) - 1)
    legs, R = val[root]
    Rd = tan[root]
    adj = {root: (legs, torch.ones_like(R))}
    dadj = {root: None}
    grads, hess = {}, {}
    for q in range(len(steps) - 1, -1, -1):
        a, b, *_ = steps[q]
        gl, g = adj.pop(("step", q))
        dg = dadj.pop(("step", q))
        for x, other in ((a, b), (b, a)):
            ol, O = val[other]
            xl, xbar = tcontract(gl, g, ol, O)
            dx = None if dg is None else tcontract(gl, dg, ol, O)[1]
            if other in tan:
                dx = _add(dx, tcontract(gl, g, ol, tan[other])[1])
            if x[0] == "leaf":
                grads[x[1]] = fused_permute(xbar, xl, val[x][0])
                hess[x[1]] = torch.zeros_like(grads[x[1]]) if dx is None else fused_permute(dx, xl, val[x][0])
            else:
                adj[x], dadj[x] = (xl, xbar), dx
        del g, dg, xbar, dx
        for s in (a, b):
            val.pop(s)
            tan.pop(s, None)
        if q == len(steps) - 1:
            val.pop(root)
            tan.pop(root, None)
    return R, Rd, grads, hess


def peak_rss_gib():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20


@pytest.mark.gpu
def test_bench_hvp_block(built_lib):
    """bench.py's Hessian-vector plan (stage, hvp; the int8 engine as bench.py runs it), element by element against
    reference_hvp, one plan at a time: (1) every leaf requested, tangents zero outside Q: Ġ_l and G_l of all 489 leaves,
    Ṙ and R; (2) wrt = Q, the same tangents: Ġ_l and G_l for l in Q.  Both with the same random complex S and Ṡ.

    Reference: one replay with seed 1 and Ṡ = 0 gives R, Ṙ, G1 and H(Ẋ); the result is a scalar, so for any (S, Ṡ)
    G = S·G1 and Ġ = Ṡ·G1 + S·H(Ẋ).  Each plan's outputs are downloaded and the plan destroyed (its 36.5 GB workspace)
    before the replay runs on the host.

    What this reaches that the pair tests and the aggregates do not: the seed tangent's term at scale, one-sided tangent
    pairs and backward pairs with no tangent on the other operand (wrt = Q), the liveness of forward tangents up to the
    backward-tangent pair that reads them and the seed-tangent slot in memory the forward levels freed (any leaf whose Ġ
    reads a clobbered slot fails), the tangent sums, and both gathers' permutations into each leaf's leg order.

    Units: max_e |ref_l| per leaf, as test_gpu_backward_pairs.test_bench_gradient_block argues (the sum of |terms| is no
    usable scale for a random circuit's amplitude).  tau: every pair's bound is normwise (int8: K 2^-49 max|b| max|a|
    per entry, FP64 pairs far tighter) and a Ġ element passes through at most four roles x the tree's depth of 18 pairs,
    whose normwise relative errors add to first order: 72 * 2^-49 * kappa, kappa = K max|b| max|a| / max|C| a pair's
    cancellation; that stays below tau = 1e-10 for kappa up to 7.8e2.  The measured worst is 4.6e-14 (Ġ) and 8.0e-14
    (G), and tau = 1e-10 keeps the checks below meaningful: a transposed sx Ġ and a 1e-8 relative change of one element
    both lie far outside it.

    The engine counters of each hvp call equal hvp_pairs' prediction, pair for pair."""
    import torch
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from test_gpu_vjp import leaf_array
    tn, path = bench_net()
    lv = leaves(tn)
    assert len(lv) == len(tn.tensors) == 489
    xs = [leaf_array(l) for l in lv]
    steps = forward_steps(tn.tensors, path)
    assert 4 * 18 * 16 * 2.0 ** -49 <= TAU / 40
    rng = np.random.default_rng(43)
    crandn = lambda shape: rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    tans = {i: crandn(xs[i].shape) for i in Q}
    S, Sd = (np.asarray(complex(crandn(()))) for _ in range(2))
    t0 = time.perf_counter()
    ctx = tb.Context(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    runs, ws_peak = [], 0
    try:
        for wrt in (None, Q):
            plan = NetworkPlan.for_hvp(tn, path, wrt, ctx=ctx)
            plan.stage(tn)
            ctx.synchronize()
            ctx.reset_stats()
            out = plan.hvp(tans, S, Sd)
            ctx.synchronize()
            ec = ctx.engine_counts()
            ws_peak = max(ws_peak, ctx.stats()["arena_peak_bytes"])
            ctx._l.tncb_plan_destroy(plan.handle)      # its workspace goes back before the next plan
            plan.handle = None
            ctx.trim()
            want = predicted_engines(hvp_pairs(steps, range(len(lv)) if wrt is None else wrt), sms)
            runs.append((wrt, out, ec, want))
    finally:
        ctx.close()
    t_plan = time.perf_counter() - t0
    for wrt, _, ec, want in runs:
        print(f"\n[bench hvp] wrt {'every leaf' if wrt is None else f'Q ({len(wrt)} leaves)'}: engines {ec}", flush=True)
    print(f"[bench hvp] two plans, stage + hvp: {t_plan:.1f} s, arena peak {ws_peak / 2**30:.2f} GiB", flush=True)
    for wrt, _, ec, want in runs:
        assert ec == want, (wrt is None, ec, want)
        assert ec["k1_tcgen05"] >= 1

    t1 = time.perf_counter()
    with torch.no_grad():
        R, Rd, g1, h = reference_hvp(tn.tensors, path, [torch.from_numpy(x) for x in xs],
                                     {i: torch.from_numpy(t) for i, t in tans.items()})
        R, Rd = complex(R.item()), complex(Rd.item())
        g1 = {l: v.numpy() for l, v in g1.items()}
        h = {l: v.numpy() for l, v in h.items()}
    s, sd = complex(S), complex(Sd)
    G_ref = {l: s * v for l, v in g1.items()}
    Gd_ref = {l: sd * g1[l] + s * h[l] for l in g1}
    print(f"[bench hvp] reference replay {time.perf_counter() - t1:.1f} s, peak RSS {peak_rss_gib():.1f} GiB; "
          f"total {time.perf_counter() - t0:.1f} s", flush=True)
    assert all(np.abs(h[l]).max() > 0 for l in h)              # every leaf's Ġ has a Hessian term
    for wrt, (val, tan, G, Gd), _, _ in runs:
        sel = sorted(G_ref) if wrt is None else sorted(wrt)
        print(f"[bench hvp] wrt {'every leaf' if wrt is None else 'Q'}: worst |Ġ_l - ref_l| / max|ref_l| "
              f"{worst(Gd, {l: Gd_ref[l] for l in sel}):.2e}, G {worst(G, {l: G_ref[l] for l in sel}):.2e}, "
              f"Ṙ {abs(complex(tan) - Rd) / abs(Rd):.2e}", flush=True)
        assert sorted(Gd) == sorted(G) == sel
        assert all(Gd[l].shape == Gd_ref[l].shape for l in sel)
        assert abs(complex(val) - R) <= TAU * abs(R)
        assert abs(complex(tan) - Rd) <= TAU * abs(Rd)
        bad = outside(Gd, {l: Gd_ref[l] for l in sel})
        assert not bad, (bad[:8], worst(Gd, {l: Gd_ref[l] for l in sel}))
        bad = outside(G, {l: G_ref[l] for l in sel})
        assert not bad, (bad[:8], worst(G, {l: G_ref[l] for l in sel}))

    # the comparator rejects one sx leaf's Ġ transposed ...
    Gd = runs[0][1][3]
    sx = next(l for l, t in enumerate(lv) if t.tensordata.kind == "gate" and t.tensordata.gate[0] == "sx"
              and np.abs(Gd[l] - Gd[l].T).max() > 1e-3 * np.abs(Gd[l]).max())
    bad = dict(Gd)
    bad[sx] = Gd[sx].T.copy()
    assert outside(bad, Gd_ref) == [sx]
    # ... and one element of an fsim leaf's Ġ off by 1e-8 relative: its largest
    l = next(l for l, t in enumerate(lv) if t.tensordata.kind == "gate" and t.tensordata.gate[0] == "fsim")
    e = int(np.argmax(np.abs(Gd[l])))
    off = dict(Gd)
    off[l] = Gd[l].copy()
    off[l].flat[e] *= 1 + 1e-8
    assert outside(off, Gd_ref) == [l]


# ================================================================================================================
# 3. the reference against torch
# ================================================================================================================
def test_reference_against_torch_func():
    """reference_hvp on a 12-qubit amplitude network, tangents on the first half of the leaves, against torch.func.jvp
    of torch.func.vjp of the TTGT replay (test_gpu_hvp.reference_hvp) for a random S and Ṡ: Ṙ, G = S·G1 and
    Ġ = Ṡ·G1 + S·H, every leaf, within 1e-12 of the terms' magnitude; R against the replay."""
    import torch
    from tnc_b200.tensornetwork import leaves
    from test_gpu_hvp import amplitude_net, close, crandn, greedy, leaf_array, reference_hvp as torch_hvp, replay
    tn = amplitude_net(12, 6, 5)
    path = greedy(tn)
    lv = leaves(tn)
    assert list(lv) == list(tn.tensors) and not path.nested
    xs = [leaf_array(l) for l in lv]
    rng = np.random.default_rng(44)
    q = range(len(lv) // 2)
    tans = {i: crandn(rng, xs[i].shape) for i in q}
    S, Sd = crandn(rng, ()), crandn(rng, ())
    with torch.no_grad():
        R, Rd, g1, h = reference_hvp(tn.tensors, path, [torch.from_numpy(x) for x in xs],
                                     {i: torch.from_numpy(t) for i, t in tans.items()})
    ts = [tans.get(i, np.zeros_like(x)) for i, x in enumerate(xs)]
    every = list(range(len(lv)))
    Rd_t, G_t, Gd_t, sRd, sGd = torch_hvp(tn, path, xs, ts, S, Sd, every)
    R_t = replay(tn, path, [torch.from_numpy(x) for x in xs])[1]
    assert abs(complex(R) - complex(R_t)) <= 1e-12 * abs(complex(R_t))
    assert close(Rd.numpy(), Rd_t, sRd)
    for l in every:
        G1, H = g1[l].numpy(), h[l].numpy()
        assert G1.shape == H.shape == xs[l].shape
        assert np.abs(S * G1 - G_t[l]).max() <= 1e-12 * np.abs(G_t[l]).max(), l
        assert close(Sd * G1 + S * H, Gd_t[l], sGd[l]), (l, np.abs(Sd * G1 + S * H - Gd_t[l]).max())
    assert any(np.abs(h[l].numpy()).max() > 0 for l in every if l not in q)   # cross terms reach leaves outside Q
