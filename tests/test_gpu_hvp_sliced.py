"""Sliced tangent and Hessian-vector plans (tncb_plan_create_jvp_sliced / _hvp_sliced, tncb_plan_jvp_sliced /
_hvp_sliced, SlicedPlan.for_tangents / for_hvp):

  1. R, Ṙ, G and Ġ against torch (torch.func.jvp of the holomorphic vjp of a complex128 replay of the UNSLICED network)
     with a random seed tangent: 12-qubit amplitudes at 1 and 2 sliced legs and with every leg of a two-qubit gate leaf
     sliced, a network with a sliced leg of dimension 3, one whose adjoints need more leg groups than an accumulate item
     holds (K3 first), and a statevector network with open legs and a seed tensor;
  2. bit identities: zero legs equal tncb_plan_jvp / tncb_plan_hvp, the value equals run_slices and SlicedPlan.run, G
     equals vjp_sliced's and Ṙ jvp_sliced's, Ġ with zero leaf tangents equals vjp_sliced(Ṡ), G and Ġ equal the
     slice-order fold of unsliced Hessian-vector passes over the host-sliced networks, and calls repeat;
  3. the identities sum_r S Ṙ = sum_l <G_l, Ẋ_l> and <Ẏ, Ġ(Ẋ)> = <Ẋ, Ġ(Ẏ)> (Ṡ = 0);
  4. partial ranges (world = 2, 3) add up to the whole, an empty range gives zeros;
  5. bench.py's network at 2 sliced legs against its unsliced Hessian-vector plan, on the int8 engine;
  6. the error codes, with the arena's live bytes unchanged."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from test_gpu_hvp import amplitude_net, close, counted, crandn, greedy, leaf_array, reference_hvp, replay, statevector_net
from test_gpu_vjp_sliced import whole_leaf_legs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_UNSUPPORTED = -1, -2, -9


@pytest.fixture(scope="module")
def ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()


def sliced(ctx, kind, tn, path, legs, wrt=None):
    from tnc_b200.contractionpath.slicing import SlicedPlan
    p = {"vjp": SlicedPlan.for_gradients, "jvp": SlicedPlan.for_tangents, "hvp": SlicedPlan.for_hvp}[kind](tn, path, legs, wrt=wrt, ctx=ctx)
    p.stage(tn)
    return p


def group_net(extra=3):
    """X (10 legs of 2 and one of `extra`) and Y (11 legs of 2, X's reversed) plus a matrix M on leg 20 and leg 10: X's
    adjoint comes out in Y's order, 9 leg groups after slicing leg 4 -> K3 before the accumulates"""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(4)
    legs = list(range(10))

    def leaf(ls, dims):
        t = Tensor(ls, dims)
        t.set_tensor_data(TensorData.Matrix(crandn(rng, dims)))
        return t
    x = leaf(legs + [20], [2] * 10 + [extra])
    y = leaf([10] + legs[::-1], [2] * 11)
    m = leaf([20, 10], [extra, 2])
    return Tensor.new_composite([x, m, y]), ContractionPath.simple([(0, 1), (0, 2)])


def check_against_reference(ctx, tn, path, legs, seed=1, wrt=None):
    """R, Ṙ, G and Ġ of the sliced Hessian-vector plan, and Ṙ of the sliced tangent plan, against the unsliced replay"""
    import torch
    from tnc_b200.tensornetwork import leaves
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    wrt = [i for i, x in enumerate(xs) if x is not None] if wrt is None else wrt
    rng = np.random.default_rng(seed)
    tans = {i: crandn(rng, xs[i].shape) for i in wrt}
    ts = [tans[i] if i in tans else np.zeros_like(xs[i]) for i in range(len(lv))]
    plan = sliced(ctx, "hvp", tn, path, legs, wrt)
    rdims = plan.plan.result_dims
    S, Sd = crandn(rng, rdims), crandn(rng, rdims)
    (val, tan, G, Gd), ec = counted(ctx, lambda: plan.hvp(tans, S, Sd))
    R = replay(tn, path, [torch.tensor(x) for x in xs])[1].numpy()
    assert np.abs(val - R).max() <= 1e-12 * np.abs(R).max()
    Rd, Gr, Gdr, sRd, sGd = reference_hvp(tn, path, xs, ts, S, Sd, wrt)
    assert tan.shape == Rd.shape and close(tan, Rd, sRd), np.abs(tan - Rd).max()
    assert sorted(G) == sorted(Gd) == sorted(wrt)
    for k, i in enumerate(wrt):
        assert Gd[i].shape == Gdr[k].shape == xs[i].shape
        assert close(Gd[i], Gdr[k], sGd[k]), (i, np.abs(Gd[i] - Gdr[k]).max(), sGd[k].max())
        assert np.abs(G[i] - Gr[k]).max() <= 1e-12 * max(np.abs(Gr[k]).max(), 1e-300) * 1e3
    tp = sliced(ctx, "jvp", tn, path, legs, wrt)
    res, tan2 = tp.jvp(tans)
    assert res.legs == plan.plan.result_legs
    assert close(tan2, Rd, sRd)
    return plan, ec


# ================================================================================================================
# 1. against an independent reference
# ================================================================================================================
@pytest.mark.parametrize("n_legs", [1, 2])
def test_amplitude_against_torch(ctx, n_legs):
    from tnc_b200.contractionpath.slicing import find_slices
    tn = amplitude_net(12, 6, 5)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=2 ** n_legs)
    plan, ec = check_against_reference(ctx, tn, path, legs)
    assert plan.n_slices == 2 ** n_legs
    assert ec["k0"] > 0, ec


def test_every_leg_of_a_leaf_sliced(ctx):
    """the four legs of one two-qubit gate: that leaf is rank 0 in every slice, 16 slices, a wrt subset"""
    tn = amplitude_net(12, 6, 7)
    path = greedy(tn)
    legs = whole_leaf_legs(tn, 4)
    whole = next(i for i, t in enumerate(tn.tensors) if list(t.legs) == legs)
    plan, _ = check_against_reference(ctx, tn, path, legs, wrt=sorted({0, 5, whole, len(tn.tensors) - 1}))
    assert plan.n_slices == 16


def test_dimension_three_leg(ctx):
    """a sliced leg of dimension 3 (leg 20) with a binary one: 6 slices, digits of mixed radix"""
    tn, path = group_net()
    plan, _ = check_against_reference(ctx, tn, path, [20, 4])
    assert plan.n_slices == 6


def test_many_group_route(ctx):
    """X's adjoint and adjoint tangent need 9 leg groups: K3 for both, per slice, before the accumulates"""
    tn, path = group_net()
    plan, ec = check_against_reference(ctx, tn, path, [4])
    assert ec["permute"] >= 2 * plan.n_slices, ec


def test_statevector_against_torch(ctx):
    """a result with 13 open legs, a seed tensor and a seed tangent; one sliced leg"""
    from tnc_b200.contractionpath.slicing import find_slices
    tn = statevector_net(1)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=2)
    _, ec = check_against_reference(ctx, tn, path, legs, seed=3)
    assert ec["k0"] >= 1 and ec["k2"] >= 1, ec


# ================================================================================================================
# 2. bit identities
# ================================================================================================================
def bits(a):
    return np.ascontiguousarray(a).tobytes()


def test_zero_legs_equal_unsliced(ctx):
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = amplitude_net(12, 6, 8)
    path = greedy(tn)
    xs = [leaf_array(l) for l in leaves(tn)]
    rng = np.random.default_rng(1)
    tans = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    S, Sd = np.asarray(crandn(rng, ())), np.asarray(crandn(rng, ()))
    j = NetworkPlan.for_tangents(tn, path, ctx=ctx)
    j.stage(tn)
    v0, t0 = j.jvp(tans)
    v1, t1 = sliced(ctx, "jvp", tn, path, []).jvp(tans)
    assert bits(v0.to_numpy()) == bits(v1.to_numpy()) and bits(t0) == bits(t1)
    h = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    h.stage(tn)
    a = h.hvp(tans, S, Sd)
    b = sliced(ctx, "hvp", tn, path, []).hvp(tans, S, Sd)
    assert bits(a[0]) == bits(b[0]) and bits(a[1]) == bits(b[1])
    for k in (2, 3):
        assert sorted(a[k]) == sorted(b[k])
        for i in a[k]:
            assert np.array_equal(a[k][i], b[k][i]), (k, i)      # == : -0.0 and +0.0 compare equal


def embed(lf, legs, assignment, block):
    """`block` (slice q's leaf) placed into q's sub-block of a zero full-shape leaf"""
    val = dict(zip(legs, assignment))
    out = np.zeros([int(d) for d in lf.bond_dims], dtype=np.complex128)
    out[tuple(val[l] if l in val else slice(None) for l in lf.legs)] = block
    return out


def test_bit_identities(ctx):
    from tnc_b200.contractionpath.slicing import SlicedNetwork, SlicedPlan, find_slices
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = amplitude_net(12, 6, 3)
    path = greedy(tn)
    lv = leaves(tn)
    legs = find_slices(tn, path, min_slices=8)
    xs = [leaf_array(l) for l in lv]
    rng = np.random.default_rng(2)
    tans = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    S, Sd = np.asarray(crandn(rng, ())), np.asarray(crandn(rng, ()))
    run = SlicedPlan(tn, path, legs, ctx=ctx).run().to_numpy()
    hp = sliced(ctx, "hvp", tn, path, legs)
    jp = sliced(ctx, "jvp", tn, path, legs)
    gp = sliced(ctx, "vjp", tn, path, legs)
    val, tan, G, Gd = hp.hvp(tans, S, Sd)
    # the value: run_slices of every plan kind, SlicedPlan.run, jvp_sliced's and vjp_sliced's
    for p in (hp, jp, gp):
        assert bits(p.run().to_numpy()) == bits(run)
    assert bits(val) == bits(run)
    jv, jt = jp.jvp(tans)
    assert bits(jv.to_numpy()) == bits(run) and bits(jt) == bits(tan)
    gv, Gv = gp.vjp(S)
    assert bits(gv.to_numpy()) == bits(run)
    for i in G:
        assert bits(G[i]) == bits(Gv[i]), i
    # zero leaf tangents: Ġ is the gradient with seed Ṡ
    _, _, _, Gd0 = hp.hvp({}, S, Sd)
    _, GSd = gp.vjp(Sd)
    for i in Gd0:
        assert np.array_equal(Gd0[i], GSd[i]), i
    # the fold of unsliced Hessian-vector passes over the host-sliced networks, in slice order
    sn = SlicedNetwork(tn, legs)
    fv = ft = None
    fG = {i: np.zeros_like(x) for i, x in enumerate(xs)}
    fGd = {i: np.zeros_like(x) for i, x in enumerate(xs)}
    for a in sn.assignments:
        net = sn.slice(a)
        val_of = dict(zip(legs, a))
        sub = lambda i: tuple(val_of[l] if l in val_of else slice(None) for l in lv[i].legs)
        p = NetworkPlan.for_hvp(net, path, ctx=ctx)
        p.stage(net)
        v, t, g, gd = p.hvp({i: np.ascontiguousarray(tans[i][sub(i)]) for i in tans}, S, Sd)
        fv, ft = (v, t) if fv is None else (fv + v, ft + t)
        for i in g:
            fG[i] = fG[i] + embed(lv[i], legs, a, g[i])
            fGd[i] = fGd[i] + embed(lv[i], legs, a, gd[i])
        del p
    assert bits(fv) == bits(val) and bits(ft) == bits(tan)
    for i in G:
        assert bits(fG[i]) == bits(G[i]), i
        assert bits(fGd[i]) == bits(Gd[i]), i
    # repeated calls
    again = hp.hvp(tans, S, Sd)
    assert bits(again[0]) == bits(val) and bits(again[1]) == bits(tan)
    for i in G:
        assert bits(again[2][i]) == bits(G[i]) and bits(again[3][i]) == bits(Gd[i]), i


# ================================================================================================================
# 3. identities
# ================================================================================================================
def test_identities(ctx):
    """transpose and symmetry on a statevector network with a seed tensor, two sliced legs"""
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    tn = statevector_net(2)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    xs = [leaf_array(l) for l in leaves(tn)]
    hp = sliced(ctx, "hvp", tn, path, legs)
    rng = np.random.default_rng(6)
    S = crandn(rng, hp.plan.result_dims)
    V = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    W = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    _, Rd, G, HV = hp.hvp(V, S)
    lhs, rhs = np.sum(S * Rd), sum(np.sum(G[i] * V[i]) for i in V)
    assert abs(lhs - rhs) <= 1e-12 * (np.sum(np.abs(S * Rd)) + sum(np.sum(np.abs(G[i] * V[i])) for i in V))
    HW = hp.hvp(W, S)[3]
    lhs = sum(np.sum(W[i] * HV[i]) for i in V)
    rhs = sum(np.sum(V[i] * HW[i]) for i in V)
    mag = sum(np.sum(np.abs(W[i]) * np.abs(HV[i])) + np.sum(np.abs(V[i]) * np.abs(HW[i])) for i in V)
    assert abs(lhs - rhs) <= 1e-12 * mag, (lhs, rhs, mag)


# ================================================================================================================
# 4. partial ranges
# ================================================================================================================
def test_partial_ranges_add_up(ctx):
    from tnc_b200.contractionpath.slicing import find_slices
    from tnc_b200.tensornetwork import leaves
    tn = amplitude_net(12, 6, 9)
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    xs = [leaf_array(l) for l in leaves(tn)]
    rng = np.random.default_rng(4)
    tans = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    S, Sd = np.asarray(crandn(rng, ())), np.asarray(crandn(rng, ()))
    hp = sliced(ctx, "hvp", tn, path, legs)
    jp = sliced(ctx, "jvp", tn, path, legs)
    whole = hp.hvp(tans, S, Sd)
    for world in (2, 3):
        parts = [hp.hvp(tans, S, Sd, rank=r, world=world, allreduce=False) for r in range(world)]
        for k in (0, 1):
            assert abs(sum(complex(p[k]) for p in parts) - complex(whole[k])) <= 1e-13 * abs(complex(whole[k]))
        for k in (2, 3):
            scale = max(np.abs(g).max() for g in whole[k].values())
            for i in whole[k]:
                assert np.abs(sum(p[k][i] for p in parts) - whole[k][i]).max() <= 1e-13 * scale, (world, k, i)
        jparts = [jp.jvp(tans, rank=r, world=world, allreduce=False)[1] for r in range(world)]
        assert abs(sum(complex(t) for t in jparts) - complex(whole[1])) <= 1e-13 * abs(complex(whole[1]))
    empty = hp.hvp(tans, S, Sd, rank=hp.n_slices, world=hp.n_slices + 1, allreduce=False)
    assert complex(empty[0]) == 0 and complex(empty[1]) == 0
    assert all(not g.any() for k in (2, 3) for g in empty[k].values())
    jv, jt = jp.jvp(tans, rank=jp.n_slices, world=jp.n_slices + 1, allreduce=False)
    assert complex(jv.to_numpy()) == 0 and complex(jt) == 0


# ================================================================================================================
# 5. bench scale, int8 engine
# ================================================================================================================
def test_bench_network_two_legs(ctx):
    sys.path.insert(0, ROOT)
    import bench
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = bench.build_network()
    path = bench.greedy_path(tn)
    lv = leaves(tn)
    xs = [leaf_array(l) for l in lv]
    rng = np.random.default_rng(8)
    V = {i: crandn(rng, x.shape) for i, x in enumerate(xs)}
    S, Sd = np.asarray(crandn(rng, ())), np.asarray(crandn(rng, ()))
    ctx.trim()
    hp = sliced(ctx, "hvp", tn, path, [149, 156])
    assert hp.info()["peak_bytes"] == 10248070144
    (val, tan, G, Gd), ec = counted(ctx, lambda: hp.hvp(V, S, Sd))
    assert ec["k1_tcgen05"] >= 1, ec                   # the int8 engine
    assert len(G) == len(Gd) == len(lv) == 489
    del hp
    ctx.trim()
    full = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    full.stage(tn)
    v0, t0, G0, Gd0 = full.hvp(V, S, Sd)
    del full
    ctx.trim()
    assert abs(complex(val) - complex(v0)) <= 1e-9 * abs(complex(v0))
    assert abs(complex(tan) - complex(t0)) <= 1e-9 * abs(complex(t0))
    for ref, got in ((G0, G), (Gd0, Gd)):
        scale = max(np.abs(g).max() for g in ref.values())
        for i in ref:
            assert np.abs(got[i] - ref[i]).max() <= 1e-9 * scale, i


# ================================================================================================================
# 6. errors
# ================================================================================================================
def raw_hvp_sliced(c, handle, tangents, seed=None, seed_tangent=None, first=0, stride=1):
    outs = [C.c_void_p() for _ in range(4)]
    return c._l.tncb_plan_hvp_sliced(c.handle, handle, first, stride, tangents.handle if tangents is not None else None,
                                     seed.handle if seed is not None else None,
                                     seed_tangent.handle if seed_tangent is not None else None, *[C.byref(o) for o in outs])


def test_errors(ctx):
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    amp = amplitude_net(10, 4, 6)
    path = greedy(amp)
    legs = find_slices(amp, path, min_slices=2)
    sv = statevector_net(3)
    sv_path = greedy(sv)
    sv_legs = find_slices(sv, sv_path, min_slices=2)
    hp = SlicedPlan.for_hvp(amp, path, legs, ctx=ctx)
    jp = SlicedPlan.for_tangents(amp, path, legs, ctx=ctx)
    s_sv = sliced(ctx, "hvp", sv, sv_path, sv_legs)
    n = sum(int(np.prod(t.bond_dims)) for t in amp.tensors)
    good = DeviceTensor.from_numpy(ctx, np.ones(n, dtype=np.complex128))
    short = DeviceTensor.from_numpy(ctx, np.ones(n - 1, dtype=np.complex128))
    n_sv = sum(int(np.prod(t.bond_dims)) for t in sv.tensors)
    sv_tan = DeviceTensor.from_numpy(ctx, np.ones(n_sv, dtype=np.complex128))
    wrong = DeviceTensor.from_numpy(ctx, np.ones([2] * 12, dtype=np.complex128))
    scalar_wrong = DeviceTensor.from_numpy(ctx, np.ones(3, dtype=np.complex128))
    other = tb.Context(0)
    try:
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]

        def expect(rc, want):
            assert rc == want, (rc, want, ctx._l.tncb_last_error())
            assert ctx.stats()["arena_live_bytes"] == live

        h, j = hp.plan.handle, jp.plan.handle
        v, t = C.c_void_p(), C.c_void_p()
        expect(raw_hvp_sliced(ctx, h, good), ERR_INVALID)                                  # not staged
        expect(ctx._l.tncb_plan_jvp_sliced(ctx.handle, j, 0, 1, good.handle, C.byref(v), C.byref(t)), ERR_INVALID)
        hp.stage(amp)
        jp.stage(amp)
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]
        expect(raw_hvp_sliced(ctx, h, short), ERR_SHAPE)                                   # tangent block size
        expect(ctx._l.tncb_plan_jvp_sliced(ctx.handle, j, 0, 1, short.handle, C.byref(v), C.byref(t)), ERR_SHAPE)
        expect(raw_hvp_sliced(ctx, h, None), ERR_INVALID)                                  # no tangents
        expect(raw_hvp_sliced(ctx, h, good, stride=0), ERR_INVALID)                        # stride 0
        expect(raw_hvp_sliced(other, h, good), ERR_INVALID)                                # another context
        expect(ctx._l.tncb_plan_jvp_sliced(other.handle, j, 0, 1, good.handle, C.byref(v), C.byref(t)), ERR_INVALID)
        expect(raw_hvp_sliced(ctx, h, good, seed=scalar_wrong), ERR_SHAPE)                 # a scalar result's seed
        expect(raw_hvp_sliced(ctx, h, good, seed_tangent=scalar_wrong), ERR_SHAPE)
        expect(raw_hvp_sliced(ctx, s_sv.plan.handle, sv_tan), ERR_INVALID)                 # no seed for a rank-13 result
        expect(raw_hvp_sliced(ctx, s_sv.plan.handle, sv_tan, seed=wrong), ERR_SHAPE)       # seed dims differ
        expect(raw_hvp_sliced(ctx, j, good), ERR_INVALID)                                  # the other sliced kind
        expect(ctx._l.tncb_plan_jvp_sliced(ctx.handle, h, 0, 1, good.handle, C.byref(v), C.byref(t)), ERR_INVALID)
        expect(ctx._l.tncb_plan_hvp(ctx.handle, h, good.handle, None, None, C.byref(v), None, None, None), ERR_UNSUPPORTED)
        expect(ctx._l.tncb_plan_jvp(ctx.handle, j, good.handle, C.byref(v), None), ERR_UNSUPPORTED)
        expect(ctx._l.tncb_plan_set_leaves(ctx.handle, h, 0, None, None), ERR_UNSUPPORTED)
        expect(ctx._l.tncb_plan_vjp_sliced(ctx.handle, h, 0, 1, None, C.byref(v), C.byref(t)), ERR_UNSUPPORTED)
        # still usable after all of that; outputs may be NULL
        val, tan, G, Gd = hp.hvp({})
        assert len(G) == len(amp.tensors)
        outs = hp.hvp_blocks({}, outputs=(False, False, False, True))
        assert outs[:3] == [None, None, None]
        outs[3].free()
    finally:
        for x in (good, short, sv_tan, wrong, scalar_wrong):
            x.free()
        other.close()
