"""Instance-batched Hessian-vector products (tncb_plan_hvp_batch, NetworkPlan.hvp_batch):

  1. bit identities: every row of all six outputs against tncb_plan_set_leaves + tncb_plan_hvp of that instance, the
     sums as the left folds of the rows, on K0 and its level batches, K1 DMMA (16 qubits x 8 rounds), K2 (a 13-qubit
     statevector with non-scalar seeds and seed tangents), a pair on the int8 engine and leaves that take the K3 gather;
     with n = 0 (many directions of the staged network) and with device payloads at non-zero and zero stride;
  2. several passes (a lowered static-workspace limit) give the one-pass bits;
  3. the full Hessian of a small network (hvp_batch over the identity) against torch.func.hessian of a TTGT replay on the
     CPU, symmetric with zero diagonal leaf blocks, and equal to the column-by-column loop of hvp;
  4. a sampled loss over bitstrings from one [B, q, 2] device tensor: rows, the fold of Ġ, Euler's identity per row;
  5. the plan's staged state is left alone: hvp before and after gives the same bits, and so does hvp_batch repeated;
  6. every error, with the arena's live bytes unchanged."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_SHAPE, ERR_OOM = -1, -2, -5


@pytest.fixture(scope="module")
def ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def counted(ctx, fn):
    ctx.reset_stats()
    res = fn()
    ctx.synchronize()
    return res, ctx.engine_counts()


def leaf_array(t):
    td = t.tensordata
    if td.kind == "gate":
        d = orc.OTensor(list(t.legs), list(t.bond_dims), ("gate", td.gate[0], td.gate[1], td.gate[2])).materialise()
    else:
        d = np.asarray(td.matrix)
    return np.asarray(d, dtype=np.complex128).reshape([int(x) for x in t.bond_dims])


def crandn(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


# ------------------------------------------------------------------------------------------------ networks
def amplitude_net(qubits, rounds, seed):
    from tnc_b200.builders import random_circuit_builder
    c = random_circuit_builder(qubits, rounds, 0.5, 0.5, np.random.default_rng(seed))
    return c.into_amplitude_network("0" * qubits)[0]


def matrix_net(specs, seed):
    """a network of Matrix leaves with random payloads; specs = [(legs, dims)]"""
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(seed)
    ts = []
    for legs, dims in specs:
        t = Tensor(legs, dims)
        t.set_tensor_data(TensorData.Matrix(crandn(rng, dims)))
        ts.append(t)
    return Tensor.new_composite(ts)


def statevector_net(seed):
    """13 qubits, 4 rounds, random normalised input states as Matrix leaves: K0 steps and one K2 step"""
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn, _ = random_circuit_builder(13, 4, 0.5, 0.5, np.random.default_rng(4)).into_statevector_network()
    rng = np.random.default_rng(seed)
    out = []
    for t in tn.tensors:
        if len(t.legs) == 1:
            v = crandn(rng, 2)
            t = Tensor(t.legs, t.bond_dims)
            t.set_tensor_data(TensorData.Matrix(v / np.linalg.norm(v)))
        out.append(t)
    return Tensor.new_composite(out)


def pair_net(m=2048, k=256, n=2048, seed=3):
    """A[m, k] x B[k, n]: M N K = 2^30, a pair for the int8 engine"""
    from tnc_b200.contractionpath import ContractionPath
    return matrix_net([([0, 1], [m, k]), ([1, 2], [k, n])], seed), ContractionPath.simple([(0, 1)])


def many_group_net():
    """X (11 legs) and Y (the same legs reversed) plus a matrix on two of them: the adjoints come out in the other leaf's
    order, more leg groups than a gather item holds -> K3"""
    from tnc_b200.contractionpath import ContractionPath
    legs = list(range(11))
    tn = matrix_net([(legs[:10] + [20], [2] * 10 + [3]), ([20, 10], [3, 2]), ([10] + legs[:10][::-1], [2] * 11)], 9)
    return tn, ContractionPath.simple([(0, 1), (0, 2)])


# ------------------------------------------------------------------------------------------------ the check
def packed_size(plan):
    offs = plan.grad_offsets()
    return sum(int(np.prod(s)) for o, s in zip(offs, plan.leaf_shapes) if o >= 0)


def row_dict(plan, row):
    """a packed tangent row as {leaf: leaf-shaped tangent}"""
    return {i: row[o:o + int(np.prod(s))].reshape(s) for i, (o, s) in enumerate(zip(plan.grad_offsets(), plan.leaf_shapes))
            if o >= 0}


def instance_payloads(payloads, i, shapes):
    return {leaf: (x[i] if tuple(x.shape) != tuple(shapes[leaf]) else x) for leaf, x in payloads.items()}


def fold(rows):
    return functools.reduce(np.add, list(rows), np.zeros(rows.shape[1:], np.complex128))


def check_rows(ctx, plan, tn, count, tangents, seeds=None, seed_tans=None, payloads=None):
    """hvp_batch (all six outputs) against set_leaves + hvp of every instance, bit for bit, and the sums against the
    left folds of the rows; the staged network is restored afterwards.  Returns the batched outputs and the engine
    counts of the batched call and of instance 0."""
    batched, ec = counted(ctx, lambda: plan.hvp_batch(count, tangents, seeds, seed_tans, payloads))
    legs, vals, tans, G, Gs, Gd, Gds = batched
    assert legs == plan.result_legs
    assert vals.shape == tans.shape == (count,) + tuple(plan.result_dims)
    ec1 = None
    for i in range(count):
        if payloads:
            plan.set_leaves(instance_payloads(payloads, i, plan.leaf_shapes))
        (v, t, g, gd), e = counted(ctx, lambda: plan.hvp(row_dict(plan, tangents[i]), None if seeds is None else seeds[i],
                                                         None if seed_tans is None else seed_tans[i]))
        ec1 = ec1 or e
        assert np.array_equal(vals[i], v) and np.array_equal(tans[i], t), i
        assert sorted(g) == sorted(G) == sorted(Gd)
        for leaf in g:
            assert np.array_equal(G[leaf][i], g[leaf]), (i, leaf)
            assert np.array_equal(Gd[leaf][i], gd[leaf]), (i, leaf)
    for leaf in G:
        assert np.array_equal(Gs[leaf], fold(G[leaf])), leaf
        assert np.array_equal(Gds[leaf], fold(Gd[leaf])), leaf
    if payloads:
        plan.stage(tn)
    return batched, ec, ec1


def directions(plan, count, seed):
    return crandn(np.random.default_rng(seed), (count, packed_size(plan)))


# ================================================================================================================
# 1. bit identities on every route
# ================================================================================================================
ROUTES = ["amp12", "amp16", "statevector", "int8_pair", "many_groups"]


def route(name):
    """(network, path, wrt, the engine instance 0 must reach, payload leaves)"""
    if name == "amp12":
        tn = amplitude_net(12, 6, 5)
        return tn, greedy(tn), None, "k0", list(range(len(tn.tensors) - 12, len(tn.tensors)))
    if name == "amp16":
        tn = amplitude_net(16, 8, 5)
        return tn, greedy(tn), list(range(len(tn.tensors)))[::2], "k1_dmma", [len(tn.tensors) - 1, len(tn.tensors) - 2]
    if name == "statevector":
        tn = statevector_net(1)
        return tn, greedy(tn), None, "k2", [k for k, t in enumerate(tn.tensors) if len(t.legs) == 1][:4]
    if name == "int8_pair":
        tn, path = pair_net()
        return tn, path, None, "k1_tcgen05", [0]
    tn, path = many_group_net()
    return tn, path, None, "permute", [1]


@pytest.mark.parametrize("name", ROUTES)
def test_bit_identities(ctx, name):
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path, wrt, engine, pl = route(name)
    plan = NetworkPlan.for_hvp(tn, path, wrt, ctx=ctx)
    plan.stage(tn)
    count = 2 if name == "int8_pair" else 4
    rng = np.random.default_rng(7)
    rdims = (count,) + tuple(plan.result_dims)
    seeds = None if name == "amp12" else crandn(rng, rdims)                  # amp12: a scalar result, every seed 1
    seed_tans = None if name == "amp16" else crandn(rng, rdims)              # amp16: zero seed tangents
    # n = 0: many directions of the staged network
    _, ec, ec1 = check_rows(ctx, plan, tn, count, directions(plan, count, 1), seeds, seed_tans)
    assert ec1[engine] >= 1, ec1
    want = {k: count * v for k, v in ec1.items()}
    want["permute"] *= 2                                  # K3 leaves: one permute into the row, one for the sum
    assert ec == want, (ec, ec1)
    # device payloads: the first payload leaf per instance (non-zero stride), the others shared (stride 0)
    dev = torch.device("cuda", ctx.device)
    payloads = {}
    for k, leaf in enumerate(pl):
        shape = plan.leaf_shapes[leaf]
        payloads[leaf] = torch.tensor(crandn(rng, ((count,) if k == 0 else ()) + shape), device=dev)
    check_rows(ctx, plan, tn, count, directions(plan, count, 2), seeds, seed_tans, payloads)
    del plan
    ctx.trim()


def test_dict_tangents_equal_packed(ctx):
    """jvp_batch-style {leaf: rows or shared} tangents and torch / DeviceTensor blocks give the packed ndarray's bits"""
    import torch
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan
    tn = amplitude_net(12, 6, 5)
    plan = NetworkPlan.for_hvp(tn, greedy(tn), ctx=ctx)
    plan.stage(tn)
    rng = np.random.default_rng(3)
    count = 3
    tans = {0: crandn(rng, (count,) + plan.leaf_shapes[0]), 5: crandn(rng, plan.leaf_shapes[5])}
    offs = plan.grad_offsets()
    packed = np.zeros((count, packed_size(plan)), np.complex128)
    packed[:, offs[0]:offs[0] + 2] = tans[0].reshape(count, -1)
    packed[:, offs[5]:offs[5] + tans[5].size] = tans[5].reshape(-1)
    ref = plan.hvp_batch(count, packed)
    dev = torch.device("cuda", ctx.device)
    block = DeviceTensor.from_numpy(ctx, packed)
    for got in (plan.hvp_batch(count, tans), plan.hvp_batch(count, torch.tensor(packed, device=dev)),
                plan.hvp_batch(count, block)):
        for a, b in zip(ref[1:3] + ref[3:], got[1:3] + got[3:]):
            if isinstance(a, dict):
                assert all(np.array_equal(a[k], b[k]) for k in a)
            else:
                assert np.array_equal(a, b)
    block.free()
    # outputs left out are None; the forward outputs alone skip the backward levels
    _, v, t, g, gs, gd, gds = plan.hvp_batch(count, packed, outputs=(True, True, False, False, False, False))
    assert np.array_equal(v, ref[1]) and np.array_equal(t, ref[2]) and g is gs is gd is gds is None
    _, v, t, g, gs, gd, gds = plan.hvp_batch(count, packed, outputs=(False, False, False, True, False, False))
    assert v is t is g is gd is gds is None and all(np.array_equal(gs[k], ref[4][k]) for k in gs)


# ================================================================================================================
# 2. several passes
# ================================================================================================================
def test_several_passes(ctx, monkeypatch):
    """the int8 pair's 0.33 GiB workspace under a 1 GiB limit: 3 copies per pass, 7 instances in 3 passes"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = pair_net()
    plan = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    ws = plan.info()["peak_bytes"]
    assert 3 * ws <= 1 << 30 < 4 * ws, ws
    plan.stage(tn)
    rng = np.random.default_rng(11)
    count = 7
    rdims = (count,) + tuple(plan.result_dims)
    args = (count, directions(plan, count, 4), crandn(rng, rdims), crandn(rng, rdims),
            {0: torch.tensor(crandn(rng, (count,) + plan.leaf_shapes[0]), device=torch.device("cuda", ctx.device))})
    one_pass = plan.hvp_batch(*args)
    monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")
    passes = plan.hvp_batch(*args)
    monkeypatch.delenv("TNCB_PLAN_WS_GB")
    for a, b in zip(one_pass[1:], passes[1:]):
        if isinstance(a, dict):
            assert sorted(a) == sorted(b) and all(np.array_equal(a[k], b[k]) for k in a)
        else:
            assert np.array_equal(a, b)
    del plan
    ctx.trim()


# ================================================================================================================
# 3. the full Hessian of a small network
# ================================================================================================================
def ttgt(a_legs, A, b_legs, B):
    import torch
    shared = [l for l in a_legs if l in b_legs]
    am = [l for l in a_legs if l not in b_legs]
    bn = [l for l in b_legs if l not in a_legs]
    dim = dict(zip(a_legs, A.shape)) | dict(zip(b_legs, B.shape))
    size = lambda ls: int(np.prod([dim[l] for l in ls], dtype=np.int64))
    At = A.permute([a_legs.index(l) for l in shared + am]).reshape(size(shared), size(am))
    Bt = B.permute([b_legs.index(l) for l in bn + shared]).reshape(size(bn), size(shared))
    return bn + am, torch.matmul(Bt, At).reshape([dim[l] for l in bn + am])


def replay(tn, path, xs):
    it = iter(xs)

    def walk(t, p):
        if not t.tensors:
            return list(t.legs), next(it)
        slots = [walk(c, p.nested.get(i) if c.tensors else None) for i, c in enumerate(t.tensors)]
        for i, j in p.toplevel:
            slots[i] = ttgt(*slots[i], *slots[j])
            slots[j] = None
        return next(s for s in slots if s is not None)
    return walk(tn, path)


def test_full_hessian(ctx):
    """5 qubits x 3 rounds, 21 leaves, 124 tangent elements: hvp_batch over the identity is H = d²(S R)/dX dX"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    tn = amplitude_net(5, 3, 1)
    path = greedy(tn)
    lv = leaves(tn)
    plan = NetworkPlan.for_hvp(tn, path, ctx=ctx)
    plan.stage(tn)
    offs = plan.grad_offsets()
    te = packed_size(plan)
    assert te == 124 and all(o >= 0 for o in offs)
    S = np.array([0.6 - 0.8j])
    _, _, _, _, _, Gd, _ = plan.hvp_batch(te, np.eye(te), np.repeat(S, te), outputs=(False,) * 4 + (True, False))
    H = np.concatenate([Gd[i].reshape(te, -1) for i in range(len(lv))], axis=1)      # row p: H e_p
    # the holomorphic Hessian of S R on the CPU replay: along real directions, real and imaginary parts apart
    x0 = torch.tensor(np.concatenate([leaf_array(l).ravel() for l in lv]))

    def loss(a):
        x = x0 + a
        xs = [x[o:o + int(np.prod(s))].reshape(s) for o, s in zip(offs, plan.leaf_shapes)]
        return complex(S[0]) * replay(tn, path, xs)[1]
    a0 = torch.zeros(te, dtype=torch.float64)
    H_ref = (torch.func.hessian(lambda a: loss(a).real)(a0) + 1j * torch.func.hessian(lambda a: loss(a).imag)(a0)).numpy()
    mag = torch.func.hessian(lambda a: (complex(abs(S[0])) * replay(tn, path, [
        (x0.abs() + a)[o:o + int(np.prod(s))].reshape(s).to(torch.complex128) for o, s in zip(offs, plan.leaf_shapes)])[1]).real)(a0)
    scale = np.maximum(np.abs(mag.numpy()), np.abs(mag.numpy()).max() * 1e-3)
    assert (np.abs(H - H_ref) <= 1e-12 * scale + 1e-300).all(), np.abs(H - H_ref).max()
    assert np.abs(H - H.T).max() <= 1e-12 * np.abs(H).max()
    for o, s in zip(offs, plan.leaf_shapes):                                             # multilinear: zero diagonal blocks
        n = int(np.prod(s))
        assert not H[o:o + n, o:o + n].any()
    for p in range(te):                                                                   # the column-by-column loop
        gd = plan.hvp(row_dict(plan, np.eye(te)[p]), S[0])[3]
        assert np.array_equal(np.concatenate([gd[i].ravel() for i in range(len(lv))]), H[p]), p


# ================================================================================================================
# 4. a sampled loss over bitstrings
# ================================================================================================================
def test_sampled_bitstrings(ctx):
    """B = 6 output bitstrings of a 12-qubit amplitude network from one [B, q, 2] device tensor (strided views, no
    copies), per-instance seeds and seed tangents; then Ẋ = X and Ṡ = 0 with every leaf requested: Euler's identity
    for the multilinear R, Ġ_l = (k - 1) G_l and Ṙ = k R, row by row"""
    import torch
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    q, B = 12, 6
    tn = amplitude_net(q, 6, 5)
    lv = leaves(tn)
    k = len(lv)
    bit_leaves = list(range(k - q, k))
    plan = NetworkPlan.for_hvp(tn, greedy(tn), ctx=ctx)
    plan.stage(tn)
    rng = np.random.default_rng(9)
    bits = rng.integers(0, 2, (B, q))
    onehot = np.zeros((B, q, 2), np.complex128)
    onehot[np.arange(B)[:, None], np.arange(q)[None, :], bits] = 1.0
    dev_bits = torch.tensor(onehot, device=torch.device("cuda", ctx.device))
    payloads = {leaf: dev_bits[:, j, :] for j, leaf in enumerate(bit_leaves)}
    seeds, seed_tans = crandn(rng, (B,)), crandn(rng, (B,))
    check_rows(ctx, plan, tn, B, directions(plan, B, 5), seeds, seed_tans, payloads)
    # Euler: the tangent of instance i is its own leaves, packed
    offs = plan.grad_offsets()
    X = np.zeros((B, packed_size(plan)), np.complex128)
    for i, l in enumerate(lv):
        X[:, offs[i]:offs[i] + int(np.prod(l.bond_dims))] = leaf_array(l).ravel()
    for j, leaf in enumerate(bit_leaves):
        X[:, offs[leaf]:offs[leaf] + 2] = onehot[:, j, :]
    (_, vals, tans, G, _, Gd, Gds), _, _ = check_rows(ctx, plan, tn, B, X, seeds, None, payloads)
    for i in range(B):
        r = complex(vals[i])
        assert abs(complex(tans[i]) - k * r) <= 1e-9 * k * abs(r), (i, complex(tans[i]), k * r)
        gb = np.concatenate([G[l][i].ravel() for l in range(k)])
        gdb = np.concatenate([Gd[l][i].ravel() for l in range(k)])
        assert np.linalg.norm(gdb - (k - 1) * gb) <= 1e-9 * (k - 1) * np.linalg.norm(gb), i
    assert sorted(Gds) == list(range(k))


# ================================================================================================================
# 5. the plan's state
# ================================================================================================================
def test_plan_state_untouched(ctx):
    import torch
    from tnc_b200.tensornetwork import NetworkPlan
    tn = statevector_net(2)
    plan = NetworkPlan.for_hvp(tn, greedy(tn), ctx=ctx)
    plan.stage(tn)
    rng = np.random.default_rng(13)
    row = directions(plan, 1, 6)[0]
    S, Sd = crandn(rng, plan.result_dims), crandn(rng, plan.result_dims)
    before = plan.hvp(row_dict(plan, row), S, Sd)
    count = 5
    rdims = (count,) + tuple(plan.result_dims)
    leaf = next(i for i, t in enumerate(tn.tensors) if len(t.legs) == 1)
    args = (count, directions(plan, count, 7), crandn(rng, rdims), crandn(rng, rdims),
            {leaf: torch.tensor(crandn(rng, (count, 2)), device=torch.device("cuda", ctx.device))})
    first = plan.hvp_batch(*args)
    after = plan.hvp(row_dict(plan, row), S, Sd)
    again = plan.hvp_batch(*args)
    for a, b in zip(before, after):
        if isinstance(a, dict):
            assert all(np.array_equal(a[k], b[k]) for k in a)
        else:
            assert np.array_equal(a, b)
    for a, b in zip(first[1:], again[1:]):
        if isinstance(a, dict):
            assert all(np.array_equal(a[k], b[k]) for k in a)
        else:
            assert np.array_equal(a, b)


# ================================================================================================================
# 6. errors
# ================================================================================================================
def raw(c, handle, count, tangents, seeds=None, seed_tans=None, items=(), outs=(True,) * 6):
    """tncb_plan_hvp_batch with device sources items = [(leaf, address, stride)]"""
    from tnc_b200._lib import u64_array
    idx = u64_array([i for i, _, _ in items])
    src = (C.c_void_p * max(len(items), 1))(*[p for _, p, _ in items])
    st = u64_array([s for _, _, s in items])
    o = [C.c_void_p() for _ in outs]
    h = lambda t: t.handle if t is not None else None
    rc = c._l.tncb_plan_hvp_batch(c.handle, handle, count, len(items), idx, src, st, h(tangents), h(seeds), h(seed_tans),
                                  *[C.byref(x) if w else None for x, w in zip(o, outs)])
    if rc == 0:
        from tnc_b200 import DeviceTensor
        for x, w in zip(o, outs):
            if w:
                DeviceTensor.adopt(c, x).free()
    return rc


def rank64_net():
    """A x B over one shared leg, 64 open legs of dimension 1 in the result"""
    from tnc_b200.contractionpath import ContractionPath
    tn = matrix_net([(list(range(32)) + [100], [1] * 32 + [2]), ([100] + list(range(32, 64)), [2] + [1] * 32)], 12)
    return tn, ContractionPath.simple([(0, 1)])


def outer_net(d):
    """u[i] v[j] u'[i] v'[j]: a scalar result, a d x d outer product inside (1.5 GiB of Hessian-vector workspace at
    d = 4096)"""
    from tnc_b200.contractionpath import ContractionPath
    return matrix_net([([0], [d]), ([1], [d]), ([0], [d]), ([1], [d])], 14), ContractionPath.simple([(0, 1), (0, 2), (0, 3)])


def test_errors(ctx, monkeypatch):
    import torch
    import tnc_b200 as tb
    from tnc_b200 import DeviceTensor
    from tnc_b200.tensornetwork import NetworkPlan
    sv = statevector_net(2)
    sv_path = greedy(sv)
    h = NetworkPlan.for_hvp(sv, sv_path, ctx=ctx)
    unstaged = NetworkPlan.for_hvp(sv, sv_path, ctx=ctx)
    plain = NetworkPlan(sv, sv_path, ctx=ctx)
    plain.stage(sv)
    g = NetworkPlan.for_gradients(sv, sv_path, ctx=ctx)
    g.stage(sv)
    r64, r64_path = rank64_net()
    h64 = NetworkPlan.for_hvp(r64, r64_path, ctx=ctx)
    assert len(h64.result_legs) == 64
    h64.stage(r64)
    big, big_path = outer_net(4096)
    hbig = NetworkPlan.for_hvp(big, big_path, ctx=ctx)
    assert hbig.info()["peak_bytes"] > 1 << 30
    hbig.stage(big)
    h.stage(sv)
    te = packed_size(h)
    count = 2
    rdims = (count,) + tuple(h.result_dims)
    dev = torch.device("cuda", ctx.device)
    good = DeviceTensor.from_numpy(ctx, np.ones((count, te), np.complex128))
    wrong = [DeviceTensor.from_numpy(ctx, np.ones(s, np.complex128)) for s in ((count, te + 1), (count + 1, te), (te,))]
    seeds = DeviceTensor.from_numpy(ctx, np.ones(rdims, np.complex128))
    bad_seeds = [DeviceTensor.from_numpy(ctx, np.ones(s, np.complex128)) for s in (rdims[1:], (count + 1,) + rdims[1:])]
    t64 = DeviceTensor.from_numpy(ctx, np.ones((1, packed_size(h64)), np.complex128))
    tbig = DeviceTensor.from_numpy(ctx, np.ones((1, packed_size(hbig)), np.complex128))
    leaf = next(i for i, t in enumerate(sv.tensors) if len(t.legs) == 1)
    other_leaf = next(i for i, t in enumerate(sv.tensors) if len(t.legs) == 1 and i != leaf)
    pay = torch.ones((count, 2), dtype=torch.complex128, device=dev)
    host = np.ones((count, 2), np.complex128)
    p = pay.data_ptr()
    other = tb.Context(0)
    try:
        ctx.synchronize()
        live = ctx.stats()["arena_live_bytes"]

        def expect(rc, want):
            assert rc == want, (rc, want, ctx._l.tncb_last_error())
            ctx.synchronize()
            assert ctx.stats()["arena_live_bytes"] == live

        expect(raw(ctx, plain.handle, count, good, seeds), ERR_INVALID)             # not a Hessian-vector plan
        expect(raw(ctx, g.handle, count, good, seeds), ERR_INVALID)
        expect(raw(ctx, unstaged.handle, count, good, seeds), ERR_INVALID)          # nothing staged
        expect(raw(other, h.handle, count, good, seeds), ERR_INVALID)               # another context
        expect(raw(ctx, h.handle, 0, good, seeds), ERR_INVALID)                     # count 0
        expect(raw(ctx, h.handle, count, good, seeds, outs=(False,) * 6), ERR_INVALID)   # no output
        expect(raw(ctx, h.handle, count, None, seeds), ERR_INVALID)                 # no tangents
        expect(raw(ctx, h.handle, count, good, None), ERR_INVALID)                  # no seeds for a rank-13 result
        expect(raw(ctx, h64.handle, 1, t64, None), ERR_INVALID)                     # rank 64: no instance dimension
        for w in wrong:
            expect(raw(ctx, h.handle, count, w, seeds), ERR_SHAPE)
        for b in bad_seeds:
            expect(raw(ctx, h.handle, count, good, b), ERR_SHAPE)
            expect(raw(ctx, h.handle, count, good, seeds, b), ERR_SHAPE)
        for items in ([(len(sv.tensors), p, 2)],                                    # no such leaf
                      [(leaf, p, 2), (leaf, p, 2)],                                 # listed twice
                      [(leaf, p, 1)],                                               # stride below the leaf's 2 elements
                      [(leaf, 0, 2)],                                               # null source
                      [(leaf, p + 8, 2)],                                           # not 16-byte aligned
                      [(leaf, host.ctypes.data, 2)],                                # host memory
                      [(other_leaf, p, 0), (leaf, p, 1)]):                          # the second source is refused
            expect(raw(ctx, h.handle, count, good, seeds, items=items), ERR_INVALID)
        monkeypatch.setenv("TNCB_PLAN_WS_GB", "1")                                  # not one copy fits
        expect(raw(ctx, hbig.handle, 1, tbig, None), ERR_OOM)
        monkeypatch.delenv("TNCB_PLAN_WS_GB")
        # the legal calls next to them work: one output alone, shared and per-instance sources
        for k in range(6):
            expect(raw(ctx, h.handle, count, good, seeds, items=[(leaf, p, 2), (other_leaf, p, 0)],
                       outs=tuple(j == k for j in range(6))), 0)
    finally:
        other.close()
        for t in [good, seeds, t64, tbig] + wrong + bad_seeds:
            t.free()
