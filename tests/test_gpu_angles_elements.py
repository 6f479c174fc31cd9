"""The device's gate-angle table element by element, the angle kernels' edges, and exact parameter shifts of all six
angle gates on the H100 (tncb_angles_gates / tangents / pullback, tnc_b200.angles).

Single entries are read off the device through maps whose reads are exact (every angle its own parameter, scale 1):
gates rows give U; tangents(θ, e_p) and pullback(θ, identity rows) give dU/da_s (the kernels add 0 + u·1); pullback with
identity rows, zero Ġ and direction e_q gives d²U/da_s da_t.  They are compared with the 50-digit reference of
tests/test_angles_table_host.py at the arguments the kernels form, within 9·2^-53 per component (CUDA's double sin and
cos are within 2 ulp), and at the nominal angles within that plus the argument rounding.  General maps (one parameter on
several slots and leaves, scales negative and 0, slots that keep their own angle) are compared with the 50-digit chain
rule within (n_terms + 9)·2^-53·Σ|terms|.  The edges: more rows than the grid's y dimension, several x-blocks, elements
outside the referenced leaves, row strides and shared rows, non-finite θ.  Last, a 14-qubit circuit with every angle
gate and both adjoint flags: gradient, Jacobian and Hessian against exact parameter shifts evaluated through a plain
plan's batched run."""
import ctypes as C
import math

import numpy as np
import pytest

from test_angles_table_host import (ANGLES, DEVICE_UNITS, DIM, N_ANG, TINY, U53, M, adjointed, angle_tuples, compare,
                                    reference, split, _structure)
from test_gpu_angles import cuda, greedy, hvp_batch_rows

pytestmark = pytest.mark.gpu
WORST = {}


def note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k in sorted(WORST):
        print(f"worst ratio to the bound, {k}: {WORST[k]:.3g}")


def gate_circuit(gates, qubits=2, own=0.1):
    """one leaf per (gate, adjoint) on `qubits` qubits; returns (tn, [(leaf, gate, adjoint)])"""
    from tnc_b200.builders import Circuit
    from tnc_b200.tensornetwork import leaves
    c = Circuit()
    q = c.allocate_register(qubits)
    for i, (g, adj) in enumerate(gates):
        qs = [q[i % qubits]] if DIM[g] == 2 else [q[i % qubits], q[(i + 1) % qubits]]
        c.append_gate(g, [own] * N_ANG[g], qs, adjoint=adj)
    tn = c.into_amplitude_network("0" * qubits)[0]
    gl = [i for i, t in enumerate(leaves(tn)) if t.tensordata.kind == "gate"]
    return tn, [(l, g, adj) for l, (g, adj) in zip(gl, gates)]


ALL12 = [(g, adj) for g in sorted(N_ANG) for adj in (False, True)]


@pytest.fixture(scope="module")
def table_map(ctx):
    """the twelve leaves (six gates, both flags), every angle its own parameter; θ row i puts angle_tuples(g)[i] on
    each leaf of gate g (cycling), so the rows run through every angle set of the host test"""
    from tnc_b200.angles import AngleMap, Angles
    tn, lv = gate_circuit(ALL12)
    amap = AngleMap.every_angle(tn)
    ang = Angles(ctx, tn, amap)
    params, p = {}, 0
    for l, g, _ in lv:
        params[l] = list(range(p, p + N_ANG[g]))
        p += N_ANG[g]
    assert p == amap.n_params
    count = max(len(angle_tuples(g)) for g in N_ANG)
    theta = np.zeros((count, p))
    tup = {}
    for l, g, _ in lv:
        ts = angle_tuples(g)
        for i in range(count):
            tup[i, l] = ts[i % len(ts)]
            theta[i, params[l]] = ts[i % len(ts)]
    return ang, lv, params, theta, tup


def span(ang, l, g):
    return slice(ang.offsets[l], ang.offsets[l] + DIM[g] ** 2)


# ------------------------------------------------------------------------------------------------ 1. the table
def test_gate_rows_against_50_digits(table_map):
    ang, lv, params, theta, tup = table_map
    rows = ang.gates(cuda(theta)).to_numpy()
    for i in range(len(theta)):
        for l, g, adj in lv:
            rf, rn = compare(rows[i, span(ang, l, g)], g, tup[i, l], (), adj, DEVICE_UNITS)
            note("U at the formed arguments", rf)
            note("U at the nominal angles", rn)


def test_first_derivatives_against_50_digits(ctx, table_map):
    import torch
    from tnc_b200 import DeviceTensor
    ang, lv, params, theta, tup = table_map
    count, P, E = len(theta), ang.n_params, ang.block_elems
    leaf_of = {p: (l, g, adj, s) for l, g, adj in lv for s, p in enumerate(params[l])}
    # tangents(θ, e_p): row i holds dU/da_{s_p} of p's leaf, zeros elsewhere
    for p in range(P):
        l, g, adj, s = leaf_of[p]
        rows = ang.tangents(cuda(theta), cuda(np.eye(P)[p])).to_numpy()
        sp = span(ang, l, g)
        for i in range(count):
            note("dU (tangents)", compare(rows[i, sp], g, tup[i, l], (s,), adj, DEVICE_UNITS)[0])
        rest = np.delete(rows, np.arange(E)[sp], axis=1)
        assert np.all(rest == 0), p
    # pullback(θ, identity rows): entry [k][p] = dU[k]/da_{s_p}; θ_i repeated over the E identity rows
    th = torch.repeat_interleave(cuda(theta), E, dim=0)
    eye = torch.eye(E, dtype=torch.complex128, device="cuda").repeat(count, 1)
    G = DeviceTensor.from_torch(ctx, eye)
    out = ang.pullback(th, G)[0].to_numpy().reshape(count, E, P)
    for p in range(P):
        l, g, adj, s = leaf_of[p]
        sp = span(ang, l, g)
        for i in range(count):
            note("dU (pullback)", compare(out[i, sp, p], g, tup[i, l], (s,), adj, DEVICE_UNITS)[0])
        assert np.all(np.delete(out[:, :, p], np.arange(E)[sp], axis=1) == 0), p
    # the Hessian entries: identity rows, zero Ġ, direction e_q: [k][p] = d²U[k]/da_{s_p} da_{s_q} on a shared leaf
    Gd = DeviceTensor.from_torch(ctx, torch.zeros_like(eye))
    for q in range(P):
        lq, _, _, sq = leaf_of[q]
        out = ang.pullback(th, G, Gd, cuda(np.eye(P)[q]))[0].to_numpy().reshape(count, E, P)
        for p in range(P):
            l, g, adj, s = leaf_of[p]
            if l != lq:
                assert np.all(out[:, :, p] == 0), (p, q)
                continue
            sp = span(ang, l, g)
            for i in range(count):
                note("d2U (pullback)", compare(out[i, sp, p], g, tup[i, l], (s, sq), adj, DEVICE_UNITS)[0])
            assert np.all(np.delete(out[:, :, p], np.arange(E)[sp], axis=1) == 0), (p, q)


# ------------------------------------------------------------------------------------------------ 2. general maps
def chain_map():
    """u and fsim leaves with one parameter on two slots (scales of both signs and 0), one parameter over ten leaves,
    leaves whose other slots keep their own angle; returns (tn, AngleMap, {leaf: gate, adjoint, own angles})"""
    from tnc_b200.angles import AngleMap
    gates = [("u", False), ("fsim", True), ("rx", False), ("ry", True), ("rz", False), ("cp", True), ("u", True),
             ("rz", True), ("rx", True), ("cp", False), ("ry", False), ("fsim", False), ("u", False)]
    tn, lv = gate_circuit(gates, qubits=3, own=0.45)
    L = [l for l, _, _ in lv]
    refs = [(L[0], 1, 0, 0.7), (L[0], 2, 0, -1.3), (L[0], 0, 2, 1.0),             # u: φ and λ tied
            (L[1], 0, 0, 2.0), (L[1], 1, 0, 0.0),                                  # fsim: θ and φ tied, one scale 0
            (L[2], 0, 1, 1.5), (L[3], 0, 1, -0.25), (L[4], 0, 1, 3.0), (L[5], 0, 1, -1.0), (L[6], 0, 1, 0.5),
            (L[7], 0, 1, 1e-3), (L[8], 0, 1, 7.0), (L[9], 0, 1, -2.5), (L[10], 0, 1, 0.0), (L[11], 1, 1, -0.75),
            (L[6], 2, 2, -1.0),                                                    # u: φ keeps its own angle
            (L[11], 0, 3, 1.0), (L[12], 2, 3, 0.3)]                                # u: θ and φ keep their own
    own = {l: (g, adj, [0.45] * N_ANG[g]) for l, g, adj in lv}
    return tn, AngleMap(refs, 4), own


def chain_reference(g, adj, a, pairs, roundings=1):
    """Σ_j c_j d^{|D_j|} U / da_{D_j} at slot values a (the formed ones), adjointed when asked, c_j a product of
    scales (exact in 50 digits): (hi, lo, Σ|terms|, structurally nonzero, the roundings the kernel makes) per component
    [d*d, 2].  The kernel scales each term `roundings` times and adds the terms up: with the element's own error that
    is within (n_terms - 1 + roundings + 9)·2^-53·Σ|terms| to first order."""
    d = DIM[g]
    tot = [M.mpc(0)] * (d * d)
    mags = np.zeros((d * d, 2))
    st = np.zeros((d * d, 2), dtype=bool)
    for cs, D in pairs:
        c = M.fprod(M.mpf(x) for x in cs)
        vals = reference(g, tuple(a), tuple(D))[0]
        s = _structure(g, tuple(D))
        if adj:
            vals = adjointed(vals, d)
            s = s[[cc * d + r for r in range(d) for cc in range(d)]]
        tot = [x + c * y for x, y in zip(tot, vals)]
        hi, _ = split([c * y for y in vals])
        mags += np.abs(hi)
        st |= s
    hi, lo = split(tot)
    return hi, lo, mags, st, max(len(pairs) - 1 + roundings, 0)


def check_chain(got, ref, what):
    hi, lo, mags, st, n = ref
    g = np.stack([got.real, got.imag], axis=1)
    assert np.all(g[~st] == 0), (what, g[~st])
    err = np.abs((g - hi) - lo)
    tol = (n + DEVICE_UNITS) * U53 * mags + n * TINY
    assert np.all(err <= tol), (what, g, hi, err, tol)
    if (tol > 0).any():
        note("chain rule sums", float((err[tol > 0] / tol[tol > 0]).max()))


def test_chain_rule_maps(ctx):
    import torch
    from tnc_b200 import DeviceTensor
    from tnc_b200.angles import Angles
    tn, amap, own = chain_map()
    ang = Angles(ctx, tn, amap)
    P, E = amap.n_params, ang.block_elems
    rng = np.random.default_rng(11)
    theta = np.concatenate([rng.uniform(-4, 4, (12, P)), [[1e3, -123.456, 1e5, 2.0 ** 31 + 1], [0.0, -0.0, 1e-300, math.pi]]])
    count = len(theta)
    by_leaf = {}
    for l, s, p, c in amap.refs:
        by_leaf.setdefault(l, []).append((s, p, c))

    def slots(i, l):
        g, _, a = own[l]
        a = list(a)
        for s, p, c in by_leaf[l]:
            a[s] = c * theta[i, p]                 # fl(c·θ), as the kernels form it
        return tuple(a)

    th = torch.repeat_interleave(cuda(theta), E, dim=0)
    eye = torch.eye(E, dtype=torch.complex128, device="cuda").repeat(count, 1)
    G, Gd = DeviceTensor.from_torch(ctx, eye), DeviceTensor.from_torch(ctx, torch.zeros_like(eye))
    grad = ang.pullback(th, G)[0].to_numpy().reshape(count, E, P)
    hess = [ang.pullback(th, G, Gd, cuda(np.eye(P)[q]))[0].to_numpy().reshape(count, E, P) for q in range(P)]
    for p in range(P):
        tan = ang.tangents(cuda(theta), cuda(np.eye(P)[p])).to_numpy()
        for l, rs in by_leaf.items():
            g, adj, _ = own[l]
            sp = span(ang, l, g)
            first = [((c,), (s,)) for s, pp, c in rs if pp == p]
            for i in range(count):
                a = slots(i, l)
                ref = chain_reference(g, adj, a, first)
                check_chain(tan[i, sp], ref, ("tangents", p, l, i))
                check_chain(grad[i, sp, p], ref, ("pullback", p, l, i))
                for q in range(P):
                    second = [((c, c2), (s, s2)) for s, pp, c in rs if pp == p for s2, qq, c2 in rs if qq == q]
                    check_chain(hess[q][i, sp, p], chain_reference(g, adj, a, second, 2), ("hessian", p, q, l, i))


# ------------------------------------------------------------------------------------------------ 3. kernel edges
def test_rows_past_the_grid(ctx, table_map):
    """count = 65537: the rows past the grid's y dimension (65535) equal the same calls on that row alone"""
    import torch
    from tnc_b200 import DeviceTensor
    ang, lv, params, theta, tup = table_map
    P, E, n = ang.n_params, ang.block_elems, 65537
    gen = torch.Generator(device="cuda").manual_seed(5)
    TH = (torch.rand((n, P), dtype=torch.float64, device="cuda", generator=gen) - 0.5) * 8
    D = torch.randn((n, P), dtype=torch.float64, device="cuda", generator=gen)
    V = torch.randn((n, P), dtype=torch.float64, device="cuda", generator=gen)
    Gt = torch.randn((n, E), dtype=torch.complex128, device="cuda", generator=gen)
    Gdt = torch.randn((n, E), dtype=torch.complex128, device="cuda", generator=gen)
    G, Gd = DeviceTensor.from_torch(ctx, Gt), DeviceTensor.from_torch(ctx, Gdt)
    gates = ang.gates(TH).to_torch()[n - 2:].cpu().numpy()
    tans = ang.tangents(TH, D).to_torch()[n - 2:].cpu().numpy()
    prow, psum = ang.pullback(TH, G, rows=True, sum=True)
    prow, psum = prow.to_numpy(), psum.to_numpy()
    hrow = ang.pullback(TH, G, Gd, V)[0].to_torch()[n - 2:].cpu().numpy()
    for j, i in enumerate((n - 2, n - 1)):
        Gi, Gdi = DeviceTensor.from_torch(ctx, Gt[i]), DeviceTensor.from_torch(ctx, Gdt[i])
        assert np.array_equal(gates[j], ang.gates(TH[i]).to_numpy()[0])
        assert np.array_equal(tans[j], ang.tangents(TH[i:i + 1], D[i:i + 1]).to_numpy()[0])
        assert np.array_equal(prow[i], ang.pullback(TH[i], Gi)[0].to_numpy()[0])
        assert np.array_equal(hrow[j], ang.pullback(TH[i], Gi, Gdi, V[i])[0].to_numpy()[0])
    fold = np.zeros(P, dtype=np.complex128)
    for i in range(n):                           # the left fold 0 + row_0 + row_1 + ..., one vector add per row
        fold = fold + prow[i]
    assert np.array_equal(psum, fold)


def wide_circuit(qubits=10, layers=14):
    """h gates, every angle gate and both adjoint flags over `qubits` qubits; every seventh angle leaf left out of the
    map; returns (tn, AngleMap, [(leaf, gate, adjoint, params)])"""
    from tnc_b200.angles import AngleMap
    from tnc_b200.builders import Circuit
    from tnc_b200.tensornetwork import leaves
    rng = np.random.default_rng(8)
    c = Circuit()
    q = c.allocate_register(qubits)
    for i in range(qubits):
        c.append_gate("h", [], [q[i]])
    singles = ["u", "rx", "ry", "rz", "u"]
    for layer in range(layers):
        for i in range(qubits):
            g = singles[(i + layer) % len(singles)]
            c.append_gate(g, list(rng.uniform(-2, 2, N_ANG[g])), [q[i]], adjoint=(i + layer) % 3 == 0)
        for i in range(layer % 2, qubits - 1, 2):
            g = "fsim" if (i // 2 + layer) % 2 else "cp"
            c.append_gate(g, list(rng.uniform(-2, 2, N_ANG[g])), [q[i], q[i + 1]], adjoint=(i + layer) % 4 == 1)
        c.append_gate("h", [], [q[layer % qubits]])
    tn = c.into_amplitude_network("0" * qubits)[0]
    lv = leaves(tn)
    angle_leaves = [i for i, t in enumerate(lv) if t.tensordata.kind == "gate" and t.tensordata.gate[0] in N_ANG]
    refs, info = [], []
    for k, l in enumerate(angle_leaves):
        if k % 7 == 3:
            continue                             # an angle gate the map does not reference
        name, _, adj = lv[l].tensordata.gate
        ps = list(range(len(refs), len(refs) + N_ANG[name]))
        refs += [(l, s, p, 1.0) for s, p in enumerate(ps)]
        info.append((l, name, bool(adj), ps))
    return tn, AngleMap(refs, len(refs)), info


@pytest.fixture(scope="module")
def wide(ctx):
    from tnc_b200.angles import Angles
    from tnc_b200.tensornetwork import NetworkPlan
    tn, amap, info = wide_circuit()
    gp = NetworkPlan.for_gradients(tn, greedy(tn), ctx=ctx)          # every leaf: h gates and states in the block too
    ang = Angles(ctx, tn, amap, gp)
    P = amap.n_params
    assert 256 < P < 384 and P % 128 and len(info) > 8
    inside = np.zeros(ang.block_elems, dtype=bool)
    for l, g, _, _ in info:
        inside[span(ang, l, g)] = True
    assert not inside.all()
    return ang, info, inside


def test_many_params_and_untouched_elements(ctx, wide):
    import torch
    from tnc_b200 import DeviceTensor
    ang, info, inside = wide
    P, E = ang.n_params, ang.block_elems
    rng = np.random.default_rng(21)
    theta = np.concatenate([rng.uniform(-4, 4, (3, P)), rng.choice(ANGLES, (1, P))])
    rows = ang.gates(cuda(theta)).to_numpy()
    assert np.all(rows[:, ~inside] == 0)
    for i in range(len(theta)):
        for l, g, adj, ps in info:
            note("U, 300 parameters", compare(rows[i, span(ang, l, g)], g, tuple(theta[i, ps]), (), adj, DEVICE_UNITS)[0])
    # tangents along every e_p at θ_0: row p is dU/da_{s_p} on p's leaf and zero everywhere else
    tan = ang.tangents(cuda(theta[0]), cuda(np.eye(P))).to_numpy()
    for l, g, adj, ps in info:
        sp = span(ang, l, g)
        for s, p in enumerate(ps):
            note("dU, 300 parameters", compare(tan[p, sp], g, tuple(theta[0, ps]), (s,), adj, DEVICE_UNITS)[0])
            tan[p, sp] = 0
    assert np.all(tan == 0)
    # pullback: G and Ġ NaN outside the referenced spans leave every row as with zeros there
    Gz = rng.standard_normal((4, E)) + 1j * rng.standard_normal((4, E))
    Gdz = rng.standard_normal((4, E)) + 1j * rng.standard_normal((4, E))
    Gz[:, ~inside] = 0
    Gdz[:, ~inside] = 0
    Gn, Gdn = Gz.copy(), Gdz.copy()
    Gn[:, ~inside] = np.nan
    Gdn[:, ~inside] = complex(np.nan, np.nan)
    V = rng.standard_normal((4, P))
    up = lambda a: DeviceTensor.from_numpy(ctx, a)
    for args in [(), "hvp"]:
        extra_z = (up(Gdz), cuda(V)) if args else ()
        extra_n = (up(Gdn), cuda(V)) if args else ()
        rz_, sz = ang.pullback(cuda(theta), up(Gz), *extra_z, rows=True, sum=True)
        rn, sn = ang.pullback(cuda(theta), up(Gn), *extra_n, rows=True, sum=True)
        rz_, rn = rz_.to_numpy(), rn.to_numpy()
        assert np.isfinite(rz_).all()
        assert rz_.tobytes() == rn.tobytes() and sz.to_numpy().tobytes() == sn.to_numpy().tobytes()
        fold = np.zeros(P, dtype=np.complex128)
        for i in range(4):
            fold = fold + rz_[i]
        assert np.array_equal(sn.to_numpy(), fold)
    # pullback of identity rows over the whole block: dU[k]/da_{s_p} inside p's span, zero elsewhere
    eye = DeviceTensor.from_torch(ctx, torch.eye(E, dtype=torch.complex128, device="cuda"))
    out = ang.pullback(cuda(theta[1]), eye)[0].to_numpy()
    for l, g, adj, ps in info:
        sp = span(ang, l, g)
        for s, p in enumerate(ps):
            note("dU, 300 parameters", compare(out[sp, p], g, tuple(theta[1, ps]), (s,), adj, DEVICE_UNITS)[0])
            out[sp, p] = 0
    assert np.all(out == 0)


def test_row_strides_and_shared_rows(ctx, wide):
    import torch
    from tnc_b200 import DeviceTensor
    ang, info, inside = wide
    P, E, n = ang.n_params, ang.block_elems, 5
    gen = torch.Generator(device="cuda").manual_seed(9)
    W = (torch.rand((n, P + 7), dtype=torch.float64, device="cuda", generator=gen) - 0.5) * 8
    TH = W[:, 3:3 + P]                           # row stride P + 7
    assert TH.stride(0) == P + 7
    THc = TH.contiguous()
    D = torch.randn((n, P), dtype=torch.float64, device="cuda", generator=gen)
    V = torch.randn((n, P), dtype=torch.float64, device="cuda", generator=gen)
    Gt = torch.randn((n, E), dtype=torch.complex128, device="cuda", generator=gen)
    Gdt = torch.randn((n, E), dtype=torch.complex128, device="cuda", generator=gen)
    dt = lambda x: DeviceTensor.from_torch(ctx, x)
    same = lambda a, b: a.to_numpy().tobytes() == b.to_numpy().tobytes()
    assert same(ang.gates(TH), ang.gates(THc))
    assert same(ang.tangents(TH, D), ang.tangents(THc, D))
    assert same(ang.pullback(TH, dt(Gt), dt(Gdt), V)[0], ang.pullback(THc, dt(Gt), dt(Gdt), V)[0])
    # one θ for every row of G, one G for every row of θ, one direction for every row
    rep = lambda x: x.unsqueeze(0).repeat((n,) + (1,) * x.dim()).contiguous()
    assert same(ang.pullback(THc[0], dt(Gt))[0], ang.pullback(rep(THc[0]), dt(Gt))[0])
    assert same(ang.pullback(THc[0], dt(Gt), dt(Gdt), V)[0], ang.pullback(rep(THc[0]), dt(Gt), dt(Gdt), V)[0])
    assert same(ang.pullback(THc, dt(Gt[0]))[0], ang.pullback(THc, dt(rep(Gt[0])))[0])
    assert same(ang.pullback(THc, dt(Gt[0]), dt(Gdt[0]), V)[0], ang.pullback(THc, dt(rep(Gt[0])), dt(rep(Gdt[0])), V)[0])
    assert same(ang.pullback(THc, dt(Gt), dt(Gdt), V[0])[0], ang.pullback(THc, dt(Gt), dt(Gdt), rep(V[0]))[0])
    assert same(ang.tangents(THc, D[0]), ang.tangents(THc, rep(D[0])))
    assert same(ang.tangents(THc[0], D), ang.tangents(rep(THc[0]), D))


def test_non_finite_angles(ctx, wide):
    import torch
    from tnc_b200 import DeviceTensor
    ang, info, inside = wide
    P, E, n = ang.n_params, ang.block_elems, 4
    rng = np.random.default_rng(13)
    theta = rng.uniform(-4, 4, (n, P))
    (la, ga, _, pa), (lb, gb, _, pb) = info[3], info[10]
    bad = theta.copy()
    bad[1, pa[-1]] = np.inf
    bad[2, pb[0]] = np.nan
    leaf_params = {(1, la): pa, (2, lb): pb}
    D = rng.standard_normal((n, P))
    V = rng.standard_normal((n, P))
    G = DeviceTensor.from_numpy(ctx, rng.standard_normal((n, E)) + 1j * rng.standard_normal((n, E)))
    Gd = DeviceTensor.from_numpy(ctx, rng.standard_normal((n, E)) + 1j * rng.standard_normal((n, E)))
    for call in (lambda t: ang.gates(cuda(t)), lambda t: ang.tangents(cuda(t), cuda(D))):
        good, got = call(theta).to_numpy(), call(bad).to_numpy()
        for (i, l), g in [((1, la), ga), ((2, lb), gb)]:
            sp = span(ang, l, g)
            assert not np.isfinite(got[i, sp]).all()
            got[i, sp] = good[i, sp]
        assert got.tobytes() == good.tobytes()
    for extra in [(), (Gd, cuda(V))]:
        good = ang.pullback(cuda(theta), G, *extra)[0].to_numpy()
        got = ang.pullback(cuda(bad), G, *extra)[0].to_numpy()
        for (i, l), ps in leaf_params.items():
            assert not np.isfinite(got[i, ps]).all()
            got[i, ps] = good[i, ps]
        assert got.tobytes() == good.tobytes()


# ------------------------------------------------------------------------------------------------ 4. parameter shifts
OMEGA = {"u": (0.5, 1.0, 1.0), "rx": (0.5,), "ry": (0.5,), "rz": (0.5,), "cp": (1.0,), "fsim": (1.0, 1.0)}


def shift_circuit(qubits=14, layers=3):
    from tnc_b200.builders import Circuit
    rng = np.random.default_rng(17)
    c = Circuit()
    q = c.allocate_register(qubits)
    for i in range(qubits):
        c.append_gate("h", [], [q[i]])
    singles = ["u", "rx", "ry", "rz"]
    for layer in range(layers):
        for i in range(qubits):
            g = singles[(i + layer) % 4]
            c.append_gate(g, list(rng.uniform(-3, 3, N_ANG[g])), [q[i]], adjoint=(i + layer) % 2 == 1)
            if g != "u":
                c.append_gate("u", list(rng.uniform(-3, 3, 3)), [q[i]], adjoint=i % 3 == 0)
        for i in range(layer % 2, qubits - 1, 2):
            g = "fsim" if (i // 2) % 2 == 0 else "cp"
            c.append_gate(g, list(rng.uniform(-3, 3, N_ANG[g])), [q[i], q[i + 1]], adjoint=(i + layer) % 3 == 0)
    return c.into_amplitude_network("0" * qubits)[0]


def test_exact_parameter_shifts(ctx):
    import torch
    from tnc_b200 import DeviceTensor
    from tnc_b200.angles import AngleMap, Angles
    from tnc_b200.tensornetwork import NetworkPlan, leaves
    from tnc_b200.tensornetwork.tensordata import TensorData
    tn = shift_circuit()
    path = greedy(tn)
    amap = AngleMap.every_angle(tn)
    P = amap.n_params
    assert P > 128
    lv = leaves(tn)
    omega = np.array([OMEGA[lv[l].tensordata.gate[0]][s] for l, s, _, _ in amap.refs])
    h = math.pi / (2 * omega)
    th0 = amap.theta0.copy()
    rng = np.random.default_rng(23)
    # shifted angle sets: ±h_p, +2h_p, and (±h_p, ±h_q) for 64 pairs, 16 of them on one leaf
    leaf_of = np.array([l for l, _, _, _ in amap.refs])
    same = [(p, q) for p in range(P) for q in range(p + 1, P) if leaf_of[p] == leaf_of[q]]
    other = [(p, q) for p in range(P) for q in range(p + 1, P) if leaf_of[p] != leaf_of[q]]
    pairs = [same[i] for i in rng.choice(len(same), 16, replace=False)] + [other[i] for i in rng.choice(len(other), 48, replace=False)]
    sets = [th0]
    for p in range(P):
        for sh in (h[p], -h[p], 2 * h[p]):
            t = th0.copy()
            t[p] += sh
            sets.append(t)
    for p, q in pairs:
        for sp_, sq_ in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
            t = th0.copy()
            t[p] += sp_ * h[p]
            t[q] += sq_ * h[q]
            sets.append(t)
    sets = np.array(sets)
    plain = NetworkPlan(tn, path, ctx=ctx)
    packed = Angles(ctx, tn, amap)
    packed.stage_instances(plain, tn, cuda(sets))
    R = plain.run_batch()[1].to_numpy().reshape(-1)
    scale = np.abs(R).max()
    assert abs(R[0]) > 1e-3 * scale
    # a few of them host-staged as Gate networks
    for k in (0, 1, 3 * P + 1):
        saved = {l: lv[l].tensordata for l in amap.leaves()}
        a = {l: list(td.gate[1]) for l, td in saved.items()}
        for l, s, p, _ in amap.refs:
            a[l][s] = sets[k, p]
        try:
            for l, td in saved.items():
                lv[l].set_tensor_data(TensorData.Gate(td.gate[0], tuple(a[l]), td.gate[2]))
            ref = complex(NetworkPlan(tn, path, ctx=ctx).execute(tn).to_numpy())
        finally:
            for l, td in saved.items():
                lv[l].set_tensor_data(td)
        assert abs(R[k] - ref) <= 1e-13 * scale, (k, R[k], ref)
    Rp, Rm, R2 = R[1:3 * P + 1:3], R[2:3 * P + 1:3], R[3:3 * P + 1:3]
    g_ref = omega * (Rp - Rm) / 2
    Hd_ref = -omega ** 2 * (R[0] - R2) / 2
    quad = R[3 * P + 1:].reshape(len(pairs), 4)
    Hpq_ref = np.array([omega[p] * omega[q] * (x[0] - x[1] - x[2] + x[3]) / 4 for (p, q), x in zip(pairs, quad)])
    tol = 1e-12 * scale
    T = cuda(th0)
    # the gradient: vjp + pullback
    gp = NetworkPlan.for_gradients(tn, path, wrt=amap.leaves(), ctx=ctx)
    gp.stage(tn)
    ag = Angles(ctx, tn, amap, gp)
    ag.set_leaves(gp, T)
    assert abs(complex(gp.run().to_numpy()) - R[0]) <= 1e-13 * scale
    g = ag.pullback(T, gp.vjp_block())[0].to_numpy()[0]
    note("parameter shift, gradient (1e-12 max|R|)", np.abs(g - g_ref).max() / tol)
    assert np.abs(g - g_ref).max() <= tol
    # the Jacobian: tangents(θ, eye(P)) + jvp_batch over P instances of the network at θ
    tp = NetworkPlan.for_tangents(tn, path, wrt=amap.leaves(), ctx=ctx)
    at = Angles(ctx, tn, amap, tp)
    at.stage_instances(tp, tn, cuda(np.repeat(th0[None], P, axis=0)))
    trows = at.tangents(T, cuda(np.eye(P)))
    out = C.c_void_p()
    assert ctx._l.tncb_plan_jvp_batch(ctx.handle, tp.handle, 0, P, trows.handle, None, C.byref(out)) == 0, ctx._l.tncb_last_error()
    J = DeviceTensor.adopt(ctx, out).to_numpy().reshape(-1)
    note("parameter shift, Jacobian (1e-12 max|R|)", np.abs(J - g_ref).max() / tol)
    assert np.abs(J - g_ref).max() <= tol
    # the Hessian: hvp_batch over the P directions e_p + one pullback
    hp = NetworkPlan.for_hvp(tn, path, wrt=amap.leaves(), ctx=ctx)
    hp.stage(tn)
    ah = Angles(ctx, tn, amap, hp)
    ah.set_leaves(hp, T)
    hrows = ah.tangents(T, cuda(np.eye(P)))
    Gr, Gdr = hvp_batch_rows(ctx, hp, P, hrows)
    H = ah.pullback(T, Gr, Gdr, cuda(np.eye(P)))[0].to_numpy()
    err = max(np.abs(np.diag(H) - Hd_ref).max(), max(abs(H[p, q] - r) for (p, q), r in zip(pairs, Hpq_ref)),
              max(abs(H[q, p] - r) for (p, q), r in zip(pairs, Hpq_ref)))
    note("parameter shift, Hessian (1e-12 max|R|)", err / tol)
    assert err <= tol
    note("Hessian symmetry (1e-12 max|R|)", np.abs(H - H.T).max() / tol)
    assert np.abs(H - H.T).max() <= tol
