"""The executors that serve repeated contractions, checked against the oracle and against the pair-by-pair executor.

A plan with a static layout (csrc/network.cpp: plan_static_layout / execute_static) re-orders its steps by tree level,
keeps every slot at a fixed offset of one workspace, runs all eligible tiny K0 pairs of a level as one k0_batch_kernel
launch, gives K0 split-K plan-owned scratch and, without K1 steps, replays CUDA graphs.  The pair-by-pair executor
(execute) is the reference: a plan created with TNCB_NO_STATIC=1 set uses it for every call, whatever the plan cache
has seen before.  The kernels are deterministic (fixed-order split-K, no atomics) and the batch kernel sums in the
order of k0_kernel, so the two executors must agree bit for bit.

  1. bench.py's network (36 qubits, 488 pairs) in every form the benchmark times: staged + run, execute, the cached
     plan behind contract_tensor_network, DMMA only, and sliced (run_slices with stride > 1, a rank with no slice).
  2. k0_batch_kernel at its edges: lane counts G = 1..32, K around the 1024-entry chunk of k0_kernel and the 4096 cap,
     M N K at the 2^22 cap, 8 and 9 fused leg groups, dim-1 legs, permuted strides, levels that mix batched and
     unbatched pairs, and a level with a single eligible pair.
  3. Graph replay while the payload changes between execute (graph with the upload) and stage + run (graph on resident
     leaves), and a sliced plan that replays its graph after the per-slice leaf copy."""
import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu


def to_oracle(t):
    if t.is_composite():
        return orc.OTensor(children=[to_oracle(c) for c in t.tensors])
    td = t.tensordata
    if td.kind == "gate":
        d = ("gate", td.gate[0], td.gate[1], td.gate[2])
    elif td.kind == "matrix":
        d = np.asarray(td.matrix)
    else:
        d = None
    return orc.OTensor(list(t.legs), list(t.bond_dims), d)


def to_opath(p):
    return orc.OPath(list(p.toplevel), {i: to_opath(q) for i, q in p.nested.items()})


def greedy(tn):
    from tnc_b200.contractionpath.paths import Cotengrust
    opt = Cotengrust(tn)
    opt.find_path()
    return opt.get_best_replace_path()


def pair_by_pair_plan(monkeypatch, tn, path, ctx):
    """A plan without a static layout: plan.execute runs the pair-by-pair executor.  plan_static_layout reads
    TNCB_NO_STATIC on every plan creation."""
    from tnc_b200.tensornetwork import NetworkPlan
    monkeypatch.setenv("TNCB_NO_STATIC", "1")
    try:
        return NetworkPlan(tn, path, ctx=ctx)
    finally:
        monkeypatch.delenv("TNCB_NO_STATIC")


def run_counted(ctx, fn):
    """(result as an array, engine counts, kernel launches) of one call"""
    ctx.reset_stats()
    res = fn().to_numpy()
    return res, ctx.engine_counts(), ctx.stats()["kernel_launches"]


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def replay_steps(built_lib, tn, path):
    """(a legs, a dims, b legs, b dims, kernel class, level) of every step of a flat replace-left path; level = 1 + the
    deepest level among the operands' producers (leaves: 0), as plan_static_layout computes it"""
    from tnc_b200._lib import u64_array
    assert not path.nested
    ts = [(list(t.legs), list(t.bond_dims), 0) for t in tn.tensors]
    out = []
    for i, j in path.toplevel:
        (al, ad, la), (bl, bd, lb) = ts[i], ts[j]
        cls = built_lib.tncb_pair_kernel_class(len(al), u64_array(al), u64_array(ad), len(bl), u64_array(bl), u64_array(bd))
        lv = max(la, lb) + 1
        out.append((al, ad, bl, bd, cls, lv))
        ts[i] = ([l for l in bl if l not in al] + [l for l in al if l not in bl],
                 [d for l, d in zip(bl, bd) if l not in al] + [d for l, d in zip(al, ad) if l not in bl], lv)
        ts[j] = None
    return out


# ================================================================================================================
# 1. the benchmark network through every executor
# ================================================================================================================
@pytest.fixture(scope="module")
def bench_net(built_lib):
    import bench
    tn = bench.build_network()
    return tn, bench.greedy_path(tn)


@pytest.fixture(scope="module")
def bench_oracle(bench_net):
    import torch
    tn, path = bench_net
    torch.set_num_threads(max(1, min(16, torch.get_num_threads())))
    return complex(orc.contract_tensor_network(to_oracle(tn), to_opath(path), backend="torch").data)


@pytest.fixture(scope="module")
def bench_pair_by_pair(bench_net):
    """The pair-by-pair executor on the benchmark network: default engines, then DMMA only."""
    import tnc_b200 as tb
    tn, path = bench_net
    c = tb.Context(0)
    try:
        with pytest.MonkeyPatch.context() as mp:
            plan = pair_by_pair_plan(mp, tn, path, c)
        amp, ec, launches = run_counted(c, lambda: plan.execute(tn))
        c.set_tcgen05_slices(0)
        amp_dmma, ec_dmma, _ = run_counted(c, lambda: plan.execute(tn))
        del plan
    finally:
        c.close()
    return {"amp": complex(amp), "ec": ec, "launches": launches, "amp_dmma": complex(amp_dmma), "ec_dmma": ec_dmma}


def close_to(got, ref, rel):
    return abs(got - ref) <= rel * abs(ref)


def test_bench_pair_by_pair_reference(bench_oracle, bench_pair_by_pair):
    r = bench_pair_by_pair
    assert close_to(r["amp"], bench_oracle, 1e-9), (r["amp"], bench_oracle)        # rel 1e-9 on amplitudes (SURVEY 8d)
    assert close_to(r["amp_dmma"], bench_oracle, 1e-9), (r["amp_dmma"], bench_oracle)
    ec = r["ec"]
    assert ec["k1_tcgen05"] >= 1 and ec["k1_dmma_splitk"] >= 1 and ec["k0_splitk"] >= 1, ec
    assert r["ec_dmma"]["k1_tcgen05"] == 0 and r["ec_dmma"]["k1_dmma"] >= 1, r["ec_dmma"]
    assert r["launches"] >= 488, r["launches"]


def test_bench_static_plan_resident_and_upload(bench_net, bench_oracle, bench_pair_by_pair):
    """bench.py's `value`: NetworkPlan + stage + run (three times), the DMMA-only run of the `dmma_only` extra, then
    execute (with the upload; it replaces the staged leaves), all on one static plan."""
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import NetworkPlan
    tn, path = bench_net
    ref = bench_pair_by_pair
    c = tb.Context(0)
    try:
        plan = NetworkPlan(tn, path, ctx=c)
        plan.stage(tn)
        runs = [run_counted(c, plan.run) for _ in range(3)]
        c.set_tcgen05_slices(0)
        try:
            dmma, ec_dmma, _ = run_counted(c, plan.run)
        finally:
            c.set_tcgen05_slices(8)
        up = complex(plan.execute(tn).to_numpy())
        del plan
    finally:
        c.close()
    for amp, ec, launches in runs:
        amp = complex(amp)
        assert close_to(amp, bench_oracle, 1e-9), (amp, bench_oracle)
        assert amp == ref["amp"], (amp, ref["amp"])                          # same kernels, same sums
        assert ec == ref["ec"], (ec, ref["ec"])                               # no engine fell back inside the static workspace
        assert launches < ref["launches"], (launches, ref["launches"])        # the tiny pairs ran in batches
    assert up == ref["amp"], (up, ref["amp"])
    dmma = complex(dmma)
    assert ec_dmma["k1_tcgen05"] == 0, ec_dmma
    assert close_to(dmma, bench_oracle, 1e-9), (dmma, bench_oracle)
    assert dmma == ref["amp_dmma"], (dmma, ref["amp_dmma"])


def test_bench_cached_plan_e2e(bench_net, bench_oracle, bench_pair_by_pair):
    """bench.py's `e2e`: repeated contract_tensor_network calls; from the second sighting of the structure on, the
    context's plan cache serves them with a static plan."""
    import tnc_b200 as tb
    from tnc_b200.tensornetwork import contract_tensor_network
    tn, path = bench_net
    ref = bench_pair_by_pair
    c = tb.Context(0)
    try:
        runs = [run_counted(c, lambda: contract_tensor_network(tn, path, ctx=c)) for _ in range(3)]
    finally:
        c.close()
    for amp, _, _ in runs:
        assert complex(amp) == ref["amp"], (complex(amp), ref["amp"])
    assert runs[2][1] == ref["ec"], (runs[2][1], ref["ec"])
    assert runs[2][2] < ref["launches"], (runs[2][2], ref["launches"])       # the cached static plan ran it


def test_bench_sliced_plan(bench_net, bench_oracle):
    """bench.py's `sliced8_on_1gpu`: the slice loop inside the library, all slices and round-robin subsets of them."""
    import tnc_b200 as tb
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    tn, path = bench_net
    c = tb.Context(0)
    try:
        sp = SlicedPlan(tn, path, find_slices(tn, path, min_slices=8), ctx=c)
        assert sp.n_slices >= 8
        total = sp.run().to_numpy()
        parts = [sp.plan.run_slices(r, 3).to_numpy() for r in range(3)]
        # a rank past the last slice: an earlier result's freed block is the first candidate for its output
        sp.plan.run_slices(1, 1).tensordata.matrix.free()
        empty = sp.plan.run_slices(sp.n_slices, 1).to_numpy()
        del sp
    finally:
        c.close()
    amp = complex(total)
    assert close_to(amp, bench_oracle, 1e-9), (amp, bench_oracle)
    s = complex(parts[0] + parts[1] + parts[2])
    assert close_to(s, amp, 1e-12), (s, amp)
    assert empty.shape == total.shape and not np.any(empty), empty


# ================================================================================================================
# 2. k0_batch_kernel at its edges
# ================================================================================================================
BATCH_GROUPS = 8          # kBatchGroups
BATCH_MAX_K = 4096
BATCH_MAX_MNK = 1 << 22


def k0_config(sms, M, N, K):
    """kernels.cu k0_config: (G lanes per output, K ranges)"""
    MN, target = M * N, sms * 1024
    G = 1
    while G < 32 and MN * G < target and G * 2 <= K:
        G *= 2
    ksplit, per_lane = 1, K // G
    if MN * G < target and per_lane > 64:
        ksplit = max(1, min(min(target // max(1, MN * G), per_lane // 32), 1024))
    kchunk = (K + ksplit - 1) // ksplit
    return G, (K + kchunk - 1) // kchunk


def fused_groups(al, ad, bl, bd):
    """plan.cpp plan_pair: fused leg groups of the m, n and k lists (dim-1 legs dropped, neighbours that are contiguous
    in every operand they index merged; the k list in a's or b's order, whichever fuses into fewer groups)"""
    def strides(dims):
        s, out = 1, [0] * len(dims)
        for i in range(len(dims) - 1, -1, -1):
            out[i] = s
            s *= dims[i]
        return out

    def fuse(v, use_b):
        out = []
        for d, s1, s2 in v:
            if d == 1:
                continue
            if out and out[-1][1] == s1 * d and (not use_b or out[-1][2] == s2 * d):
                out[-1] = (out[-1][0] * d, s1, s2)
                continue
            out.append((d, s1, s2))
        return out
    sa, sb = strides(ad), strides(bd)
    m = fuse([(d, s, 0) for l, d, s in zip(al, ad, sa) if l not in bl], False)
    n = fuse([(d, s, 0) for l, d, s in zip(bl, bd, sb) if l not in al], False)
    ka = fuse([(d, s, sb[bl.index(l)]) for l, d, s in zip(al, ad, sa) if l in bl], True)
    kb = fuse([(ad[al.index(l)], sa[al.index(l)], s) for l, s in zip(bl, sb) if l in al], True)
    return len(m), len(n), len(kb) if len(kb) < len(ka) else len(ka)


def mnk(al, ad, bl, bd):
    M = int(np.prod([d for l, d in zip(al, ad) if l not in bl], dtype=np.int64))
    N = int(np.prod([d for l, d in zip(bl, bd) if l not in al], dtype=np.int64))
    K = int(np.prod([d for l, d in zip(al, ad) if l in bl], dtype=np.int64))
    return M, N, K


def batch_landing(sms, al, ad, bl, bd, cls):
    """kernels.cu k0_batch_eligible + the G of the batch item: (batched, G, K ranges)"""
    M, N, K = mnk(al, ad, bl, bd)
    G, ksplit = k0_config(sms, M, N, K)
    ok = (cls == 0 and M * N > 0 and max(fused_groups(al, ad, bl, bd)) <= BATCH_GROUPS and K <= BATCH_MAX_K
          and M * N * K <= BATCH_MAX_MNK and ksplit == 1)
    return ok, G, ksplit


def interleaved(free, kname, n):
    """f0 k0 f1 k1 ... : no two free legs and no two shared legs are neighbours, so none of them fuse"""
    return " ".join(f"{free}{i} {kname}{i}" for i in range(n))


def two(prefix, n):
    return {f"{prefix}{i}": 2 for i in range(n)}


# (name, a legs, b legs, dims, intended (batched, G)).  Legs named m* are a's free legs, n* b's, everything else shared.
# M N K and G on a 132-SM H100; the shapes stay K0 (M < 16, N < 16 or M N K < 2^17) and off K2.
CASES = {
    "G1_K1": ("m0", "n0", {"m0": 37, "n0": 11}, (True, 1)),                                      # M N = 407
    "G2": ("m0 k0", "k0 n0", {"m0": 50, "n0": 9, "k0": 3}, (True, 2)),                           # M N = 450
    "G4": ("k0 m0", "n0 k0", {"m0": 33, "n0": 3, "k0": 5}, (True, 4)),
    "G8_permuted": ("k1 m1 k0 m0", "n1 k0 n0 k1", {"m0": 4, "m1": 5, "n0": 2, "n1": 3, "k0": 3, "k1": 4}, (True, 8)),
    "G16_dim1": ("m0 u0 k0 m1", "k0 n0 u0 n1", {"m0": 7, "m1": 1, "n0": 13, "n1": 1, "k0": 24, "u0": 1}, (True, 16)),
    "G16_by_MN": ("m0 k0", "k0 n0", {"m0": 1250, "n0": 8, "k0": 64}, (True, 16)),                # M N G reaches the target
    "G32": ("m0 k0", "n0 k0", {"m0": 129, "n0": 7, "k0": 64}, (True, 32)),
    "K1023": ("m0 k0", "k0 n0", {"m0": 300, "n0": 3, "k0": 1023}, (True, 32)),
    "K1024_permuted": ("k0 m0 k1", "k1 n0 k0", {"m0": 100, "n0": 5, "k0": 32, "k1": 32}, (True, 32)),
    "K1025": ("m0 k0 k1", "k0 k1 n0", {"m0": 64, "n0": 9, "k0": 5, "k1": 205}, (True, 32)),
    "MNK_2p22": ("m0 k0 m1", "k0", {"m0": 64, "m1": 64, "k0": 1024}, (True, 32)),                # M N K = 2^22 exactly
    "MNK_above": ("m0 k0", "k0", {"m0": 4097, "k0": 1024}, (False, 32)),                         # 2^22 + 1024
    "K4096_splitk": ("m0 k0 k1", "n0 k1 k0", {"m0": 3, "n0": 5, "k0": 64, "k1": 64}, (False, 32)),   # split-K: never batched
    "K4097": ("k0 m0", "n0 k0", {"m0": 2, "n0": 3, "k0": 4097}, (False, 32)),
    "MN1": ("k0 k1", "k1 k0", {"k0": 6, "k1": 7}, (True, 32)),                                   # scalar output
    "groups_m8": (interleaved("m", "k", 8), "n0 " + " ".join(f"k{i}" for i in (5, 2, 7, 0, 3, 6, 1, 4)),
                  {**two("m", 8), **two("k", 8), "n0": 2}, (True, 32)),
    "groups_n8": ("m0 " + " ".join(f"k{i}" for i in (3, 7, 1, 5, 0, 4, 2, 6)), interleaved("n", "k", 8),
                  {**two("n", 8), **two("k", 8), "m0": 2}, (True, 32)),
    "groups_m9": (interleaved("m", "k", 9), "n0 " + " ".join(f"k{i}" for i in (8, 4, 0, 6, 2, 7, 3, 5, 1)),
                  {**two("m", 9), **two("k", 9), "n0": 2}, (False, 32)),
}

# Each network's first level mixes batched and unbatched pairs; the probe pairs form the second batched level.
BATCH_NETWORKS = {
    "lanes": ["G1_K1", "G2", "G4", "G8_permuted", "G16_dim1", "G32", "MNK_above"],
    "long_k": ["G16_by_MN", "K1023", "K1024_permuted", "K1025", "K4096_splitk", "K4097"],
    "caps_groups": ["MNK_2p22", "MN1", "groups_m8", "groups_n8", "groups_m9"],
    "single_eligible": ["G32", "groups_m9"],                 # level 1 holds one eligible pair: a plain launch
}


def batch_network(names, seed):
    """Leaves a_c, b_c of every case, then one probe per case.  Level 1: the case pairs.  Level 2: each case output
    against its probe, a random tensor over all of the output's legs and one new dim-2 witness leg, so every output
    entry reaches the witness vector with two random weights.  Then the witness vectors' outer products, pairwise, up to
    2^len(names) entries."""
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(seed)

    def leaf(legs, dims):
        t = Tensor(legs, dims)
        t.set_tensor_data(TensorData.Matrix(rng.standard_normal(dims) + 1j * rng.standard_normal(dims)))
        return t

    pairs, probes, next_id = [], [], 0
    for name in names:
        a_spec, b_spec, dims, _ = CASES[name]
        ids = {}
        for leg in (a_spec + " " + b_spec).split():
            if leg not in ids:
                ids[leg] = next_id
                next_id += 1
        al, bl = [ids[l] for l in a_spec.split()], [ids[l] for l in b_spec.split()]
        ad, bd = [dims[l] for l in a_spec.split()], [dims[l] for l in b_spec.split()]
        pairs += [leaf(al, ad), leaf(bl, bd)]
        out = [(l, d) for l, d in zip(bl, bd) if l not in al] + [(l, d) for l, d in zip(al, ad) if l not in bl]
        probes.append(leaf([next_id] + [l for l, _ in out], [2] + [d for _, d in out]))    # (one k group: batchable)
        next_id += 1
    n = len(names)
    steps = [(2 * c, 2 * c + 1) for c in range(n)] + [(2 * c, 2 * n + c) for c in range(n)]
    slots = [2 * c for c in range(n)]
    while len(slots) > 1:
        steps += [(slots[q], slots[q + 1]) for q in range(0, len(slots) - 1, 2)]
        slots = slots[::2]
    return Tensor.new_composite(pairs + probes), ContractionPath.simple(steps)


@pytest.fixture(scope="module")
def small_ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    yield c
    c.close()


def test_batch_cases_land_where_intended(built_lib):
    """The mirror of k0_config / k0_batch_eligible puts every case where its name says, and the set covers every G."""
    sms = sm_count()
    pair = {}
    for name, (_, _, _, want) in CASES.items():
        tn, path = batch_network([name], 0)
        al, ad, bl, bd, cls, _ = pair[name] = replay_steps(built_lib, tn, path)[0]
        assert cls == 0, (name, cls)
        ok, G, ksplit = batch_landing(sms, al, ad, bl, bd, cls)
        assert (ok, G) == want, (name, ok, G, ksplit, mnk(al, ad, bl, bd))
    assert {w[1] for *_, w in CASES.values() if w[0]} == {1, 2, 4, 8, 16, 32}
    groups = {name: fused_groups(*pair[name][:4]) for name in ("groups_m8", "groups_n8", "groups_m9", "G16_dim1")}
    assert groups == {"groups_m8": (8, 1, 8), "groups_n8": (1, 8, 8), "groups_m9": (9, 1, 9), "G16_dim1": (1, 1, 1)}, groups
    assert mnk(*pair["MNK_2p22"][:4]) == (4096, 1, 1024) and mnk(*pair["MN1"][:4])[:2] == (1, 1)
    assert batch_landing(sms, *pair["K4096_splitk"][:5])[2] > 1                # K0 split-K on plan-owned scratch


@pytest.mark.parametrize("net", list(BATCH_NETWORKS))
def test_k0_batch_network(built_lib, small_ctx, monkeypatch, net):
    """The static plan (batched levels, graph replay) against the pair-by-pair executor bit for bit and against the
    numpy oracle normwise; the launch count shows which levels ran as one batch."""
    from tnc_b200.tensornetwork import NetworkPlan
    names = BATCH_NETWORKS[net]
    tn, path = batch_network(names, 17 + len(net))
    steps = replay_steps(built_lib, tn, path)
    sms = sm_count()
    assert all(s[4] == 0 for s in steps), [s[4] for s in steps]
    n_levels = max(s[5] for s in steps)
    batched = [0] * n_levels
    for al, ad, bl, bd, cls, lv in steps:
        batched[lv - 1] += batch_landing(sms, al, ad, bl, bd, cls)[0]
    batched = [b if b >= 2 else 0 for b in batched]                          # a batch of one is a plain launch
    saved = sum(b - 1 for b in batched if b)
    lvl1 = [batch_landing(sms, *s[:5])[0] for s in steps if s[5] == 1]
    if net == "single_eligible":
        assert lvl1.count(True) == 1 and batched[0] == 0, lvl1
    else:
        assert 2 <= lvl1.count(True) < len(lvl1) and batched[1] >= 2, (lvl1, batched)

    eager = pair_by_pair_plan(monkeypatch, tn, path, small_ctx)
    ref, _, l_ref = run_counted(small_ctx, lambda: eager.execute(tn))
    assert l_ref >= len(steps)
    plan = NetworkPlan(tn, path, ctx=small_ctx)
    assert plan.info()["kernels"] == len(steps) - saved, (plan.info(), saved)
    got, _, l_got = run_counted(small_ctx, lambda: plan.execute(tn))
    again = plan.execute(tn).to_numpy()
    assert l_got == l_ref - saved, (l_got, l_ref, saved)
    assert np.array_equal(got, ref) and np.array_equal(again, ref)
    exp = orc.contract_tensor_network(to_oracle(tn), to_opath(path))
    assert got.shape == exp.data.shape and got.size == 2 ** len(names)
    assert np.linalg.norm(got - exp.data) <= 1e-12 * np.linalg.norm(exp.data), np.linalg.norm(got - exp.data) / np.linalg.norm(exp.data)


# ================================================================================================================
# 3. graph replay with changing payloads
# ================================================================================================================
def statevector_payload(tn, seed):
    """The 13-qubit statevector network with random normalised input states in place of |0>: same structure, new
    payload"""
    from tnc_b200.tensornetwork import Tensor
    from tnc_b200.tensornetwork.tensordata import TensorData
    rng = np.random.default_rng(seed)
    out = []
    for t in tn.tensors:
        if len(t.legs) == 1:
            v = rng.standard_normal(2) + 1j * rng.standard_normal(2)
            t = Tensor(t.legs, t.bond_dims)
            t.set_tensor_data(TensorData.Matrix(v / np.linalg.norm(v)))
        out.append(t)
    return Tensor.new_composite(out)


@pytest.fixture(scope="module")
def replay_net(built_lib):
    """13 qubits, 4 rounds, seed 4: the greedy path has K0 steps and one K2 step (gate against the 2^13 state) and no
    K1 step, so its static plan is captured into graphs (a 12-qubit network never reaches the K2 shape, M >= 4096)."""
    from tnc_b200.builders import random_circuit_builder
    tn, _ = random_circuit_builder(13, 4, 0.5, 0.5, np.random.default_rng(4)).into_statevector_network()
    path = greedy(tn)
    classes = [s[4] for s in replay_steps(built_lib, tn, path)]
    assert set(classes) == {0, 2}, classes
    return tn, path


@pytest.mark.parametrize("order", ["upload_first", "resident_first"])
def test_graph_replay_payload_switching(replay_net, small_ctx, monkeypatch, order):
    """execute uploads the leaves inside its graph (exec[0]), stage + run replays the graph without the upload
    (exec[1]).  Every call must see its own payload, whichever graph was captured first."""
    from tnc_b200.tensornetwork import NetworkPlan
    tn0, path = replay_net
    seq = {"upload_first": ["execute", "execute", "stage", "run", "run", "execute", "stage", "run"],
           "resident_first": ["stage", "run", "execute", "execute", "stage", "run", "run", "execute"]}[order]
    eager = pair_by_pair_plan(monkeypatch, tn0, path, small_ctx)
    plan = NetworkPlan(tn0, path, ctx=small_ctx)
    seed, payload = 100, None
    for op in seq:
        if op in ("execute", "stage"):
            seed += 1
            payload = statevector_payload(tn0, seed)
        if op == "stage":
            plan.stage(payload)
            continue
        res = plan.execute(payload) if op == "execute" else plan.run()
        got = res.to_numpy()
        ref = eager.execute(payload).to_numpy()
        exp = orc.contract_tensor_network(to_oracle(payload), to_opath(path))
        assert res.legs == exp.legs
        assert np.array_equal(got, ref), (op, seed)
        assert np.abs(got - exp.data).max() <= 1e-12 * np.abs(exp.data).max() + 1e-18, (op, seed)
        assert abs(np.vdot(got, got) - 1) <= 1e-12                          # a unitary circuit on a normalised state


def test_sliced_graph_replay(built_lib, small_ctx):
    """A sliced plan without K1 steps: every slice copies its leaf block into the workspace and replays the graph on
    resident leaves."""
    from tnc_b200.builders import random_circuit_builder
    from tnc_b200.contractionpath.slicing import SlicedPlan, find_slices
    tn, _ = random_circuit_builder(12, 6, 0.5, 0.5, np.random.default_rng(9)).into_amplitude_network("010011100101")
    path = greedy(tn)
    legs = find_slices(tn, path, min_slices=4)
    sp = SlicedPlan(tn, path, legs, ctx=small_ctx)
    assert sp.n_slices >= 4
    assert {s[4] for s in replay_steps(built_lib, sp.sn.slice(sp.sn.assignments[0]), path)} == {0}
    ref = complex(orc.contract_tensor_network(to_oracle(tn), to_opath(path)).data)
    for _ in range(2):
        got = complex(sp.run().to_numpy())
        assert abs(got - ref) <= 1e-12 * abs(ref) + 1e-18, (got, ref)
    halves = complex(sp.plan.run_slices(0, 2).to_numpy()) + complex(sp.plan.run_slices(1, 2).to_numpy())
    assert abs(halves - ref) <= 1e-12 * abs(ref) + 1e-18, (halves, ref)
