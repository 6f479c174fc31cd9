"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle on the
same seeded inputs, against the reference's golden vectors, and -- at BASELINE's full C2 size --
through size-independent properties (checksum of checksums, sampled entries).

Tolerances: KATs abs 1e-14 (tnc/src/tensornetwork/contraction.rs:172,177,223); everything else
||gpu-cpu||_inf <= 1e-12 * max(1, ||cpu||_inf) (SURVEY 8d allows 1e-10)."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu
RTOL = 1e-12


def rand_c(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def check_pair(ctx, rng, a_legs, a_dims, b_legs, b_dims, tol=RTOL):
    import tnc_b200 as tb
    a, b = rand_c(rng, a_dims), rand_c(rng, b_dims)
    legs, got = tb.contract_pair(ctx, a_legs, a, b_legs, b)
    ref_legs, ref = orc.contract_pair(a_legs, a, b_legs, b)
    assert legs == ref_legs
    assert got.shape == ref.shape
    err = np.abs(got - ref).max() if ref.size else 0.0
    assert err <= tol * max(1.0, np.abs(ref).max() if ref.size else 1.0), (a_legs, a_dims, b_legs, b_dims, err)


# ---- reference KATs through the C ABI ----------------------------------------------------------
def test_kat_pairs(ctx, kat):
    import tnc_b200 as tb
    legs, got = tb.contract_pair(ctx, kat["A"]["legs"], kat["A"]["data"], kat["B"]["legs"], kat["B"]["data"])
    assert legs == kat["AxB"]["legs"] and list(got.shape) == kat["AxB"]["shape"]
    assert np.abs(got - kat["AxB"]["data"]).max() <= 1e-14
    legs, got = tb.contract_pair(ctx, kat["B"]["legs"], kat["B"]["data"], kat["C"]["legs"], kat["C"]["data"])
    assert legs == kat["BxC"]["legs"] and list(got.shape) == kat["BxC"]["shape"]
    assert np.abs(got - kat["BxC"]["data"]).max() <= 1e-14


def _leaf(t):
    from tnc_b200.tensornetwork import Tensor, TensorData
    x = Tensor(t["legs"], t["shape"])
    x.set_tensor_data(TensorData.new_from_data(t["shape"], t["data"].reshape(-1)))
    return x


def test_kat_network(ctx, kat):
    from tnc_b200.contractionpath import path
    from tnc_b200.tensornetwork import Tensor, contract_tensor_network
    tn = Tensor.new_composite([_leaf(kat["A"]), _leaf(kat["B"]), _leaf(kat["C"])])
    res = contract_tensor_network(tn, path((0, 1), (0, 2)), ctx=ctx)
    assert res.legs == kat["ABxC"]["legs"] and res.bond_dims == kat["ABxC"]["shape"]
    assert np.abs(res.to_numpy() - kat["ABxC"]["data"]).max() <= 1e-14


def test_kat_outer_product(ctx):
    from tnc_b200.contractionpath import path
    from tnc_b200.tensornetwork import Tensor, TensorData, contract_tensor_network
    t1 = Tensor([0], [3]); t1.set_tensor_data(TensorData.new_from_data([3], [1, 2 + 5j, 3 - 1j]))
    t2 = Tensor([1], [2]); t2.set_tensor_data(TensorData.new_from_data([2], [-4 + 2j, -1j]))
    res = contract_tensor_network(Tensor.new_composite([t1, t2]), path((0, 1)), ctx=ctx)
    assert res.legs == [1, 0] and res.bond_dims == [2, 3]
    exp = np.array([-4 + 2j, -18 - 16j, -10 + 10j, -1j, 5 - 2j, -1 - 3j]).reshape(2, 3)
    assert np.array_equal(res.to_numpy(), exp)  # exact small integers


# ---- pair sweeps ------------------------------------------------------------------------------
def test_pairs_edge_cases(ctx):
    rng = np.random.default_rng(1)
    check_pair(ctx, rng, [], [], [], [])                       # scalar x scalar
    check_pair(ctx, rng, [], [], [0, 1], [3, 4])               # scalar x tensor
    check_pair(ctx, rng, [0, 1], [3, 4], [], [])               # tensor x scalar
    check_pair(ctx, rng, [0], [5], [0], [5])                   # inner product -> scalar
    check_pair(ctx, rng, [0, 1], [1, 4], [1, 2], [4, 1])       # dim-1 legs
    check_pair(ctx, rng, [0, 1, 2], [2, 2, 2], [2, 1, 0], [2, 2, 2])  # full contraction, permuted
    check_pair(ctx, rng, [0, 1], [7, 3], [5, 6], [2, 5])       # outer product, odd dims
    check_pair(ctx, rng, [3, 0], [6, 5], [0], [5])             # matrix-vector
    check_pair(ctx, rng, [0], [5], [0, 3], [5, 6])             # vector-matrix


def test_pairs_random_small(ctx):
    rng = np.random.default_rng(2)
    for _ in range(60):
        na, nb = int(rng.integers(0, 6)), int(rng.integers(0, 6))
        ids = [int(x) for x in rng.permutation(10)]
        a_legs = ids[:na]
        nshared = int(rng.integers(0, min(na, nb) + 1))
        shared = [int(x) for x in rng.permutation(a_legs)[:nshared]] if na else []
        b_free = ids[na:na + nb - nshared]
        b_legs = [int(x) for x in rng.permutation(shared + b_free)]
        dim = {i: int(rng.integers(1, 6)) for i in range(10)}
        check_pair(ctx, rng, a_legs, [dim[l] for l in a_legs], b_legs, [dim[l] for l in b_legs])


def test_pairs_k0_split_k(ctx):
    rng = np.random.default_rng(3)
    # few outputs, long K: exercises G=32 lanes and the deterministic split-K reduction
    check_pair(ctx, rng, list(range(16)), [2] * 16, list(range(15, -1, -1)), [2] * 16)  # scalar, K=65536
    check_pair(ctx, rng, [0, 1, 2, 3], [2, 31, 37, 29], [3, 2, 1, 9], [29, 37, 31, 3])   # K=33263, N=3, M=2
    check_pair(ctx, rng, list(range(18)) + [30], [2] * 19, list(range(17, -1, -1)) + [31], [2] * 19)  # 2x2 out, K=2^18


def test_pairs_k0_streaming(ctx):
    rng = np.random.default_rng(4)
    # gate-application shapes: big tensor x tiny gate (low intensity, stays on K0)
    big = list(range(16))
    check_pair(ctx, rng, big, [2] * 16, [3, 7, 20, 21], [2, 2, 2, 2])
    check_pair(ctx, rng, [3, 7, 20, 21], [2, 2, 2, 2], big, [2] * 16)
    check_pair(ctx, rng, big, [2] * 16, [15, 22], [2, 2])


def test_pairs_k2_streaming_kernel(ctx, built_lib):
    """K2 (big tensor x tiny tensor, HBM-bound): power-of-two and odd dims, both orientations,
    N (or M) not a power of two, K = 1 (outer product with a big operand)."""
    from tnc_b200._lib import u64_array
    rng = np.random.default_rng(41)
    def cls(a_legs, a_dims, b_legs, b_dims):
        return built_lib.tncb_pair_kernel_class(len(a_legs), u64_array(a_legs), u64_array(a_dims), len(b_legs), u64_array(b_legs), u64_array(b_dims))
    cases = [
        (list(range(14)), [2] * 14, [3, 20, 9, 21], [2, 2, 2, 2]),            # big A, gate on legs 3 and 9
        ([3, 20, 9, 21], [2, 2, 2, 2], list(range(14)), [2] * 14),            # big B
        ([0, 1, 2, 3], [15, 17, 9, 33], [2, 9], [9, 3]),                      # odd dims: M = 15*17*33, N = 3, K = 9
        ([9, 2], [3, 9], [0, 1, 2, 3], [15, 17, 9, 33]),                      # same, big B, M = 3
        (list(range(13)), [2] * 13, [40], [5]),                               # K = 1: outer product, N = 5
        ([0, 1, 2], [64, 64, 3], [2, 5, 6], [3, 2, 3]),                       # N = 6 (not a power of two)
    ]
    for a_legs, a_dims, b_legs, b_dims in cases:
        assert cls(a_legs, a_dims, b_legs, b_dims) == 2, (a_legs, b_legs)
        check_pair(ctx, rng, a_legs, a_dims, b_legs, b_dims)


def test_pairs_k2_large_operands(ctx, built_lib):
    """K2 with >= 2^16 free elements on the big side: orientations, K = 1..16, NS = 1..16, scattered K legs, odd dims and
    a ragged last block, against the oracle.  launch_k2 caps the grid at 32 blocks of 256 threads per SM, so only the
    2^23 case (BIG >= 4 * 256 * 32 * SMs) makes every thread take several grid-stride trips."""
    import torch
    from tnc_b200._lib import u64_array
    rng = np.random.default_rng(43)
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    def cls(a_legs, a_dims, b_legs, b_dims):
        return built_lib.tncb_pair_kernel_class(len(a_legs), u64_array(a_legs), u64_array(a_dims), len(b_legs), u64_array(b_legs), u64_array(b_dims))
    cases = [
        (list(range(20)), [2] * 20, [3, 17, 9, 12, 30, 31, 32, 33], [2] * 8),         # 2^16 x 16 x 16, big A, K legs scattered
        ([3, 17, 9, 12, 30, 31, 32, 33], [2] * 8, list(range(20)), [2] * 20),         # same, big B
        (list(range(19)), [2] * 19, [18, 17, 16, 40], [2, 2, 2, 2]),                  # K = 8 on the fastest legs, NS = 2
        (list(range(18)), [2] * 18, [0, 40, 41, 42, 43], [2] * 5),                    # K = 2 on the slowest leg, NS = 16
        ([0, 1, 2, 3], [37, 41, 7, 47], [2, 9], [7, 5]),                              # odd dims: BIG = 37*41*47 = 71299 (ragged block), K = 7, NS = 8 (5 used)
        ([9, 2], [3, 11], [0, 1, 2, 3], [29, 53, 11, 59]),                            # big B, M = 3, K = 11
        (list(range(17)), [2] * 17, [40], [13]),                                      # K = 1: outer product with a 2^17 operand, NS = 16 (13 used)
        (list(range(24)), [2] * 24, [9], [2]),                                        # BIG = 2^23, K = 2 on a middle leg, NS = 1 (256 MiB)
    ]
    for a_legs, a_dims, b_legs, b_dims in cases:
        assert cls(a_legs, a_dims, b_legs, b_dims) == 2, (a_legs, b_legs)
        ctx.reset_stats()
        check_pair(ctx, rng, a_legs, a_dims, b_legs, b_dims)
        assert ctx.engine_counts()["k2"] == 1
    big = 2 ** 23
    blocks = min((big + 255) // 256, 32 * sm_count)
    assert -(-big // (256 * blocks)) >= 4, (sm_count, blocks)     # grid-stride trips per thread of the last case


@pytest.mark.parametrize("mode", ["interleaved", "a_suffix_b_prefix", "a_prefix_b_suffix", "reversed"])
def test_pairs_k1_modes(ctx, mode):
    """K1 (gather + DMMA ZGEMM) under the four loader-mode combinations, dims 2 and 4."""
    rng = np.random.default_rng(5)
    for d, nfree, nsh in [(2, 7, 6), (4, 3, 3), (2, 8, 4)]:
        sh = list(range(100, 100 + nsh)); af = list(range(nfree)); bf = list(range(50, 50 + nfree))
        if mode == "interleaved":
            a_legs = [x for p in zip(af, sh) for x in p] + af[nsh:] + sh[nfree:]
            b_legs = [x for p in zip(reversed(sh), bf) for x in p] + bf[nsh:]
        elif mode == "a_suffix_b_prefix":   # GEMM-ready: no permute needed
            a_legs = af + sh; b_legs = sh + bf
        elif mode == "a_prefix_b_suffix":
            a_legs = sh + af; b_legs = bf + sh
        else:
            a_legs = list(reversed(sh)) + list(reversed(af)); b_legs = list(reversed(bf)) + sh
        a_legs = list(dict.fromkeys(a_legs)); b_legs = list(dict.fromkeys(b_legs))
        check_pair(ctx, rng, a_legs, [d] * len(a_legs), b_legs, [d] * len(b_legs))


def test_pairs_k1_ragged(ctx):
    """K1 with M, N, K that are not multiples of the tile (predicated loads/stores)."""
    rng = np.random.default_rng(6)
    check_pair(ctx, rng, [0, 1, 2], [7, 11, 13], [2, 3, 1], [13, 23, 11])       # M=7, N=23, K=143 -> K0 (M<16)
    check_pair(ctx, rng, [0, 1, 2], [37, 11, 13], [2, 3, 1], [13, 71, 11])      # M=37, N=71, K=143
    check_pair(ctx, rng, [0, 1, 2, 3], [5, 9, 7, 3], [3, 4, 1, 5], [3, 33, 9, 5])  # M=35, N=165, K=27
    check_pair(ctx, rng, [0, 1], [130, 67], [1, 2], [67, 257])                  # M=130, N=257, K=67
    check_pair(ctx, rng, [0, 1], [1000, 5], [1, 2], [5, 300])                   # K=5 (< BK)
    check_pair(ctx, rng, [0, 1], [64, 300], [1, 2], [300, 384])                 # big-tile config candidates


def test_pair_k1_large_tile_config(ctx):
    rng = np.random.default_rng(7)
    # enough tiles for the 128x64 configuration (>= 2 waves): M=2048, N=2048, K=64
    a_legs = [0, 1, 2]; b_legs = [3, 2, 4, 0]
    check_pair(ctx, rng, a_legs, [8, 2048, 8], b_legs, [32, 8, 64, 8])
    check_pair(ctx, rng, [0, 1], [96, 2048 + 40], [2, 0], [4096 + 24, 96])


# ---- networks ---------------------------------------------------------------------------------
def chain(n):
    from tnc_b200.contractionpath import ContractionPath
    return ContractionPath.simple([(0, i) for i in range(1, n)])


def odd_circuit():
    from tnc_b200.builders import Circuit
    c = Circuit(); q = c.allocate_register(3)
    c.append_gate("rx", [0.5], [q[0]]); c.append_gate("rx", [0.2], [q[1]]); c.append_gate("rx", [0.3], [q[2]])
    c.append_gate("cx", [], [q[0], q[1]]); c.append_gate("cx", [], [q[1], q[2]])
    return c


SV8 = np.array([0.953246407214305, -0.14406910361762032j, -0.014455126269118733, -0.09564366568448116j,
                -0.024421837348497916, 0.0036909997130494475j, -0.03678688170631573, -0.24340376901515096j])


def approx_default(a, b):
    a, b = np.asarray(a), np.asarray(b)
    eps = np.finfo(np.float64).eps
    for x, y in ((a.real, b.real), (a.imag, b.imag)):
        d = np.abs(x - y)
        assert np.all((d <= eps) | (d <= 4 * np.spacing(np.maximum(np.abs(x), np.abs(y))))), d.max()


def run_sv(ctx, circuit, bitstring=None):
    from tnc_b200.tensornetwork import contract_tensor_network
    tn, perm = circuit.into_statevector_network() if bitstring is None else circuit.into_amplitude_network(bitstring)
    res = perm.apply(contract_tensor_network(tn, chain(len(tn.tensors)), ctx=ctx), ctx=ctx)
    return res.to_numpy().reshape(-1)


def test_qasm_kats(ctx):
    """io/qasm/qasm_importer.rs:171-298 with the circuits restated by hand."""
    from tnc_b200.builders import Circuit
    c = Circuit(); q = c.allocate_register(2)
    c.append_gate("h", [], [q[0]]); c.append_gate("cx", [], [q[0], q[1]])
    approx_default(run_sv(ctx, c), [orc.FRAC_1_SQRT_2, 0, 0, orc.FRAC_1_SQRT_2])
    c = Circuit(); q = c.allocate_register(2)
    c.append_gate("x", [], [q[0]])
    a, b = q[1], q[0]
    c.append_gate("cx", [], [a, b]); c.append_gate("cx", [], [b, a]); c.append_gate("cx", [], [a, b])
    approx_default(run_sv(ctx, c), [0, 1, 0, 0])
    approx_default(run_sv(ctx, odd_circuit()), SV8)
    approx_default(run_sv(ctx, odd_circuit(), "1*0"), SV8[[4, 6]])
    approx_default(run_sv(ctx, odd_circuit(), "*1*"), SV8[[2, 3, 6, 7]])


def test_circuit_builder_kats(ctx):
    """builders/circuit_builder.rs:372-427."""
    from tnc_b200.builders import Circuit
    from tnc_b200.tensornetwork import contract_tensor_network
    c = Circuit(); q = c.allocate_register(5)
    for x in q:
        c.append_gate("h", [], [x])
    tn, perm = c.into_amplitude_network("00000")
    assert perm.is_identity()
    res = contract_tensor_network(tn, chain(len(tn.tensors)), ctx=ctx)
    assert res.legs == []
    approx_default(res.to_numpy().reshape(-1), [orc.FRAC_1_SQRT_2 ** 5])
    c = Circuit(); q = c.allocate_register(2)
    c.append_gate("rx", [math.pi / 4], [q[0]]); c.append_gate("rx", [math.pi / 3], [q[1]])
    tn = c.into_expectation_value_network()
    res = contract_tensor_network(tn, chain(len(tn.tensors)), ctx=ctx)
    approx_default(res.to_numpy().reshape(-1), [orc.FRAC_1_SQRT_2 * 0.5])


def random_network(rng, n_tensors=10, n_legs=14, max_rank=4):
    """A random closed-ish network of small tensors with mixed dims (host arrays)."""
    dim = {l: int(rng.integers(2, 4)) for l in range(n_legs)}
    uses = {l: 0 for l in range(n_legs)}
    tensors = []
    for _ in range(n_tensors):
        avail = [l for l in range(n_legs) if uses[l] < 2]
        r = int(min(len(avail), rng.integers(1, max_rank + 1)))
        legs = [int(x) for x in rng.permutation(avail)[:r]]
        for l in legs:
            uses[l] += 1
        tensors.append((legs, [dim[l] for l in legs]))
    return tensors


def test_network_random_vs_oracle(ctx):
    from tnc_b200.contractionpath import ContractionPath
    from tnc_b200.tensornetwork import Tensor, TensorData, contract_tensor_network
    rng = np.random.default_rng(11)
    for trial in range(8):
        spec = random_network(rng)
        datas = [rand_c(rng, d) for _, d in spec]
        n = len(spec)
        order = [int(x) for x in rng.permutation(n)]
        pairs = [(order[0], j) for j in order[1:]]
        tn = Tensor.new_composite([])
        for (l, d), x in zip(spec, datas):
            t = Tensor(l, d); t.set_tensor_data(TensorData.new_from_data(d, x.reshape(-1))); tn.push_tensor(t)
        res = contract_tensor_network(tn, ContractionPath.simple(pairs), ctx=ctx)
        otn = orc.OTensor(children=[orc.OTensor(list(l), list(d), x) for (l, d), x in zip(spec, datas)])
        ref = orc.contract_tensor_network(otn, orc.OPath(pairs))
        assert res.legs == ref.legs and res.bond_dims == ref.dims
        got = res.to_numpy()
        assert np.abs(got - ref.data).max() <= 1e-12 * max(1.0, np.abs(ref.data).max())


def test_network_nested_equals_flat(ctx):
    """integration_tests.rs:22-83 property: partitioned == flat (and == oracle)."""
    from tnc_b200.contractionpath import path
    from tnc_b200.tensornetwork import Tensor, TensorData, contract_tensor_network
    rng = np.random.default_rng(12)
    def rt(legs, dims):
        t = Tensor(legs, dims); t.set_tensor_data(TensorData.new_from_data(dims, rand_c(rng, dims).reshape(-1))); return t
    ts = [rt([0, 1, 8], [2, 3, 2]), rt([1, 2], [3, 4]), rt([2, 3, 9], [4, 2, 3]), rt([3, 0], [2, 2]), rt([8, 9], [2, 3])]
    flat = contract_tensor_network(Tensor.new_composite(list(ts)), path((0, 1), (0, 2), (0, 3), (0, 4)), ctx=ctx)
    nested_tn = Tensor.new_composite([Tensor.new_composite(ts[:2]), Tensor.new_composite(ts[2:4]), ts[4]])
    nested = contract_tensor_network(nested_tn, path((0, 1), (0, 2), nested={0: [(0, 1)], 1: [(0, 1)]}), ctx=ctx)
    a, b = complex(flat.to_numpy()), complex(nested.to_numpy())
    assert abs(a - b) <= 1e-12 * max(1, abs(a))


def test_network_errors(ctx):
    import tnc_b200 as tb
    from tnc_b200.contractionpath import path
    from tnc_b200.tensornetwork import Tensor, TensorData, contract_tensor_network
    def leaf(legs):
        t = Tensor(legs, [2] * len(legs)); t.set_tensor_data(TensorData.new_from_data([2] * len(legs), np.ones(2 ** len(legs)))); return t
    tn = lambda: Tensor.new_composite([leaf([0]), leaf([0, 1]), leaf([1])])
    import gc
    gc.collect(); ctx.synchronize()
    live_before = ctx.stats()["arena_live_bytes"]     # (workspaces of plans cached by earlier successful calls stay allocated)
    with pytest.raises(tb.TncbError) as e:   # slot 1 consumed, used again (tensordata.rs:42)
        contract_tensor_network(tn(), path((0, 1), (2, 1)), ctx=ctx)
    assert e.value.status == -3 and "uncontracted" in str(e.value)
    with pytest.raises(tb.TncbError) as e:   # "Not fully contracted" (contraction.rs:50)
        contract_tensor_network(tn(), path((0, 1)), ctx=ctx)
    assert e.value.status == -4
    with pytest.raises(tb.TncbError) as e:
        contract_tensor_network(tn(), path((0, 7)), ctx=ctx)
    assert e.value.status == -1
    bad = Tensor.new_composite([leaf([0]), Tensor([0], [3], tensordata=TensorData.new_from_data([3], np.ones(3)))])
    with pytest.raises(tb.TncbError) as e:
        contract_tensor_network(bad, path((0, 1)), ctx=ctx)
    assert e.value.status == -2
    g = Tensor([0, 1], [2, 2]); g.set_tensor_data(TensorData.Gate("foo"))
    with pytest.raises(tb.TncbError, match="Gate 'foo' not found."):
        contract_tensor_network(Tensor.new_composite([leaf([0]), g]), path((0, 1)), ctx=ctx)
    # the arena must be balanced after failures
    ctx.synchronize()
    assert ctx.stats()["arena_live_bytes"] == live_before


def test_single_leaf_and_empty(ctx):
    from tnc_b200.contractionpath import path
    from tnc_b200.tensornetwork import Tensor, TensorData, contract_tensor_network
    t = Tensor([4, 5], [2, 3]); x = np.arange(6) + 1j
    t.set_tensor_data(TensorData.new_from_data([2, 3], x))
    res = contract_tensor_network(Tensor.new_composite([t]), path(), ctx=ctx)
    assert res.legs == [4, 5] and np.array_equal(res.to_numpy().reshape(-1), x)


def test_plan_reuse(ctx):
    """Same circuit, different bitstrings: one plan, many executions."""
    from tnc_b200.tensornetwork import NetworkPlan
    tn0, _ = odd_circuit().into_amplitude_network("000")
    plan = NetworkPlan(tn0, chain(len(tn0.tensors)), ctx=ctx)
    assert plan.info()["pairs"] == len(tn0.tensors) - 1
    for i in range(8):
        bits = format(i, "03b")
        tn, _ = odd_circuit().into_amplitude_network(bits)
        amp = complex(plan.execute(tn).to_numpy())
        assert abs(amp - SV8[i]) <= 4e-16


def test_permute_and_conjugate(ctx):
    import tnc_b200 as tb
    rng = np.random.default_rng(13)
    for shape, perm in [((2, 3, 4), (2, 0, 1)), ((5,), (0,)), ((2, 2, 2, 2, 2, 2), (5, 3, 1, 0, 2, 4)), ((7, 1, 3), (1, 2, 0)), ((64, 33), (1, 0))]:
        x = rand_c(rng, shape)
        d = tb.DeviceTensor.from_numpy(ctx, x)
        out = C.c_void_p()
        tb.check(ctx._l.tncb_permute(ctx.handle, d.handle, (C.c_int * len(perm))(*perm), C.byref(out)))
        d.release()
        o = tb.DeviceTensor.adopt(ctx, out)
        assert np.array_equal(o.to_numpy(), np.transpose(x, perm))
        tb.check(ctx._l.tncb_conjugate(ctx.handle, o.handle))
        assert np.array_equal(o.to_numpy(), np.conj(np.transpose(x, perm)))


def _permute(ctx, x, perm):
    import tnc_b200 as tb
    d = tb.DeviceTensor.from_numpy(ctx, x)
    out = C.c_void_p()
    tb.check(ctx._l.tncb_permute(ctx.handle, d.handle, (C.c_int * len(perm))(*perm), C.byref(out)))
    d.release()
    return tb.DeviceTensor.adopt(ctx, out).to_numpy()


def test_contract_pair_host_pipeline(ctx):
    """tncb_contract_pair_host: 7 back-to-back asynchronous pairs with different payloads (3 slots are recycled twice)
    must give exactly the results of the synchronous tncb_contract_pair path."""
    import torch
    import tnc_b200 as tb
    rng = np.random.default_rng(23)
    a_legs, b_legs = [0, 1, 2, 3], [3, 5, 1, 4]
    a_dims, b_dims = [6, 16, 5, 32], [32, 7, 16, 9]
    jobs = []
    for j in range(7):
        ta = torch.empty(a_dims, dtype=torch.complex128, pin_memory=True); tb_ = torch.empty(b_dims, dtype=torch.complex128, pin_memory=True)
        to = torch.empty([7, 9, 6, 5], dtype=torch.complex128, pin_memory=True)
        ta.numpy()[...] = rand_c(rng, a_dims); tb_.numpy()[...] = rand_c(rng, b_dims)
        jobs.append((ta, tb_, to))
    for ta, tb_, to in jobs:
        tb.contract_pair_host(ctx, a_legs, ta.numpy(), b_legs, tb_.numpy(), to.numpy())
    ctx.synchronize()
    for ta, tb_, to in jobs:
        legs, ref = tb.contract_pair(ctx, a_legs, ta.numpy().copy(), b_legs, tb_.numpy().copy())
        assert legs == [5, 4, 0, 2] and np.array_equal(to.numpy(), ref)


def test_tiled_transpose_k3(ctx):
    """K3 (tiled transpose through shared memory, Permutor::apply circuit_builder.rs:86-114): bit-exact against
    numpy.transpose over shapes that exercise full / partial tiles, many dim-2 legs, prime dims, identity and
    inner-run-preserving permutations, and the statevector-like reversal of 22 qubit legs (8 MiB elements)."""
    rng = np.random.default_rng(17)
    cases = [((64, 65), (1, 0)), ((100, 37, 29), (2, 0, 1)), ((100, 37, 29), (1, 2, 0)), ((33, 31, 30, 7), (3, 1, 0, 2)),
             ((2,) * 14, tuple(reversed(range(14)))), ((2,) * 14, (13, 0, 12, 1, 11, 2, 10, 3, 9, 4, 8, 5, 7, 6)),
             ((4,) * 7, (6, 5, 0, 1, 2, 3, 4)), ((4,) * 7, (0, 1, 2, 3, 5, 4, 6)), ((3, 5, 7, 11, 13), (4, 2, 0, 3, 1)),
             ((1024, 3, 128), (2, 1, 0)), ((40, 2, 40, 2, 40), (3, 1, 4, 2, 0)), ((5000, 3), (1, 0)), ((3, 5000), (1, 0)),
             ((17, 4096), (0, 1))]
    for shape, perm in cases:
        x = rand_c(rng, shape)
        ctx.reset_stats()
        got = _permute(ctx, x, perm)
        assert ctx.engine_counts()["permute"] == 1
        assert np.array_equal(got, np.transpose(x, perm)), (shape, perm)
    x = rand_c(rng, (2,) * 22)
    perm = tuple(reversed(range(22)))
    assert np.array_equal(_permute(ctx, x, perm), np.transpose(x, perm))


# ---- full-size C2: size-independent properties --------------------------------------------------
def test_c2_full_size_properties(ctx):
    """BASELINE config 2: rank-12, dim-4 operands (2^24 elements each), M=N=K=4096, shared legs
    interleaved.  Checksum of checksums: sum_{n,m} C = sum_k (sum_n Bt[n,k]) (sum_m At[k,m]);
    plus sampled entries recomputed on the host."""
    import tnc_b200 as tb
    rng = np.random.default_rng(20240612)
    a_legs = list(range(12))
    sh = [1, 3, 5, 7, 9, 11]
    b_legs = [x for p in zip([11, 9, 7, 5, 3, 1][::1], range(12, 18)) for x in p]  # shared at even positions, reversed order
    a = (rng.random([4] * 12) * 2 - 1) + 1j * (rng.random([4] * 12) * 2 - 1)
    b = (rng.random([4] * 12) * 2 - 1) + 1j * (rng.random([4] * 12) * 2 - 1)
    legs, got = tb.contract_pair(ctx, a_legs, a, b_legs, b)
    assert legs == list(range(12, 18)) + [0, 2, 4, 6, 8, 10]
    a_sum = a.sum(axis=tuple(i for i, l in enumerate(a_legs) if l not in sh))      # over shared legs in a's order (1,3,..,11)
    b_sum = b.sum(axis=tuple(i for i, l in enumerate(b_legs) if l not in sh))      # shared legs in b's order (11,9,..,1)
    checksum = (a_sum * np.transpose(b_sum, (5, 4, 3, 2, 1, 0))).sum()
    total = got.sum()
    assert abs(total - checksum) <= 1e-9 * max(1.0, abs(checksum)), (total, checksum)
    # sampled entries
    for _ in range(16):
        n_idx = tuple(int(x) for x in rng.integers(0, 4, 6)); m_idx = tuple(int(x) for x in rng.integers(0, 4, 6))
        a_sl = a[tuple(x for p in zip(m_idx, [slice(None)] * 6) for x in p)]        # [k1,k3,...,k11]
        b_sl = b[tuple(x for p in zip([slice(None)] * 6, n_idx) for x in p)]        # [k11,k9,...,k1]
        ref = (a_sl * np.transpose(b_sl, (5, 4, 3, 2, 1, 0))).sum()
        assert abs(got[n_idx + m_idx] - ref) <= 1e-11 * max(1.0, abs(ref))
