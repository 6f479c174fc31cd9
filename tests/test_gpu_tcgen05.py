"""K1' (tcgen05 int8 engine) parity: against the oracle, against the FP64 DMMA path, and against its own guaranteed
bound  |C - C_exact|[n,m] <= bound(K, tol) * max|b[n,:]| * max|a[m,:]|  (tncb.h).  Default engine = modular (CRT)
emulation with the full 53-bit mantissa; the round-1 digit-slicing engine is checked as engine 1.
Tolerance of the plain comparisons: ||gpu-cpu||_inf <= 1e-12 * max(1, ||cpu||_inf)."""
import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu


def rand_c(rng, shape, scale=1.0):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) * scale


@pytest.fixture(params=[4, 3], ids=["4prod", "3prod"])
def tc_ctx(built_lib, request):
    """Every test below runs with the 4-product and with the 3-product (Gauss) form of the complex int8 GEMM."""
    import tnc_b200 as tb
    c = tb.Context(0)
    c.set_tcgen05_slices(8)
    c.set_tcgen05_threshold(1, 128)     # route every pair with M, N >= 128 and K >= 128 to the tcgen05 engine
    c.set_tcgen05_products(request.param)
    c.products = request.param
    yield c
    c.close()


ENGINES = [("4prod", 0, 4), ("3prod", 0, 3), ("digits", 1, 0)]


@pytest.fixture(params=ENGINES, ids=[e[0] for e in ENGINES])
def int8_ctx(built_lib, request):
    """The modular engine in its 4- and 3-product forms, and the digit-slicing engine (engine 1, S = 8 digits)."""
    import tnc_b200 as tb
    _, engine, products = request.param
    c = tb.Context(0)
    c.set_tcgen05_slices(8)
    c.set_tcgen05_threshold(1, 128)
    c.set_tcgen05_engine(engine)
    if engine == 0:
        c.set_tcgen05_products(products)
    c.engine, c.products, c.slices = engine, products, 8
    yield c
    c.close()


def digit_bound(K, S):
    """Engine 1's guarantee (ozaki.cu): |C - C_exact|[n,m] <= (S+1) K 2^(-7S) * 4 max|b[n,:]| max|a[m,:]|."""
    return (S + 1) * K * 2.0 ** (-7 * S) * 4


def engine_bound(ctx, K):
    import tnc_b200 as tb
    return tb.tcgen05_bound(K)["bound"] if ctx.engine == 0 else digit_bound(K, ctx.slices)


def absmax(x, axis):
    """max(|re|, |im|) along axis: the magnitude both engines scale a row by"""
    return np.maximum(np.abs(x.real).max(axis=axis), np.abs(x.imag).max(axis=axis))


def gemm_view(a_legs, a, b_legs, b):
    """Bt [N, K] and At [K, M] with C = Bt At, legs ordered as in oracle.contract_pair."""
    shared = [l for l in a_legs if l in b_legs]
    bf = [i for i, l in enumerate(b_legs) if l not in a_legs]
    af = [i for i, l in enumerate(a_legs) if l not in b_legs]
    bk = [b_legs.index(l) for l in shared]
    ak = [a_legs.index(l) for l in shared]
    N, M, K = (int(np.prod([x.shape[i] for i in ix], dtype=np.int64)) for x, ix in ((b, bf), (a, af), (a, ak)))
    return np.transpose(b, bf + bk).reshape(N, K), np.transpose(a, ak + af).reshape(K, M)


def edge_sample(rng, n, count=24):
    """first/last index, 63/64, 127/128, 255/256 where they exist, filled up with random indices"""
    idx = {i for i in (0, 63, 64, 127, 128, 255, 256, n - 1) if i < n}
    rest = [int(i) for i in rng.permutation(n) if int(i) not in idx]
    return np.array(sorted(idx) + rest[:max(0, count - len(idx))])


def check_bound(ctx, rng, got, a_legs, a, b_legs, b):
    """sampled entries (tile edges included) against a long-double reference, in units of the engine's own bound"""
    bt, at = gemm_view(a_legs, a, b_legs, b)
    N, K = bt.shape
    M = at.shape[1]
    ns, ms = edge_sample(rng, N), edge_sample(rng, M)
    ref = bt[ns].astype(np.clongdouble) @ at[:, ms].astype(np.clongdouble)
    scale = absmax(bt[ns], 1)[:, None] * absmax(at[:, ms], 0)[None, :]
    err = np.abs(got.reshape(N, M)[np.ix_(ns, ms)] - ref)
    ratio = float((err / (engine_bound(ctx, K) * scale)).max())
    assert ratio <= 1.0, ratio


@pytest.fixture()
def dmma_ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    c.set_tcgen05_slices(0)             # FP64 tensor pipe (DMMA) for every pair
    yield c
    c.close()


def check(ctx, rng, a_legs, a_dims, b_legs, b_dims, tol=1e-12, scale_rows=False, engine="k1_tcgen05"):
    """With the digit-slicing engine (engine 1), only pairs it takes (M, N, K >= 256) run, and they are also checked against
    that engine's own bound; the smaller cases are the modular engine's."""
    import tnc_b200 as tb
    M = int(np.prod([d for l, d in zip(a_legs, a_dims) if l not in b_legs]))
    N = int(np.prod([d for l, d in zip(b_legs, b_dims) if l not in a_legs]))
    K = int(np.prod([d for l, d in zip(a_legs, a_dims) if l in b_legs]))
    if getattr(ctx, "engine", 0) == 1 and min(M, N, K) < 256:
        return None, None
    a, b = rand_c(rng, a_dims), rand_c(rng, b_dims)
    if scale_rows:  # wildly different magnitudes per slice of the leading free legs -> per-row exponents matter
        a = a * np.exp(rng.uniform(-40, 40, size=[a_dims[0]] + [1] * (len(a_dims) - 1)))
        b = b * np.exp(rng.uniform(-40, 40, size=[b_dims[0]] + [1] * (len(b_dims) - 1)))
    ctx.reset_stats()
    legs, got = tb.contract_pair(ctx, a_legs, a, b_legs, b)
    assert ctx.engine_counts()[engine] == 1, ctx.engine_counts()
    ref_legs, ref = orc.contract_pair(a_legs, a, b_legs, b)
    assert legs == ref_legs and got.shape == ref.shape
    err = np.abs(got - ref).max()
    assert err <= tol * max(1.0, np.abs(ref).max()), err
    if getattr(ctx, "engine", 0) == 1 and engine == "k1_tcgen05":
        check_bound(ctx, rng, got, a_legs, a, b_legs, b)
    return got, ref


def test_engine_is_really_tcgen05(tc_ctx):
    """Guard against silently testing the DMMA path: the modular engine launches 6 kernels per pair
    (2 row-max + 2 residue + 1 GEMM + 1 reconstruction) after the table build, the DMMA step 1 or 2."""
    import tnc_b200 as tb
    rng = np.random.default_rng(0)
    a = tb.DeviceTensor.from_numpy(tc_ctx, rand_c(rng, (256, 256)))
    b = tb.DeviceTensor.from_numpy(tc_ctx, rand_c(rng, (256, 256)))
    c = tb.DeviceTensor.empty(tc_ctx, (256, 256))
    tb.contract_pair_into(tc_ctx, [0, 1], a, [1, 2], b, c)     # builds the offset tables
    tc_ctx.reset_stats()
    tb.contract_pair_into(tc_ctx, [0, 1], a, [1, 2], b, c)
    assert tc_ctx.stats()["kernel_launches"] == 6
    assert tc_ctx.engine_counts()["k1_tcgen05"] == 1 and tc_ctx.last_tcgen05_info()["n_moduli"] == tb.tcgen05_bound(256)["n_moduli"] == 15
    assert tc_ctx.last_tcgen05_info()["products"] == tc_ctx.products
    tc_ctx.set_tcgen05_engine(1)                               # legacy digit slicing: 2 exponent + 2 slicing + 1 GEMM
    tc_ctx.reset_stats()
    tb.contract_pair_into(tc_ctx, [0, 1], a, [1, 2], b, c)
    assert tc_ctx.stats()["kernel_launches"] == 5 and tc_ctx.engine_counts()["k1_tcgen05"] == 1
    tc_ctx.set_tcgen05_engine(0)
    tc_ctx.set_tcgen05_slices(0)
    tc_ctx.reset_stats()
    tb.contract_pair_into(tc_ctx, [0, 1], a, [1, 2], b, c)
    assert tc_ctx.stats()["kernel_launches"] <= 2      # k1_kernel (+ split-K reduce)
    ec = tc_ctx.engine_counts()
    assert ec["k1_tcgen05"] == 0 and ec["k1_dmma"] + ec["k1_dmma_splitk"] == 1
    tc_ctx.set_tcgen05_slices(8)


def test_three_and_four_products_agree(built_lib):
    """Karatsuba's three-product form takes its sums on residues (exact): it reconstructs the same integers as the
    four-product form and may differ from it only by the last rounding of the reconstruction -- far inside the engine's
    bound.  The default picks it by K (tncb_ctx_set_tcgen05_products)."""
    import tnc_b200 as tb
    ctx = tb.Context(0)
    ctx.set_tcgen05_threshold(1, 128)
    rng = np.random.default_rng(11)
    try:
        for (M, N, K) in [(256, 512, 1024), (384, 136, 2048), (130, 300, 640), (1024, 256, 128 * 33)]:
            a, b = rand_c(rng, (K, M)), rand_c(rng, (N, K))
            a *= np.exp(rng.uniform(-30, 30, size=(1, M))); b *= np.exp(rng.uniform(-30, 30, size=(N, 1)))
            out = {}
            for pr in (4, 3):
                ctx.set_tcgen05_products(pr)
                ctx.reset_stats()
                _, out[pr] = tb.contract_pair(ctx, [0, 1], a, [2, 0], b)
                assert ctx.engine_counts()["k1_tcgen05"] == 1
                assert ctx.last_tcgen05_info()["products"] == pr
            ctx.set_tcgen05_products(0, 2048)
            _, out[0] = tb.contract_pair(ctx, [0, 1], a, [2, 0], b)
            assert ctx.last_tcgen05_info()["products"] == (3 if K >= 2048 else 4)
            assert np.array_equal(out[0].view(np.float64), out[3 if K >= 2048 else 4].view(np.float64))
            scale = (np.maximum(np.abs(b.real), np.abs(b.imag)).max(axis=1)[:, None] *
                     np.maximum(np.abs(a.real), np.abs(a.imag)).max(axis=0)[None, :])
            bound = tb.tcgen05_bound(K)["bound"]
            ref = b.astype(np.clongdouble) @ a.astype(np.clongdouble)
            # same integers, last-bit rounding of the reconstruction only
            assert np.all(np.abs(out[3] - out[4]) <= 8 * np.finfo(np.float64).eps * np.abs(ref).astype(np.float64) + 1e-3 * bound * scale)
            assert np.all(np.abs(out[3] - ref) <= bound * scale) and np.all(np.abs(out[4] - ref) <= bound * scale)
    finally:
        ctx.close()


def test_tcgen05_square(tc_ctx):
    rng = np.random.default_rng(1)
    check(tc_ctx, rng, [0, 1], [256, 256], [1, 2], [256, 256])
    check(tc_ctx, rng, [0, 1], [512, 384], [1, 2], [384, 640])
    check(tc_ctx, rng, [0, 1], [128, 128], [1, 2], [128, 128])      # one tile pair, half of it padding


def test_tcgen05_ragged(int8_ctx):
    rng = np.random.default_rng(2)
    check(int8_ctx, rng, [0, 1], [300, 333], [1, 2], [333, 260])      # M, N, K not multiples of 128
    check(int8_ctx, rng, [0, 1, 2], [7, 41, 300], [2, 3, 1], [300, 257, 41], engine="k0_splitk")  # M = 7: too thin for tcgen05 -> K0 split-K
    check(int8_ctx, rng, [0, 1, 2], [133, 41, 30], [2, 3, 1], [30, 257, 41])   # permuted K legs (K = 1230), ragged everywhere
    check(int8_ctx, rng, [0, 1], [130, 129], [1, 2], [129, 131])
    check(int8_ctx, rng, [0, 1, 2], [257, 20, 15], [2, 3, 1], [15, 511, 20])   # one row past a tile, one short of it


def test_tcgen05_permuted_circuit_like(int8_ctx):
    rng = np.random.default_rng(3)
    sh = list(range(100, 109)); af = list(range(9)); bf = list(range(50, 59))
    a_legs = [x for p in zip(af, sh) for x in p]
    b_legs = [x for p in zip(reversed(sh), bf) for x in p]
    check(int8_ctx, rng, a_legs, [2] * 18, b_legs, [2] * 18)           # M = N = K = 512, all dims 2, interleaved
    # shared legs leading in a, trailing in b: both loader modes (row-fast / k-fast) of the preparation kernels
    check(int8_ctx, rng, [0, 1, 2, 3], [16, 16, 16, 16], [4, 5, 0, 1], [16, 16, 16, 16])
    check(int8_ctx, rng, [2, 3, 0, 1], [16, 16, 16, 16], [0, 1, 4, 5], [16, 16, 16, 16])
    # C2 in small: dim-4 legs, shared legs interleaved with the free ones in both operands (M = N = K = 256): the warp
    # lanes of the preparation kernels are split 4 along k x 8 along rows (a) and 8 x 4 (b)
    check(int8_ctx, rng, list(range(8)), [4] * 8, [7, 8, 5, 9, 3, 10, 1, 11], [4] * 8)
    check(int8_ctx, rng, [0, 1, 2], [160, 64, 48], [2, 3, 1], [48, 130, 64])       # fastest K leg of a is 48 long (lk = 5), of b 64


def test_tcgen05_row_scaling(int8_ctx):
    rng = np.random.default_rng(4)
    # relative tolerance per output row group: compare in scaled units
    import tnc_b200 as tb
    a = rand_c(rng, [256, 256]); b = rand_c(rng, [256, 256])
    ra = np.exp(rng.uniform(-30, 30, size=(256, 1))); rb = np.exp(rng.uniform(-30, 30, size=(1, 256)))
    a2, b2 = a * ra, b * rb                                            # a rows (M) and b columns (N) scaled
    int8_ctx.reset_stats()
    legs, got = tb.contract_pair(int8_ctx, [0, 1], a2, [1, 2], b2)
    assert int8_ctx.engine_counts()["k1_tcgen05"] == 1
    _, ref = orc.contract_pair([0, 1], a2, [1, 2], b2)
    rel = np.abs(got - ref) / (rb.T * ra.T * 16.0 * np.ones_like(np.abs(ref)))
    assert rel.max() <= 1e-12, rel.max()
    check_bound(int8_ctx, rng, got, [0, 1], a2, [1, 2], b2)


def test_tcgen05_long_k_split(int8_ctx):
    """K = 20000 with one tile pair: the modular engine splits K over CTAs (chunk residues add up in the reconstruction),
    the digit-slicing engine runs three int32-safe K chunks of 8192 (the epilogue adds each chunk into C);
    K = 70000 > 32768 needs several int32-safe chunks in any case."""
    rng = np.random.default_rng(5)
    check(int8_ctx, rng, [0, 1], [256, 20000], [1, 2], [20000, 256])
    check(int8_ctx, rng, [0, 1], [128, 70000], [1, 2], [70000, 128], tol=3e-12)


@pytest.mark.parametrize("S", [2, 4, 8])
def test_digit_slicing_digit_counts(built_lib, S):
    """The digit-slicing engine with S = 2, 4 and 8 digits, each against its own bound, on a ragged pair with per-row
    exponents.  The int8 operation count, 8 * S(S+1)/2 * Np Mp Kp, shows that S digits were used."""
    import tnc_b200 as tb
    rng = np.random.default_rng(100 + S)
    ctx = tb.Context(0)
    try:
        ctx.set_tcgen05_threshold(1, 128)
        ctx.set_tcgen05_engine(1)
        ctx.set_tcgen05_slices(S)
        ctx.engine, ctx.slices = 1, S
        M, N, K = 385, 300, 1000
        a = rand_c(rng, (M, K)) * np.exp(rng.uniform(-8, 8, size=(M, 1)))
        b = rand_c(rng, (K, N)) * np.exp(rng.uniform(-8, 8, size=(1, N)))
        ctx.reset_stats()
        _, got = tb.contract_pair(ctx, [0, 1], a, [1, 2], b)
        assert ctx.engine_counts()["k1_tcgen05"] == 1
        padded = lambda x: -(-x // 128) * 128
        assert ctx.last_tcgen05_info()["int8_ops"] == 8 * (S * (S + 1) // 2) * padded(N) * padded(M) * padded(K)
        check_bound(ctx, rng, got, [0, 1], a, [1, 2], b)
    finally:
        ctx.close()


def bound_check(ctx, rng, M, N, K, rel=0.0, n_mod=0, zero_row=False):
    """error against the exact-ish oracle, in units of the guaranteed bound"""
    import tnc_b200 as tb
    a = rand_c(rng, (M, K)) * np.exp(rng.uniform(-8, 8, size=(M, 1)))
    b = rand_c(rng, (K, N)) * np.exp(rng.uniform(-8, 8, size=(1, N)))
    if zero_row:
        a[5] = 0.0
    ctx.set_tolerance(rel); ctx.set_tcgen05_moduli(n_mod)
    ctx.reset_stats()
    _, got = tb.contract_pair(ctx, [0, 1], a, [1, 2], b)              # C[n, m] = sum_k b[k, n] a[m, k]
    info = ctx.last_tcgen05_info()
    assert ctx.engine_counts()["k1_tcgen05"] == 1
    ctx.set_tolerance(0.0); ctx.set_tcgen05_moduli(0)
    bd = tb.tcgen05_bound(K, rel, n_mod)
    assert info["n_moduli"] == bd["n_moduli"]
    # long-double reference on a 24 x 24 sample of (n, m) (numpy has no long-double BLAS)
    ns, ms_ = rng.choice(N, 24, replace=False), rng.choice(M, 24, replace=False)
    if zero_row:
        ms_[0] = 5
    ref = b[:, ns].T.astype(np.clongdouble) @ a[ms_].T.astype(np.clongdouble)
    sub = got[np.ix_(ns, ms_)]
    mxa = np.maximum(np.abs(a.real), np.abs(a.imag)).max(axis=1)[ms_]; mxb = np.maximum(np.abs(b.real), np.abs(b.imag)).max(axis=0)[ns]
    scale = mxb[:, None] * np.where(mxa > 0, mxa, 1.0)[None, :]
    ratio = float((np.abs(sub - ref) / scale).max() / bd["bound"])
    assert ratio <= 1.0, (ratio, bd)
    if zero_row:
        assert np.all(got[:, 5] == 0)
    return ratio, bd, float(np.abs(sub - ref).max() / np.abs(ref).max())


@pytest.mark.parametrize("K", [1 << 14, 1 << 16, 1 << 18])
def test_tolerance_driven_modulus_count(tc_ctx, K):
    """VERDICT r1 item 4: the slice/modulus count follows a requested normwise tolerance with a proven bound,
    tested over K = 2^14 ... 2^18 (the oracle side is a long-double GEMM of 128 x 128 x K)."""
    rng = np.random.default_rng(K)
    r_full, bd_full, e_full = bound_check(tc_ctx, rng, 128, 128, K, 0.0, zero_row=True)
    r_10, bd_10, e_10 = bound_check(tc_ctx, rng, 128, 128, K, 1e-10)
    r_6, bd_6, e_6 = bound_check(tc_ctx, rng, 128, 128, K, 1e-6)
    assert bd_full["n_moduli"] >= bd_10["n_moduli"] > bd_6["n_moduli"]
    assert e_full < 1e-13 and e_10 < 1e-10 and e_6 < 1e-6
    print(f"K={K}: moduli {bd_full['n_moduli']}/{bd_10['n_moduli']}/{bd_6['n_moduli']}  err/max|C| {e_full:.1e}/{e_10:.1e}/{e_6:.1e}  "
          f"err/bound {r_full:.1e}/{r_10:.1e}/{r_6:.1e}")


def test_forced_modulus_counts(tc_ctx):
    rng = np.random.default_rng(77)
    prev = None
    import tnc_b200 as tb
    assert tb.tcgen05_bound(512, 0.0, 20)["n_moduli"] == tb.tcgen05_bound(512)["n_moduli"] == 16     # clamped to what 53 bits need
    for n in (20, 16, 12, 8, 4):
        _, bd, e = bound_check(tc_ctx, rng, 256, 128, 512, 0.0, n_mod=n)
        assert prev is None or bd["bound"] >= prev
        prev = bd["bound"]


def test_nonfinite_rows_poison_their_outputs(tc_ctx):
    """ADVICE r1: NaN / Inf must not come out as finite garbage.  A row (column) of C whose operand row contains a
    non-finite value is NaN; every other entry is unaffected."""
    import tnc_b200 as tb
    rng = np.random.default_rng(6)
    a, b = rand_c(rng, (256, 300)), rand_c(rng, (300, 256))
    a[7, 11] = np.nan; a[200, 0] = np.inf + 0j; b[5, 40] = complex(0, -np.inf)
    _, got = tb.contract_pair(tc_ctx, [0, 1], a, [1, 2], b)          # got[n, m]
    bad_m = np.zeros(256, bool); bad_m[[7, 200]] = True
    bad_n = np.zeros(256, bool); bad_n[40] = True
    bad = bad_n[:, None] | bad_m[None, :]
    assert np.all(np.isnan(got[bad].real)) and np.all(np.isnan(got[bad].imag))
    a0, b0 = np.where(np.isfinite(a), a, 0), np.where(np.isfinite(b), b, 0)
    ref = b0.T @ a0.T
    assert np.abs(got[~bad] - ref[~bad]).max() <= 1e-12 * np.abs(ref).max()


def extreme_pair(ctx, a2, b2):
    """C = b2^T a2^T on the int8 engine: every entry finite and within the engine's bound relative to
    max(|b col|, 2^-1001) * max(|a row|, 2^-1001) (the scale exponents are clamped at -1000)."""
    import tnc_b200 as tb
    ctx.reset_stats()
    _, got = tb.contract_pair(ctx, [0, 1], a2, [1, 2], b2)
    assert ctx.engine_counts()["k1_tcgen05"] == 1
    ref = b2.T.astype(np.clongdouble) @ a2.T.astype(np.clongdouble)
    assert np.all(np.isfinite(got.real)) and np.all(np.isfinite(got.imag))
    mxa = np.maximum(absmax(a2, 1), 2.0 ** -1001)
    mxb = np.maximum(absmax(b2, 0), 2.0 ** -1001)
    # outputs below 2^-1022 are denormal doubles: no FP64 result (the reference's included) can be closer than 2^-1075
    allowed = engine_bound(ctx, a2.shape[1]) * (mxb[:, None].astype(np.longdouble) * mxa[None, :].astype(np.longdouble)) + np.longdouble(2.0) ** -1070
    assert np.all(np.abs(got - ref) <= allowed), float((np.abs(got - ref) / allowed).max())
    return got, ref


def test_extreme_exponents(int8_ctx):
    """Rows near the ends of the double range.  First pair: a rows with maxima of 2^-1040 (denormal: the scale exponent is
    clamped at -1000, the row keeps ABSOLUTE accuracy 2^(-1000-53)), 2^-900, 1 and 2^+900 against b columns of
    2^-100 .. 2^+20.  Second pair: the other ends, a rows with maxima in [2^1023, 2^1024) (the largest scale exponent a finite
    row can have, 1024) against b columns of 2^-1040 and of 2^-100 .. 2^-70, and rows of 2^-60 against all of them; every
    product is finite."""
    rng = np.random.default_rng(9)
    M, N, K = 256, 256, 384
    a, b = rand_c(rng, (M, K)), rand_c(rng, (K, N))
    ea = np.zeros(M, dtype=int); ea[:64] = -1040; ea[64:128] = -900; ea[192:] = 900
    eb = rng.integers(-100, 20, size=N)
    a2 = np.ldexp(a.real, ea[:, None]) + 1j * np.ldexp(a.imag, ea[:, None])
    b2 = np.ldexp(b.real, eb[None, :]) + 1j * np.ldexp(b.imag, eb[None, :])
    got, ref = extreme_pair(int8_ctx, a2, b2)
    rel = (np.abs(got - ref)[:, 128:] / np.abs(ref)[:, 128:]).astype(np.float64)    # rows of ordinary magnitude: relative accuracy as usual
    assert np.median(rel) < 1e-14

    a, b = rand_c(rng, (M, K)), rand_c(rng, (K, N))
    a3 = a * 2.0 ** -60
    a3[:8] = a[:8] / absmax(a[:8], 1)[:, None] * (1.5 * 2.0 ** 1023)     # max(|re|, |im|) of the row = 1.5 * 2^1023
    eb = rng.integers(-100, -70, size=N); eb[:64] = -1040
    b3 = np.ldexp(b.real, eb[None, :]) + 1j * np.ldexp(b.imag, eb[None, :])
    assert absmax(a3[:8], 1).min() >= 2.0 ** 1023
    extreme_pair(int8_ctx, a3, b3)


def test_panels_when_the_workspace_is_small(tc_ctx):
    """A tiny workspace budget forces panels over M and N; results must not change."""
    import tnc_b200 as tb
    rng = np.random.default_rng(8)
    a, b = rand_c(rng, (700, 384)), rand_c(rng, (384, 900))
    _, ref = tb.contract_pair(tc_ctx, [0, 1], a, [1, 2], b)
    tc_ctx.set_tcgen05_workspace(6 << 20)
    tc_ctx.reset_stats()
    _, got = tb.contract_pair(tc_ctx, [0, 1], a, [1, 2], b)
    assert tc_ctx.stats()["kernel_launches"] > 6       # several panels
    tc_ctx.set_tcgen05_workspace(12 << 30)
    assert np.array_equal(got, ref)                    # same integers, same reconstruction


def test_full_size_c2_all_engines(tc_ctx, dmma_ctx):
    """Full-size C2 (4096^3): DMMA (really DMMA: engine counters), the modular engine and the legacy digit-slicing
    engine against each other and against a host-computed sample of entries (VERDICT r1 weak #1)."""
    import tnc_b200 as tb
    rng = np.random.default_rng(20240612)
    a_legs = list(range(12))
    b_legs = [x for p in zip([11, 9, 7, 5, 3, 1], range(12, 18)) for x in p]
    a = (rng.random([4] * 12) * 2 - 1) + 1j * (rng.random([4] * 12) * 2 - 1)
    b = (rng.random([4] * 12) * 2 - 1) + 1j * (rng.random([4] * 12) * 2 - 1)
    dmma_ctx.reset_stats()
    _, ref = tb.contract_pair(dmma_ctx, a_legs, a, b_legs, b)
    ec = dmma_ctx.engine_counts()
    assert ec["k1_tcgen05"] == 0 and ec["k1_dmma"] == 1 and dmma_ctx.stats()["kernel_launches"] <= 2, ec
    # host sample: 64 entries of C[n, m] = sum_k Bt[n, k] At[k, m] in long double
    at = a.transpose([0, 2, 4, 6, 8, 10, 11, 9, 7, 5, 3, 1]).reshape(4096, 4096)      # [m, k] with k in b's order (11, 9, ..., 1)
    bt = b.transpose([1, 3, 5, 7, 9, 11, 0, 2, 4, 6, 8, 10]).reshape(4096, 4096)      # [n, k]
    refm = ref.reshape(4096, 4096)
    idx = rng.integers(0, 4096, size=(64, 2))
    samp = np.array([np.dot(bt[n].astype(np.clongdouble), at[m].astype(np.clongdouble)) for n, m in idx])
    scale = np.abs(refm).max()
    assert np.abs(refm[idx[:, 0], idx[:, 1]] - samp).max() / scale < 1e-13        # DMMA at full size vs the host
    tc_ctx.reset_stats()
    _, got = tb.contract_pair(tc_ctx, a_legs, a, b_legs, b)
    assert tc_ctx.engine_counts()["k1_tcgen05"] == 1
    e_crt = np.abs(got - ref).max() / scale
    assert np.abs(got.reshape(4096, 4096)[idx[:, 0], idx[:, 1]] - samp).max() / scale < 1e-13
    tc_ctx.set_tcgen05_moduli(12)
    _, got12 = tb.contract_pair(tc_ctx, a_legs, a, b_legs, b)
    tc_ctx.set_tcgen05_moduli(0)
    e12 = np.abs(got12 - ref).max() / scale
    tc_ctx.set_tcgen05_engine(1)
    _, got_s8 = tb.contract_pair(tc_ctx, a_legs, a, b_legs, b)
    tc_ctx.set_tcgen05_engine(0)
    e_s8 = np.abs(got_s8 - ref).max() / scale
    assert e_crt <= 1e-13 and e_s8 <= 1e-13 and e_crt < e12 <= 1e-9, (e_crt, e12, e_s8)
    print(f"C2 vs DMMA: modular 16 moduli {e_crt:.2e}, 12 moduli {e12:.2e}, digit slicing S=8 {e_s8:.2e}")
