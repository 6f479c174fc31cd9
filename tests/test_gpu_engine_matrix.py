"""The H100 GEMM routes of launch_k1 (kernels.cu), each checked against an independent reference in units of the error
bound its engine documents, at the shapes where tiled kernels go wrong: ragged edges, K below one BK chunk, half-filled
m16n8k4 row pairs, split-K, every loader mode -- and at the benchmark network's own pair shapes.

References are long double (np.clongdouble) or exact integers; the oracle's FP64 GEMM is used for full-matrix checks with
its own rounding error counted in.  Per-entry bounds:
  FP64 (K1 DMMA, split-K):   |err| <= (2K + ksplit + 8) 2^-53 sum_k |Bt[n,k]| |At[k,m]|
  modular int8 engine:       |err| <= tcgen05_bound(K)["bound"] max|b[n,:]| max|a[m,:]|     (max over max(|re|, |im|))
Operands carry a per-row exponent spread, so that an error confined to small rows or columns cannot hide behind max|C|,
and the sampled entries include the first and last rows and columns and the tile edges 63/64, 127/128, 255/256."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import tnc_oracle as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -53
SM_COUNT = 132          # H100 SXM; the split-K mirror below reads the device's own count when a GPU is present


# ---- references and bounds ------------------------------------------------------------------------------------------
def operand(rng, dims, row_axes, integer=False):
    """complex operand, one rng call per plane; integer: |re|, |im| <= 2^10, else uniform in [-1, 1) times 2^e with one
    e in [-8, 8] per index of the free legs `row_axes` (a per-row exponent spread of the GEMM view)"""
    x = np.empty(dims, dtype=np.complex128)
    if integer:
        x.real[...] = rng.integers(-1024, 1025, size=dims)
        x.imag[...] = rng.integers(-1024, 1025, size=dims)
        return x
    for plane in (x.real, x.imag):
        t = rng.random(dims)
        t *= 2.0
        t -= 1.0
        plane[...] = t
        del t
    sdims = [d if i in row_axes else 1 for i, d in enumerate(dims)]
    x *= np.exp2(rng.integers(-8, 9, size=sdims).astype(np.float64))
    return x


class View:
    """The GEMM view C[n, m] = sum_k Bt[n, k] At[k, m] of one pair, legs ordered as in oracle.contract_pair (shared legs
    in a's order), without materialising Bt or At."""

    def __init__(self, a_legs, a, b_legs, b):
        self.a_legs, self.a, self.b_legs, self.b = list(a_legs), a, list(b_legs), b
        self.shared = [l for l in a_legs if l in b_legs]
        self.af = [l for l in a_legs if l not in b_legs]
        self.bf = [l for l in b_legs if l not in a_legs]
        dim = dict(zip(a_legs, a.shape)) | dict(zip(b_legs, b.shape))
        self.M = int(np.prod([dim[l] for l in self.af], dtype=np.int64))
        self.N = int(np.prod([dim[l] for l in self.bf], dtype=np.int64))
        self.K = int(np.prod([dim[l] for l in self.shared], dtype=np.int64))

    def _rows(self, x, legs, free, idx):
        fpos = [legs.index(l) for l in free]
        fdims = [x.shape[p] for p in fpos]
        left = [l for l in legs if l in self.shared]                     # axes left after fixing the free ones
        perm = [left.index(l) for l in self.shared]
        out = np.empty((len(idx), self.K), dtype=x.dtype)
        for r, i in enumerate(idx):
            sel = [slice(None)] * x.ndim
            for p, v in zip(fpos, np.unravel_index(int(i), fdims)):
                sel[p] = int(v)
            out[r] = np.transpose(x[tuple(sel)], perm).reshape(-1)
        return out

    def bt_rows(self, ns):
        return self._rows(self.b, self.b_legs, self.bf, ns)              # [len(ns), K]

    def at_cols(self, ms):
        return self._rows(self.a, self.a_legs, self.af, ms)              # [len(ms), K]

    def full(self):
        bt = np.transpose(self.b, [self.b_legs.index(l) for l in self.bf + self.shared]).reshape(self.N, self.K)
        at = np.transpose(self.a, [self.a_legs.index(l) for l in self.shared + self.af]).reshape(self.K, self.M)
        return bt, at

    def _absmax(self, x, legs):
        ax = tuple(legs.index(l) for l in self.shared)
        return np.maximum(np.abs(x.real).max(axis=ax), np.abs(x.imag).max(axis=ax)).reshape(-1)

    def row_max_b(self):
        return self._absmax(self.b, self.b_legs)                        # [N]: max over k of max(|re|, |im|) of Bt[n, :]

    def row_max_a(self):
        return self._absmax(self.a, self.a_legs)                        # [M]

    def _sums(self, x, legs, absolute):
        ax = tuple(legs.index(l) for l in legs if l not in self.shared)
        s = np.abs(x).sum(axis=ax) if absolute else x.sum(axis=ax)
        left = [l for l in legs if l in self.shared]
        return np.transpose(s, [left.index(l) for l in self.shared]).reshape(-1)

    def checksums(self):
        """sum_{n,m} C = sum_k (sum_n Bt[n,k]) (sum_m At[k,m]), and the same with |.| (bounds sum |C|)"""
        return ((self._sums(self.b, self.b_legs, False) * self._sums(self.a, self.a_legs, False)).sum(),
                float((self._sums(self.b, self.b_legs, True) * self._sums(self.a, self.a_legs, True)).sum()))


def edge_sample(rng, n, count=16):
    idx = {i for i in (0, 63, 64, 127, 128, 255, 256, n - 1) if i < n}
    rest = [int(i) for i in rng.choice(n, size=min(n, count + len(idx)), replace=False) if int(i) not in idx]
    return np.array(sorted(idx) + rest[:max(0, count - len(idx))])


def ld_sample(v, rng):
    """(ns, ms, exact-ish entries, sum_k |Bt||At|) on an edges-included grid of at least 16 x 16 entries, in long double"""
    ns, ms = edge_sample(rng, v.N), edge_sample(rng, v.M)
    bt = v.bt_rows(ns).astype(np.clongdouble)
    at = v.at_cols(ms).astype(np.clongdouble).T
    return ns, ms, bt @ at, np.abs(bt) @ np.abs(at)


def check_fp64(got, v, ksplit, rng, full_limit=1 << 30):
    """FP64 bound, on the sampled grid against long double and, when M N K <= full_limit, on every entry against the
    oracle's FP64 GEMM (whose own error obeys the same bound, hence the factor 2)"""
    c = got.reshape(v.N, v.M)
    gamma = (2 * v.K + ksplit + 8) * U
    if v.M * v.N * v.K <= full_limit:
        _, ref = orc.contract_pair(v.a_legs, v.a, v.b_legs, v.b)
        ref = ref.reshape(v.N, v.M)
        bt, at = v.full()
        mag = np.abs(bt) @ np.abs(at)
        assert np.all(np.abs(c - ref) <= 2 * gamma * mag), float((np.abs(c - ref) / (gamma * mag)).max())
    ns, ms, ref, mag = ld_sample(v, rng)
    err = np.abs(c[np.ix_(ns, ms)] - ref)
    assert np.all(err <= gamma * mag), float((err / (gamma * mag)).max())


def check_int8(got, v, rng):
    """modular-engine bound on the sampled grid against long double, and the checksum of checksums over all of C"""
    import tnc_b200 as tb
    c = got.reshape(v.N, v.M)
    unit = tb.tcgen05_bound(v.K)["bound"]
    mb, ma = v.row_max_b(), v.row_max_a()
    ns, ms, ref, _ = ld_sample(v, rng)
    allowed = unit * (mb[ns][:, None] * ma[ms][None, :]).astype(np.longdouble)
    err = np.abs(c[np.ix_(ns, ms)] - ref)
    assert np.all(err <= allowed), float((err / allowed).max())
    checksum, p = v.checksums()
    total = c.sum()
    # every entry within its bound, plus the rounding of the two float64 sums (pairwise: well inside 64 u sum |C|)
    assert abs(total - checksum) <= unit * float(mb.sum()) * float(ma.sum()) + 64 * U * p, (total, checksum)


# ---- the dispatch of launch_k1, mirrored --------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def sm_count():
    try:
        import torch
        return torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:
        return SM_COUNT


TILES = {"64x64": (64, 64), "32x64": (32, 64), "64x32": (64, 32), "128x64": (128, 64)}   # (BN, BM)


def k1_config(M, N, variant=0):
    if variant == 1:
        return "128x64"
    if N <= 32 < M:
        return "32x64"
    if M <= 32 < N:
        return "64x32"
    return "64x64"


def k1_ksplit(cfg, M, N, K, sms):
    """launch_k1_modes: split K when there are fewer than 2 tiles per SM and at least 16 BK = 16 chunks"""
    bn, bm = TILES[cfg]
    tiles = -(-M // bm) * -(-N // bn)
    nk = -(-K // 16)
    if tiles >= 2 * sms or nk < 16:
        return 1
    ks = min(-(-2 * sms // tiles), nk // 8)
    ks = max(1, min(ks, (1 << 30) // 16 // max(1, M * N)))
    if ks <= 1:
        return 1
    per = -(-nk // ks)
    return -(-nk // per)


def pair_mnk(a_legs, a_dims, b_legs, b_dims):
    M = int(np.prod([d for l, d in zip(a_legs, a_dims) if l not in b_legs], dtype=np.int64))
    N = int(np.prod([d for l, d in zip(b_legs, b_dims) if l not in a_legs], dtype=np.int64))
    K = int(np.prod([d for l, d in zip(a_legs, a_dims) if l in b_legs], dtype=np.int64))
    return M, N, K


def int8_route(M, N, K):
    """default context: the modular engine for M, N >= 128, K >= 256 and M N K >= 2^28"""
    return M >= 128 and N >= 128 and K >= 256 and M * N * K >= (1 << 28)


# ---- K1 DMMA matrix -------------------------------------------------------------------------------------------------
MODES = [(True, True), (True, False), (False, True), (False, False)]
MODE_IDS = ["akf-bkf", "akf-bnf", "amf-bkf", "amf-bnf"]       # k-fast (kf) or free-index-fast (mf / nf) loader per operand
KS = [4, 8, 15, 16, 17, 143]
K_LEGS = {4: [2, 2], 8: [2, 4], 15: [3, 5], 16: [4, 4], 17: [17], 143: [11, 13], 1000: [8, 125], 777: [7, 111], 999: [27, 37]}
# (M, N): one row or column past a tile and one short of it; N (32x64) or M (64x32) in 16..24 fills only the first 8-row
# half of an m16n8k4 row pair (64x64: the last n tile holds 20 rows).  M N >= 2^15 keeps K = 4 on K1.
SHAPES = {"64x64": [(257, 191), (255, 148)], "32x64": [(2049, 20), (1025, 32)], "64x32": [(24, 1473), (31, 1087)]}
SPLIT = {"64x64": (200, 190, 1000), "32x64": (1000, 24, 777), "64x32": (20, 700, 999)}


def k1_pair(M, N, kdims, akf, bkf):
    """legs of a pair whose loader modes are set by leg order: a = [m, k...] is k-fast, [k..., m] row-fast; b likewise
    with n, and b lists the shared legs in reverse (a gathered, non-contiguous K)"""
    ks = [100 + i for i in range(len(kdims))]
    a_legs, a_dims = ([0] + ks, [M] + kdims) if akf else (ks + [0], kdims + [M])
    bk, bkd = ks[::-1], kdims[::-1]
    b_legs, b_dims = ([1] + bk, [N] + bkd) if bkf else (bk + [1], bkd + [N])
    return a_legs, a_dims, b_legs, b_dims


def k1_cases(cfg):
    """(M, N, K, integer inputs) of one tile config: every K on both shapes, the split-K case, and integer-valued inputs on
    the split-K case and on K = 143"""
    cases = [(M, N, K, False) for (M, N) in SHAPES[cfg] for K in KS]
    M, N, K = SPLIT[cfg]
    cases += [(M, N, K, False), (M, N, K, True), (*SHAPES[cfg][0], 143, True)]
    return cases


def run_k1_case(ctx, rng, M, N, K, akf, bkf, integer):
    import tnc_b200 as tb
    a_legs, a_dims, b_legs, b_dims = k1_pair(M, N, K_LEGS[K], akf, bkf)
    a = operand(rng, a_dims, [a_legs.index(0)], integer)
    b = operand(rng, b_dims, [b_legs.index(1)], integer)
    _, first = tb.contract_pair(ctx, a_legs, a, b_legs, b)              # builds the offset tables
    ctx.reset_stats()
    _, got = tb.contract_pair(ctx, a_legs, a, b_legs, b)
    return a_legs, a, b_legs, b, first, got


def check_k1_case(got, ec, launches, a_legs, a, b_legs, b, cfg, integer, rng, first=None):
    v = View(a_legs, a, b_legs, b)
    ks = k1_ksplit(cfg, v.M, v.N, v.K, sm_count())
    where = (cfg, v.M, v.N, v.K, ks, integer)
    assert ec["k1_dmma_splitk" if ks > 1 else "k1_dmma"] == 1 and sum(ec.values()) == 1, (where, ec)
    assert launches == 1 + (ks > 1), (where, launches)                 # k1_kernel (+ the split-K reduction)
    if first is not None:
        assert np.array_equal(got.view(np.float64), first.view(np.float64)), where     # deterministic, split-K included
    if integer:
        # |x| <= 2^10, K <= 2^12: every partial sum is an integer below 2^33, exact in any order and any split
        bt, at = v.full()
        btr, bti, atr, ati = (np.rint(x).astype(np.int64) for x in (bt.real, bt.imag, at.real, at.imag))
        exact = (btr @ atr - bti @ ati) + 1j * (btr @ ati + bti @ atr)
        assert np.array_equal(got.reshape(v.N, v.M), exact.astype(np.complex128)), where
    else:
        check_fp64(got, v, ks, rng)


@pytest.fixture(scope="module")
def dmma_ctx(built_lib):
    import tnc_b200 as tb
    c = tb.Context(0)
    c.set_tcgen05_slices(0)
    yield c
    c.close()


@pytest.mark.parametrize("mode", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("cfg", ["64x64", "32x64", "64x32"])
def test_k1_dmma_matrix(dmma_ctx, cfg, mode):
    """K1 tile config x loader modes: K = 4 .. 143 (one partial BK chunk up to nine), ragged M and N, a split-K case, and
    integer-valued inputs whose product is exact whatever the tiling."""
    akf, bkf = mode
    rng = np.random.default_rng(10 * list(SHAPES).index(cfg) + MODES.index(mode))
    for M, N, K, integer in k1_cases(cfg):
        assert k1_config(M, N) == cfg
        a_legs, a, b_legs, b, first, got = run_k1_case(dmma_ctx, rng, M, N, K, akf, bkf, integer)
        check_k1_case(got, dmma_ctx.engine_counts(), dmma_ctx.stats()["kernel_launches"], a_legs, a, b_legs, b, cfg,
                      integer, rng, first)


_VARIANT_CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import tnc_b200 as tb
d = sys.argv[2]
cases = json.load(open(d + "/cases.json"))
ctx = tb.Context(0)
ctx.set_tcgen05_slices(0)
stats = []
for i, c in enumerate(cases):
    z = np.load(f"{d}/in{i}.npz")
    _, first = tb.contract_pair(ctx, c["a_legs"], z["a"], c["b_legs"], z["b"])
    ctx.reset_stats()
    _, got = tb.contract_pair(ctx, c["a_legs"], z["a"], c["b_legs"], z["b"])
    np.savez(f"{d}/out{i}.npz", first=first, got=got)
    stats.append({"engines": ctx.engine_counts(), "launches": ctx.stats()["kernel_launches"]})
ctx.close()
json.dump(stats, open(d + "/stats.json", "w"))
"""


def test_k1_variant_128x64(built_lib, tmp_path):
    """TNCB_K1_VARIANT=1 (128x64 tiles, 4 stages) is read once per process: the same matrix runs in a child process over
    every loader mode, the skinny shapes included, and is checked here against the same references."""
    rng = np.random.default_rng(128)
    cases = []
    for mode in MODES:
        for M, N in SHAPES["64x64"] + [SHAPES["32x64"][0], SHAPES["64x32"][0]]:
            for K in (4, 15, 17, 143):
                cases.append((M, N, K, mode, False))
        cases.append((*SPLIT["64x64"], mode, False))
        cases.append((*SPLIT["32x64"], mode, True))
    meta = []
    for i, (M, N, K, (akf, bkf), integer) in enumerate(cases):
        a_legs, a_dims, b_legs, b_dims = k1_pair(M, N, K_LEGS[K], akf, bkf)
        a = operand(rng, a_dims, [a_legs.index(0)], integer)
        b = operand(rng, b_dims, [b_legs.index(1)], integer)
        np.savez(tmp_path / f"in{i}.npz", a=a, b=b)
        meta.append({"a_legs": a_legs, "b_legs": b_legs})
    (tmp_path / "cases.json").write_text(json.dumps(meta))
    env = dict(os.environ, TNCB_K1_VARIANT="1")
    r = subprocess.run([sys.executable, "-s", "-c", _VARIANT_CHILD, ROOT, str(tmp_path)], env=env, timeout=600,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    assert r.returncode == 0, r.stdout.decode()[-4000:]
    stats = json.loads((tmp_path / "stats.json").read_text())
    assert len(stats) == len(cases)
    for i, (M, N, K, mode, integer) in enumerate(cases):
        z_in, z_out = np.load(tmp_path / f"in{i}.npz"), np.load(tmp_path / f"out{i}.npz")
        check_k1_case(z_out["got"], stats[i]["engines"], stats[i]["launches"], meta[i]["a_legs"], z_in["a"],
                      meta[i]["b_legs"], z_in["b"], "128x64", integer, rng, z_out["first"])


# ---- the benchmark network's own pairs ------------------------------------------------------------------------------
N_BENCH_PAIRS = 29


@pytest.fixture(scope="module")
def bench_pairs(built_lib):
    """bench.py's network (random_circuit(36, 10, 0.5, 0.5, seed 1), greedy Cotengrust path), the path replayed on leg
    metadata; the steps tncb_pair_kernel_class puts in class 1 (K1 / K1') or 2 (K2) as (a legs, a dims, b legs, b dims)."""
    from tnc_b200._lib import u64_array
    from tnc_b200.builders import random_circuit
    from tnc_b200.contractionpath.paths import Cotengrust
    tn = random_circuit(36, 10, 0.5, 0.5, np.random.default_rng(1))
    opt = Cotengrust(tn)
    opt.find_path()
    path = opt.get_best_replace_path()
    assert not path.nested
    ts = [(list(t.legs), list(t.bond_dims)) for t in tn.tensors]
    out = []
    for i, j in path.toplevel:
        (al, ad), (bl, bd) = ts[i], ts[j]
        cls = built_lib.tncb_pair_kernel_class(len(al), u64_array(al), u64_array(ad), len(bl), u64_array(bl), u64_array(bd))
        if cls in (1, 2):
            out.append((cls, al, ad, bl, bd))
        ts[i] = ([l for l in bl if l not in al] + [l for l in al if l not in bl],
                 [d for l, d in zip(bl, bd) if l not in al] + [d for l, d in zip(al, ad) if l not in bl])
        ts[j] = None
    return out


def test_bench_network_pair_inventory(bench_pairs):
    """29 GEMM-like steps today: 6 on the modular int8 engine, 23 on K1 DMMA (one split-K, two on 32x64 tiles)."""
    shapes = [pair_mnk(al, ad, bl, bd) for _, al, ad, bl, bd in bench_pairs]
    assert len(bench_pairs) == N_BENCH_PAIRS and all(c == 1 for c, *_ in bench_pairs)
    dmma = [(M, N, K) for M, N, K in shapes if not int8_route(M, N, K)]
    n_split = sum(k1_ksplit(k1_config(M, N), M, N, K, sm_count()) > 1 for M, N, K in dmma)
    assert (len(shapes) - len(dmma), len(dmma), n_split) == (6, 23, 1)
    assert sum(k1_config(M, N) == "32x64" for M, N, K in dmma) == 2   # the two M = 1024, N = 32, K = 32 steps


@pytest.mark.parametrize("idx", range(N_BENCH_PAIRS))
def test_bench_network_pair(bench_pairs, idx):
    """One GEMM-like step of the benchmark network with its exact legs and dims, on random operands, through
    contract_pair with the default engine choice.  Pairs with M N K <= 2^30 are checked on every entry, larger ones on an
    edges-included sample of >= 256 entries and by the checksum of checksums.  The largest, 65536 x 4096 x 2048, holds
    2 GiB of A and 4 GiB of C on the host; with the temporaries of the checks this test peaks at about 8 GiB of host
    memory (the split-K pair, 256 x 64 x 2^20, holds 4 GiB of A and 1 GiB of B)."""
    import tnc_b200 as tb
    cls, al, ad, bl, bd = bench_pairs[idx]
    rng = np.random.default_rng(1000 + idx)
    a = operand(rng, ad, [i for i, l in enumerate(al) if l not in bl])
    b = operand(rng, bd, [i for i, l in enumerate(bl) if l not in al])
    v = View(al, a, bl, b)
    ctx = tb.Context(0)                                                 # fresh: the offset tables are built once here
    try:
        _, got = tb.contract_pair(ctx, al, a, bl, b)
        ec, launches = ctx.engine_counts(), ctx.stats()["kernel_launches"]
        info = ctx.last_tcgen05_info()
    finally:
        ctx.close()
    where = (idx, v.M, v.N, v.K)
    if int8_route(v.M, v.N, v.K):
        assert ec["k1_tcgen05"] == 1 and sum(ec.values()) == 1, (where, ec)
        assert info["n_moduli"] == tb.tcgen05_bound(v.K)["n_moduli"], (where, info)
        assert info["products"] == (3 if v.K >= 2048 else 4), (where, info)
        if (v.M, v.N, v.K) == (65536, 4096, 2048):
            assert launches > 7, (where, launches)                     # panels: the residue workspace exceeds 12 GiB
        else:
            assert launches == 7, (where, launches)                    # tables + 2 row-max + 2 residue + GEMM + reconstruction
        check_int8(got, v, rng)
    else:
        cfg = k1_config(v.M, v.N)
        ks = k1_ksplit(cfg, v.M, v.N, v.K, sm_count())
        assert ec["k1_dmma_splitk" if ks > 1 else "k1_dmma"] == 1 and sum(ec.values()) == 1, (where, cfg, ec)
        assert launches == 2 + (ks > 1), (where, cfg, launches)       # tables + k1_kernel (+ split-K reduction)
        check_fp64(got, v, ks, rng)
        if v.M * v.N * v.K > (1 << 30):
            checksum, p = v.checksums()
            gamma = (2 * v.K + ks + 8) * U
            assert abs(got.sum() - checksum) <= (gamma + 64 * U) * p, where
