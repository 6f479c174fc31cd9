"""The modular int8 engine (csrc/crt.cu) is exact integer arithmetic up to its CRT reconstruction, so its output is a
function of the inputs alone: a change to the GEMM's pipeline (stage ring, stage depth, epilogue) must leave every output
bit unchanged.  Each case contracts one seeded pair through the engine and compares a SHA-256 digest of the complex128
output with tests/golden/crt_digests.json, recorded on an H100 by the library before its GEMM moved to 64-byte stages
and a register-only epilogue.  A loose comparison with numpy guards the fixture itself.

The cases cover both product forms; K with K % 128 in {1, 64, 65} (zero padding inside the last 128-byte block, at and
after a 64-byte stage boundary); K long enough for several K chunks, and a split-K case; M and N at a tile edge +- 1; a
panelled pair (small workspace); and pairs with many items per CTA whose stage count is not a multiple of the ring depth,
so that items start at an offset within the ring.

Regenerate the fixture with the library that defines the expected bits:
    python tests/test_gpu_crt_pipeline.py --write tests/golden/crt_digests.json [--lib path/to/libtncb200.so]"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "crt_digests.json")

# name: (M, N, K, products, workspace bytes or 0 for the default)
CASES = {
    "p4_k129": (256, 256, 129, 4, 0),
    "p3_k192": (512, 256, 192, 3, 0),
    "p4_k321": (384, 128, 321, 4, 0),
    "p3_k2113": (256, 384, 2113, 3, 0),
    "p4_k2112": (384, 256, 2112, 4, 0),
    "p3_edges_m255_n129": (255, 129, 1024, 3, 0),
    "p3_edges_m257_n255": (257, 255, 640, 3, 0),
    "p4_edges_m129_n257": (129, 257, 640, 4, 0),
    "p4_edges_m383_n129": (383, 129, 448, 4, 0),
    "p4_kchunks_k33000": (128, 128, 33000, 4, 0),
    "p3_kchunks_k33000": (256, 128, 33000, 3, 0),
    "p4_splitk": (256, 256, 4096, 4, 0),
    "p3_splitk": (256, 256, 4160, 3, 0),
    "p4_panels": (1024, 512, 512, 4, 8 << 20),
    "p3_panels": (1024, 512, 576, 3, 8 << 20),
    "p4_wrap_k704": (1024, 1024, 704, 4, 0),
    "p3_wrap_k704": (1024, 1024, 704, 3, 0),
    "p3_wrap_k1088": (1536, 512, 1088, 3, 0),
}


def operands(name, M, N, K):
    rng = np.random.default_rng(int.from_bytes(hashlib.sha256(name.encode()).digest()[:4], "little"))
    a = rng.standard_normal((K, M)) + 1j * rng.standard_normal((K, M))
    b = rng.standard_normal((N, K)) + 1j * rng.standard_normal((N, K))
    return a, b


def run_case(tb, ctx, name):
    """(digest of the output, rel. error against numpy, products used, number of int8 GEMM launches)"""
    M, N, K, products, ws = CASES[name]
    a, b = operands(name, M, N, K)
    ctx.set_tcgen05_products(products)
    ctx.set_tcgen05_workspace(ws if ws else 12 << 30)
    ctx.time_gemm(2)
    before = ctx.engine_counts()["k1_tcgen05"]
    legs, got = tb.contract_pair(ctx, [0, 1], a, [2, 0], b)
    launches = ctx.gemm_totals()["launches"]
    ctx.time_gemm(0)
    assert ctx.engine_counts()["k1_tcgen05"] == before + 1, f"{name} did not take the int8 engine"
    assert legs == [2, 1], legs
    got = np.ascontiguousarray(got, dtype=np.complex128)
    ref = b @ a
    err = float(np.abs(got - ref).max() / np.abs(ref).max())
    return hashlib.sha256(got.tobytes()).hexdigest(), err, ctx.last_tcgen05_info()["products"], launches


def make_ctx(tb):
    ctx = tb.Context(0)
    ctx.set_tcgen05_slices(8)
    ctx.set_tcgen05_threshold(1, 128)   # every pair with M, N >= 128 and K >= 128 takes the int8 engine
    return ctx


@pytest.fixture(scope="module")
def crt_ctx(built_lib):
    import tnc_b200 as tb
    c = make_ctx(tb)
    yield c
    c.close()


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_crt_output_bits(crt_ctx, golden, name):
    import tnc_b200 as tb
    digest, err, products, launches = run_case(tb, crt_ctx, name)
    assert products == CASES[name][3]
    assert err < 1e-12, err
    if CASES[name][4]:
        assert launches > 1, "the small workspace should split the pair into panels"
    assert digest == golden[name]["sha256"], f"{name}: output bits differ from the recorded ones"


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", required=True, help="JSON file for the digests")
    ap.add_argument("--lib", default=None, help="libtncb200.so to record (default: the tree's own build)")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import tnc_b200 as tb
    import tnc_b200._lib as tl
    if a.lib:
        tl.LIB_PATH = os.path.abspath(a.lib)
    ctx = make_ctx(tb)
    out = {}
    for name in CASES:
        digest, err, products, launches = run_case(tb, ctx, name)
        out[name] = {"sha256": digest, "rel_err_vs_numpy": err, "products": products, "gemm_launches": launches}
        print(name, out[name], flush=True)
    with open(a.write, "w") as f:
        json.dump({"library": tb.lib().tncb_version().decode(), "cases": out}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
