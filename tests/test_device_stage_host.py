"""Device staging without a GPU: the two entry points are declared with the signatures the header gives them, and torch
payloads that are not CUDA tensors are refused in Python before the library is called."""
import ctypes as C
import os
import re
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# C parameter types of include/tncb.h -> the ctypes the binding declares
CTYPES = {"tncb_ctx*": C.c_void_p, "tncb_plan*": C.c_void_p, "size_t": C.c_size_t, "const uint64_t*": "u64p",
          "const void* const*": "vpp", "const tncb_tn*": "tn*"}


def header_params(name):
    with open(os.path.join(ROOT, "include", "tncb.h")) as f:
        text = f.read()
    m = re.search(r"int\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    return [re.sub(r"\s*\w+$", "", p).replace(" *", "*") for p in params]


@pytest.mark.parametrize("name", ["tncb_plan_set_leaves", "tncb_plan_stage_instances"])
def test_signatures_match_header(name):
    from tnc_b200._lib import SIGNATURES, TncbTn, u64p, vpp
    resolve = {"u64p": u64p, "vpp": vpp, "tn*": C.POINTER(TncbTn)}
    want = [resolve.get(CTYPES[p], CTYPES[p]) for p in header_params(name)]
    res, args = SIGNATURES[name]
    assert res is C.c_int
    assert args == want, (args, want)


def test_cpu_payloads_refused():
    torch = pytest.importorskip("torch")
    from tnc_b200 import check_cuda_tensor
    from tnc_b200.tensornetwork.contraction import _device_sources
    ctx = types.SimpleNamespace(device=0)
    with pytest.raises(ValueError, match="CUDA"):
        check_cuda_tensor(ctx, torch.zeros(2, dtype=torch.complex128), "x")
    with pytest.raises(ValueError, match="CUDA"):
        check_cuda_tensor(ctx, [0.0, 1.0], "x")
    with pytest.raises(ValueError, match="CUDA"):
        _device_sources(ctx, [(2,)], {0: torch.zeros(2, dtype=torch.complex128)})
    with pytest.raises(IndexError):
        _device_sources(ctx, [(2,)], {1: torch.zeros(2, dtype=torch.complex128)})
