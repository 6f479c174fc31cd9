"""tnc_b200 -- H100-native pairwise tensor-contraction hot path of qc-tum/TNC.

Host-side mirror (Python, over the C ABI in include/tncb.h) of the reference's interface for
this path: `tensornetwork.tensor.Tensor`, `tensornetwork.tensordata.TensorData`,
`contractionpath.ContractionPath`, `tensornetwork.contraction.contract_tensor_network`,
`builders.circuit_builder.Circuit` / `Permutor`, and `dist.communication` for the
partitioned fan-in (tnc::mpi::communication).  All numerics run in libtncb200 (CUDA, sm_90a);
nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from ._lib import TncbError, check, lib, u64_array

__all__ = ["Context", "DeviceTensor", "Expectation", "PauliSum", "Sampler", "Samples", "TncbError", "contract_pair", "contract_pair_into", "default_context",
           "lib"]


class Context:
    """One device + stream + arena (tncb_ctx)."""

    def __init__(self, device: int = 0, arena_bytes: int = 0):
        self._l = lib()
        h = C.c_void_p()
        check(self._l.tncb_ctx_create(device, arena_bytes, C.byref(h)))
        self.handle = h
        self.device = device

    def synchronize(self) -> None:
        check(self._l.tncb_ctx_synchronize(self.handle))

    @property
    def stream(self) -> int:
        return int(self._l.tncb_ctx_stream(self.handle) or 0)

    def stats(self) -> dict:
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(self._l.tncb_ctx_stats(self.handle, C.byref(a), C.byref(b), C.byref(c)))
        return {"kernel_launches": a.value, "arena_peak_bytes": b.value, "arena_live_bytes": c.value}

    def set_tcgen05_slices(self, slices: int) -> None:
        """0: FP64 tensor pipe (DMMA) for every pair.  2..8: the int8 tensor-core engine (K1') takes large pairs."""
        check(self._l.tncb_ctx_set_tcgen05_slices(self.handle, int(slices)))

    def set_tcgen05_engine(self, engine: int) -> None:
        """0: modular (CRT) int8 engine (default).  1: the 7-bit digit-slicing engine of round 1."""
        check(self._l.tncb_ctx_set_tcgen05_engine(self.handle, int(engine)))

    def set_tolerance(self, rel: float) -> None:
        """Normwise tolerance of K1' (0 = full FP64 mantissa), see tncb.h."""
        check(self._l.tncb_ctx_set_tolerance(self.handle, float(rel)))

    def set_tcgen05_moduli(self, n: int) -> None:
        check(self._l.tncb_ctx_set_tcgen05_moduli(self.handle, int(n)))

    def trim(self) -> dict:
        """Give unused arena slabs back to the driver (tncb_ctx_trim)."""
        f, r = C.c_uint64(), C.c_uint64()
        check(self._l.tncb_ctx_trim(self.handle, C.byref(f), C.byref(r)))
        return {"freed_bytes": f.value, "reserved_bytes": r.value}

    def set_tcgen05_products(self, products: int = 0, min_k3: int = 0) -> None:
        """3 / 4 real int8 products per complex product (0 = by K), see tncb.h; both forms give identical bits."""
        check(self._l.tncb_ctx_set_tcgen05_products(self.handle, int(products), int(min_k3)))

    def set_tcgen05_workspace(self, nbytes: int) -> None:
        check(self._l.tncb_ctx_set_tcgen05_workspace(self.handle, int(nbytes)))

    def engine_counts(self) -> dict:
        arr = (C.c_uint64 * 8)()
        check(self._l.tncb_ctx_engine_counts(self.handle, arr))
        names = ["k0", "k0_splitk", "k1_dmma", "k1_dmma_splitk", "k1_tcgen05", "k2", "permute", "reserved"]
        return {n: int(arr[i]) for i, n in enumerate(names)}

    def last_tcgen05_info(self) -> dict:
        ops, n = C.c_double(), C.c_int()
        check(self._l.tncb_ctx_last_tcgen05_info(self.handle, C.byref(ops), C.byref(n)))
        pr = C.c_int()
        check(self._l.tncb_ctx_last_tcgen05_products(self.handle, C.byref(pr)))
        return {"int8_ops": ops.value, "n_moduli": n.value, "products": pr.value}

    def set_tcgen05_threshold(self, min_tiles: int, min_k: int) -> None:
        check(self._l.tncb_ctx_set_tcgen05_threshold(self.handle, int(min_tiles), int(min_k)))

    def time_gemm(self, enable=True) -> None:
        """False/0 off, True/1 last launch of the dominant GEMM kernel, 2 accumulate every int8 GEMM launch."""
        check(self._l.tncb_ctx_time_gemm(self.handle, int(enable)))

    def gemm_totals(self) -> dict:
        ms, ops, n = C.c_double(), C.c_double(), C.c_uint64()
        check(self._l.tncb_ctx_gemm_totals(self.handle, C.byref(ms), C.byref(ops), C.byref(n)))
        return {"ms": ms.value, "int8_ops": ops.value, "launches": n.value}

    def last_gemm_ms(self) -> float:
        ms = C.c_float()
        check(self._l.tncb_ctx_last_gemm_ms(self.handle, C.byref(ms)))
        return float(ms.value)

    def reset_stats(self) -> None:
        check(self._l.tncb_ctx_reset_stats(self.handle))

    def close(self) -> None:
        if getattr(self, "handle", None):
            self._l.tncb_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


class DeviceTensor:
    """A device-resident complex128 tensor (tncb_tensor), row-major."""

    def __init__(self, ctx: Context, handle, shape: Sequence[int]):
        self.ctx = ctx
        self.handle = handle
        self.shape = tuple(int(s) for s in shape)

    @classmethod
    def from_numpy(cls, ctx: Context, arr: np.ndarray) -> "DeviceTensor":
        a = np.asarray(arr, dtype=np.complex128, order="C")  # (ascontiguousarray would promote 0-d to 1-d)
        h = C.c_void_p()
        check(ctx._l.tncb_tensor_upload(ctx.handle, a.ndim, u64_array(a.shape), a.ctypes.data_as(C.c_void_p), C.byref(h)))
        return cls(ctx, h, a.shape)

    @classmethod
    def empty(cls, ctx: Context, shape: Sequence[int]) -> "DeviceTensor":
        h = C.c_void_p()
        check(ctx._l.tncb_tensor_alloc(ctx.handle, len(shape), u64_array(shape), C.byref(h)))
        return cls(ctx, h, shape)

    @classmethod
    def adopt(cls, ctx: Context, handle) -> "DeviceTensor":
        l = ctx._l
        r = l.tncb_tensor_rank(handle)
        dims = u64_array([0] * max(r, 1))
        check(l.tncb_tensor_dims(handle, dims))
        return cls(ctx, handle, [dims[i] for i in range(r)])

    def to_numpy(self) -> np.ndarray:
        if self.handle is None:
            raise TncbError(-3, "Cannot convert uncontracted tensor to data")
        out = np.empty(self.shape, dtype=np.complex128)
        check(self.ctx._l.tncb_tensor_download(self.ctx.handle, self.handle, out.ctypes.data_as(C.c_void_p)))
        return out

    def device_ptr(self) -> int:
        return int(self.ctx._l.tncb_tensor_device_ptr(self.handle) or 0)

    def _torch_view(self):
        """float64 [elements, 2] torch view of the device memory (no copy; valid while this tensor lives)"""
        import torch
        elems = int(np.prod(self.shape, dtype=np.int64))
        return torch.as_tensor(_CudaArray(self.device_ptr(), elems), device=torch.device("cuda", self.ctx.device))

    def to_torch(self):
        """A torch complex128 tensor on the context's device with this tensor's shape: a device-to-device copy on the
        context stream, after the library's work there; torch's current stream waits for it."""
        import torch
        if self.handle is None:
            raise TncbError(-3, "Cannot convert uncontracted tensor to data")
        cur, ext = torch_streams(self.ctx)
        out = torch.empty(self.shape, dtype=torch.complex128, device=cur.device)
        if out.numel():
            ext.wait_stream(cur)                 # out's block may still be read or written by earlier torch work
            with torch.cuda.stream(ext):
                torch.view_as_real(out).view(-1, 2).copy_(self._torch_view())
            cur.wait_stream(ext)
        return out

    @classmethod
    def from_torch(cls, ctx: Context, t) -> "DeviceTensor":
        """A library tensor holding a copy of the torch CUDA tensor `t` (on the context's device; cast to complex128 on
        the device).  The copy runs on the context stream after torch's current stream, and torch's current stream then
        waits for it, so `t`'s memory is not handed to later work before the copy has read it."""
        import torch
        check_cuda_tensor(ctx, t, "the tensor")
        src = t.detach().to(torch.complex128).contiguous()
        out = cls.empty(ctx, tuple(src.shape))
        if src.numel():
            cur, ext = torch_streams(ctx)
            ext.wait_stream(cur)
            with torch.cuda.stream(ext):
                out._torch_view().copy_(torch.view_as_real(src).reshape(-1, 2))
            cur.wait_stream(ext)
        return out

    def release(self):
        """Give up ownership (the C side consumed the handle)."""
        h, self.handle = self.handle, None
        return h

    def free(self) -> None:
        if self.handle is not None and self.ctx.handle is not None:
            self.ctx._l.tncb_tensor_free(self.ctx.handle, self.handle)
        self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class _CudaArray:
    """__cuda_array_interface__ of `elems` complex128 at device address `ptr`, as float64 [elems, 2]"""

    def __init__(self, ptr: int, elems: int):
        self.__cuda_array_interface__ = {"shape": (elems, 2), "typestr": "<f8", "data": (ptr, False), "version": 3,
                                         "strides": None}


def torch_streams(ctx: Context):
    """(torch's current stream, the context stream as a torch stream) on the context's device"""
    import torch
    dev = torch.device("cuda", ctx.device)
    return torch.cuda.current_stream(dev), torch.cuda.ExternalStream(ctx.stream, device=dev)


def check_cuda_tensor(ctx: Context, t, what: str) -> None:
    """ValueError unless `t` is a torch tensor on the context's CUDA device"""
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError(f"{what} must be a torch CUDA tensor, got {type(t).__name__}"
                         + (f" on {t.device}" if isinstance(t, torch.Tensor) else ""))
    if t.device.index != ctx.device:
        raise ValueError(f"{what} is on {t.device}, the context on cuda:{ctx.device}")


def tcgen05_bound(k: int, rel: float = 0.0, n_moduli: int = 0) -> dict:
    """Host-only: what K1' does for contraction length k (tncb_tcgen05_bound)."""
    n, a, b, bd = C.c_int(), C.c_int(), C.c_int(), C.c_double()
    check(lib().tncb_tcgen05_bound(int(k), float(rel), int(n_moduli), C.byref(n), C.byref(a), C.byref(b), C.byref(bd)))
    return {"n_moduli": n.value, "bits_a": a.value, "bits_b": b.value, "bound": bd.value}


def tcgen05_tables(n_moduli: int) -> dict:
    """Host-only: moduli and split CRT weights of K1' (tncb_tcgen05_tables)."""
    m = (C.c_int * n_moduli)()
    r1, r2 = (C.c_double * n_moduli)(), (C.c_double * n_moduli)()
    lp = C.c_double()
    check(lib().tncb_tcgen05_tables(int(n_moduli), m, r1, r2, C.byref(lp)))
    return {"moduli": list(m), "rho1": list(r1), "rho2": list(r2), "log2_product": lp.value}


def contract_pair(ctx: Context, a_legs, a, b_legs, b):
    """tetra::contract equivalent for host arrays: returns (out_legs, ndarray).
    out legs = (b \\ a) ++ (a \\ b) (contraction.rs:64, tensor.rs:463-479)."""
    da = a if isinstance(a, DeviceTensor) else DeviceTensor.from_numpy(ctx, np.asarray(a))
    db = b if isinstance(b, DeviceTensor) else DeviceTensor.from_numpy(ctx, np.asarray(b))
    out_legs = [l for l in b_legs if l not in a_legs] + [l for l in a_legs if l not in b_legs]
    h = C.c_void_p()
    check(ctx._l.tncb_contract_pair(ctx.handle, len(out_legs), u64_array(out_legs),
                                    len(a_legs), u64_array(a_legs), da.handle,
                                    len(b_legs), u64_array(b_legs), db.handle, C.byref(h)))
    da.release(); db.release()
    out = DeviceTensor.adopt(ctx, h)
    return out_legs, out.to_numpy()


def contract_pair_into(ctx: Context, a_legs, da: DeviceTensor, b_legs, db: DeviceTensor, dc: DeviceTensor) -> None:
    """Device-resident pair into a pre-allocated output (operands stay alive); asynchronous on
    the context stream."""
    check(ctx._l.tncb_contract_pair_into(ctx.handle, len(a_legs), u64_array(a_legs), da.handle,
                                         len(b_legs), u64_array(b_legs), db.handle, dc.handle))


def contract_pair_host(ctx: Context, a_legs, a: np.ndarray, b_legs, b: np.ndarray, out: np.ndarray) -> None:
    """Pipelined host-buffer pair (tncb_contract_pair_host): asynchronous; `out` (C-contiguous complex128 with
    prod(out dims) elements, ideally pinned like a and b) is valid after ctx.synchronize()."""
    check(ctx._l.tncb_contract_pair_host(ctx.handle, len(a_legs), u64_array(a_legs), u64_array(a.shape), a.ctypes.data_as(C.c_void_p),
                                         len(b_legs), u64_array(b_legs), u64_array(b.shape), b.ctypes.data_as(C.c_void_p),
                                         out.ctypes.data_as(C.c_void_p)))


def upload_into(ctx: Context, host: np.ndarray, dst: DeviceTensor) -> None:
    """Asynchronous H2D of a (pinned) host array into an existing device tensor."""
    check(ctx._l.tncb_tensor_write(ctx.handle, dst.handle, host.ctypes.data_as(C.c_void_p)))


def download_into(ctx: Context, src: DeviceTensor, host: np.ndarray) -> None:
    """Asynchronous D2H into a (pinned) host array; synchronise the context before reading."""
    check(ctx._l.tncb_tensor_read(ctx.handle, src.handle, host.ctypes.data_as(C.c_void_p)))


from .sampling import Sampler, Samples  # noqa: E402  (needs Context and DeviceTensor above)
from .observables import Expectation, PauliSum, pauli_layer_matrix  # noqa: E402
