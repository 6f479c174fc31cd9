"""contract_tensor_network (tnc/src/tensornetwork/contraction.rs:30-52) over the C ABI.

The Python side only marshals the `Tensor` tree and the `ContractionPath` into the plain C
structs of include/tncb.h; schedule construction, leaf materialisation, the single host->device
upload and every pair kernel run inside libtncb200."""
from __future__ import annotations

import ctypes as C
import math
import os
from itertools import chain
from typing import List, Optional

import numpy as np

from .. import Context, DeviceTensor, default_context
from .._lib import TncbError, TncbPath, TncbTn, check, u64_array
from ..contractionpath import ContractionPath
from .tensor import Tensor
from .tensordata import TensorData

_KIND = {"uncontracted": 0, "matrix": 1, "gate": 2, "device": 3}


# TncbTn as a numpy record (same layout as the ctypes Structure / the C struct): a composite's children are filled
# column-wise instead of one ctypes object per leaf (the 36-qubit bench network has 489 leaves per call)
_TN_DTYPE = np.dtype([("n_children", np.uint64), ("children", np.uint64), ("rank", np.int32), ("legs", np.uint64), ("dims", np.uint64),
                      ("kind", np.int32), ("host_re_im", np.uint64), ("gate_name", np.uint64), ("gate_angles", np.uint64),
                      ("n_gate_angles", np.int32), ("gate_adjoint", np.int32), ("device", np.uint64),
                      ("file_path", np.uint64), ("file_adjoint", np.int32)], align=True)
assert _TN_DTYPE.itemsize == C.sizeof(TncbTn), "TncbTn layout drifted"
_GATE_NAMES = {}


def _gate_name_ptr(name: str) -> int:
    hit = _GATE_NAMES.get(name)
    if hit is None:
        buf = C.create_string_buffer(name.encode())                         # interned: stays alive for the process
        hit = _GATE_NAMES[name] = (C.addressof(buf), buf)
    return hit[0]


class _Marshal:
    """Keeps every buffer the C tree points to alive for the duration of the call."""

    def __init__(self):
        self.keep: List[object] = []
        self.device_inputs: List[DeviceTensor] = []

    def _children(self, tensors) -> int:
        """array of TncbTn for `tensors`; returns its address"""
        n = len(tensors)
        rec = np.zeros(n, dtype=_TN_DTYPE)
        self.keep.append(rec)
        ranks = [len(t.legs) for t in tensors]
        tot = sum(ranks)
        legs = np.fromiter(chain.from_iterable(t.legs for t in tensors), dtype=np.uint64, count=tot)
        dims = np.fromiter(chain.from_iterable(t.bond_dims for t in tensors), dtype=np.uint64, count=tot)
        self.keep += [legs, dims]
        off = np.zeros(n, dtype=np.uint64)
        if n > 1:
            np.cumsum(np.asarray(ranks[:-1], dtype=np.uint64), out=off[1:])
        rec["legs"] = legs.ctypes.data + 8 * off
        rec["dims"] = dims.ctypes.data + 8 * off
        # one pass over the leaves into plain lists, one column assignment per field (a numpy record setitem or an
        # ndarray.ctypes access per leaf costs more than everything else in this function)
        kind, n_children, children = [0] * n, [0] * n, [0] * n
        host, device, gate_name, gate_adj, gate_ang, n_ang = [0] * n, [0] * n, [0] * n, [0] * n, [0] * n, [0] * n
        file_path, file_adj = [0] * n, [0] * n
        ang_vals: List[float] = []
        for i, t in enumerate(tensors):
            if t.tensors:
                n_children[i] = len(t.tensors)
                children[i] = self._children(t.tensors)
                ranks[i] = 0
                continue
            td = t.tensordata
            k = td.kind
            if k == "gate":
                name, ang, adj = td.gate
                kind[i] = 2
                gate_name[i] = _gate_name_ptr(name)
                gate_adj[i] = int(adj)
                gate_ang[i] = 8 * len(ang_vals)        # byte offset into `angles`, made absolute below
                if ang:
                    n_ang[i] = len(ang)
                    ang_vals.extend(ang)
            elif k == "matrix":
                m = td.matrix
                if isinstance(m, DeviceTensor):
                    if m.handle is None:   # consumed by an earlier call (the Rust move left TensorData::Uncontracted behind)
                        raise TncbError(-3, "Cannot convert uncontracted tensor to data (device tensor already consumed)")
                    kind[i] = 3
                    device[i] = m.handle.value or 0
                    self.device_inputs.append(m)
                else:
                    arr = np.asarray(m, dtype=np.complex128, order="C")
                    if list(arr.shape) != list(t.bond_dims):
                        arr = arr.reshape(t.bond_dims)
                    self.keep.append(arr)
                    kind[i] = 1
                    host[i] = arr.__array_interface__["data"][0]
            elif k == "file":   # TensorData::File((path, adjoint)): loaded by the library while it stages the leaves
                buf = C.create_string_buffer(os.fsencode(td.file[0]))
                self.keep.append(buf)
                kind[i] = 4
                file_path[i] = C.addressof(buf)
                file_adj[i] = int(bool(td.file[1]))
        angles = np.zeros(max(len(ang_vals), 1), dtype=np.float64)
        angles[:len(ang_vals)] = ang_vals
        self.keep.append(angles)
        abase = angles.__array_interface__["data"][0]
        rec["rank"] = ranks
        rec["kind"] = kind
        rec["n_children"] = n_children
        rec["children"] = children
        rec["host_re_im"] = host
        rec["device"] = device
        rec["gate_name"] = gate_name
        rec["gate_adjoint"] = gate_adj
        rec["n_gate_angles"] = n_ang
        rec["gate_angles"] = [abase + o if kd == 2 else 0 for o, kd in zip(gate_ang, kind)]
        rec["file_path"] = file_path
        rec["file_adjoint"] = file_adj
        return rec.ctypes.data

    def tn(self, t: Tensor) -> TncbTn:
        addr = self._children([t])
        return TncbTn.from_address(addr)

    def path(self, p: ContractionPath) -> TncbPath:
        out = TncbPath()
        flat = [x for pair in p.toplevel for x in pair]
        pairs = u64_array(flat)
        self.keep.append(pairs)
        out.n_pairs = len(p.toplevel)
        out.pairs = pairs
        idx = sorted(p.nested)
        if idx:
            ni = u64_array(idx)
            arr = (TncbPath * len(idx))(*[self.path(p.nested[i]) for i in idx])
            self.keep += [ni, arr]
            out.n_nested = len(idx)
            out.nested_index = ni
            out.nested = arr
        return out


def contract_tensor_network(tn: Tensor, contract_path: ContractionPath, ctx: Optional[Context] = None) -> Tensor:
    """Fully contracts `tn` with the replace-left `contract_path`; returns the resulting
    leaf `Tensor` whose data stays on the device (`.to_numpy()` downloads it)."""
    ctx = ctx or default_context()
    m = _Marshal()
    c_tn = m.tn(tn)
    c_path = m.path(contract_path)
    return _leaf(*_contracted(ctx, "tncb_contract_tensor_network", C.byref(c_tn), C.byref(c_path), consumed=m.device_inputs))


def _contracted(ctx: Context, fn: str, *args, consumed=()):
    """ctx._l.<fn>(context, *args, out, n_out, legs), checked, for the entries that return a contracted tensor; the
    device leaves `consumed` are then given up (the call consumed them).  Returns (the result's legs, DeviceTensor or None
    when nothing is left)."""
    out, n_out, legs = C.c_void_p(), C.c_int(), u64_array([0] * 64)
    check(getattr(ctx._l, fn)(ctx.handle, *args, C.byref(out), C.byref(n_out), legs))
    for d in consumed:
        d.release()
    return [legs[i] for i in range(n_out.value)], (DeviceTensor.adopt(ctx, out) if out.value else None)


def _leaf(legs, dt: Optional[DeviceTensor]) -> Tensor:
    """the leaf Tensor with legs `legs` holding `dt`; an empty Tensor for None"""
    if dt is None:
        return Tensor()  # nothing left (empty network)
    res = Tensor(legs, dt.shape)
    res.set_tensor_data(TensorData.Matrix(dt))
    return res


def leaves(tn: Tensor) -> List[Tensor]:
    """The leaves of `tn` depth first, children in order: the leaf order that gradient plans' `wrt` and their gradients
    are indexed by."""
    if not tn.tensors:
        return [tn]
    return [leaf for child in tn.tensors for leaf in leaves(child)]


class PreparedNetwork:
    """A network marshalled once for the C ABI: the host template NetworkPlan.stage_instances can take call after call
    without walking the tree again.  The network's payloads are read by every call, so it must outlive its use."""

    def __init__(self, tn: Tensor):
        self._m = _Marshal()
        self.node = self._m.tn(tn)


def _device_sources(ctx: Context, shapes, payloads: dict, count: Optional[int] = None):
    """{leaf index: torch CUDA tensor} as (leaf indices, device addresses, instance strides in elements, the complex128
    tensors read).  count=None: one payload shaped like its leaf.  Else per instance, [count, *leaf shape] (its rows may
    lie further apart than a row's size: the stride is the tensor's own), or shared, [*leaf shape] (stride 0)."""
    import torch
    from .. import check_cuda_tensor
    idx, ptrs, strides, keep = [], [], [], []
    for leaf, x in payloads.items():
        leaf = int(leaf)
        if not 0 <= leaf < len(shapes):
            raise IndexError(f"leaf index {leaf} out of range ({len(shapes)} leaves)")
        check_cuda_tensor(ctx, x, f"the payload of leaf {leaf}")
        shape = tuple(shapes[leaf])
        elems = math.prod(shape)
        x = x.detach()
        # a lazily conjugated or negated view keeps its bit through .to and .contiguous, and its data_ptr is the
        # memory without it
        if x.dtype != torch.complex128 or x.is_conj() or x.is_neg():
            x = x.to(torch.complex128).resolve_conj().resolve_neg()
        if tuple(x.shape) == shape:
            src, stride = x.contiguous(), 0
        elif count is not None and tuple(x.shape) == (int(count),) + shape:
            src = x
            if count > 1 and src[0].is_contiguous() and src.stride(0) >= elems:
                stride = src.stride(0)
            else:
                src, stride = src.contiguous(), elems
        else:
            want = f"{shape}" if count is None else f"{(int(count),) + shape} or {shape}"
            raise ValueError(f"the payload of leaf {leaf} has shape {tuple(x.shape)}, expected {want}")
        idx.append(leaf)
        ptrs.append(src.data_ptr())
        strides.append(stride)
        keep.append(src)
    return idx, ptrs, strides, keep


def _download(blocks, convert: str = "to_numpy") -> list:
    """the DeviceTensors `blocks` converted by their method `convert` (host arrays; "to_torch": torch CUDA tensors), each
    freed; None stays None"""
    out = []
    for b in blocks:
        out.append(None if b is None else getattr(b, convert)())
        if b is not None:
            b.free()
    return out


def _addresses(ptrs):
    """device addresses as a C array (one null entry when there are none)"""
    return (C.c_void_p * max(len(ptrs), 1))(*ptrs)


def _call_after_torch(ctx: Context, keep, call) -> None:
    """`call()` (a library call that reads the torch tensors `keep` on the context stream) ordered after torch's current
    stream; torch's current stream then waits for the context stream, so the caching allocator cannot hand `keep`'s
    memory to later work before the library has read it (record_stream would tie the tensors to a stream that dies with
    the context)"""
    from .. import torch_streams
    cur, ext = torch_streams(ctx)
    ext.wait_stream(cur)
    try:
        check(call())
    finally:
        cur.wait_stream(ext)


def _library_call(ctx: Context, fn: str, args, outputs=(), keep=None, temps=()) -> list:
    """ctx._l.<fn>(*args, output pointers), checked; then `temps` are freed, whatever happened.  outputs: a flag per
    output pointer; the outputs come back as DeviceTensors, None where the flag is False.  keep: the torch tensors the call
    reads; the call is then ordered after torch's current stream (_call_after_torch)."""
    outs = [C.c_void_p() if want else None for want in outputs]
    call = lambda: getattr(ctx._l, fn)(*args, *[C.byref(o) if o is not None else None for o in outs])
    try:
        if keep is None:
            check(call())
        else:
            _call_after_torch(ctx, keep, call)
    finally:
        for t in temps:
            t.free()
    return [None if o is None else DeviceTensor.adopt(ctx, o) for o in outs]


class NetworkPlan:
    """Compile once / execute many (tncb_plan_*): same structure, new payloads."""

    def __init__(self, tn: Tensor, contract_path: ContractionPath, ctx: Optional[Context] = None):
        self._create("tncb_plan_create", tn, contract_path, ctx)

    @classmethod
    def for_gradients(cls, tn: Tensor, contract_path: ContractionPath, wrt=None, ctx: Optional[Context] = None) -> "NetworkPlan":
        """A gradient plan (tncb_plan_create_vjp): `stage` + `run` (or `execute`) contract the network as a plain plan
        does, then `vjp` returns the gradient of the result with respect to the leaves `wrt` (indices into
        `leaves(tn)`; None = every leaf with a payload) in one backward pass."""
        return cls._derivative_plan("tncb_plan_create_vjp", tn, contract_path, wrt, ctx)

    @classmethod
    def for_tangents(cls, tn: Tensor, contract_path: ContractionPath, wrt=None, ctx: Optional[Context] = None) -> "NetworkPlan":
        """A tangent plan (tncb_plan_create_jvp): after `stage`, `jvp` returns the result and its directional derivative
        along tangents of the leaves `wrt` (indices into `leaves(tn)`; None = every leaf with a payload) in one pass over
        the forward levels.  `stage_batch` / `stage_instances` + `jvp_batch` do the same for many networks, or for
        many directions of one network."""
        return cls._derivative_plan("tncb_plan_create_jvp", tn, contract_path, wrt, ctx)

    @classmethod
    def for_hvp(cls, tn: Tensor, contract_path: ContractionPath, wrt=None, ctx: Optional[Context] = None) -> "NetworkPlan":
        """A Hessian-vector plan (tncb_plan_create_hvp): after `stage`, `hvp` returns the result, its directional
        derivative, the gradient of the leaves `wrt` (indices into `leaves(tn)`; None = every leaf with a payload) and
        that gradient's directional derivative along leaf and seed tangents: Hessian-vector products, in one
        forward-over-reverse pass."""
        return cls._derivative_plan("tncb_plan_create_hvp", tn, contract_path, wrt, ctx)

    @classmethod
    def _derivative_plan(cls, create: str, tn: Tensor, contract_path: ContractionPath, wrt, ctx, *extra) -> "NetworkPlan":
        """a plan from the derivative creator `create`, called with `extra` (a sliced creator's legs) between the path and
        the mask of `wrt`"""
        self = cls.__new__(cls)
        self._create(create, tn, contract_path, ctx, *extra, wrt=wrt, masked=True)
        return self

    def _create(self, create: str, tn: Tensor, contract_path: ContractionPath, ctx, *extra, wrt=None, masked=False) -> None:
        """the plan from the creator `create`, called with `extra` after the path and, when `masked` (the derivative
        creators), the mask of the leaves `wrt` (None: no mask); then the result's legs and dims"""
        self.handle = None
        self.ctx = ctx or default_context()
        self.leaf_shapes = [tuple(int(d) for d in leaf.bond_dims) for leaf in leaves(tn)]
        mask = None
        if wrt is not None:
            mask = (C.c_uint8 * max(len(self.leaf_shapes), 1))()
            for i in wrt:
                if not 0 <= int(i) < len(self.leaf_shapes):
                    raise IndexError(f"leaf index {i} out of range ({len(self.leaf_shapes)} leaves)")
                mask[int(i)] = 1
        m = _Marshal()
        c_tn, c_path = m.tn(tn), m.path(contract_path)
        h = C.c_void_p()
        check(getattr(self.ctx._l, create)(self.ctx.handle, C.byref(c_tn), C.byref(c_path), *extra, *([mask] if masked else []),
                                           C.byref(h)))
        self.handle = h
        n_out, legs, dims = C.c_int(), u64_array([0] * 64), u64_array([0] * 64)
        check(self.ctx._l.tncb_network_out_legs(C.byref(c_tn), C.byref(c_path), C.byref(n_out), legs, dims))
        self.result_legs = [legs[i] for i in range(n_out.value)]
        self.result_dims = tuple(int(dims[i]) for i in range(n_out.value))

    def _call(self, fn: str, *args, inputs=(), payloads=None, outputs=(), keep=None) -> list:
        """_library_call of self.ctx._l.<fn>(context, plan, *args, *inputs, output pointers); DeviceTensors among `args`
        are passed as their handles.  inputs: (value, what, count) of the tensor arguments, converted in order by
        `_input`; what they upload is freed after the call, or when a later argument is refused.  payloads: ({leaf: torch
        CUDA tensor} or None, count) of a batched pass, checked after the inputs and passed before them as (n, leaf
        indices, addresses, instance strides), the call then ordered after torch's current stream."""
        tmp = []
        try:
            ts = [self._input(x, what, count, tmp) for x, what, count in inputs]
            if payloads is not None:
                p, count = payloads
                idx, ptrs, strides, keep = _device_sources(self.ctx, self.leaf_shapes, p, count) if p else ([], [], [], None)
                args += (len(idx), u64_array(idx), _addresses(ptrs), u64_array(strides))
        except BaseException:
            for t in tmp:
                t.free()
            raise
        return _library_call(self.ctx, fn, [self.ctx.handle, self.handle] + [a.handle if isinstance(a, DeviceTensor) else a
                                                                             for a in (*args, *ts)], outputs, keep, tmp)

    def _input(self, x, what: str, count: Optional[int], tmp: list):
        """The tensor argument `what` ("tangents", "seed", "seeds", "seed tangent" or "seed tangents") of a plan call as a
        DeviceTensor; None and DeviceTensors as they are (a DeviceTensor is checked by the library).  Tangents may be
        {leaf index: tangent}, packed by _tangent_block; else an array or torch CUDA tensor shaped like the tangent block
        [grad_elems] or like the result, after a leading `count` unless count is None, refused with ValueError before it
        is uploaded.  What is uploaded is appended to `tmp`."""
        one_pass_tangents = what == "tangents" and count is None
        if isinstance(x, DeviceTensor) or x is None and not one_pass_tangents:
            return x
        if isinstance(x, dict) or x is None:      # None as the tangents of one pass fails in the packing
            t = self._tangent_block(x, count)
        else:
            if what == "tangents":
                dims = (sum(math.prod(s) for off, s in zip(self.grad_offsets(), self.leaf_shapes) if off >= 0),)
            else:
                dims = tuple(self.result_dims)
            shape = dims if count is None else (int(count),) + dims
            on_device = type(x).__module__.split(".")[0] == "torch"
            if not on_device:
                x = np.asarray(x, dtype=np.complex128)
            if tuple(x.shape) != shape:
                raise ValueError(f"the {what} have shape {tuple(x.shape)}, expected {shape}" if what.endswith("s") else
                                 f"the {what} has shape {tuple(x.shape)}, the result {shape}")
            t = DeviceTensor.from_torch(self.ctx, x) if on_device else DeviceTensor.from_numpy(self.ctx, x)
        tmp.append(t)
        return t

    def _staged(self, count: int, fn: str, *args, keep=None) -> None:
        """`fn` stages `count` networks of the plan's structure: the batched calls run them"""
        self._call(fn, *args, keep=keep)
        self.n_staged = count

    def _count(self, first: int, count: Optional[int]) -> int:
        """count, or for None the staged networks from `first` on"""
        return max(0, getattr(self, "n_staged", 0) - int(first)) if count is None else int(count)

    def grad_offsets(self) -> List[int]:
        """Element offset of every leaf's gradient in the block `vjp` downloads, -1 for leaves not requested."""
        offs = (C.c_int64 * max(len(self.leaf_shapes), 1))()
        check(self.ctx._l.tncb_plan_grad_offsets(self.handle, offs))
        return [offs[i] for i in range(len(self.leaf_shapes))]

    def vjp(self, seed=None) -> dict:
        """After a forward `run`/`execute` of a gradient plan: {leaf index: G} for every requested leaf, G shaped like
        the leaf with G[e] = sum_r seed[r] dR[r]/dX[e] (no conjugation).  seed: array, torch CUDA tensor or DeviceTensor
        with the result's shape; None for a scalar result (seed 1).  One device-to-host copy of the whole gradient block."""
        (flat,) = _download([self.vjp_block(seed)])
        return self._unpack(self.grad_offsets(), flat, ())

    def vjp_block(self, seed=None) -> DeviceTensor:
        """`vjp` left on the device: the rank-1 block of every requested leaf's G at grad_offsets()"""
        return self._call("tncb_plan_vjp", inputs=[(seed, "seed", None)], outputs=(True,))[0]

    def _tangent_block(self, tangents: dict, count: Optional[int] = None) -> DeviceTensor:
        """{leaf index: tangent} packed at grad_offsets() into a [tangent_elems] (count=None) or [count, tangent_elems]
        block on the device; leaves left out have zero tangent.  A tangent is shaped like its leaf (with count: shared by
        every instance) or, with count, [count, *leaf shape].  Any torch CUDA tensor among them: packed by torch on the
        context's device (host arrays are uploaded first), nothing goes through the host; else packed on the host, one
        upload."""
        offs = self.grad_offsets()
        sizes = [int(np.prod(s, dtype=np.int64)) for s in self.leaf_shapes]
        elems = sum(sz for off, sz in zip(offs, sizes) if off >= 0)
        lead = () if count is None else (int(count),)
        on_device = any(type(x).__module__.split(".")[0] == "torch" for x in tangents.values())
        if on_device:
            import torch
            from .. import check_cuda_tensor
            block = torch.zeros(lead + (elems,), dtype=torch.complex128, device=torch.device("cuda", self.ctx.device))
        else:
            block = np.zeros(lead + (elems,), dtype=np.complex128)
        for leaf, x in tangents.items():
            leaf = int(leaf)
            if not 0 <= leaf < len(offs):
                raise IndexError(f"leaf index {leaf} out of range ({len(offs)} leaves)")
            if offs[leaf] < 0:
                raise ValueError(f"leaf {leaf} is not requested by this tangent plan")
            shape = tuple(self.leaf_shapes[leaf])
            if on_device:
                if isinstance(x, torch.Tensor):
                    check_cuda_tensor(self.ctx, x, f"the tangent of leaf {leaf}")
                    x = x.detach().to(torch.complex128)
                else:
                    x = torch.as_tensor(np.asarray(x, dtype=np.complex128), device=block.device)
            else:
                x = np.asarray(x, dtype=np.complex128)
            got = tuple(x.shape)
            if got != shape and (count is None or got != lead + shape):
                want = f"{shape}" if count is None else f"{lead + shape} or {shape}"
                raise ValueError(f"the tangent of leaf {leaf} has shape {got}, expected {want}")
            block[..., offs[leaf]:offs[leaf] + sizes[leaf]] = x.reshape(lead + (sizes[leaf],) if got != shape else (sizes[leaf],))
        return DeviceTensor.from_torch(self.ctx, block) if on_device else DeviceTensor.from_numpy(self.ctx, block)

    def jvp_block(self, tangents):
        """One forward-mode pass on the staged leaves (tncb_plan_jvp), left on the device: (value, tangent) DeviceTensors
        with the result's shape.  tangents: {leaf index: array or torch CUDA tensor shaped like the leaf}, requested
        leaves left out having zero tangent, or the tangents already packed at grad_offsets(): a [grad_elems] array,
        torch CUDA tensor or DeviceTensor (Angles.tangents).  The value equals a plain plan's run bit for bit; a call
        repeats bit for bit."""
        return tuple(self._call("tncb_plan_jvp", inputs=[(tangents, "tangents", None)], outputs=(True, True)))

    def _jvp_tangent(self, tangents) -> DeviceTensor:
        """jvp_block's tangent alone: the library is given no value output to fill"""
        return self._call("tncb_plan_jvp", inputs=[(tangents, "tangents", None)], outputs=(False, True))[1]

    def jvp(self, tangents):
        """`jvp_block` with the derivative downloaded: (value Tensor on the device with the result's legs, tangent
        ndarray), tangent[r] = sum_l sum_e dR[r]/dX_l[e] tangents[l][e] (no conjugation)."""
        val, tan = self.jvp_block(tangents)
        return _leaf(list(self.result_legs), val), _download([tan])[0]

    def hvp_blocks(self, tangents, seed=None, seed_tangent=None, outputs=(True, True, True, True)):
        """One forward-over-reverse pass on the staged leaves of a Hessian-vector plan (tncb_plan_hvp), left on the
        device: [value, tangent, grads, grad_tangents] as DeviceTensors, None where `outputs` is False.  value and
        tangent have the result's shape (R and Ṙ, as jvp_block); grads and grad_tangents are [grad_elems] blocks at
        grad_offsets() (G = vjp(seed) and Ġ, its derivative along the leaf tangents and the seed tangent).
        tangents: {leaf index: array or torch CUDA tensor shaped like the leaf}, requested leaves left out having zero
        tangent, or a packed [grad_elems] block as jvp_block takes it; seed / seed_tangent: array, torch CUDA tensor or
        DeviceTensor with the result's shape, seed None for a scalar result (seed 1), seed_tangent None = zero.  No
        conjugation anywhere; a call repeats bit for bit."""
        return self._hvp("tncb_plan_hvp", (), tangents, seed, seed_tangent, outputs)

    def _hvp(self, fn: str, lead, tangents, seed, seed_tangent, outputs) -> list:
        """the forward-over-reverse pass `fn` (tncb_plan_hvp, or a sliced one with lead = (rank, world))"""
        return self._call(fn, *lead, inputs=[(tangents, "tangents", None), (seed, "seed", None),
                                             (seed_tangent, "seed tangent", None)], outputs=outputs)

    def hvp(self, tangents, seed=None, seed_tangent=None):
        """`hvp_blocks` downloaded: (value, tangent, {leaf: G}, {leaf: Ġ}) as host arrays, value and tangent with the
        result's shape, G and Ġ shaped like their leaf, for every requested leaf.  Ġ_l = sum_r Ṡ[r] dR[r]/dX_l +
        sum_r S[r] sum_m d²R[r]/dX_l dX_m · Ẋ_m: with Ṡ = 0 that is the Hessian of sum_r S[r] R[r] times the tangents."""
        value, tangent, g, dg = _download(self.hvp_blocks(tangents, seed, seed_tangent))
        offs = self.grad_offsets()
        return value, tangent, self._unpack(offs, g, ()), self._unpack(offs, dg, ())

    def hvp_batch_blocks(self, count: int, tangents, seeds=None, seed_tangents=None, payloads: Optional[dict] = None,
                         outputs=(True,) * 6):
        """`count` forward-over-reverse passes in one walk over the levels (tncb_plan_hvp_batch), left on the device:
        [values, tangent_rows, grad_rows, grad_sum, grad_tangent_rows, grad_tangent_sum] as DeviceTensors, None where
        `outputs` is False.  Values and tangent rows are [count, *result dims] (R, Ṙ), the G / Ġ rows [count, grad_elems]
        at grad_offsets(), the sums [grad_elems] (the left fold of the rows in instance order).
        Instance i is the staged network, with payloads = {leaf: torch CUDA tensor [count, *leaf shape] (row i for
        instance i) or [*leaf shape] (shared)} replacing leaves from device memory.
        tangents: {leaf: [count, *leaf shape] or [*leaf shape]} as jvp_batch takes them, or an already packed
        [count, grad_elems] array, torch CUDA tensor or DeviceTensor (a Hessian block: np.eye(grad_elems)[rows]).
        seeds / seed_tangents: [count, *result dims] array, torch CUDA tensor or DeviceTensor; seeds None for a scalar
        result (every seed 1), seed_tangents None = zero.  Row i equals set_leaves(instance i's payloads) + hvp(tangent
        row i, seed i, seed tangent i) bit for bit; the plan's staged leaves are left as they are."""
        count = int(count)
        return self._call("tncb_plan_hvp_batch", count, inputs=[(tangents, "tangents", count), (seeds, "seeds", count),
                                                                (seed_tangents, "seed tangents", count)],
                          payloads=(payloads, count), outputs=outputs)

    def hvp_batch(self, count: int, tangents, seeds=None, seed_tangents=None, payloads: Optional[dict] = None,
                  outputs=(True,) * 6):
        """`hvp_batch_blocks` downloaded: (legs of one instance, values [count, *dims], tangent rows [count, *dims],
        {leaf: G rows [count, *leaf shape]}, {leaf: G sum}, {leaf: Ġ rows}, {leaf: Ġ sum}) as host arrays, None where
        not requested."""
        host = _download(self.hvp_batch_blocks(count, tangents, seeds, seed_tangents, payloads, outputs))
        offs = self.grad_offsets()
        rows, one = (int(count),), ()
        return (list(self.result_legs), host[0], host[1], self._unpack(offs, host[2], rows), self._unpack(offs, host[3], one),
                self._unpack(offs, host[4], rows), self._unpack(offs, host[5], one))

    def jvp_batch_blocks(self, first: int = 0, count: Optional[int] = None, tangents=None, values: bool = True):
        """`jvp_batch` left on the device: [values [count, *dims] or None, tangents [count, *dims]] as DeviceTensors"""
        count = self._count(first, count)
        return self._call("tncb_plan_jvp_batch", int(first), count, inputs=[({} if tangents is None else tangents, "tangents", count)],
                          outputs=(values, True))

    def jvp_batch(self, first: int = 0, count: Optional[int] = None, tangents=None, values: bool = True):
        """Forward mode over the staged networks first .. first + count - 1 (stage_batch / stage_instances), each with
        its own tangents, the instances a grid dimension of every kernel (tncb_plan_jvp_batch).  tangents: {leaf index:
        [count, *leaf shape] (a row per instance) or [*leaf shape] (the same for every instance)}, or the tangent rows
        already packed at grad_offsets(): a [count, grad_elems] array, torch CUDA tensor or DeviceTensor
        (Angles.tangents).  Returns (legs of one instance, values [count, *dims] or None, tangents [count, *dims]); row i
        equals jvp of instance i with its tangent rows, bit for bit.  Many directions of one network: stage_instances of
        it with count copies, one tangent row per direction."""
        vals, tans = _download(self.jvp_batch_blocks(first, count, tangents, values))
        return list(self.result_legs), vals, tans

    def set_leaves(self, payloads: dict) -> None:
        """New payloads for leaves of the staged network straight from device memory (tncb_plan_set_leaves): {leaf index
        (into leaves(tn)): torch CUDA tensor shaped like the leaf}, on the context's device, cast to complex128 there.
        One copy kernel on the context stream, after torch's current stream; the next run / vjp reads them.  A gradient
        plan needs a new run before vjp."""
        idx, ptrs, _, keep = _device_sources(self.ctx, self.leaf_shapes, payloads)
        self._set_leaves(idx, ptrs, keep)

    def _set_leaves(self, idx, ptrs, keep=None) -> None:
        """tncb_plan_set_leaves: the leaves `idx` from the device addresses `ptrs`; keep: the torch tensors they lie in"""
        self._call("tncb_plan_set_leaves", len(idx), u64_array(idx), _addresses(ptrs), keep=keep)

    def stage_instances(self, template, payloads: dict, count: int) -> None:
        """Stage `count` networks of the plan's structure from device memory (tncb_plan_stage_instances): every leaf from
        `template` (a Tensor of the plan's structure, or a PreparedNetwork of one), except the leaves in `payloads`,
        {leaf index: torch CUDA tensor}, [count, *leaf shape] for a payload per instance or [*leaf shape] for one shared
        by all.  The host work does not grow with count.  Plain plans: feeds run_slices / run_batch, as stage_slices does;
        gradient plans: feeds vjp_batch, as stage_batch does."""
        tmpl = template if isinstance(template, PreparedNetwork) else PreparedNetwork(template)
        self._stage_instances(tmpl, int(count), *_device_sources(self.ctx, self.leaf_shapes, payloads, int(count)))

    def _stage_instances(self, template: PreparedNetwork, count: int, idx, ptrs, strides, keep=None) -> None:
        """tncb_plan_stage_instances: `count` copies of `template` with the leaves `idx` from the device addresses `ptrs`,
        instance i at ptr + i * stride elements; keep: the torch tensors they lie in"""
        self._staged(count, "tncb_plan_stage_instances", C.byref(template.node), count, len(idx), u64_array(idx),
                     _addresses(ptrs), u64_array(strides), keep=keep)

    def stage_batch(self, nets) -> None:
        """Materialise + upload the leaves of many networks of a gradient plan's structure once (tncb_plan_stage_batch):
        bitstrings, angle sets or input states for `vjp_batch`.  The plan's own staged leaves stay as they are."""
        m = _Marshal()
        nodes = [m.tn(t) for t in nets]
        ptrs = (C.POINTER(TncbTn) * max(len(nodes), 1))(*[C.pointer(n) for n in nodes])
        self._staged(len(nodes), "tncb_plan_stage_batch", len(nodes), ptrs)

    def vjp_batch(self, first: int = 0, count: Optional[int] = None, seeds=None, rows: bool = True, sum: bool = False,
                  values: bool = True):
        """Forward and backward of the staged networks first .. first + count - 1, each on its own, the instances as a
        grid dimension of every kernel (tncb_plan_vjp_batch).  count=None: every staged network from `first` on.
        seeds: [count, *result dims] array, torch CUDA tensor or DeviceTensor; None for a scalar result (seed 1) or
        without gradients.  Returns (legs of one instance, values [count, *dims] or None, {leaf: [count, *leaf shape]} or
        None, {leaf: leaf-shaped sum over the instances} or None).  Row i equals stage(net_i) + run + vjp(seed_i) bit for
        bit; the sum is the left fold of the rows in instance order, also bit for bit."""
        count = self._count(first, count)
        vals, row_block, sum_block = _download(self.vjp_batch_blocks(first, count, seeds, rows, sum, values))
        offs = self.grad_offsets()
        return (list(self.result_legs), vals, self._unpack(offs, row_block, (count,)), self._unpack(offs, sum_block, ()))

    def _unpack(self, offs, block, lead):
        """{leaf: lead + leaf shape} views of a host block [*lead, grad_elems] at the offsets `offs`; None stays None"""
        if block is None:
            return None
        out = {}
        for i, (off, shape) in enumerate(zip(offs, self.leaf_shapes)):
            if off >= 0:
                size = int(np.prod(shape, dtype=np.int64))
                out[i] = block[..., off:off + size].reshape(lead + tuple(shape))
        return out

    def vjp_batch_blocks(self, first: int = 0, count: Optional[int] = None, seeds=None, rows: bool = True,
                         sum: bool = False, values: bool = True):
        """`vjp_batch` left on the device: [values [count, *dims], rows [count, grad_elems], sum [grad_elems]] as
        DeviceTensors, None where not requested"""
        count = self._count(first, count)
        return self._call("tncb_plan_vjp_batch", int(first), count, inputs=[(seeds, "seeds", count)], outputs=(values, rows, sum))

    def info(self) -> dict:
        n, k = C.c_uint64(), C.c_uint64()
        pk = C.c_uint64()
        fl, by = C.c_double(), C.c_double()
        check(self.ctx._l.tncb_plan_info(self.handle, C.byref(n), C.byref(fl), C.byref(by), C.byref(pk), C.byref(k)))
        return {"pairs": n.value, "flops": fl.value, "bytes": by.value, "peak_bytes": pk.value, "kernels": k.value}

    def stage(self, tn: Tensor) -> None:
        """Materialise + upload the leaves once (tncb_plan_stage); `run()` then needs no host data."""
        m = _Marshal()
        c_tn = m.tn(tn)
        self._call("tncb_plan_stage", C.byref(c_tn))

    def run(self) -> Tensor:
        return _leaf(*_contracted(self.ctx, "tncb_plan_run", self.handle))

    def stage_slices(self, slice_tns) -> None:
        """Materialise + upload the leaf blocks of many networks of the plan's structure once (tncb_plan_stage_slices):
        slices, other bitstrings or angle sets."""
        m = _Marshal()
        nodes = [m.tn(t) for t in slice_tns]
        ptrs = (C.POINTER(TncbTn) * len(nodes))(*[C.pointer(n) for n in nodes])
        self._staged(len(nodes), "tncb_plan_stage_slices", len(nodes), ptrs)

    def run_batch(self, first: int = 0, count: Optional[int] = None):
        """Contract the staged networks first .. first + count - 1 each on its own, the instances as a grid dimension of
        every kernel (tncb_plan_run_batch).  count=None: every staged network from `first` on.  Returns (legs of one
        instance, DeviceTensor of shape (count, *dims)); row i is bit-identical to run_slices(first + i, n_staged)."""
        return _contracted(self.ctx, "tncb_plan_run_batch", self.handle, int(first), self._count(first, count))

    def run_slices(self, first: int = 0, stride: int = 1) -> Tensor:
        """Sum of the slices first, first + stride, ... on the device, no host work per slice."""
        return _leaf(*_contracted(self.ctx, "tncb_plan_run_slices", self.handle, int(first), int(stride)))

    def execute(self, tn: Tensor) -> Tensor:
        m = _Marshal()
        c_tn = m.tn(tn)
        return _leaf(*_contracted(self.ctx, "tncb_plan_execute", self.handle, C.byref(c_tn), consumed=m.device_inputs))

    def __del__(self):
        try:
            if self.handle:
                self.ctx._l.tncb_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
