"""Slicing: the data-parallel mode the reference lists as future work
(book/src/future_work.md:9-11, book/src/parallelization.md:16-24).

Fixing the value of a leg that is summed over splits one contraction into dim(leg) independent
contractions of smaller networks whose results add up.  With S sliced legs of dimension 2 there are
2^S independent units: they bound the peak memory, and they shard over GPUs with a single
all-reduce at the end (`contract_sliced`).  The same replace-left path is used for every slice."""
from __future__ import annotations

import itertools
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from ..tensornetwork.tensor import Tensor
from ..tensornetwork.tensordata import TensorData
from . import ContractionPath


def _flat(tn: Tensor) -> List[Tensor]:
    assert all(t.is_leaf() for t in tn.tensors), "slicing works on flat networks"
    return tn.tensors


def path_cost(tensors: Sequence[Tuple[Sequence[int], Sequence[int]]], path: ContractionPath, sliced: Iterable[int] = ()):
    """(flops 8MNK summed, peak intermediate elements, legs of the largest intermediate) with the
    `sliced` legs removed."""
    sl = set(sliced)
    ts: List[Optional[Dict[int, int]]] = [{l: d for l, d in zip(legs, dims) if l not in sl} for legs, dims in tensors]
    flops, peak, peak_legs = 0.0, 0.0, []
    for (i, j) in path.toplevel:
        a, b = ts[i], ts[j]
        out = {l: d for l, d in b.items() if l not in a}
        out.update({l: d for l, d in a.items() if l not in b})
        f = 8.0
        for l, d in a.items():
            f *= d
        for l, d in b.items():
            if l not in a:
                f *= d
        flops += f
        sz = 1.0
        for d in out.values():
            sz *= d
        if sz > peak:
            peak, peak_legs = sz, list(out)
        ts[i], ts[j] = out, None
    return flops, peak, peak_legs


def path_time(tensors: Sequence[Tuple[Sequence[int], Sequence[int]]], path: ContractionPath, sliced: Iterable[int] = ()) -> float:
    """Predicted device seconds of one slice (contraction_cost.gpu_time_tensors per pair): unlike the flop count it
    sees that halving K of the dominant pair costs the int8 engine efficiency while halving M or N does not."""
    from ..tensornetwork.tensor import Tensor as _T
    from .contraction_cost import gpu_time_tensors
    sl = set(sliced)
    ts: List[Optional[_T]] = [_T([l for l in legs if l not in sl], [d for l, d in zip(legs, dims) if l not in sl]) for legs, dims in tensors]
    total = 0.0
    for (i, j) in path.toplevel:
        total += gpu_time_tensors(ts[i], ts[j])
        ts[i], ts[j] = ts[j] ^ ts[i], None
    return total


def find_slices(tn: Tensor, path: ContractionPath, min_slices: int = 1, max_peak_elements: Optional[float] = None,
                objective: str = "flops") -> List[int]:
    """Greedy slice finder: repeatedly slice the leg of the currently largest intermediate that
    minimises the total work (slices x flops, or slices x predicted device time with objective="time"), until there
    are at least `min_slices` slices and the largest intermediate has at most `max_peak_elements` elements.
    Output legs are never sliced."""
    leaves = _flat(tn)
    meta = [(t.legs, t.bond_dims) for t in leaves]
    count: Dict[int, int] = {}
    dim: Dict[int, int] = {}
    for legs, dims in meta:
        for l, d in zip(legs, dims):
            count[l] = count.get(l, 0) + 1
            dim[l] = d
    sliced: List[int] = []
    n_slices = 1
    while True:
        flops, peak, peak_legs = path_cost(meta, path, sliced)
        if n_slices >= min_slices and (max_peak_elements is None or peak <= max_peak_elements):
            return sliced
        cands = [l for l in peak_legs if count.get(l, 0) >= 2 and dim[l] > 1]
        if not cands:
            cands = [l for l in dim if count[l] >= 2 and dim[l] > 1 and l not in sliced]
        if not cands:
            return sliced
        best, best_cost = None, None
        for l in cands:
            f, p, _ = path_cost(meta, path, sliced + [l])
            if objective == "time":
                f = path_time(meta, path, sliced + [l])
            cost = (f * n_slices * dim[l], p)
            if best_cost is None or cost < best_cost:
                best, best_cost = l, cost
        sliced.append(best)
        n_slices *= dim[best]


def slice_assignments(tn: Tensor, legs: Sequence[int]) -> List[Tuple[int, ...]]:
    dim = {l: d for t in _flat(tn) for l, d in t.edges()}
    return list(itertools.product(*[range(dim[l]) for l in legs]))


def _leaf_array(t: Tensor) -> np.ndarray:
    td = t.tensordata
    if td.kind == "gate":
        from ..gates import load_gate, load_gate_adjoint
        name, angles, adj = td.gate
        return (load_gate_adjoint if adj else load_gate)(name, angles).reshape(t.bond_dims)
    if td.kind == "matrix":
        m = td.matrix
        return (m if isinstance(m, np.ndarray) else m.to_numpy()).reshape(t.bond_dims)
    raise RuntimeError("Cannot convert uncontracted tensor to data")


class SlicedNetwork:
    """Pre-extracts the leaves that contain sliced legs so that building slice number s is a few
    tiny numpy index operations; all other leaves are shared between slices."""

    def __init__(self, tn: Tensor, legs: Sequence[int]):
        self.tn, self.legs = tn, list(legs)
        self.leaves = list(_flat(tn))
        self.touched = {}
        for idx, t in enumerate(self.leaves):
            if any(l in t.legs for l in self.legs):
                self.touched[idx] = _leaf_array(t)
            elif t.tensordata.kind == "matrix" and not isinstance(t.tensordata.matrix, np.ndarray):
                # a device-resident leaf shared by every slice would be consumed by the first one:
                # download it once, every slice then uploads its own copy with the leaf block
                nt = Tensor(t.legs, t.bond_dims)
                nt.set_tensor_data(TensorData.Matrix(_leaf_array(t)))
                self.leaves[idx] = nt
        self.assignments = slice_assignments(tn, self.legs)

    def slice(self, assignment: Sequence[int]) -> Tensor:
        val = dict(zip(self.legs, assignment))
        out = []
        for idx, t in enumerate(self.leaves):
            if idx not in self.touched:
                out.append(t)
                continue
            arr = self.touched[idx]
            index = tuple(val[l] if l in val else slice(None) for l in t.legs)
            keep = [(l, d) for l, d in t.edges() if l not in val]
            nt = Tensor([l for l, _ in keep], [d for _, d in keep])
            nt.set_tensor_data(TensorData.Matrix(np.ascontiguousarray(arr[index])))
            out.append(nt)
        return Tensor.new_composite(out)


class SlicedPlan:
    """Compile + stage once, run many: the sliced contraction with every slice's leaf block resident on the device and
    the slice loop inside libtncb200 (tncb_plan_stage_slices / tncb_plan_run_slices)."""

    def __init__(self, tn: Tensor, path: ContractionPath, legs: Sequence[int], ctx=None):
        from .. import default_context
        from ..tensornetwork.contraction import NetworkPlan
        self.ctx = ctx or default_context()
        self.sn = SlicedNetwork(tn, legs)
        nets = [self.sn.slice(a) for a in self.sn.assignments]
        self.n_slices = len(nets)
        self.plan = NetworkPlan(nets[0], path, ctx=self.ctx)
        self.plan.stage_slices(nets)

    @classmethod
    def for_gradients(cls, tn: Tensor, path: ContractionPath, legs: Sequence[int], wrt=None, ctx=None) -> "SlicedPlan":
        """A sliced gradient plan (tncb_plan_create_vjp_sliced): compiled for the FULL network `tn` and the legs to slice;
        `stage(tn)` uploads the full leaves once, `run` sums the slices' results and `vjp` also returns every requested
        leaf's gradient in the full leaf's shape, each slice extracted and accumulated on the device.  wrt: indices into
        `leaves(tn)`; None = every leaf with a payload.  Slice q is the row-major digit vector of q over `legs`, last leg
        fastest (the order of `slice_assignments`)."""
        return cls._derivative("tncb_plan_create_vjp_sliced", tn, path, legs, wrt, ctx)

    @classmethod
    def for_tangents(cls, tn: Tensor, path: ContractionPath, legs: Sequence[int], wrt=None, ctx=None) -> "SlicedPlan":
        """A sliced tangent plan (tncb_plan_create_jvp_sliced), built like `for_gradients`: after `stage(tn)`, `jvp`
        returns the sum of the slices' results and of their directional derivatives along full-shape leaf tangents, each
        slice's tangents extracted on the device.  `run` sums the slices' results."""
        return cls._derivative("tncb_plan_create_jvp_sliced", tn, path, legs, wrt, ctx)

    @classmethod
    def for_hvp(cls, tn: Tensor, path: ContractionPath, legs: Sequence[int], wrt=None, ctx=None) -> "SlicedPlan":
        """A sliced Hessian-vector plan (tncb_plan_create_hvp_sliced), built like `for_gradients`: after `stage(tn)`,
        `hvp` returns R, Ṙ and every requested leaf's G and Ġ in the full leaf's shape, summed over the slices, each
        slice's forward-over-reverse pass on the device.  `run` sums the slices' results."""
        return cls._derivative("tncb_plan_create_hvp_sliced", tn, path, legs, wrt, ctx)

    @classmethod
    def _derivative(cls, create: str, tn: Tensor, path: ContractionPath, legs: Sequence[int], wrt, ctx) -> "SlicedPlan":
        from .. import default_context
        from .._lib import u64_array
        from ..tensornetwork.contraction import NetworkPlan, leaves
        self = cls.__new__(cls)
        self.ctx = ctx or default_context()
        self.sn = None
        legs = [int(l) for l in legs]
        self.plan = NetworkPlan._derivative_plan(create, tn, path, wrt, self.ctx, len(legs), u64_array(legs or [0]))
        dim = {l: int(d) for t in leaves(tn) for l, d in zip(t.legs, t.bond_dims)}
        self.n_slices = int(np.prod([dim[l] for l in legs], dtype=object)) if legs else 1
        return self

    def stage(self, tn: Tensor) -> None:
        """Upload the full network's leaves once (a sliced gradient plan); re-staging replaces them."""
        self.plan.stage(tn)

    def grad_offsets(self) -> List[int]:
        return self.plan.grad_offsets()

    def info(self) -> dict:
        """One slice's pass: pairs, flops, bytes, peak_bytes (the per-slice workspace), kernels."""
        return self.plan.info()

    def vjp(self, seed=None, rank: int = 0, world: int = 1, allreduce: bool = True):
        """(value, {leaf index: G}) summed over the slices rank, rank + world, ...: value is bit-identical to `run`, G has
        the full leaf's shape with G[e] = sum_r seed[r] dR[r]/dX[e] (no conjugation).  seed: array, torch CUDA tensor or
        DeviceTensor with the result's shape, None for a scalar result.  With world > 1 and allreduce, both are summed
        over the ranks."""
        from ..tensornetwork.contraction import _download, _leaf
        value, block = self.vjp_blocks(seed, rank, world, allreduce)
        (flat,) = _download([block])
        return _leaf(list(self.plan.result_legs), value), self.plan._unpack(self.plan.grad_offsets(), flat, ())

    def vjp_blocks(self, seed=None, rank: int = 0, world: int = 1, allreduce: bool = True):
        """`vjp` left on the device: (value, rank-1 gradient block at grad_offsets()) as DeviceTensors"""
        return tuple(self._allreduce(self.plan._call("tncb_plan_vjp_sliced", int(rank), int(world), inputs=[(seed, "seed", None)],
                                                     outputs=(True, True)), world, allreduce))

    def _allreduce(self, blocks, world: int, allreduce: bool):
        from .._lib import check
        if world > 1 and allreduce:
            for b in blocks:
                if b is not None:
                    check(self.ctx._l.tncb_comm_allreduce_sum(self.ctx.handle, b.handle))
        return blocks

    def jvp_block(self, tangents, rank: int = 0, world: int = 1, allreduce: bool = True):
        """A sliced tangent plan's forward-mode pass over the slices rank, rank + world, ... (tncb_plan_jvp_sliced), left on
        the device: (value, tangent) DeviceTensors with the result's shape.  tangents: {leaf index: array or torch CUDA
        tensor shaped like the FULL leaf}, requested leaves left out having zero tangent, or the tangents already packed
        at grad_offsets() (see NetworkPlan.jvp_block).  value equals `run` bit for bit.  With world > 1 and allreduce,
        both are summed over the ranks."""
        return tuple(self._allreduce(self.plan._call("tncb_plan_jvp_sliced", int(rank), int(world),
                                                     inputs=[(tangents, "tangents", None)], outputs=(True, True)), world, allreduce))

    def jvp(self, tangents, rank: int = 0, world: int = 1, allreduce: bool = True):
        """`jvp_block` with the derivative downloaded: (value Tensor on the device with the result's legs, tangent
        ndarray), tangent[r] = sum_l sum_e dR[r]/dX_l[e] tangents[l][e] over the full leaves (no conjugation)."""
        from ..tensornetwork.contraction import _download, _leaf
        val, tan = self.jvp_block(tangents, rank, world, allreduce)
        return _leaf(list(self.plan.result_legs), val), _download([tan])[0]

    def hvp_blocks(self, tangents, seed=None, seed_tangent=None, rank: int = 0, world: int = 1, allreduce: bool = True,
                   outputs=(True, True, True, True)):
        """A sliced Hessian-vector plan's forward-over-reverse pass over the slices rank, rank + world, ...
        (tncb_plan_hvp_sliced), left on the device: [value, tangent, grads, grad_tangents] as DeviceTensors, None where
        `outputs` is False; grads and grad_tangents are full-shape blocks at grad_offsets().  Arguments as
        NetworkPlan.hvp_blocks, with tangents shaped like the FULL leaves, or already packed.  With world > 1 and
        allreduce, every returned block is summed over the ranks."""
        return self._allreduce(self.plan._hvp("tncb_plan_hvp_sliced", (int(rank), int(world)), tangents, seed, seed_tangent,
                                              outputs), world, allreduce)

    def hvp(self, tangents, seed=None, seed_tangent=None, rank: int = 0, world: int = 1, allreduce: bool = True):
        """`hvp_blocks` downloaded: (value, tangent, {leaf: G}, {leaf: Ġ}) as host arrays, G and Ġ shaped like the full
        leaf, for every requested leaf (see NetworkPlan.hvp)."""
        from ..tensornetwork.contraction import _download
        value, tangent, g, dg = _download(self.hvp_blocks(tangents, seed, seed_tangent, rank, world, allreduce))
        offs = self.plan.grad_offsets()
        return value, tangent, self.plan._unpack(offs, g, ()), self.plan._unpack(offs, dg, ())

    def set_leaves(self, payloads: dict) -> None:
        """New payloads for leaves of the staged FULL network straight from device memory ({leaf index: torch CUDA tensor
        shaped like the full leaf}, see NetworkPlan.set_leaves); the next run / vjp slices them on the device.  Sliced
        gradient plans only (SlicedPlan.for_gradients)."""
        if self.sn is not None:
            raise TypeError("set_leaves needs a sliced gradient plan (SlicedPlan.for_gradients); this plan stages every slice on the host")
        self.plan.set_leaves(payloads)

    def run(self, rank: int = 0, world: int = 1, allreduce: bool = True) -> Tensor:
        total = self.plan.run_slices(rank, world)
        self._allreduce([total.tensordata.matrix], world, allreduce)
        return total


def contract_sliced(tn: Tensor, path: ContractionPath, legs: Sequence[int], ctx=None, rank: int = 0, world: int = 1,
                    allreduce: bool = True) -> Tensor:
    """Contracts every slice assigned to this rank (round-robin: slices rank, rank + world, ...), accumulates on the
    device and, with world > 1, sums over ranks with one NCCL all-reduce (`tncb_comm_allreduce_sum`; the communicator must
    have been set up with `dist.init_device_comm`).  One schedule is compiled, all slice payloads are uploaded once and
    the slice loop runs inside the library; `SlicedPlan` keeps that state for repeated runs."""
    return SlicedPlan(tn, path, legs, ctx).run(rank, world, allreduce)
