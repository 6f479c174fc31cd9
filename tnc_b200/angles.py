"""Gate angles as parameters: a circuit's Gate leaves as functions of a real vector θ, on the device (tncb_angles_*).

    amap = AngleMap.every_angle(tn)                  # each angle slot of each angle gate its own parameter
    plan = NetworkPlan.for_gradients(tn, path, wrt=amap.leaves())
    plan.stage(tn)
    ang = Angles(ctx, tn, amap, plan)                # the plan's gradient-block layout
    ang.set_leaves(plan, theta)                      # theta: torch CUDA float64 [P]
    plan.run(); G = plan.vjp_block(seed)
    g = ang.pullback(theta, G)                       # sum_r seed[r] dR[r]/dθ, [1, P] complex

The tables of a map are uploaded once per context; every call is asynchronous on the context stream and ordered after
torch's current stream.  See include/tncb.h for the definitions of the three calls and how they compose with plans."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import Context, DeviceTensor, check_cuda_tensor, default_context
from ._lib import check
from .tensornetwork.contraction import PreparedNetwork, _library_call

ANGLE_GATES = {"u": 3, "rx": 1, "ry": 1, "rz": 1, "cp": 1, "fsim": 2}


class _Ref(C.Structure):
    _fields_ = [("leaf", C.c_uint64), ("slot", C.c_uint32), ("param", C.c_uint32), ("scale", C.c_double)]


class AngleMap:
    """refs (leaf, slot, param, scale): angle slot `slot` of Gate leaf `leaf` (an index into leaves(tn)) is
    scale * θ[param].  Slots no ref names keep the leaf's own angle.  theta0: an initial θ (None if not known)."""

    def __init__(self, refs: Sequence[Tuple[int, int, int, float]], n_params: int, theta0: Optional[Sequence[float]] = None):
        self.refs = [(int(r[0]), int(r[1]), int(r[2]), float(r[3]) if len(r) > 3 else 1.0) for r in refs]
        self.n_params = int(n_params)
        self.theta0 = None if theta0 is None else np.asarray(theta0, dtype=np.float64)

    @classmethod
    def every_angle(cls, tn) -> "AngleMap":
        """Every angle slot of every Gate leaf of u, rx, ry, rz, cp or fsim its own parameter, in leaf order then slot
        order, scale 1; theta0 holds the leaves' own angles."""
        from .tensornetwork import leaves
        refs, theta0 = [], []
        for i, leaf in enumerate(leaves(tn)):
            td = leaf.tensordata
            if td is None or td.kind != "gate":
                continue
            name, ang, _ = td.gate
            for s in range(ANGLE_GATES.get(name, 0)):
                refs.append((i, s, len(theta0), 1.0))
                theta0.append(float(ang[s]))
        return cls(refs, len(theta0), theta0)

    def leaves(self) -> List[int]:
        """The referenced leaves, ascending: the `wrt` of a plan whose gradient block the map should read."""
        return sorted({l for l, _, _, _ in self.refs})


def _vector(rows: DeviceTensor) -> DeviceTensor:
    """a [1, n] tensor as a new [n] one: a device-to-device copy on the context stream"""
    import torch
    from . import torch_streams
    out = DeviceTensor.empty(rows.ctx, [rows.shape[1]])
    _, ext = torch_streams(rows.ctx)
    with torch.cuda.stream(ext):
        out._torch_view().copy_(rows._torch_view())
    rows.free()
    return out


def _block_size(offsets, shapes) -> int:
    return max([o + int(np.prod(s, dtype=np.int64)) for o, s in zip(offsets, shapes) if o >= 0], default=0)


class Angles:
    """An angle map compiled for the network `tn` (tncb_angles_create).  With `plan` (a NetworkPlan or SlicedPlan of
    `tn` whose requested leaves include every referenced one), the blocks take the plan's grad_offsets() layout, so
    gate rows, tangent blocks, G and Ġ are interchangeable with the plan's; without, the referenced leaves are packed in
    leaf order."""

    def __init__(self, ctx: Optional[Context], tn, angle_map: AngleMap, plan=None):
        from .tensornetwork import leaves
        from .tensornetwork.contraction import _Marshal
        self.ctx = ctx or default_context()
        self.handle = None
        self.map = angle_map
        shapes = [tuple(int(d) for d in leaf.bond_dims) for leaf in leaves(tn)]
        offs, block = None, 0
        if plan is not None:
            o = plan.grad_offsets()
            offs = (C.c_int64 * max(len(o), 1))(*o)
            block = _block_size(o, shapes)
        refs = (_Ref * max(len(angle_map.refs), 1))(*[_Ref(*r) for r in angle_map.refs])
        m = _Marshal()
        c_tn = m.tn(tn)
        h = C.c_void_p()
        check(self.ctx._l.tncb_angles_create(C.byref(c_tn), angle_map.n_params, len(angle_map.refs), refs, offs, block, C.byref(h)))
        self.handle = h
        n_p, n_b = C.c_size_t(), C.c_size_t()
        lay = (C.c_int64 * max(len(shapes), 1))()
        check(self.ctx._l.tncb_angles_layout(h, C.byref(n_p), C.byref(n_b), lay))
        self.n_params, self.block_elems = n_p.value, n_b.value
        self.offsets = [lay[i] for i in range(len(shapes))]
        self.leaf_index = angle_map.leaves()

    # ---- arguments ----
    def _rows(self, x, what: str, count: Optional[int] = None):
        """(tensor, row stride in elements, count) of a torch CUDA float64 [P] (one row) or [count, P] tensor"""
        import torch
        check_cuda_tensor(self.ctx, x, what)
        if x.dtype != torch.float64:
            raise ValueError(f"{what} must be float64, got {x.dtype}")
        P = self.n_params
        if x.dim() == 1 and x.shape[0] == P:
            x = x.detach().contiguous()
            return x, 0, 1 if count is None else count
        if x.dim() == 2 and x.shape[1] == P and x.shape[0] >= 1 and (count is None or x.shape[0] == count):
            x = x.detach()
            if x.stride(1) != 1 or (x.shape[0] > 1 and x.stride(0) < P):
                x = x.contiguous()
            return x, x.stride(0) if x.shape[0] > 1 else 0, x.shape[0]
        want = f"[{P}] or [count, {P}]" if count is None else f"[{P}] or [{count}, {P}]"
        raise ValueError(f"{what} has shape {tuple(x.shape)}, expected {want}")

    # ---- the three calls ----
    def gates(self, theta) -> DeviceTensor:
        """[count, block_elems] rows: row i holds every referenced leaf's gate at θ_i, zeros elsewhere"""
        th, st, n = self._rows(theta, "theta")
        return _library_call(self.ctx, "tncb_angles_gates", [self.ctx.handle, self.handle, C.c_void_p(th.data_ptr()), st, n],
                             (True,), [th])[0]

    def tangents(self, theta, theta_dot) -> DeviceTensor:
        """[count, block_elems] rows of leaf tangents Ẋ_l = sum_{r on l} scale_r θ̇[param_r] dU_l/da_{slot_r}; theta and
        theta_dot may each be one shared row.  When both are one row ([P]), one [block_elems] block: the tangents
        argument of a plan's jvp / hvp"""
        td, sd, nd = self._rows(theta_dot, "theta_dot")
        th, st, n = self._rows(theta, "theta", nd if nd > 1 else None)
        n = max(n, nd)
        if nd == 1:
            sd = 0
        rows = _library_call(self.ctx, "tncb_angles_tangents", [self.ctx.handle, self.handle, C.c_void_p(th.data_ptr()), st,
                                                                C.c_void_p(td.data_ptr()), sd, n], (True,), [th, td])[0]
        if theta.dim() == 1 and theta_dot.dim() == 1:
            return _vector(rows)
        return rows

    def pullback(self, theta, grads: DeviceTensor, grad_tangents: Optional[DeviceTensor] = None, direction=None,
                 rows: bool = True, sum: bool = False):
        """(rows [count, n_params], sum [n_params]) DeviceTensors, None where not requested: g[p] = sum over p's refs of
        scale_r <G_l, dU_l/da_{slot_r}>; with grad_tangents (Ġ) and direction (v), its derivative along v instead, the
        Hessian-vector product (H_θ v)[p] when G and Ġ come from a plan's hvp on tangents(θ, v).
        grads: [block_elems] (shared) or [count, block_elems]; count is theta's row count, or grads' when theta is one
        row."""
        count = grads.shape[0] if len(grads.shape) == 2 else None
        th, st, n = self._rows(theta, "theta", count)
        keep = [th]
        dv, sv = None, 0
        if direction is not None:
            dv, sv, nv = self._rows(direction, "direction", n if n > 1 else None)
            if nv == 1:
                sv = 0
            keep.append(dv)
        return tuple(_library_call(self.ctx, "tncb_angles_pullback", [
            self.ctx.handle, self.handle, C.c_void_p(th.data_ptr()), st, n, grads.handle,
            grad_tangents.handle if grad_tangents is not None else None, C.c_void_p(dv.data_ptr()) if dv is not None else None,
            sv], (rows, sum), keep))

    # ---- into plans ----
    def _gate_ptrs(self, rows: DeviceTensor) -> list:
        """the device address of every referenced leaf's gate in each row of `rows`"""
        base = rows.device_ptr()
        return [base + 16 * self.offsets[l] for l in self.leaf_index]

    def set_leaves(self, plan, theta) -> None:
        """The referenced leaves of the staged `plan` (NetworkPlan or sliced gradient SlicedPlan) set to their gates at
        θ ([P]), on the device: gates + tncb_plan_set_leaves"""
        plan = getattr(plan, "plan", plan)
        rows = self.gates(theta)
        try:
            plan._set_leaves(self.leaf_index, self._gate_ptrs(rows))
        finally:
            rows.free()                  # (the arena reuses it in stream order, after the copy)

    def stage_instances(self, plan, template, theta_rows) -> None:
        """count = len(theta_rows) instances of `plan`: every leaf from `template` (a Tensor or PreparedNetwork of the
        plan's structure) except the referenced leaves, which take their gates at θ_i: gates + tncb_plan_stage_instances"""
        tmpl = template if isinstance(template, PreparedNetwork) else PreparedNetwork(template)
        rows = self.gates(theta_rows)
        try:
            plan._stage_instances(tmpl, rows.shape[0], self.leaf_index, self._gate_ptrs(rows),
                                  [self.block_elems] * len(self.leaf_index))
        finally:
            rows.free()

    def __del__(self):
        try:
            if self.handle:
                self.ctx._l.tncb_angles_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
