"""PyTorch autograd over a gradient plan (NetworkPlan.for_gradients): `.backward()` through a contracted network.

    f = network_function(tn, path, wrt=[3, 7])      # leaves 3 and 7 of leaves(tn) become inputs
    amp = f(u3, u7)                                 # torch complex128 tensors shaped like those leaves
    (amp.abs() ** 2).backward()                     # u3.grad, u7.grad

Gate angles differentiate either through ordinary torch code that builds the gate matrices as Matrix leaves, or with
circuit_function (at the end of this module), which takes the angles themselves and computes the gates and their
derivatives on the device (tnc_b200.angles).  One backward pass gives the gradient of every input, at about two forward passes of cost.
With `sliced_legs`, a network whose gradient workspace does not fit unsliced runs slice by slice (SlicedPlan.for_gradients).
With `batched`, B networks that differ in some leaves (bitstrings, input states) run in one batched pass
(NetworkPlan.vjp_batch) and the result gets a leading dimension B.  With `on_device=True`, CUDA inputs are copied into the
staged plan on the device and the result and gradients come back as CUDA tensors.

Forward mode (torch.autograd.forward_ad, torch.func.jvp) runs on a tangent plan (NetworkPlan.for_tangents).  Without
`batched` or `sliced_legs`, the backward is itself differentiable: `grad(..., create_graph=True)` followed by another
`grad`, torch.autograd.functional.hvp / hessian and torch.func.jvp of torch.func.grad get the second-order terms that
pass through the network from Hessian-vector products of a forward-over-reverse plan (NetworkPlan.for_hvp)."""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import numpy as np
import torch

from . import Context, DeviceTensor, check_cuda_tensor, default_context
from ._lib import check
from .contractionpath import ContractionPath
from .contractionpath.slicing import SlicedPlan
from .tensornetwork import NetworkPlan, PreparedNetwork, Tensor, leaves
from .tensornetwork.tensordata import TensorData


def _with_payloads(tn: Tensor, payloads: dict, counter: list) -> Tensor:
    """copy of the tree structure of `tn` whose leaves numbered in `payloads` (collect order) hold those arrays"""
    if not tn.tensors:
        i = counter[0]
        counter[0] += 1
        if i not in payloads:
            return tn
        t = Tensor(list(tn.legs), list(tn.bond_dims))
        t.set_tensor_data(TensorData.Matrix(payloads[i]))
        return t
    return Tensor.new_composite([_with_payloads(c, payloads, counter) for c in tn.tensors])


class _NetworkFn(torch.autograd.Function):
    # forward / setup_context (rather than forward(ctx, ...)) so that torch.func transforms (torch.func.jvp) accept it
    @staticmethod
    def forward(runner, *xs):
        runner._forward_device(xs) if runner.on_device else runner._forward(xs)
        return runner._result

    @staticmethod
    def setup_context(ctx, inputs, output):
        runner, xs = inputs[0], inputs[1:]
        ctx.runner = runner
        ctx.token = runner._token        # the staging the forward just did
        ctx.save_for_backward(*xs)
        ctx.save_for_forward(*xs)
        ctx.out_meta = (tuple(output.shape), output.device)

    @staticmethod
    def jvp(ctx, _runner_tangent, *tangents):
        # torch.func.jvp calls this inside its transform, where reading a tensor's storage (numpy, the library's
        # device copies) is refused; the work here is outside torch's tracing anyway
        with torch._C._DisableFuncTorch():
            return ctx.runner._jvp(ctx.saved_tensors, tangents, ctx.out_meta)

    @staticmethod
    def backward(ctx, grad_out):
        xs = ctx.saved_tensors           # raises on a second backward through a graph that was not retained
        runner = ctx.runner
        if not runner.batched and not runner.sliced:
            # G through a differentiable Function of (seed, xs), so that create_graph=True keeps the second-order terms
            g = _GradFn.apply(runner, ctx, torch.conj_physical(grad_out), *xs)
            return (None,) + tuple(torch.conj_physical(x) for x in g)
        if torch.is_grad_enabled():      # create_graph=True: the gradients would have no graph back to the inputs
            what = "batched inputs" if runner.batched else "sliced_legs"
            raise NotImplementedError(f"second-order derivatives (create_graph=True) are not supported with {what}: "
                                      "Hessian-vector plans are neither batched nor sliced")
        if runner.on_device:
            return (None,) + runner._backward_device(ctx, grad_out, xs)
        seed = np.conj(grad_out.detach().to(torch.complex128).cpu().numpy())
        if runner.batched:               # vjp_batch runs forward and backward of every instance: it only needs them staged
            if runner._token != ctx.token:
                ctx.token = runner._stage_batch(xs)
            return (None,) + runner._batch_grads(seed, xs)
        # sliced: vjp_sliced re-runs every slice's forward, it only needs these inputs staged
        if runner._token != ctx.token:
            ctx.token = runner._stage(xs)
        g = runner.plan.vjp(seed)[1]
        return (None,) + tuple(torch.from_numpy(np.conj(g[i])).to(x.device) for i, x in zip(runner.wrt, xs))


class _GradFn(torch.autograd.Function):
    """(seed, *xs) -> G of an unbatched, unsliced network_function: G_i = sum_r seed[r] dR[r]/dx_i, holomorphic in the
    seed and the inputs (no conjugation).  forward is the gradient plan's run + vjp.  Second derivatives are symmetric,
    so the vjp of this map with cotangent W is (Ṙ, Ġ) of a Hessian-vector pass with leaf tangents W and no seed tangent
    (_HessFn, itself differentiable in W), and its jvp is Ġ: one NetworkPlan.hvp_blocks call each (torch's
    conjugations for a holomorphic map around them)."""

    @staticmethod
    def forward(runner, fctx, seed, *xs):
        return runner._grads(fctx, seed, xs)

    @staticmethod
    def setup_context(ctx, inputs, output):
        runner, seed, xs = inputs[0], inputs[2], inputs[3:]
        ctx.runner = runner
        ctx.save_for_backward(seed, *xs)
        ctx.save_for_forward(seed, *xs)

    @staticmethod
    def backward(ctx, *w):
        seed, *xs = ctx.saved_tensors
        us = [torch.zeros_like(x) if t is None else torch.conj_physical(t) for x, t in zip(xs, w)]
        rdot, *gdot = _HessFn.apply(ctx.runner, seed, *xs, *us)
        return (None, None, torch.conj_physical(rdot)) + tuple(torch.conj_physical(g) for g in gdot)

    @staticmethod
    def jvp(ctx, _runner_tangent, _fctx_tangent, seed_tangent, *tangents):
        seed, *xs = ctx.saved_tensors
        runner = ctx.runner
        with torch._C._DisableFuncTorch():   # (see _NetworkFn.jvp)
            tans = {i: t for i, t in zip(runner.wrt, tangents) if t is not None}
            _, gdot = runner._hvp(xs, seed, tans, seed_tangent, want_rdot=False)
        return gdot


class _HessFn(torch.autograd.Function):
    """(seed, xs, us) -> (Ṙ, Ġ_i) of a Hessian-vector pass with leaf tangents us and no seed tangent: the holomorphic
    vjp of _GradFn, linear in us.  Its own vjp with respect to us, which torch.autograd.functional.hvp needs (it
    differentiates a backward with respect to its cotangent), is its transpose: Ġ of one pass with leaf tangents from
    the cotangent of Ġ and the seed tangent from the cotangent of Ṙ.  No gradient flows to the seed and the inputs
    through it: derivatives of third order are not computed."""

    @staticmethod
    def forward(runner, seed, *xs_us):
        n = len(xs_us) // 2
        rdot, gdot = runner._hvp(xs_us[:n], seed, dict(zip(runner.wrt, xs_us[n:])), None, want_rdot=True)
        return (rdot,) + gdot

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.runner = inputs[0]
        ctx.save_for_backward(*inputs[1:len(inputs) - (len(inputs) - 2) // 2])

    @staticmethod
    def backward(ctx, a, *b):
        seed, *xs = ctx.saved_tensors
        runner = ctx.runner
        with torch._C._DisableFuncTorch():   # (see _NetworkFn.jvp)
            tans = {i: torch.conj_physical(t) for i, t in zip(runner.wrt, b) if t is not None}
            _, gdot = runner._hvp(xs, seed, tans, None if a is None else torch.conj_physical(a), want_rdot=False)
        return (None, None) + (None,) * len(xs) + tuple(torch.conj_physical(g) for g in gdot)


class NetworkFunction:
    """The callable network_function returns: inputs -> contracted result, differentiable in every input."""

    def __init__(self, tn: Tensor, path: ContractionPath, wrt: Sequence[int], ctx: Optional[Context] = None,
                 sliced_legs: Sequence[int] = (), batched: Sequence[int] = (), on_device: bool = False):
        self.wrt = [int(i) for i in wrt]
        lv = leaves(tn)
        for i in self.wrt:
            if not 0 <= i < len(lv) or lv[i].tensordata.kind != "matrix":
                raise ValueError(f"leaf {i} is not a Matrix leaf of the network (wrt must name Matrix leaves)")
        self.batched = [int(i) for i in batched]
        for i in self.batched:
            if not 0 <= i < len(lv) or lv[i].tensordata.kind != "matrix":
                raise ValueError(f"leaf {i} is not a Matrix leaf of the network (batched must name Matrix leaves)")
        if len(set(self.batched)) != len(self.batched):
            raise ValueError("batched names a leaf twice")
        if self.batched and len(sliced_legs) > 0:
            raise ValueError("batched inputs and sliced_legs cannot be combined")
        # the inputs: one per wrt leaf, then one per batched leaf that is not in wrt
        self.inputs = self.wrt + [i for i in self.batched if i not in self.wrt]
        self.shapes = [tuple(int(d) for d in lv[i].bond_dims) for i in self.inputs]
        self.tn, self.path = tn, path
        self.sliced = len(sliced_legs) > 0
        if self.sliced:
            self.plan = SlicedPlan.for_gradients(tn, path, sliced_legs, self.wrt, ctx=ctx or default_context())
        else:
            self.plan = NetworkPlan.for_gradients(tn, path, self.wrt, ctx=ctx or default_context())
        self._token, self._count, self._result = None, 0, None
        self.on_device = bool(on_device)
        self._staged = False             # on_device: the template network is staged (unbatched and sliced)
        self._template = None            # on_device, batched: the network marshalled once
        self._offsets = None
        self._ctx = ctx or default_context()
        self._sliced_legs = tuple(sliced_legs)
        self._tplan = None               # the tangent plan, compiled on the first forward-mode call
        self._tstaged = False            # on_device, unbatched: the tangent plan has `tn` staged
        self._hplan = None               # the Hessian-vector plan, compiled on the first second-order call
        self._hstaged = False            # on_device: the Hessian-vector plan has `tn` staged

    # ---- on_device: inputs, results and gradients stay on the GPU ----
    def _check_device(self, xs):
        for i, x in zip(self.inputs, xs):
            check_cuda_tensor(self.plan.ctx, x, f"input for leaf {i}")

    def _set_device(self, xs):
        """the inputs as the wrt leaves' payloads, copied on the device into the staged network (staged once, from the
        network's own payloads, on first use)"""
        self._check_device(xs)
        for i, shape, x in zip(self.wrt, self.shapes, xs):
            if tuple(x.shape) != shape:
                raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, the leaf {shape}")
        if not self._staged:
            self.plan.stage(self.tn)
            self._staged = True
        self.plan.set_leaves(dict(zip(self.wrt, xs)))
        self._count += 1
        self._token = self._count
        return self._token

    def _stage_instances(self, xs):
        """B instances staged from device memory: batched inputs row by row, the others shared"""
        self._check_device(xs)
        b = self._batch_size(xs)
        if self._template is None:
            self._template = PreparedNetwork(self.tn)
        self.plan.stage_instances(self._template, dict(zip(self.inputs, xs)), b)
        self._count += 1
        self._token = self._count
        return self._token

    def _split(self, block, lead=()):
        """{wrt leaf: its slice of a [..., grad_elems] torch gradient block, shaped lead + leaf shape}"""
        if self._offsets is None:
            self._offsets = self.plan.grad_offsets()
        out = {}
        for i, shape in zip(self.wrt, self.shapes):
            off = self._offsets[i]
            out[i] = block[..., off:off + int(np.prod(shape, dtype=np.int64))].reshape(tuple(lead) + shape)
        return out

    def _forward_device(self, xs):
        if self.batched:
            token = self._stage_instances(xs)
            vals = self.plan.vjp_batch_blocks(0, None, rows=False, sum=False, values=True)[0]
        else:
            token = self._set_device(xs)
            vals = self.plan.run().tensordata.matrix
        self._result = vals.to_torch()
        vals.free()
        return token

    def _backward_device(self, fctx, grad_out, xs):
        """the gradients of batched or sliced inputs (torch's convention, conj of the holomorphic vjp)"""
        seed = DeviceTensor.from_torch(self.plan.ctx, torch.conj_physical(grad_out.detach().to(torch.complex128)))
        try:
            if self.batched:
                if self._token != fctx.token:
                    fctx.token = self._stage_instances(xs)
                return self._batch_grads_device(seed, xs)
            if self._token != fctx.token:
                fctx.token = self._set_device(xs)
            value, block = self.plan.vjp_blocks(seed)
            value.free()
            flat = torch.conj_physical(block.to_torch())
            block.free()
        finally:
            seed.free()
        g = self._split(flat)
        return tuple(g[i] for i in self.wrt)

    def _grads(self, fctx, seed, xs):
        """G_i = sum_r seed[r] dR[r]/dx_i (holomorphic, no conjugation) of the unbatched, unsliced plan, one per wrt input:
        the forward of the _NetworkFn call `fctx` (re-run when another call used the plan's state since), then vjp"""
        seed = seed.detach().to(torch.complex128)
        if self.on_device:
            s = DeviceTensor.from_torch(self.plan.ctx, seed)
            try:
                if self._token != fctx.token:
                    fctx.token = self._forward_device(xs)
                self._token = None
                block = self.plan.vjp_block(s)
                flat = block.to_torch()
                block.free()
            finally:
                s.free()
            g = self._split(flat)
            return tuple(g[i] for i in self.wrt)
        if self._token != fctx.token:    # another forward (or an earlier backward) used the plan's state since
            fctx.token = self._forward(xs)
        self._token = None               # the backward levels overwrite the forward state
        g = self.plan.vjp(seed.cpu().numpy())
        return tuple(torch.from_numpy(g[i]).to(x.device) for i, x in zip(self.wrt, xs))

    # ---- second order (create_graph=True, torch.autograd.functional.hvp / hessian, torch.func.jvp of torch.func.grad):
    # a Hessian-vector plan, compiled on the first second-order call ----
    def _hvp(self, xs, seed, tangents: dict, seed_tangent, want_rdot: bool):
        """(Ṙ or None, (Ġ_i per wrt input)) of one NetworkPlan.hvp_blocks pass on the inputs xs with seed `seed`, leaf
        tangents {wrt leaf: tensor} (left out: zero) and seed tangent `seed_tangent` (None: zero); no conjugation"""
        if self._hplan is None:
            self._hplan = NetworkPlan.for_hvp(self.tn, self.path, self.wrt, ctx=self._ctx)
        plan = self._hplan
        for i, shape, x in zip(self.wrt, self.shapes, xs):
            if tuple(x.shape) != shape:
                raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, the leaf {shape}")
        outputs = (False, want_rdot, False, True)

        def phys(t):
            return t.detach().to(torch.complex128).resolve_conj()
        if self.on_device:
            self._check_device(xs)
            for i, t in tangents.items():
                check_cuda_tensor(plan.ctx, t, f"tangent for leaf {i}")
            if not self._hstaged:
                plan.stage(self.tn)
                self._hstaged = True
            plan.set_leaves(dict(zip(self.wrt, xs)))
            _, rdot, _, gdot = plan.hvp_blocks({i: phys(t) for i, t in tangents.items()}, phys(seed),
                                               None if seed_tangent is None else phys(seed_tangent), outputs)
            out = []
            for dt in (rdot, gdot):
                out.append(None if dt is None else dt.to_torch())
                if dt is not None:
                    dt.free()
            g = self._split(out[1])
            return out[0], tuple(g[i] for i in self.wrt)

        def host(t):                     # (np.ascontiguousarray would make a rank-0 seed rank 1)
            return phys(t).contiguous().cpu().numpy()
        plan.stage(_with_payloads(self.tn, {i: host(x) for i, x in zip(self.wrt, xs)}, [0]))
        _, rdot, _, gdot = plan.hvp_blocks({i: host(t) for i, t in tangents.items()}, host(seed),
                                           None if seed_tangent is None else host(seed_tangent), outputs)
        out = []
        for dt in (rdot, gdot):
            out.append(None if dt is None else torch.from_numpy(dt.to_numpy()).to(seed.device))
            if dt is not None:
                dt.free()
        g = self._split(out[1])
        return out[0], tuple(g[i].to(x.device) for i, x in zip(self.wrt, xs))

    def _batch_grads_device(self, seed, xs):
        want_rows = any(i in self.batched for i in self.wrt)
        want_sum = any(i not in self.batched for i in self.wrt)
        _, rows, total = self.plan.vjp_batch_blocks(0, None, seeds=seed, rows=want_rows, sum=want_sum, values=False)
        blocks = []
        for dt in (rows, total):
            blocks.append(None if dt is None else torch.conj_physical(dt.to_torch()))
            if dt is not None:
                dt.free()
        rows_g = self._split(blocks[0], (self.plan.n_staged,)) if want_rows else {}
        sum_g = self._split(blocks[1]) if want_sum else {}
        grads = []
        for i in self.inputs:
            if i not in self.wrt:
                grads.append(None)
            else:
                grads.append(rows_g[i] if i in self.batched else sum_g[i])
        return tuple(grads)

    def _stage(self, xs):
        """stage the inputs as the wrt leaves' payloads (through the host)"""
        pay = {}
        for i, shape, x in zip(self.wrt, self.shapes, xs):
            if tuple(x.shape) != shape:
                raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, the leaf {shape}")
            pay[i] = np.ascontiguousarray(x.detach().to(torch.complex128).cpu().numpy())
        self.plan.stage(_with_payloads(self.tn, pay, [0]))
        self._count += 1
        self._token = self._count
        return self._token

    def _batch_size(self, xs) -> int:
        """the common leading dimension B of the batched inputs; every input's shape checked"""
        b = None
        for i, shape, x in zip(self.inputs, self.shapes, xs):
            want = shape
            if i in self.batched:
                if x.dim() < 1:
                    raise ValueError(f"batched input for leaf {i} needs a leading batch dimension")
                if b is None:
                    b = int(x.shape[0])
                elif int(x.shape[0]) != b:
                    raise ValueError(f"batched input for leaf {i} has {int(x.shape[0])} instances, an earlier one {b}")
                want = (b,) + shape
            if tuple(x.shape) != want:
                raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, expected {want}")
        if b == 0:
            raise ValueError("batched inputs hold no instance")
        return b

    def _stage_batch(self, xs):
        """stage B networks: batched leaves take their row b, the others the same payload in every instance"""
        b = self._batch_size(xs)
        arrs = [np.ascontiguousarray(x.detach().to(torch.complex128).cpu().numpy()) for x in xs]
        nets = []
        for k in range(b):
            pay = {i: (a[k] if i in self.batched else a) for i, a in zip(self.inputs, arrs)}
            nets.append(_with_payloads(self.tn, pay, [0]))
        self.plan.stage_batch(nets)
        self._count += 1
        self._token = self._count
        return self._token

    def _batch_grads(self, seed, xs):
        """conj of the rows (batched leaves in wrt) or of the sum (shared leaves in wrt); None for the other inputs"""
        want_rows = any(i in self.batched for i in self.wrt)
        want_sum = any(i not in self.batched for i in self.wrt)
        _, _, rows, total = self.plan.vjp_batch(0, None, seeds=seed, rows=want_rows, sum=want_sum, values=False)
        grads = []
        for i, x in zip(self.inputs, xs):
            if i not in self.wrt:
                grads.append(None)
            else:
                g = rows[i] if i in self.batched else total[i]
                grads.append(torch.from_numpy(np.conj(g)).to(x.device))
        return tuple(grads)

    def _forward(self, xs):
        """stage the inputs and run the forward levels (every slice's, summed, on a sliced plan; every instance's, one
        per row, with batched inputs)"""
        if self.batched:
            token = self._stage_batch(xs)
            _, vals, _, _ = self.plan.vjp_batch(0, None, rows=False, sum=False, values=True)
            self._result = torch.from_numpy(np.asarray(vals).copy())
            return token
        token = self._stage(xs)
        res = self.plan.run()
        self._result = torch.from_numpy(np.asarray(res.to_numpy()).copy())
        return token

    # ---- forward mode (torch.autograd.forward_ad, torch.func.jvp): a tangent plan, compiled on first use ----
    def _jvp(self, xs, tangents, out_meta):
        """Ṙ for the tangents of the inputs (None = zero; tangents of inputs not in wrt are ignored, as backward gives
        them no gradient): the tangent plan staged with the inputs, then NetworkPlan.jvp / jvp_batch"""
        if self.sliced:
            raise NotImplementedError("forward-mode AD (jvp) is not supported with sliced_legs: tangent plans are not sliced")
        shape, device = out_meta
        tans = {i: t for i, t in zip(self.inputs, tangents) if t is not None and i in self.wrt}
        if not tans:
            return torch.zeros(shape, dtype=torch.complex128, device=device)
        if self._tplan is None:
            self._tplan = NetworkPlan.for_tangents(self.tn, self.path, self.wrt, ctx=self._ctx)
        plan = self._tplan
        if self.on_device:
            self._check_device(xs)
            for i, t in tans.items():
                check_cuda_tensor(plan.ctx, t, f"tangent for leaf {i}")
            if self.batched:
                if self._template is None:
                    self._template = PreparedNetwork(self.tn)
                plan.stage_instances(self._template, dict(zip(self.inputs, xs)), self._batch_size(xs))
                _, rows = plan.jvp_batch_blocks(0, None, tans, values=False)
                out = rows.to_torch()
                rows.free()
                return out
            for i, shape_i, x in zip(self.wrt, self.shapes, xs):
                if tuple(x.shape) != shape_i:
                    raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, the leaf {shape_i}")
            if not self._tstaged:
                plan.stage(self.tn)
                self._tstaged = True
            plan.set_leaves(dict(zip(self.wrt, xs)))
            val, tan = plan.jvp_block(tans)
            val.free()
            out = tan.to_torch()
            tan.free()
            return out
        host = {i: np.ascontiguousarray(t.detach().to(torch.complex128).resolve_conj().cpu().numpy()) for i, t in tans.items()}
        if self.batched:
            b = self._batch_size(xs)
            arrs = [np.ascontiguousarray(x.detach().to(torch.complex128).resolve_conj().cpu().numpy()) for x in xs]
            plan.stage_batch([_with_payloads(self.tn, {i: (a[k] if i in self.batched else a) for i, a in zip(self.inputs, arrs)}, [0])
                              for k in range(b)])
            _, _, rows = plan.jvp_batch(0, None, host, values=False)
            return torch.from_numpy(rows).to(device)
        pay = {}
        for i, shape_i, x in zip(self.wrt, self.shapes, xs):
            if tuple(x.shape) != shape_i:
                raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, the leaf {shape_i}")
            pay[i] = np.ascontiguousarray(x.detach().to(torch.complex128).resolve_conj().cpu().numpy())
        plan.stage(_with_payloads(self.tn, pay, [0]))
        _, tan = plan.jvp(host)
        return torch.from_numpy(tan).to(device)

    def __call__(self, *xs: torch.Tensor) -> torch.Tensor:
        if len(xs) != len(self.inputs):
            raise TypeError(f"expected {len(self.inputs)} inputs, got {len(xs)}")
        return _NetworkFn.apply(self, *xs)


def network_function(tn: Tensor, path: ContractionPath, wrt: Sequence[int], ctx: Optional[Context] = None,
                     sliced_legs: Sequence[int] = (), batched: Sequence[int] = (), on_device: bool = False) -> NetworkFunction:
    """A torch.autograd.Function over the network `tn` contracted along `path`: the returned callable takes one torch
    complex128 tensor per leaf index in `wrt` (indices into leaves(tn); each must be a Matrix leaf) and returns the
    contracted result as a torch tensor.  Its backward is conj(vjp(conj(grad_out))) of the gradient plan, torch's
    convention for complex inputs.

    Forward = stage + run: the inputs are copied to the host and staged the way NetworkPlan.stage stages any payload
    (with on_device=False, the default; see below).  A backward needs the plan's forward state: when another call of the
    same function ran in between, or a retained graph is differentiated again, the backward re-runs the forward from
    the saved inputs first.  A second backward through a graph that was not retained raises torch's error.

    sliced_legs: legs of `tn` to slice (e.g. from contractionpath.slicing.find_slices), for networks whose gradient
    workspace does not fit unsliced.  Forward = stage + the forward levels of every slice, summed on the device;
    backward = SlicedPlan.vjp with the seed.  No workspace holds all slices' forward state, so the backward runs every
    slice's forward again before its backward levels: about 4 forward passes in all, against about 3 unsliced.  The
    backward needs only the staged inputs, so it re-stages (without a forward) when another call ran in between.

    batched: Matrix leaves whose payload differs per instance, e.g. bitstring projectors or per-sample input states; they
    may include leaves not in `wrt`.  The callable then takes one tensor per `wrt` leaf followed by one per batched leaf
    not in `wrt`, in the order given; a batched leaf's tensor is [B, *leaf shape] with one B for all of them, the others
    are [*leaf shape] and shared by every instance.  It returns [B, *result].  Forward = stage_batch + the forward pass
    of every instance (NetworkPlan.vjp_batch, values only); backward = vjp_batch with seeds conj(grad_out), a forward
    plus backward pass of every instance: per-instance gradient rows for batched inputs in `wrt`, their sum over the
    instances for shared ones.  About 4 forward passes per forward + backward in all, against about 3 for one
    unbatched network; the instances share every launch.  Not combinable with sliced_legs.

    Forward mode: torch.autograd.forward_ad dual inputs and torch.func.jvp(f, inputs, tangents) give Ṙ = sum over the
    inputs of dR/dx · ẋ (the plain directional derivative, torch's forward-mode convention for holomorphic functions), from
    a tangent plan (NetworkPlan.for_tangents) compiled on the first forward-mode call.  With `batched`, tangents of
    batched inputs are [B, *leaf shape], those of shared inputs [*leaf shape] and the same for every instance; the
    instances run in one NetworkPlan.jvp_batch pass.  Tangents of inputs not in `wrt` are ignored, as their gradients are
    None.  sliced_legs with forward mode raises NotImplementedError.

    Second order (unbatched and unsliced, on_device False or True): the backward computes G = vjp(conj(grad_out)) through
    a holomorphic autograd.Function of (conj(grad_out), inputs), so with create_graph=True the gradients have a graph
    back to the inputs and to grad_out.  Differentiating them again (a second torch.autograd.grad,
    torch.autograd.functional.hvp / hessian, torch.func.jvp of torch.func.grad) makes one Hessian-vector pass per
    call (NetworkPlan.hvp_blocks) on a plan compiled on the first second-order call; it costs about nine forward passes
    with every input requested.  First-order gradients keep their bits with and without create_graph.  With `batched`
    or `sliced_legs`, a backward with create_graph=True raises NotImplementedError rather than return gradients
    without a graph.  torch.func.hessian / jacrev / jacfwd need a vmap rule the function does not have.

    on_device=True: the inputs must be torch CUDA tensors on the context's device (else ValueError), and the result and
    the gradients are CUDA tensors there; no payload, result or gradient goes through the host.  The first call stages
    `tn` itself; every call then copies the inputs into the staged network on the device (NetworkPlan.set_leaves, or
    NetworkPlan.stage_instances of the network marshalled once with `batched`), ordered against torch's current stream
    both ways.  Values and gradients equal those of on_device=False bit for bit."""
    return NetworkFunction(tn, path, wrt, ctx, sliced_legs, batched, on_device)


class _CircuitFn(torch.autograd.Function):
    @staticmethod
    def forward(runner, theta):
        return runner._forward(theta)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.runner = inputs[0]
        ctx.save_for_backward(inputs[1])
        ctx.save_for_forward(inputs[1])

    @staticmethod
    def jvp(ctx, _runner_tangent, theta_dot):
        with torch._C._DisableFuncTorch():   # (see _NetworkFn.jvp)
            return ctx.runner._jvp(ctx.saved_tensors[0], theta_dot)

    @staticmethod
    def backward(ctx, grad_out):
        (theta,) = ctx.saved_tensors
        if torch.is_grad_enabled():
            raise NotImplementedError("second-order derivatives (create_graph=True) are not supported by circuit_function")
        return None, ctx.runner._backward(theta, grad_out)


class CircuitFunction:
    """See circuit_function."""

    def __init__(self, tn: Tensor, path: ContractionPath, angle_map, ctx: Optional[Context] = None, sliced_legs: Sequence[int] = ()):
        from .angles import Angles
        self.ctx = ctx or default_context()
        self.tn, self.path, self.map = tn, path, angle_map
        self.sliced_legs = [int(l) for l in sliced_legs]
        wrt = angle_map.leaves()
        if self.sliced_legs:
            self.plan = SlicedPlan.for_gradients(tn, path, self.sliced_legs, wrt=wrt, ctx=self.ctx)
        else:
            self.plan = NetworkPlan.for_gradients(tn, path, wrt=wrt, ctx=self.ctx)
        self.plan.stage(tn)
        self.angles = Angles(self.ctx, tn, angle_map, self.plan)
        self.template = PreparedNetwork(tn)
        self.result_dims = tuple(self.plan.plan.result_dims if self.sliced_legs else self.plan.result_dims)
        self._tplan = self._tangles = None

    def _theta(self, theta) -> int:
        """the batch size B of a [B, P] θ, 0 for a [P] one; ValueError for anything else"""
        check_cuda_tensor(self.ctx, theta, "theta")
        P = self.angles.n_params
        if theta.dtype != torch.float64:
            raise ValueError(f"theta must be float64, got {theta.dtype}")
        if theta.dim() == 1 and theta.shape[0] == P:
            return 0
        if theta.dim() == 2 and theta.shape[1] == P and theta.shape[0] >= 1:
            if self.sliced_legs:
                raise ValueError("theta must be [P] with sliced_legs")
            return int(theta.shape[0])
        raise ValueError(f"theta has shape {tuple(theta.shape)}, expected [{P}] or [B, {P}]")

    def _forward(self, theta):
        B = self._theta(theta)
        if B:
            self.angles.stage_instances(self.plan, self.template, theta)
            vals = self.plan.vjp_batch_blocks(0, B, rows=False, sum=False, values=True)[0]
            return vals.to_torch()
        self.angles.set_leaves(self.plan, theta)
        return self.plan.run().tensordata.matrix.to_torch()

    def _backward(self, theta, grad_out):
        B = self._theta(theta)
        seed = DeviceTensor.from_torch(self.ctx, torch.conj_physical(grad_out.to(torch.complex128)))
        try:
            if B:
                self.angles.stage_instances(self.plan, self.template, theta)
                G = self.plan.vjp_batch_blocks(0, B, seeds=seed, rows=True, sum=False, values=False)[1]
            else:
                self.angles.set_leaves(self.plan, theta)
                if self.sliced_legs:
                    value, G = self.plan.vjp_blocks(seed)
                    value.free()
                else:
                    self.plan.run()
                    G = self.plan.vjp_block(seed)
            rows = self.angles.pullback(theta, G)[0]
            G.free()
        finally:
            seed.free()
        g = rows.to_torch().real
        rows.free()
        return g if B else g[0]

    def _jvp(self, theta, theta_dot):
        from .angles import Angles
        if self.sliced_legs:
            raise NotImplementedError("forward mode is not supported by circuit_function with sliced_legs")
        B = self._theta(theta)
        if theta_dot is None:
            theta_dot = torch.zeros_like(theta)
        if self._tplan is None:
            self._tplan = NetworkPlan.for_tangents(self.tn, self.path, wrt=self.map.leaves(), ctx=self.ctx)
            self._tplan.stage(self.tn)
            self._tangles = Angles(self.ctx, self.tn, self.map, self._tplan)
        tdot = theta_dot.detach().to(torch.float64)
        l, plan = self.ctx._l, self._tplan
        out = ctypes.c_void_p()
        if B:
            self._tangles.stage_instances(plan, self.template, theta)
            tan = self._tangles.tangents(theta, tdot)
            rc = l.tncb_plan_jvp_batch(self.ctx.handle, plan.handle, 0, B, tan.handle, None, ctypes.byref(out))
        else:
            self._tangles.set_leaves(plan, theta)
            tan = self._tangles.tangents(theta, tdot)
            rc = l.tncb_plan_jvp(self.ctx.handle, plan.handle, tan.handle, None, ctypes.byref(out))
        tan.free()
        check(rc)
        rdot = DeviceTensor.adopt(self.ctx, out)
        res = rdot.to_torch()
        rdot.free()
        return res

    def __call__(self, theta: torch.Tensor) -> torch.Tensor:
        return _CircuitFn.apply(self, theta)


def circuit_function(tn: Tensor, path: ContractionPath, angle_map, ctx: Optional[Context] = None,
                     sliced_legs: Sequence[int] = ()) -> CircuitFunction:
    """A torch.autograd.Function of the gate angles of the circuit network `tn` contracted along `path`: the returned
    callable takes θ, a CUDA float64 tensor [P] (P = angle_map.n_params, see tnc_b200.angles.AngleMap), and returns R(θ)
    as a complex128 CUDA tensor; θ of shape [B, P] runs B angle sets as instances of one batched pass and returns
    [B, *R].  Nothing goes through the host: the Gate leaves are computed on the device (Angles.gates) and copied into
    a gradient plan staged once.

    Backward (torch's convention for a real input): grad_θ = Re(pullback(vjp(conj(grad_out)))), through the plan's vjp,
    vjp_batch rows for [B, P], or vjp_sliced with `sliced_legs`.  The backward re-stages the angles and runs the forward
    again, so it is right whatever ran in between.  Forward mode (torch.autograd.forward_ad, torch.func.jvp) runs
    Angles.tangents and a tangent plan's jvp / jvp_batch, compiled on first use.  Second order (create_graph=True) and
    forward mode with sliced_legs raise NotImplementedError; vmap is not supported."""
    return CircuitFunction(tn, path, angle_map, ctx, sliced_legs)
