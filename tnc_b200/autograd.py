"""PyTorch autograd over a gradient plan (NetworkPlan.for_gradients): `.backward()` through a contracted network.

    f = network_function(tn, path, wrt=[3, 7])      # leaves 3 and 7 of leaves(tn) become inputs
    amp = f(u3, u7)                                 # torch complex128 tensors shaped like those leaves
    (amp.abs() ** 2).backward()                     # u3.grad, u7.grad

Gate angles differentiate either through ordinary torch code that builds the gate matrices as Matrix leaves, or with
circuit_function (at the end of this module), which takes the angles themselves and computes the gates and their
derivatives on the device (tnc_b200.angles).  One backward pass gives the gradient of every input, at about two forward passes of cost.
With `sliced_legs`, a network whose gradient workspace does not fit unsliced runs slice by slice (SlicedPlan.for_gradients).
With `batched`, B networks that differ in some leaves (bitstrings, input states) run in one batched pass
(NetworkPlan.vjp_batch) and the result gets a leading dimension B.  The network is staged once; every call copies the
inputs into the staged plan on the device, CPU inputs after one upload of them all.  With `on_device=True`, the inputs
must be CUDA tensors and the result and gradients come back as CUDA tensors.

Forward mode (torch.autograd.forward_ad, torch.func.jvp) runs on a tangent plan (NetworkPlan.for_tangents).  Without
`batched` or `sliced_legs`, the backward is itself differentiable: `grad(..., create_graph=True)` followed by another
`grad`, torch.autograd.functional.hvp / hessian and torch.func.jvp of torch.func.grad get the second-order terms that
pass through the network from Hessian-vector products of a forward-over-reverse plan (NetworkPlan.for_hvp)."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from . import Context, check_cuda_tensor, default_context
from .contractionpath import ContractionPath
from .contractionpath.slicing import SlicedPlan
from .tensornetwork import NetworkPlan, PreparedNetwork, Tensor, leaves
from .tensornetwork.contraction import _download
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
        return runner._forward(xs)

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
        return (None,) + runner._backward(ctx, grad_out, xs)


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
        self._ctx = ctx or default_context()
        self.sliced = len(sliced_legs) > 0
        if self.sliced:
            self.plan = SlicedPlan.for_gradients(tn, path, sliced_legs, self.wrt, ctx=self._ctx)
        else:
            self.plan = NetworkPlan.for_gradients(tn, path, self.wrt, ctx=self._ctx)
        self._token = None               # the staging the gradient plan's state belongs to
        self.on_device = bool(on_device)
        self._staged = []                # the plans `tn` is staged in (unbatched and sliced)
        self._template = None            # batched: the network marshalled once
        self._offsets = None
        self._tplan = None               # the tangent plan, compiled on the first forward-mode call
        self._hplan = None               # the Hessian-vector plan, compiled on the first second-order call

    # ---- inputs, staging and gradients: the plans run on the context's device, whatever device the inputs are on ----
    def _to_ctx(self, ts, names) -> list:
        """the torch tensors `ts` as physical complex128 tensors on the context's device.  on_device: each must be there
        already (else ValueError, naming it from `names`).  Else the ones elsewhere are packed into one buffer per
        device they are on, moved in one copy and split into views: networks have hundreds of inputs, and a copy each
        would cost more than the contraction of a small one."""
        if self.on_device:
            for t, name in zip(ts, names):
                check_cuda_tensor(self._ctx, t, name)
        dev = torch.device("cuda", self._ctx.device)
        out, away = [], {}
        for k, t in enumerate(ts):
            if t.dtype != torch.complex128 or t.is_conj() or t.is_neg():
                t = t.detach().to(torch.complex128).resolve_conj().resolve_neg()
            out.append(t)
            if t.device != dev:
                away.setdefault(t.device, []).append(k)
        for ks in away.values():
            buf = torch.cat([out[k].reshape(-1) for k in ks]).to(dev)
            for k, part in zip(ks, buf.split([out[k].numel() for k in ks])):
                out[k] = part.view(out[k].shape)
        return out

    def _inputs(self, xs):
        """(the inputs on the context's device, B or None without `batched`), every shape checked: a wrt leaf's input
        shaped like the leaf, a batched leaf's [B, *leaf shape] with one B >= 1 for all of them"""
        dxs = self._to_ctx(xs, [f"input for leaf {i}" for i in self.inputs])
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
                raise ValueError(f"input for leaf {i} has shape {tuple(x.shape)}, "
                                 + (f"expected {want}" if self.batched else f"the leaf {shape}"))
        if b == 0:
            raise ValueError("batched inputs hold no instance")
        return dxs, b

    def _stage(self, plan, xs) -> None:
        """the inputs into `plan`: with `batched`, B instances of the network marshalled once (stage_instances), batched
        inputs row by row, the others shared; else `tn` itself, staged on the plan's first use, with the wrt leaves
        copied in on the device (set_leaves)"""
        dxs, b = self._inputs(xs)
        if self.batched:
            if self._template is None:
                self._template = PreparedNetwork(self.tn)
            plan.stage_instances(self._template, dict(zip(self.inputs, dxs)), b)
            return
        if plan not in self._staged:
            plan.stage(self.tn)
            self._staged.append(plan)
        plan.set_leaves(dict(zip(self.wrt, dxs)))

    def _split(self, block, inputs: dict, lead=()) -> dict:
        """{leaf: its slice of a [*lead, grad_elems] torch gradient block, shaped lead + leaf shape} for the leaves of
        `inputs` ({wrt leaf: input}), each on its input's device: the whole block is copied once to each other device"""
        if self._offsets is None:
            self._offsets = self.plan.grad_offsets()
        shapes = dict(zip(self.inputs, self.shapes))
        blocks = {block.device: block}
        out = {}
        for i, x in inputs.items():
            if x.device not in blocks:
                blocks[x.device] = block.to(x.device)
            off, shape = self._offsets[i], shapes[i]
            out[i] = blocks[x.device][..., off:off + math.prod(shape)].reshape(tuple(lead) + shape)
        return out

    def _forward(self, xs):
        """stage the inputs and run the forward levels (every slice's, summed, on a sliced plan; every instance's, one
        per row, with batched inputs); returns the result, on the host unless on_device.  Not kept here: the result's
        graph refers to this object, and a reference back would make a cycle that holds the plans' device memory until
        the garbage collector runs."""
        self._stage(self.plan, xs)
        self._token = object()
        if self.batched:
            vals = self.plan.vjp_batch_blocks(0, None, rows=False, sum=False, values=True)[0]
        else:
            vals = self.plan.run().tensordata.matrix
        (res,) = _download([vals], "to_torch")
        return res if self.on_device else res.cpu()

    def _backward(self, fctx, grad_out, xs):
        """the gradients of batched or sliced inputs (torch's convention, conj of the holomorphic vjp), None for batched
        inputs not in wrt: per-instance rows for batched inputs, their sum over the instances for shared ones"""
        (seed,) = self._to_ctx([torch.conj_physical(grad_out)], ["the seed"])
        # vjp_batch and vjp_sliced re-run every forward: they only need these inputs staged
        if self._token != fctx.token:
            self._stage(self.plan, xs)
            fctx.token = self._token = object()
        if self.batched:
            _, rows, total = self.plan.vjp_batch_blocks(0, None, seeds=seed, rows=any(i in self.batched for i in self.wrt),
                                                        sum=any(i not in self.batched for i in self.wrt), values=False)
        else:
            value, total = self.plan.vjp_blocks(seed)
            value.free()
            rows = None
        rows, total = (None if b is None else torch.conj_physical(b) for b in _download([rows, total], "to_torch"))
        wrt = dict(zip(self.wrt, xs))
        g = {}
        if rows is not None:
            g.update(self._split(rows, {i: x for i, x in wrt.items() if i in self.batched}, (self.plan.n_staged,)))
        if total is not None:
            g.update(self._split(total, {i: x for i, x in wrt.items() if i not in self.batched}))
        return tuple(g.get(i) for i in self.inputs)

    def _grads(self, fctx, seed, xs):
        """G_i = sum_r seed[r] dR[r]/dx_i (holomorphic, no conjugation) of the unbatched, unsliced plan, one per wrt input:
        the forward of the _NetworkFn call `fctx` (re-run when another call used the plan's state since), then vjp"""
        (s,) = self._to_ctx([seed], ["the seed"])
        if self._token != fctx.token:
            self._forward(xs)
            fctx.token = self._token
        self._token = None               # the backward levels overwrite the forward state
        (flat,) = _download([self.plan.vjp_block(s)], "to_torch")
        return tuple(self._split(flat, dict(zip(self.wrt, xs))).values())

    # ---- second order (create_graph=True, torch.autograd.functional.hvp / hessian, torch.func.jvp of torch.func.grad):
    # a Hessian-vector plan, compiled on the first second-order call ----
    def _hvp(self, xs, seed, tangents: dict, seed_tangent, want_rdot: bool):
        """(Ṙ or None, (Ġ_i per wrt input)) of one NetworkPlan.hvp_blocks pass on the inputs xs with seed `seed`, leaf
        tangents {wrt leaf: tensor} (left out: zero) and seed tangent `seed_tangent` (None: zero); no conjugation.  Ṙ
        comes back on the seed's device, Ġ_i on its input's."""
        if self._hplan is None:
            self._hplan = NetworkPlan.for_hvp(self.tn, self.path, self.wrt, ctx=self._ctx)
        self._stage(self._hplan, xs)
        n = len(tangents)
        ts = self._to_ctx(list(tangents.values()) + [seed] + ([] if seed_tangent is None else [seed_tangent]),
                          [f"tangent for leaf {i}" for i in tangents] + ["the seed", "the seed tangent"])
        _, rdot, _, gdot = self._hplan.hvp_blocks(dict(zip(tangents, ts[:n])), ts[n], ts[n + 1] if seed_tangent is not None else None,
                                                  (False, want_rdot, False, True))
        rdot, gdot = _download([rdot, gdot], "to_torch")
        g = self._split(gdot, dict(zip(self.wrt, xs)))
        return None if rdot is None else rdot.to(seed.device), tuple(g.values())

    # ---- forward mode (torch.autograd.forward_ad, torch.func.jvp): a tangent plan, compiled on first use ----
    def _jvp(self, xs, tangents, out_meta):
        """Ṙ for the tangents of the inputs (None = zero; tangents of inputs not in wrt are ignored, as backward gives
        them no gradient) on the result's device: the tangent plan staged with the inputs, then NetworkPlan.jvp_block /
        jvp_batch_blocks"""
        if self.sliced:
            raise NotImplementedError("forward-mode AD (jvp) is not supported with sliced_legs: tangent plans are not sliced")
        shape, device = out_meta
        tans = {i: t for i, t in zip(self.inputs, tangents) if t is not None and i in self.wrt}
        if not tans:
            return torch.zeros(shape, dtype=torch.complex128, device=device)
        if self._tplan is None:
            self._tplan = NetworkPlan.for_tangents(self.tn, self.path, self.wrt, ctx=self._ctx)
        self._stage(self._tplan, xs)
        tans = dict(zip(tans, self._to_ctx(list(tans.values()), [f"tangent for leaf {i}" for i in tans])))
        if self.batched:
            _, tan = self._tplan.jvp_batch_blocks(0, None, tans, values=False)
        else:
            val, tan = self._tplan.jvp_block(tans)
            val.free()
        return _download([tan], "to_torch")[0].to(device)

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

    Forward = stage + run, on the context's device whatever device the inputs are on.  The first call stages `tn`
    itself; every call then copies the inputs into the staged network on the device (NetworkPlan.set_leaves, or
    NetworkPlan.stage_instances of the network marshalled once with `batched`), ordered against torch's current stream
    both ways.  So the payloads of the leaves that are not inputs are read once, at the first call: changing them in
    `tn` afterwards does not change the function.  With on_device=False (the default), inputs may be on any device:
    those elsewhere are packed into one buffer and arrive in one copy.  The result comes back on the CPU, each gradient
    on its input's device and a forward-mode tangent on the result's.  A backward needs the plan's forward state: when
    another call of the same function ran in between, or a retained graph is differentiated again, the backward re-runs
    the forward from the saved inputs first.  A second backward through a graph that was not retained raises torch's
    error.

    sliced_legs: legs of `tn` to slice (e.g. from contractionpath.slicing.find_slices), for networks whose gradient
    workspace does not fit unsliced.  Forward = stage + the forward levels of every slice, summed on the device;
    backward = SlicedPlan.vjp with the seed.  No workspace holds all slices' forward state, so the backward runs every
    slice's forward again before its backward levels: about 4 forward passes in all, against about 3 unsliced.  The
    backward needs only the staged inputs, so it re-stages (without a forward) when another call ran in between.

    batched: Matrix leaves whose payload differs per instance, e.g. bitstring projectors or per-sample input states; they
    may include leaves not in `wrt`.  The callable then takes one tensor per `wrt` leaf followed by one per batched leaf
    not in `wrt`, in the order given; a batched leaf's tensor is [B, *leaf shape] with one B for all of them, the others
    are [*leaf shape] and shared by every instance.  It returns [B, *result].  Forward = stage_instances + the forward
    pass of every instance (NetworkPlan.vjp_batch, values only); backward = vjp_batch with seeds conj(grad_out), a forward
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
    the gradients are CUDA tensors there; no payload, result or gradient goes through the host.  Values and gradients
    equal those of on_device=False bit for bit."""
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
        seed = torch.conj_physical(grad_out.to(torch.complex128))
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
        plan = self._tplan
        if B:
            self._tangles.stage_instances(plan, self.template, theta)
        else:
            self._tangles.set_leaves(plan, theta)
        tan = self._tangles.tangents(theta, tdot)
        try:
            rdot = plan.jvp_batch_blocks(0, B, tan, values=False)[1] if B else plan._jvp_tangent(tan)
        finally:
            tan.free()
        return _download([rdot], "to_torch")[0]

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


class _ExpectFn(torch.autograd.Function):
    @staticmethod
    def forward(runner, theta):
        return runner._forward(theta)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.runner = inputs[0]
        ctx.save_for_backward(inputs[1])

    @staticmethod
    def jvp(ctx, *tangents):
        raise NotImplementedError("forward mode is not supported by expectation_function")

    @staticmethod
    def backward(ctx, grad_out):
        (theta,) = ctx.saved_tensors
        if torch.is_grad_enabled():
            raise NotImplementedError("second-order derivatives (create_graph=True) are not supported by expectation_function")
        return None, grad_out * ctx.runner._grad(theta)


class ExpectationFunction:
    """See expectation_function."""

    def __init__(self, exp):
        if exp.angles is None:
            raise ValueError("expectation_function needs an Expectation built with an angle_map")
        self.exp = exp

    def _check(self, theta) -> None:
        check_cuda_tensor(self.exp.ctx, theta, "theta")
        P = self.exp.angles.n_params
        if theta.dtype != torch.float64:
            raise ValueError(f"theta must be float64, got {theta.dtype}")
        if theta.dim() == 2 and theta.shape[1] == P:
            raise NotImplementedError("expectation_function takes one θ [P]; batches of θ are not supported")
        if theta.dim() != 1 or theta.shape[0] != P:
            raise ValueError(f"theta has shape {tuple(theta.shape)}, expected [{P}]")

    def _forward(self, theta):
        self._check(theta)
        e, _ = self.exp.values(theta.detach())
        return torch.tensor(e.real, dtype=torch.float64, device=theta.device)

    def _grad(self, theta):
        return self.exp.value_and_grad(theta.detach())[1]

    def __call__(self, theta: torch.Tensor) -> torch.Tensor:
        return _ExpectFn.apply(self, theta)


def expectation_function(exp) -> ExpectationFunction:
    """A torch.autograd.Function of the gate angles: the returned callable takes θ, a CUDA float64 tensor [P] (P =
    the angle map's n_params of `exp`, an observables.Expectation built with an angle_map), and returns E(θ) =
    sum_k c_k <psi(θ)|P_k|psi(θ)> as a float64 CUDA scalar (the real part of Expectation.values).  Backward:
    grad_θ = grad_out * Re(dE/dθ) (Expectation.value_and_grad, which re-stages θ and runs the forward pass again).
    Forward mode, second order (create_graph=True) and θ of shape [B, P] raise NotImplementedError."""
    return ExpectationFunction(exp)
