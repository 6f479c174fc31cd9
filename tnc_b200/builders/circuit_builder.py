"""Circuit -> tensor network (tnc/src/builders/circuit_builder.rs:135-335) and Permutor (:72-129)."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .. import Context, DeviceTensor, default_context
from .._lib import check
from ..tensornetwork.tensor import Tensor
from ..tensornetwork.tensordata import TensorData


class Permutor:
    def __init__(self, target_legs: Sequence[int]):
        self.target_leg_order = list(target_legs)

    def is_identity(self) -> bool:
        return not self.target_leg_order

    @staticmethod
    def permutation_between(given: Sequence[int], target: Sequence[int]) -> List[int]:
        """circuit_builder.rs:125-129: the permutation p with [given[p[i]] for i] == target (`given` and `target` are equal
        up to order) -- the axis order handed to tncb_permute."""
        pos = {l: i for i, l in enumerate(given)}
        assert len(pos) == len(given) == len(target) and set(pos) == set(target), "given and target must be permutations of each other"
        return [pos[l] for l in target]

    def apply(self, tensor: Tensor, ctx: Optional[Context] = None) -> Tensor:
        """Transposes the (device) data so that the legs appear in the target order
        (circuit_builder.rs:86-114); one tncb_permute launch."""
        assert tensor.is_leaf()
        if self.is_identity():
            return tensor
        ctx = ctx or default_context()
        perm = self.permutation_between(tensor.legs, self.target_leg_order)
        m = tensor.tensordata.matrix
        dt = m if isinstance(m, DeviceTensor) else DeviceTensor.from_numpy(ctx, np.asarray(m).reshape(tensor.bond_dims))
        out = C.c_void_p()
        parr = (C.c_int * max(len(perm), 1))(*perm)
        check(ctx._l.tncb_permute(ctx.handle, dt.handle, parr, C.byref(out)))
        dt.release()
        res = Tensor(self.target_leg_order, [tensor.bond_dims[p] for p in perm])
        res.set_tensor_data(TensorData.Matrix(DeviceTensor.adopt(ctx, out)))
        return res


class Circuit:
    def __init__(self):
        self.open_edges: List[int] = []
        self.next_edge = 0
        self.tensors: List[Tensor] = []

    @staticmethod
    def _ket(bit: int) -> TensorData:
        return TensorData.new_from_data([2], [1, 0] if bit == 0 else [0, 1])

    def num_qubits(self) -> int:
        return len(self.open_edges)

    def allocate_register(self, size: int) -> List[int]:
        base = self.num_qubits()
        for _ in range(size):
            e = self.next_edge
            self.next_edge += 1
            self.open_edges.append(e)
            t = Tensor.new_from_const([e], 2)
            t.set_tensor_data(self._ket(0))
            self.tensors.append(t)
        return list(range(base, base + size))

    def append_gate(self, gate, angles: Sequence[float] = (), qubits: Sequence[int] = (), adjoint: bool = False) -> None:
        """append_gate(TensorData.Gate(...), qubits=[...]) or append_gate("h", [], [q])."""
        td = gate if isinstance(gate, TensorData) else TensorData.Gate(gate, angles, adjoint)
        if len(set(qubits)) != len(qubits):
            raise ValueError("Qubit arguments must be unique")
        old = [self.open_edges[q] for q in qubits]
        new = [self.next_edge + e for e in range(len(qubits))]
        self.next_edge += len(qubits)
        for q, e in zip(qubits, new):
            self.open_edges[q] = e
        t = Tensor.new_from_const(old + new, 2)
        t.set_tensor_data(td)
        self.tensors.append(t)

    def into_amplitude_network(self, bitstring: str) -> Tuple[Tensor, Permutor]:
        assert len(bitstring) == self.num_qubits()
        tensors = list(self.tensors)
        final_legs = []
        for c, e in zip(bitstring, self.open_edges):
            if c == "*":
                final_legs.append(e)
                continue
            if c not in "01":
                raise ValueError("Only 0, 1 and * are allowed in bitstring")
            t = Tensor.new_from_const([e], 2)
            t.set_tensor_data(self._ket(int(c)))
            tensors.append(t)
        return Tensor.new_composite(tensors), Permutor(final_legs)

    def into_statevector_network(self) -> Tuple[Tensor, Permutor]:
        return self.into_amplitude_network("*" * self.num_qubits())

    def into_expectation_value_network(self) -> Tensor:
        offset = self.next_edge
        tensors = list(self.tensors)
        for t in self.tensors:
            half = len(t.legs) // 2
            legs = [l + offset for l in (t.legs[half:] + t.legs[:half])]
            dims = t.bond_dims[half:] + t.bond_dims[:half]
            adj = Tensor(legs, dims)
            adj.set_tensor_data(t.tensordata.adjoint())
            tensors.append(adj)
        for e in self.open_edges:
            z = Tensor.new_from_const([e, e + offset], 2)
            z.set_tensor_data(TensorData.Gate("z"))
            tensors.append(z)
        return Tensor.new_composite(tensors)

    def tensor_qubits(self) -> List[List[int]]:
        """The qubits of every tensor of `tensors`: a ket's qubit, a gate's qubits in argument order."""
        qubit_of, out, kets = {}, [], 0
        for t in self.tensors:
            if len(t.legs) == 1:             # allocate_register's kets, in qubit order
                qubit_of[t.legs[0]] = kets
                out.append([kets])
                kets += 1
                continue
            half = len(t.legs) // 2
            qs = [qubit_of[l] for l in t.legs[:half]]
            for q, l in zip(qs, t.legs[half:]):
                qubit_of[l] = q
            out.append(qs)
        return out

    def into_pauli_expectation_network(self, support: Sequence[int]) -> "PauliNetwork":
        """<psi|L|psi> with one observable ("layer") leaf per qubit of `support`, pruned to the light cone of `support`.

        Leaves: the kept circuit tensors, their adjoint mirror images (built as into_expectation_value_network builds
        them: legs rotated by half, offset next_edge, TensorData.adjoint()), then per qubit q of `support`, ascending, a
        layer leaf with legs [e, e + offset] (e = open_edges[q]) holding the 2x2 identity, so that a staged plan
        contracts to <psi|psi>; tncb_plan_expect writes each term's payload there instead.
        Light cone: the gates are walked from last to first; a gate touching a qubit already in the cone is kept and adds
        its qubits to the cone.  A gate not kept cancels against its mirror image, and both are dropped.  A qubit of the
        cone outside `support` loses its later gates: its ket wire is joined to its bra wire (the bra copy takes the ket's
        leg id, no leaf is added).  Qubits never in the cone lose their ket and its mirror (<0|0> = 1).  With `support` =
        every qubit nothing is pruned, and the network is into_expectation_value_network()'s with I in place of Z."""
        n = self.num_qubits()
        sup = sorted({int(q) for q in support})
        if not sup or any(not 0 <= q < n for q in sup):
            raise ValueError(f"support {list(support)} must be a non-empty set of qubits of the {n}-qubit circuit")
        qubits = self.tensor_qubits()
        cone, keep = set(sup), [False] * len(self.tensors)
        for i in reversed(range(len(self.tensors))):
            if len(self.tensors[i].legs) > 1 and cone.intersection(qubits[i]):
                keep[i] = True
                cone.update(qubits[i])
        for i, t in enumerate(self.tensors):
            if len(t.legs) == 1:
                keep[i] = qubits[i][0] in cone
        # the output wire of each cone qubit's last kept tensor: joined to its mirror unless the qubit is in the support
        last = {}
        for i, t in enumerate(self.tensors):
            if keep[i]:
                half = len(t.legs) // 2
                for q, l in zip(qubits[i], t.legs[half:]):
                    last[q] = l
        joined = {l for q, l in last.items() if q not in set(sup)}
        offset = self.next_edge
        kept = [i for i in range(len(self.tensors)) if keep[i]]
        tensors = [self.tensors[i] for i in kept]
        for i in kept:
            t = self.tensors[i]
            half = len(t.legs) // 2
            legs = [l if l in joined else l + offset for l in (t.legs[half:] + t.legs[:half])]
            adj = Tensor(legs, t.bond_dims[half:] + t.bond_dims[:half])
            adj.set_tensor_data(t.tensordata.adjoint())
            tensors.append(adj)
        layer_leaf = []
        for q in sup:
            e = self.open_edges[q]
            layer = Tensor.new_from_const([e, e + offset], 2)
            layer.set_tensor_data(TensorData.new_from_data([2, 2], [1, 0, 0, 1]))
            layer_leaf.append(len(tensors))
            tensors.append(layer)
        k = len(kept)
        return PauliNetwork(Tensor.new_composite(tensors), layer_leaf, sup, {k + j: j for j in range(k)}, kept)


class PauliNetwork:
    """The network of Circuit.into_pauli_expectation_network.

    tn:          the network; its leaves are leaves(tn) in order
    layer_leaf:  the leaf index of the layer leaf of qubit layer_qubit[j]
    layer_qubit: the support, ascending
    ket_of:      {bra-copy leaf: its ket leaf}
    kept:        kept[i] is the index into circuit.tensors of ket leaf i"""

    def __init__(self, tn: Tensor, layer_leaf: List[int], layer_qubit: List[int], ket_of: dict, kept: List[int]):
        self.tn, self.layer_leaf, self.layer_qubit, self.ket_of, self.kept = tn, layer_leaf, layer_qubit, ket_of, kept

    def angle_map(self, circuit_map):
        """An AngleMap of this network from `circuit_map`, whose refs name circuit.tensors indices: each ref on a kept
        gate becomes a ref on its ket copy and one on its bra copy, with the same param and scale; refs on pruned gates
        are dropped, so their params get zero gradient.  n_params and theta0 stay the circuit's."""
        from ..angles import AngleMap
        leaf_of = {c: i for i, c in enumerate(self.kept)}
        bra_of = {k: b for b, k in self.ket_of.items()}
        refs = []
        for leaf, slot, param, scale in circuit_map.refs:
            if leaf in leaf_of:
                i = leaf_of[leaf]
                refs += [(i, slot, param, scale), (bra_of[i], slot, param, scale)]
        return AngleMap(refs, circuit_map.n_params, circuit_map.theta0)
