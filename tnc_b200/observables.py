"""Expectation values of Pauli-sum observables on the device (tncb_plan_expect).

    H = PauliSum([(0.5, "Z0 Z1"), (-1.0, "X2"), (0.25, "Y0 Y3")], n_qubits=circuit.num_qubits())
    exp = Expectation(circuit, H, angle_map=amap)     # amap: refs on circuit.tensors indices
    E, dE = exp.value_and_grad(theta)                  # theta: torch CUDA float64 [P]

The network is <psi|L|psi> pruned to the light cone of the Hamiltonian's support (Circuit.into_pauli_expectation_network),
compiled and staged once.  Every call writes each term's layer payloads on the device and contracts all terms as the
instances of one batched pass; E = sum_k c_k <psi|P_k|psi> and sum_k c_k dR_k/dleaf are folded on the device in term
order, and the leaf gradient is pulled back to the gate angles (Angles.pullback).

One Expectation covers all terms with the light cone of their union.  A Hamiltonian whose terms act on distant qubits
can instead be split into groups, one Expectation per group, each with a smaller light cone; the energies and gradients
add up.  That trades one batched pass over one larger network for several passes over smaller ones: which is cheaper
depends on the circuit, and each plan's `plan.info()` shows its cost before anything runs."""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import Context
from ._lib import TncbPauliLayer, u64_array
from .tensornetwork.contraction import NetworkPlan, _library_call

_BITS = {"I": (0, 0), "X": (1, 0), "Z": (0, 1), "Y": (1, 1)}


def pauli_layer_matrix(x: int, z: int) -> np.ndarray:
    """The layer payload of one qubit of a term: sigma(x, z)^T as a 2x2 complex128 array with legs [ket, bra], sigma(0,0)
    = I, (1,0) = X, (0,1) = Z, (1,1) = Y.  The expectation network contracts to sum_ab psi_a M[a, b] conj(psi_b), so the
    transpose makes it <psi|sigma|psi>; the device writes the same bits (expect.cu)."""
    m = np.zeros((2, 2), dtype=np.complex128)
    if not x:
        m[0, 0], m[1, 1] = 1.0, (-1.0 if z else 1.0)
    elif not z:
        m[0, 1] = m[1, 0] = 1.0
    else:
        m[0, 1], m[1, 0] = complex(0.0, 1.0), complex(0.0, -1.0)
    return m


class PauliSum:
    """H = sum_k c_k P_k on `n_qubits` qubits (1..64), from terms (coeff, "X0 Z3 Y7") or (coeff, {qubit: "X" | "Y" | "Z"}).
    An empty string or dict is the identity.  Terms keep their order and duplicates are not merged: the energy is
    folded in this order.  Non-real or non-finite coefficients, qubits outside 0 .. n_qubits - 1, a qubit named twice in
    a term and letters other than I, X, Y, Z raise ValueError."""

    def __init__(self, terms: Sequence[Tuple[float, Union[str, Dict[int, str]]]], n_qubits: int):
        n_qubits = int(n_qubits)
        if not 1 <= n_qubits <= 64:
            raise ValueError(f"a Pauli sum acts on 1..64 qubits, not {n_qubits}")
        self.n_qubits = n_qubits
        self.terms: List[Tuple[float, Dict[int, str]]] = []
        for k, term in enumerate(terms):
            if len(term) != 2:
                raise ValueError(f"term {k} is not a (coefficient, Pauli string) pair")
            self.terms.append((self._coeff(k, term[0]), self._paulis(k, term[1])))
        if not self.terms:
            raise ValueError("a Pauli sum needs at least one term")

    @staticmethod
    def _coeff(k: int, c) -> float:
        if isinstance(c, (bool, np.bool_)) or not isinstance(c, numbers.Number):
            raise ValueError(f"the coefficient of term {k} is not a number: {c!r}")
        if isinstance(c, numbers.Complex) and not isinstance(c, numbers.Real):
            if complex(c).imag != 0:
                raise ValueError(f"the coefficient of term {k} is not real: {c!r}")
            c = complex(c).real
        c = float(c)
        if not math.isfinite(c):
            raise ValueError(f"the coefficient of term {k} is not finite: {c!r}")
        return c

    def _paulis(self, k: int, p) -> Dict[int, str]:
        if isinstance(p, str):
            pairs = []
            for tok in p.split():
                if len(tok) < 2 or not tok[1:].isdigit():
                    raise ValueError(f"term {k}: {tok!r} is not a letter followed by a qubit")
                pairs.append((int(tok[1:]), tok[0]))
        elif isinstance(p, dict):
            pairs = list(p.items())
        else:
            raise ValueError(f"term {k}: the Paulis must be a string or a {{qubit: letter}} dict, not {type(p).__name__}")
        out: Dict[int, str] = {}
        for q, letter in pairs:
            if not isinstance(letter, str) or letter not in _BITS:
                raise ValueError(f"term {k}: unknown Pauli {letter!r} (I, X, Y or Z)")
            if isinstance(q, (bool, np.bool_)) or not isinstance(q, numbers.Integral) or not 0 <= int(q) < self.n_qubits:
                raise ValueError(f"term {k}: qubit {q!r} is outside the {self.n_qubits}-qubit circuit")
            if int(q) in out:
                raise ValueError(f"term {k}: qubit {int(q)} is named twice")
            out[int(q)] = letter
        return {q: l for q, l in out.items() if l != "I"}

    def __len__(self) -> int:
        return len(self.terms)

    def masks(self) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(x masks uint64 [K], z masks uint64 [K], coefficients float64 [K]): bit q of term k's masks is qubit q's
        Pauli, (x, z) = (0, 0) I, (1, 0) X, (0, 1) Z, (1, 1) Y -- the host arrays tncb_plan_expect takes"""
        x = np.zeros(len(self.terms), dtype=np.uint64)
        z = np.zeros(len(self.terms), dtype=np.uint64)
        for k, (_, paulis) in enumerate(self.terms):
            for q, letter in paulis.items():
                bx, bz = _BITS[letter]
                x[k] |= np.uint64(bx << q)
                z[k] |= np.uint64(bz << q)
        return x, z, np.array([c for c, _ in self.terms], dtype=np.float64)

    def support(self) -> List[int]:
        """the qubits some term acts on (not as I), ascending"""
        return sorted({q for _, paulis in self.terms for q in paulis})


class Expectation:
    """E(θ) = sum_k c_k <psi(θ)|P_k|psi(θ)> of `hamiltonian` (a PauliSum) on `circuit`, on the device.

    The network is circuit.into_pauli_expectation_network(support), support defaulting to the terms' union, on the
    greedy Cotengrust path unless `path` is given.  Without `angle_map` the plan is a plain plan and `values` evaluates
    the circuit as built; with it (refs naming circuit.tensors indices, see angles.AngleMap) it is a gradient plan whose
    requested leaves are the translated map's (PauliNetwork.angle_map), and both methods take θ.  `plan.info()` shows
    the cost before any run; `plan.run()` contracts <psi|psi> (the staged layer holds identities).
    After value_and_grad, `max_imag` is the largest |Im| of the energy and the gradient before their real parts were
    taken: rounding leaves a small one, a large one means the network is not <psi|H|psi>."""

    def __init__(self, circuit, hamiltonian: PauliSum, angle_map=None, path=None, support: Optional[Sequence[int]] = None,
                 ctx: Optional[Context] = None):
        n = circuit.num_qubits()
        if hamiltonian.n_qubits != n:
            raise ValueError(f"the Pauli sum acts on {hamiltonian.n_qubits} qubits, the circuit has {n}")
        need = hamiltonian.support()
        sup = need if support is None else sorted({int(q) for q in support})
        if support is not None and not set(need) <= set(sup):
            raise ValueError(f"support {sup} does not hold the terms' qubits {need}")
        if not sup:
            raise ValueError("every term is the identity: there is no qubit to build the observable on")
        self.n_qubits, self.hamiltonian = n, hamiltonian
        self.network = circuit.into_pauli_expectation_network(sup)
        tn = self.network.tn
        if path is None:
            from .contractionpath.paths import Cotengrust
            opt = Cotengrust(tn)
            opt.find_path()
            path = opt.get_best_replace_path()
        self.path = path
        self.angle_map, self.angles = None, None
        if angle_map is None:
            self.plan = NetworkPlan(tn, path, ctx)
        else:
            self.angle_map = self.network.angle_map(angle_map)
            if not self.angle_map.refs:
                raise ValueError("no angle of angle_map lies in the light cone of the support")
            self.plan = NetworkPlan.for_gradients(tn, path, wrt=self.angle_map.leaves(), ctx=ctx)
        self.plan.stage(tn)
        self.ctx = self.plan.ctx
        if angle_map is not None:
            from .angles import Angles
            self.angles = Angles(self.ctx, tn, self.angle_map, self.plan)
        x, z, c = hamiltonian.masks()
        self._terms = (u64_array(x.tolist()), u64_array(z.tolist()), (C.c_double * len(c))(*c.tolist()))
        self._keep = (u64_array(self.network.layer_leaf), (C.c_int * len(self.network.layer_qubit))(*self.network.layer_qubit))
        self._layer = TncbPauliLayer(n, len(self.network.layer_leaf), *self._keep)
        self.max_imag = 0.0

    def _expect(self, theta, outputs, batch: Optional[int]):
        """θ into the plan (with an angle map), then tncb_plan_expect with `outputs` (values, energy, grad_sum)"""
        if theta is not None:
            if self.angles is None:
                raise ValueError("theta needs an angle_map")
            self.angles.set_leaves(self.plan, theta)
        return _library_call(self.ctx, "tncb_plan_expect", [self.ctx.handle, self.plan.handle, C.byref(self._layer),
                                                            len(self.hamiltonian), *self._terms, int(batch or 0)], outputs)

    def values(self, theta=None, batch: Optional[int] = None):
        """(E as a complex, the term values <psi|P_k|psi> as a CUDA complex128 tensor [K]); theta: torch CUDA float64 [P]
        (an angle_map's parameters; None: the angles the plan holds).  batch: terms per pass (None: as many as fit)."""
        vals, energy, _ = self._expect(theta, (True, True, False), batch)
        e = complex(energy.to_numpy().reshape(()))
        energy.free()
        return e, vals.to_torch()

    def value_and_grad(self, theta, batch: Optional[int] = None):
        """(E(θ) as a float, dE/dθ as a CUDA float64 tensor [P]): Angles.set_leaves, tncb_plan_expect, Angles.pullback of
        sum_k c_k G_k, then the real parts (max_imag keeps what they drop).  Params whose refs were all pruned get 0."""
        if self.angles is None:
            raise ValueError("value_and_grad needs an angle_map")
        _, energy, g = self._expect(theta, (False, True, True), batch)
        try:
            rows = self.angles.pullback(theta, g)[0]
        finally:
            g.free()
        e = complex(energy.to_numpy().reshape(()))
        energy.free()
        grad = rows.to_torch()[0]
        rows.free()
        self.max_imag = max(abs(e.imag), float(grad.imag.abs().max()) if grad.numel() else 0.0)
        return e.real, grad.real.contiguous()
