"""Gate table access: mirrors tnc::gates::{load_gate, load_gate_adjoint, is_gate_known}
(tnc/src/gates.rs:50-73) on top of tncb_gate_matrix."""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from ._lib import check, lib

KNOWN_GATES = ("x", "y", "z", "h", "t", "u", "sx", "sy", "sz", "rx", "ry", "rz", "cx", "cz", "swap", "cp", "iswap", "fsim")


def _load(name: str, angles: Sequence[float], adjoint: bool) -> np.ndarray:
    buf = (C.c_double * 32)()
    rank = C.c_int()
    ang = (C.c_double * max(len(angles), 1))(*[float(x) for x in angles])
    check(lib().tncb_gate_matrix(name.encode(), ang, len(angles), int(adjoint), buf, C.byref(rank)))
    n = 4 if rank.value == 2 else 16
    flat = np.frombuffer(buf, dtype=np.float64, count=2 * n).copy().view(np.complex128)
    return flat.reshape([2] * rank.value)


def load_gate(gate: str, angles: Sequence[float] = ()) -> np.ndarray:
    return _load(gate, angles, False)


def load_gate_adjoint(gate: str, angles: Sequence[float] = ()) -> np.ndarray:
    return _load(gate, angles, True)


def load_gate_derivative(gate: str, angles: Sequence[float], slot: int, slot2: int = -1, adjoint: bool = False) -> np.ndarray:
    """dU/da_slot (slot2 < 0) or d²U/da_slot da_slot2 of a gate that takes angles (u, rx, ry, rz, cp, fsim), shaped like
    the gate, of its adjoint when `adjoint` is set (tncb_gate_derivative)"""
    buf = (C.c_double * 32)()
    rank = C.c_int()
    ang = (C.c_double * max(len(angles), 1))(*[float(x) for x in angles])
    check(lib().tncb_gate_derivative(gate.encode(), ang, len(angles), int(adjoint), int(slot), int(slot2), buf, C.byref(rank)))
    n = 4 if rank.value == 2 else 16
    flat = np.frombuffer(buf, dtype=np.float64, count=2 * n).copy().view(np.complex128)
    return flat.reshape([2] * rank.value)


def is_gate_known(gate: str) -> bool:
    return gate in KNOWN_GATES
