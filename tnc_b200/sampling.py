"""Bitstrings drawn from a circuit's output distribution on the device (tncb_plan_sample).

Candidate i of a seed fixes the closed qubits Q from a Philox4x64-10 stream; the plan contracts the amplitude network
with those bras and the open qubits O as result legs, giving the 2^k amplitudes of every outcome of O at once.  The
candidate is accepted with probability min(1, q 2^(n-k) / m), q being the closed assignment's exact marginal, and an
accepted candidate picks O's bits from its 2^k probabilities by inverse CDF.  While no ratio q 2^(n-k) / m exceeds 1 the
samples are exact and i.i.d.; include/tncb.h and DESIGN §5 give the algorithm and the stream contract.

With `sliced_legs` the open amplitude network is sliced on those legs and every candidate's amplitudes are the sum of
its slices' results, formed on the device (tncb_plan_sample_slices): circuits whose amplitude only contracts sliced can
be sampled too.  `open_path` reuses a path of the closed amplitude network for the open one."""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Optional, Sequence

from . import Context
from ._lib import TncbSampleSpec, TncbSampleStats, u64_array
from .contractionpath import ContractionPath
from .tensornetwork.contraction import NetworkPlan, _library_call, leaves


@dataclass
class Samples:
    """The samples of one `Sampler.sample` call, in candidate order.

    bits:           torch int64 CUDA [S], bit q of each word is qubit q
    probabilities:  torch float64 CUDA [S], |amplitude|^2 of each sample (not normalised: the network's own scale)
    candidates:     candidates consumed; next_candidate = first + candidates continues the same stream
    clipped:        consumed candidates whose ratio q 2^(n-k) / m exceeded 1 (their closed assignment is under-sampled)
    max_ratio:      the largest ratio q 2^(n-k) / m among the consumed candidates
    passes:         contraction passes the call ran
    """
    bits: object
    probabilities: object
    candidates: int
    clipped: int
    max_ratio: float
    next_candidate: int
    n_qubits: int
    passes: int = 0

    def bitstrings(self) -> List[str]:
        """The samples as host strings in Circuit.into_amplitude_network's character order: character q is qubit q."""
        words = self.bits.cpu().tolist()
        return ["".join("1" if (w >> q) & 1 else "0" for q in range(self.n_qubits)) for w in words]


class Sampler:
    """Samples bitstrings of `circuit`, with the qubits `open_qubits` contracted open (k of them) and the others closed.

    The plan is the amplitude network with '0' on the closed and '*' on the open qubits (Circuit.into_amplitude_network),
    on the greedy Cotengrust path unless `path` is given, created and staged once; `sampler.plan` is that NetworkPlan, so
    `sampler.plan.info()` shows the cost before sampling.  Which qubits are open changes that cost a great deal (open legs
    can stop the path from contracting a region early): choose them, or the path, with the open legs in mind.  More open
    qubits bring the acceptance rate 1/m towards 1 at a higher cost per contraction.

    sliced_legs: legs of that network to slice (SlicedNetwork), each shared by two leaves and on neither a closed qubit's
    bra nor an open qubit's leg.  The plan is then compiled for one slice, every slice is staged once (stage_slices), and
    each candidate's amplitudes are the sum over the slices in slice order, bit-identical to run_slices on that
    candidate's sliced networks; `plan.info()` is one slice's pass and `n_slices` the number of slices.  When no
    workspace copy fits beside the plan's own, a sampling call runs one candidate at a time in the plan's workspace, and
    `plan.run()` then needs `plan.stage` again (include/tncb.h, tncb_plan_sample_slices)."""

    def __init__(self, circuit, open_qubits: Sequence[int], path=None, ctx: Optional[Context] = None,
                 sliced_legs: Optional[Sequence[int]] = None):
        n = circuit.num_qubits()
        opened = _open_qubits(n, open_qubits)
        self.n_qubits = n
        self.open_qubits = sorted(opened)
        self.closed_qubits = [q for q in range(n) if q not in set(opened)]
        tn, _ = circuit.into_amplitude_network("".join("*" if q in set(opened) else "0" for q in range(n)))
        # into_amplitude_network appends the closed qubits' bras after the circuit's tensors, in qubit order
        index = {id(t): i for i, t in enumerate(leaves(tn))}
        self.closed_leaves = [index[id(t)] for t in tn.tensors[len(circuit.tensors):]]
        self.sliced_legs = None if sliced_legs is None else _check_sliced_legs(circuit, tn, self.open_qubits, sliced_legs)
        if path is None:
            from .contractionpath.paths import Cotengrust
            opt = Cotengrust(tn)
            opt.find_path()
            path = opt.get_best_replace_path()
        if self.sliced_legs is None:
            self.n_slices = 1
            self.plan = NetworkPlan(tn, path, ctx)
            self.plan.stage(tn)
        else:
            from .contractionpath.slicing import SlicedNetwork
            sn = SlicedNetwork(tn, self.sliced_legs)
            nets = [sn.slice(a) for a in sn.assignments]
            self.n_slices = len(nets)
            self.plan = NetworkPlan(nets[0], path, ctx)
            self.plan.stage_slices(nets)
        qubit_of = {e: q for q, e in enumerate(circuit.open_edges)}
        self.result_qubits = [qubit_of[int(e)] for e in self.plan.result_legs]
        self._keep = (u64_array(self.closed_leaves), (C.c_int * max(len(self.closed_qubits), 1))(*self.closed_qubits),
                      (C.c_int * max(len(self.result_qubits), 1))(*self.result_qubits))
        self._spec = TncbSampleSpec(n, len(self.closed_qubits), *self._keep)

    def sample(self, n_samples: int, m: float, seed: int = 0, first: int = 0, max_candidates: Optional[int] = None,
               batch: Optional[int] = None) -> Samples:
        """Up to `n_samples` samples from candidates first, first + 1, ... of `seed`, in passes of `batch` candidates
        (None: as many workspace copies as fit).  The call stops at n_samples samples or after max_candidates candidates;
        the default, ceil(16 m n_samples) + 1024, is sixteen times the count a normalised state needs on average (a
        candidate is accepted with probability 1/m), so an unreachable target ends.

        m has no default.  The samples are exact while every ratio q 2^(n-k) / m stays at or below 1; the returned
        max_ratio is the largest seen and `clipped` counts the candidates above 1.  m = 2^(n-k) never clips a normalised
        state (q <= 1) but accepts rarely; a pilot run with any m reports max_ratio, and m a little above max_ratio times
        the pilot's m clips none of the candidates it saw.  Re-run with a larger m if clipped is not 0.

        The output is a function of (seed, first, candidates consumed) alone: the pass size and the split into calls
        do not change it, and sample(a) followed by sample(b, first=next_candidate) equals sample(a + b).  Ranks of a
        multi-GPU job draw from disjoint candidate ranges through `first`.  The call runs on the context stream after
        torch's current stream, which then waits for it."""
        import torch
        n_samples, first = int(n_samples), int(first)
        if n_samples < 1:
            raise ValueError(f"n_samples must be at least 1, not {n_samples}")
        if max_candidates is None:
            finite = math.isfinite(float(m)) and m > 0      # (else the library refuses m)
            max_candidates = min(math.ceil(16 * float(m) * n_samples) + 1024, (1 << 64) - 1) if finite else 0
        ctx = self.plan.ctx
        dev = torch.device("cuda", ctx.device)
        bits = torch.empty(n_samples, dtype=torch.int64, device=dev)
        probs = torch.empty(n_samples, dtype=torch.float64, device=dev)
        stats = TncbSampleStats()
        fn = "tncb_plan_sample" if self.sliced_legs is None else "tncb_plan_sample_slices"
        _library_call(ctx, fn, [ctx.handle, self.plan.handle, C.byref(self._spec), int(seed), first,
                                  int(max_candidates), n_samples, float(m), int(batch or 0), bits.data_ptr(), probs.data_ptr(),
                                  C.byref(stats)], keep=[bits, probs])
        s = int(stats.samples)
        return Samples(bits[:s], probs[:s], int(stats.candidates), int(stats.clipped), float(stats.max_ratio),
                       first + int(stats.candidates), self.n_qubits, int(stats.passes))


def _open_qubits(n: int, open_qubits: Sequence[int]) -> List[int]:
    opened = [int(q) for q in open_qubits]
    if len(set(opened)) != len(opened) or any(not 0 <= q < n for q in opened):
        raise ValueError(f"open qubits {list(open_qubits)} must be distinct qubits of the {n}-qubit circuit")
    if not 1 <= n <= 64:
        raise ValueError(f"sampling takes circuits of 1..64 qubits, not {n}")
    return opened


def _check_sliced_legs(circuit, tn, open_qubits: Sequence[int], sliced_legs: Sequence[int]) -> List[int]:
    """the legs to slice of the open amplitude network `tn`, or ValueError: a leg listed twice, on a closed qubit's bra,
    on an open qubit, or not shared by two leaves"""
    legs = [int(l) for l in sliced_legs]
    count = {}
    for t in leaves(tn):
        for l in t.legs:
            count[l] = count.get(l, 0) + 1
    bra = {int(circuit.open_edges[q]): q for q in range(circuit.num_qubits()) if q not in set(open_qubits)}
    opened = {int(circuit.open_edges[q]): q for q in open_qubits}
    for i, l in enumerate(legs):
        if l in legs[:i]:
            raise ValueError(f"sliced leg {l} is listed twice")
        if l in bra:
            raise ValueError(f"sliced leg {l} lies on the bra of closed qubit {bra[l]}: a candidate's bit fixes it")
        if l in opened:
            raise ValueError(f"sliced leg {l} is the open leg of qubit {opened[l]}")
        if count.get(l, 0) != 2:
            raise ValueError(f"sliced leg {l} is not shared by two leaves of the amplitude network")
    return legs


def open_path(circuit, path: ContractionPath, open_qubits: Sequence[int]) -> ContractionPath:
    """The path of the open amplitude network (into_amplitude_network with '*' on `open_qubits`, '0' elsewhere) derived
    from `path`, a flat replace-left path of the closed one (into_amplitude_network("0" * n)).  The open qubits' bras are
    dropped: a pair whose left slot holds a dropped bra passes its right operand into that slot, a pair whose right
    operand is a dropped bra is left out, and later leaves move down.  The other pairs keep their order, so a tree whose
    open qubits' bras join near its root keeps its cost (slicing.path_cost)."""
    n = circuit.num_qubits()
    opened = set(_open_qubits(n, open_qubits))
    if not path.is_simple():
        raise ValueError("open_path takes a flat path; this one has nested paths")
    g = len(circuit.tensors)
    where: List[Optional[int]] = []      # closed slot -> open slot, None: nothing (a dropped bra, or consumed)
    kept = 0
    for i in range(g + n):
        if i >= g and i - g in opened:
            where.append(None)
        else:
            where.append(kept)
            kept += 1
    pairs = []
    for a, b in path.toplevel:
        if not (0 <= a < g + n and 0 <= b < g + n):
            raise ValueError(f"pair ({a}, {b}) is outside the closed network's {g + n} leaves")
        x, y = where[a], where[b]
        if x is None:
            where[a] = y
        elif y is not None:
            pairs.append((x, y))
        where[b] = None
    return ContractionPath.simple(pairs)
