"""The angle table of gate_angles.h against 50 digits, without a GPU: U, every dU/da_s and every d²U/da_s da_t of u, rx,
ry, rz, cp and fsim, both adjoint flags, from tncb_gate_matrix and tncb_gate_derivative, real and imaginary parts
apart.  The reference writes each gate out from its definition with mpmath and is evaluated twice: at the double
arguments the table forms (a/2, -a/2, -a, a1 + a2, each one IEEE rounding of the exact value), where every component
must lie within a few units of 2^-53 of it, and at the nominal angles, where the rounding of those arguments adds
at most 2^-53 |x| + 2^-1075 per argument.  Structural zeros must be exactly zero; d²/da_s da_t = d²/da_t da_s bit for
bit.  tests/test_gpu_angles_elements.py reads the device's table against the same reference."""
import functools
import itertools
import math

import mpmath
import numpy as np
import pytest

M = mpmath.MPContext()
M.dps = 60
U53 = 2.0 ** -53
TINY = 2.0 ** -1074                              # one rounding in the subnormal range
N_ANG = {"u": 3, "rx": 1, "ry": 1, "rz": 1, "cp": 1, "fsim": 2}
DIM = {"u": 2, "rx": 2, "ry": 2, "rz": 2, "cp": 4, "fsim": 4}
# per component, relative to the reference at the formed arguments: a product of two sines or cosines, each within 1 ulp
# (glibc) or 2 ulp (CUDA) of its value, with exact factors (powers of two, signs) and one rounding: 5 or 9 units 2^-53
HOST_UNITS, DEVICE_UNITS = 5, 9

rng = np.random.default_rng(2024)
ANGLES = ([0.0, -0.0, math.pi, -math.pi, math.pi / 2, -math.pi / 2, 1e-300, 5e-324]
          + [float(x) for x in rng.uniform(-4, 4, 8)]
          + [1e3, -1e3, 123.456, 1e5, 105615.0, 2.0 ** 31 + 1, 1e15, 1e22, 1e300])


def angle_tuples(gate):
    """the angle sets a gate is checked at: every value for one-angle gates, every pair for fsim, and every (φ, λ) pair
    for u with θ running through every value as well"""
    n, V = N_ANG[gate], ANGLES
    if n == 1:
        return [(a,) for a in V]
    pairs = list(itertools.product(range(len(V)), repeat=2))
    if n == 2:
        return [(V[i], V[j]) for i, j in pairs]
    return [(V[(3 * i + 5 * j) % len(V)], V[i], V[j]) for i, j in pairs]


# ---- the gates from their definitions ----
# An entry is a list of terms (coefficient, factors); a factor (f, {slot: k}) is f(sum_s k a_s) with f cos, sin or cis
# (x -> e^{ix}).  Entries not listed are zero.
def _c(k):
    return ("cos", k)


def _s(k):
    return ("sin", k)


def _e(k):
    return ("cis", k)


H0 = {0: 0.5}
GATES = {
    # [[cos θ/2, -e^{iλ} sin θ/2], [e^{iφ} sin θ/2, e^{i(φ+λ)} cos θ/2]]
    "u": {0: [(1, [_c(H0)])], 1: [(-1, [_e({2: 1}), _s(H0)])], 2: [(1, [_e({1: 1}), _s(H0)])],
          3: [(1, [_e({1: 1, 2: 1}), _c(H0)])]},
    # [[cos θ/2, -i sin θ/2], [-i sin θ/2, cos θ/2]]
    "rx": {0: [(1, [_c(H0)])], 1: [(-1j, [_s(H0)])], 2: [(-1j, [_s(H0)])], 3: [(1, [_c(H0)])]},
    # [[cos θ/2, -sin θ/2], [sin θ/2, cos θ/2]]
    "ry": {0: [(1, [_c(H0)])], 1: [(-1, [_s(H0)])], 2: [(1, [_s(H0)])], 3: [(1, [_c(H0)])]},
    # diag(e^{-iθ/2}, e^{iθ/2})
    "rz": {0: [(1, [_e({0: -0.5})])], 3: [(1, [_e({0: 0.5})])]},
    # diag(1, 1, 1, e^{iθ})
    "cp": {0: [(1, [])], 5: [(1, [])], 10: [(1, [])], 15: [(1, [_e({0: 1})])]},
    # 1 ⊕ [[cos θ, -i sin θ], [-i sin θ, cos θ]] ⊕ e^{-iφ}
    "fsim": {0: [(1, [])], 5: [(1, [_c({0: 1})])], 6: [(-1j, [_s({0: 1})])], 9: [(-1j, [_s({0: 1})])],
             10: [(1, [_c({0: 1})])], 15: [(1, [_e({1: -1})])]},
}


def formed(k, a):
    """the double the table computes for sum_s k_s a_s: k a (k = ±1, ±1/2: exact but for halving a subnormal) or
    a_1 + a_2, one IEEE rounding either way"""
    terms = [kk * a[s] for s, kk in sorted(k.items())]
    x = terms[0]
    for t in terms[1:]:
        x = x + t
    return x


def nominal(k, a):
    return M.fsum(M.mpf(kk) * M.mpf(a[s]) for s, kk in k.items())


def rounds(k):
    """whether forming the argument can round: a sum, or a halving (of a subnormal)"""
    return len(k) > 1 or any(abs(kk) != 1 for kk in k.values())


@functools.lru_cache(maxsize=None)
def _cos_sin(x):
    return M.cos(x), M.sin(x)


def _factor(f, x, n):
    """the n-th derivative of f at x (mp)"""
    c, s = _cos_sin(x)
    if f == "cis":
        return M.mpc(c, s) * (1j ** n)
    if f == "cos":
        return [c, -s, -c][n]
    return [s, c, -s][n]


def _term_derivs(factors, D):
    """the product rule: every way to hand the slots D to the factors, as (multiplier, [(factor index, order)])"""
    out = []
    for assign in itertools.product(range(len(factors)), repeat=len(D)):
        mult, order = 1.0, [0] * len(factors)
        for slot, fi in zip(D, assign):
            mult *= factors[fi][1].get(slot, 0.0)
            order[fi] += 1
        if mult != 0.0:
            out.append((mult, order))
    return out


def _structure(gate, D):
    """per entry (re, im): False where that component is zero whatever the angles"""
    d = DIM[gate]
    st = np.zeros((d * d, 2), dtype=bool)
    for e, terms in GATES[gate].items():
        for coef, factors in terms:
            for mult, order in _term_derivs(factors, D):
                if any(f == "cis" for f, _ in factors):
                    st[e] = True
                    continue
                # real factors: the phase is the coefficient times the signs of the derivatives
                z = complex(coef) * mult
                st[e, 0] |= z.real != 0
                st[e, 1] |= z.imag != 0
    return st


@functools.lru_cache(maxsize=None)
def reference(gate, a, D):
    """d^|D| U / da_D (D a tuple of at most two slots) at the angles a (a tuple of doubles), before the adjoint:
    (at the formed arguments [d*d] mpc, at the nominal angles [d*d] mpc, argument-rounding bound [d*d] float)"""
    d = DIM[gate]
    at_formed, at_nominal, arg_bound = [M.mpc(0)] * (d * d), [M.mpc(0)] * (d * d), [0.0] * (d * d)
    for e, terms in GATES[gate].items():
        vf, vn, bound = M.mpc(0), M.mpc(0), 0.0
        for coef, factors in terms:
            xf = [M.mpf(formed(k, a)) for _, k in factors]
            xn = [nominal(k, a) for _, k in factors]
            for mult, order in _term_derivs(factors, D):
                pf, pn = M.mpc(coef) * mult, M.mpc(coef) * mult
                for (f, _), x1, x2, n in zip(factors, xf, xn, order):
                    pf *= _factor(f, x1, n)
                    pn *= _factor(f, x2, n)
                vf += pf
                vn += pn
                # every factor has modulus <= 1 and is 1-Lipschitz in its argument, |mult| <= 1
                bound += sum(U53 * abs(float(x2)) + 2.0 ** -1075 for (_, k), x2 in zip(factors, xn) if rounds(k))
        at_formed[e], at_nominal[e], arg_bound[e] = vf, vn, bound
    return at_formed, at_nominal, arg_bound


def adjointed(vals, d):
    """the adjoint of a row-major [d*d] list"""
    return [M.conj(vals[c * d + r]) for r in range(d) for c in range(d)]


def split(vals):
    """[n] mpc -> [n, 2] (hi, lo) doubles per component, so that hi + lo carries ~106 bits"""
    hi = np.zeros((len(vals), 2))
    lo = np.zeros((len(vals), 2))
    for i, v in enumerate(vals):
        for j, x in enumerate((v.real, v.imag)):
            hi[i, j] = float(x)
            lo[i, j] = float(x - hi[i, j])
    return hi, lo


@functools.lru_cache(maxsize=None)
def expected(gate, a, D, adjoint):
    """the reference of element e of d^|D| U(a) (adjointed when asked) as arrays [d*d, 2] over (re, im): (formed hi,
    formed lo, nominal hi, nominal lo, argument bound, structurally nonzero)"""
    d = DIM[gate]
    f, n, b = reference(gate, tuple(a), tuple(D))
    st = _structure(gate, tuple(D))
    b = np.repeat(np.asarray(b)[:, None], 2, axis=1)
    if adjoint:
        f, n = adjointed(f, d), adjointed(n, d)
        idx = [c * d + r for r in range(d) for c in range(d)]
        b, st = b[idx], st[idx]
    return split(f) + split(n) + (b, st)


def compare(got, gate, a, D, adjoint, units):
    """ratios of |got - reference| to the bounds of the module docstring for one matrix (complex [d*d]): (worst ratio at
    the formed arguments, worst at the nominal angles); asserts structural zeros and the two bounds"""
    fh, fl, nh, nl, ab, st = expected(gate, tuple(a), tuple(D), bool(adjoint))
    g = np.stack([got.real, got.imag], axis=1)
    what = (gate, a, D, adjoint)
    assert np.all(g[~st] == 0), (what, "structural zero", g[~st])
    err = np.abs((g - fh) - fl)
    tol = units * U53 * np.abs(fh) + TINY
    assert np.all(err <= tol), (what, g, fh, err / tol)
    err_n = np.abs((g - nh) - nl)
    tol_n = tol + ab
    assert np.all(err_n <= tol_n), (what, g, nh, err_n / tol_n)
    return float((err / tol).max()), float((err_n / tol_n).max())


def derivative_sets(gate):
    n = N_ANG[gate]
    return [()] + [(s,) for s in range(n)] + [(s, t) for s in range(n) for t in range(n)]


# ---- the host table ----
def _host(gate, a, D, adjoint):
    from tnc_b200.gates import load_gate, load_gate_adjoint, load_gate_derivative
    if not D:
        return (load_gate_adjoint if adjoint else load_gate)(gate, a).reshape(-1)
    return load_gate_derivative(gate, a, D[0], D[1] if len(D) > 1 else -1, adjoint).reshape(-1)


def test_reference_matches_closed_forms():
    """the reference itself at a few points where the entries are known in closed form"""
    f, _, _ = reference("u", (math.pi, 0.0, 0.0), ())
    assert abs(f[0] - M.cos(M.mpf(math.pi) / 2)) < 1e-55 and abs(f[1] + 1) < 1e-30
    f, _, _ = reference("rz", (1.0,), (0, 0))
    assert abs(f[0] + M.exp(-0.5j) / 4) < 1e-55
    f, _, _ = reference("u", (0.3, 0.7, -1.1), (1, 2))
    assert abs(f[3] + M.exp(1j * M.mpf(0.7 + -1.1)) * M.cos(M.mpf(0.3) / 2)) < 1e-55 and f[0] == 0 and f[1] == 0 and f[2] == 0
    _, n, b = reference("u", (0.0, 1e3, -1e3 + 1e-9), ())
    assert b[3] > 0 and b[0] == 0                # only the sum rounds


@pytest.mark.parametrize("gate", sorted(N_ANG))
def test_table_against_50_digits(built_lib, gate):
    worst_f = worst_n = 0.0
    for a in angle_tuples(gate):
        for adj in (False, True):
            for D in derivative_sets(gate):
                rf, rn = compare(_host(gate, a, D, adj), gate, a, D, adj, HOST_UNITS)
                worst_f, worst_n = max(worst_f, rf), max(worst_n, rn)
    print(f"{gate}: worst ratio to the bound {worst_f:.3f} at the formed arguments, {worst_n:.3g} at the nominal angles")


@pytest.mark.parametrize("gate", sorted(N_ANG))
def test_second_derivatives_symmetric(built_lib, gate):
    n = N_ANG[gate]
    for a in angle_tuples(gate)[::7]:
        for adj in (False, True):
            for s in range(n):
                for t in range(s + 1, n):
                    assert _host(gate, a, (s, t), adj).tobytes() == _host(gate, a, (t, s), adj).tobytes(), (gate, a, s, t)
