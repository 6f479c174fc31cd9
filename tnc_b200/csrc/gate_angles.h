// The six gates of the table that take angles (u, rx, ry, rz, cp, fsim): U(a), dU/da_s and d²U/da_s da_t, element by
// element in the gate's row-major order, for the host (gates.cpp: tncb_gate_matrix, tncb_gate_derivative) and the
// device (angles.cu) alike, so that U has one source.  Plain double arithmetic: each value entry is formed exactly as
// the std::complex expressions of the reference table form it (a complex times a real scales both parts, so -i * s has
// the real part -0.0 * s), which keeps tncb_gate_matrix bit for bit.  The adjoint flag transposes and conjugates; the
// angles are real, so the derivative of U† is (dU)†.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define TNCB_HD __host__ __device__ __forceinline__
#else
#define TNCB_HD inline
#endif

namespace tncb {
namespace ga {

enum Gate { kU = 0, kRx, kRy, kRz, kCp, kFsim, kGates };

struct Cplx { double re, im; };

TNCB_HD int n_angles(int g) { return g == kU ? 3 : g == kFsim ? 2 : 1; }
TNCB_HD int dim(int g) { return g == kCp || g == kFsim ? 4 : 2; }    // matrix rows: 4 or 16 elements

// cos and sin of the (at most four) arguments a gate's entries use, computed once per angle set
struct Trig { double c[4], s[4]; };
TNCB_HD void trig_of(double x, Trig& T, int k) { T.c[k] = cos(x); T.s[k] = sin(x); }
TNCB_HD Trig trig(int g, double a0, double a1, double a2) {
  Trig T{};
  switch (g) {
    case kU: trig_of(a0 / 2, T, 0); trig_of(a1, T, 1); trig_of(a2, T, 2); trig_of(a1 + a2, T, 3); break;
    case kRx: case kRy: trig_of(a0 / 2, T, 0); break;
    case kRz: trig_of(-a0 / 2, T, 0); trig_of(a0 / 2, T, 1); break;
    case kCp: trig_of(a0, T, 0); break;
    case kFsim: trig_of(a0, T, 0); trig_of(-a1, T, 1); break;
  }
  return T;
}

// the n-th derivative (n <= 2) with respect to a of cos(k a), sin(k a) and e^{i k a}, from c = cos(k a), s = sin(k a)
TNCB_HD double dcos(double c, double s, double k, int n) { return n == 0 ? c : n == 1 ? -k * s : -(k * k) * c; }
TNCB_HD double dsin(double c, double s, double k, int n) { return n == 0 ? s : n == 1 ? k * c : -(k * k) * s; }
TNCB_HD Cplx dexpi(const Trig& T, int j, double k, int n) { return {dcos(T.c[j], T.s[j], k, n), dsin(T.c[j], T.s[j], k, n)}; }
TNCB_HD Cplx scale(Cplx z, double r) { return {z.re * r, z.im * r}; }
TNCB_HD Cplx neg(Cplx z) { return {-z.re, -z.im}; }

// Element e of d^(o0+o1+o2) U / da0^o0 da1^o1 da2^o2 (total order <= 2), before the adjoint; T = trig(g, a0, a1, a2).
TNCB_HD Cplx entry(int g, const Trig& T, int o0, int o1, int o2, int e) {
  const Cplx z{0.0, 0.0}, one{1.0, 0.0};
  switch (g) {
    case kU: {                         // [[c, -e^{iλ} s], [e^{iφ} s, e^{i(φ+λ)} c]], c, s of θ/2; (θ, φ, λ) = (a0, a1, a2)
      const double c = dcos(T.c[0], T.s[0], 0.5, o0), s = dsin(T.c[0], T.s[0], 0.5, o0);
      if (e == 0) return o1 || o2 ? z : Cplx{c, 0.0};
      if (e == 1) return o1 ? z : scale(neg(dexpi(T, 2, 1.0, o2)), s);
      if (e == 2) return o2 ? z : scale(dexpi(T, 1, 1.0, o1), s);
      return scale(dexpi(T, 3, 1.0, o1 + o2), c);
    }
    case kRx: {                        // [[c, -i s], [-i s, c]]
      if (e == 0 || e == 3) return scale(one, dcos(T.c[0], T.s[0], 0.5, o0));
      return scale(Cplx{-0.0, -1.0}, dsin(T.c[0], T.s[0], 0.5, o0));
    }
    case kRy: {                        // [[c, -s], [s, c]]
      if (e == 0 || e == 3) return scale(one, dcos(T.c[0], T.s[0], 0.5, o0));
      return scale(e == 1 ? Cplx{-1.0, -0.0} : one, dsin(T.c[0], T.s[0], 0.5, o0));
    }
    case kRz:                          // diag(e^{-ia/2}, e^{ia/2})
      if (e == 0) return dexpi(T, 0, -0.5, o0);
      if (e == 3) return dexpi(T, 1, 0.5, o0);
      return z;
    case kCp:                          // diag(1, 1, 1, e^{ia})
      if (e == 15) return dexpi(T, 0, 1.0, o0);
      return !o0 && (e == 0 || e == 5 || e == 10) ? one : z;
    case kFsim:                        // [[1], [cos θ, -i sin θ], [-i sin θ, cos θ], [e^{-iφ}]]; (θ, φ) = (a0, a1)
      if (o0 && o1) return z;
      if (e == 0) return o0 || o1 ? z : one;
      if (e == 5 || e == 10) return o1 ? z : Cplx{dcos(T.c[0], T.s[0], 1.0, o0), 0.0};
      if (e == 6 || e == 9) return o1 ? z : Cplx{0.0, -dsin(T.c[0], T.s[0], 1.0, o0)};
      if (e == 15) return o0 ? z : dexpi(T, 1, -1.0, o1);
      return z;
  }
  return z;
}

// Element e (row-major) of U (s < 0), dU/da_s (t < 0) or d²U/da_s da_t of gate g with T = trig(g, angles), adjointed
// when `adjoint` is set.  Slots past the gate's angle count must not be passed.
TNCB_HD Cplx element(int g, const Trig& T, int s, int t, bool adjoint, int e) {
  const int o0 = (s == 0) + (t == 0), o1 = (s == 1) + (t == 1), o2 = (s == 2) + (t == 2);
  if (!adjoint) return entry(g, T, o0, o1, o2, e);
  const int d = dim(g);
  const Cplx v = entry(g, T, o0, o1, o2, (e % d) * d + e / d);
  return {v.re, -v.im};
}

}  // namespace ga
}  // namespace tncb
