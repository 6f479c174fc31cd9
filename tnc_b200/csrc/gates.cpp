// Host-side gate table: replaces load_gate / load_gate_adjoint (tnc/src/gates.rs:50-66) and
// the 18 Gate impls (gates.rs:147-627).  Gate tensors are 4 or 16 complex numbers; they are
// materialised on the host and travel to the device inside the single leaf upload of a
// network (network.cpp), not one call per pair as in the reference (tensordata.rs:50-56).
#include "internal.h"
#include "gate_angles.h"
#include <cmath>
#include <complex>
#include <cstring>

namespace tncb {

typedef std::complex<double> cd;

// the table index of a gate that takes angles (gate_angles.h), -1 for the others
int angle_gate(const char* name) {
  static const char* const names[ga::kGates] = {"u", "rx", "ry", "rz", "cp", "fsim"};
  for (int g = 0; g < ga::kGates; g++) if (name && std::strcmp(name, names[g]) == 0) return g;
  return -1;
}

// every entry of U (s < 0), dU/da_s (t < 0) or d²U/da_s da_t of angle gate g into out; returns 4 or 16
static int angle_entries(int g, const double* ang, int s, int t, bool adjoint, cd* out) {
  const int cnt = ga::dim(g) * ga::dim(g), n = ga::n_angles(g);
  const ga::Trig T = ga::trig(g, ang[0], n > 1 ? ang[1] : 0.0, n > 2 ? ang[2] : 0.0);
  for (int e = 0; e < cnt; e++) {
    const ga::Cplx v = ga::element(g, T, s, t, adjoint, e);
    out[e] = cd(v.re, v.im);
  }
  return cnt;
}

// Returns number of complex entries written (4 or 16) or a negative status.
int gate_matrix(const char* name, const double* ang, int n_ang, bool adjoint, cd* out) {
  const cd z(0, 0), o(1, 0), i(0, 1);
  const double h = 0.70710678118654752440; // FRAC_1_SQRT_2
  auto need = [&](int n) -> bool {
    if (n_ang != n) { fail(TNCB_ERR_GATE, "Expected " + std::to_string(n) + " angles, but got " + std::to_string(n_ang) + "."); return false; }
    return true;
  };
  int cnt = 0;
  auto set4 = [&](cd a, cd b, cd c, cd d) { out[0] = a; out[1] = b; out[2] = c; out[3] = d; cnt = 4; };
  auto set16 = [&](const cd (&m)[16]) { for (int q = 0; q < 16; q++) out[q] = m[q]; cnt = 16; };
  std::string g(name ? name : "");
  const int ag = angle_gate(name);
  if (ag >= 0) {                       // u, rx, ry, rz, cp, fsim: gate_angles.h, adjoint included
    if (!need(ga::n_angles(ag))) return TNCB_ERR_GATE;
    return angle_entries(ag, ang, -1, -1, adjoint, out);
  }
  if (g == "x") { if (!need(0)) return TNCB_ERR_GATE; set4(z, o, o, z); }
  else if (g == "y") { if (!need(0)) return TNCB_ERR_GATE; set4(z, -i, i, z); }
  else if (g == "z") { if (!need(0)) return TNCB_ERR_GATE; set4(o, z, z, -o); }
  else if (g == "h") { if (!need(0)) return TNCB_ERR_GATE; set4(cd(h, 0), cd(h, 0), cd(h, 0), cd(-h, 0)); }
  else if (g == "t") { if (!need(0)) return TNCB_ERR_GATE; set4(o, z, z, cd(h, h)); }
  else if (g == "sx") { if (!need(0)) return TNCB_ERR_GATE; set4(cd(.5, .5), cd(.5, -.5), cd(.5, -.5), cd(.5, .5)); }
  else if (g == "sy") { if (!need(0)) return TNCB_ERR_GATE; set4(cd(.5, .5), cd(-.5, -.5), cd(.5, .5), cd(.5, .5)); }
  else if (g == "sz") { if (!need(0)) return TNCB_ERR_GATE; set4(o, z, z, i); }
  else if (g == "cx") { if (!need(0)) return TNCB_ERR_GATE; const cd m[16] = {o, z, z, z, z, o, z, z, z, z, z, o, z, z, o, z}; set16(m); }
  else if (g == "cz") { if (!need(0)) return TNCB_ERR_GATE; const cd m[16] = {o, z, z, z, z, o, z, z, z, z, o, z, z, z, z, -o}; set16(m); }
  else if (g == "swap") { if (!need(0)) return TNCB_ERR_GATE; const cd m[16] = {o, z, z, z, z, z, o, z, z, o, z, z, z, z, z, o}; set16(m); }
  else if (g == "iswap") { if (!need(0)) return TNCB_ERR_GATE; const cd m[16] = {o, z, z, z, z, z, i, z, z, i, z, z, z, z, z, o}; set16(m); }
  else return fail(TNCB_ERR_GATE, "Gate '" + g + "' not found.");
  if (adjoint) { // matrix_adjoint_inplace, gates.rs:82-99: swap dim halves, conjugate
    const int d = cnt == 4 ? 2 : 4;
    cd tmp[16];
    for (int r = 0; r < d; r++) for (int c = 0; c < d; c++) tmp[r * d + c] = std::conj(out[c * d + r]);
    std::memcpy(out, tmp, sizeof(cd) * cnt);
  }
  return cnt;
}

} // namespace tncb

extern "C" int tncb_gate_matrix(const char* name, const double* angles, int n_angles, int adjoint,
                                double* out_re_im, int* rank) {
  if (!name || !out_re_im || (n_angles > 0 && !angles)) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  tncb::cd buf[16];
  int cnt = tncb::gate_matrix(name, angles, n_angles, adjoint != 0, buf);
  if (cnt < 0) return cnt;
  for (int q = 0; q < cnt; q++) { out_re_im[2 * q] = buf[q].real(); out_re_im[2 * q + 1] = buf[q].imag(); }
  if (rank) *rank = cnt == 4 ? 2 : 4;
  return TNCB_OK;
}

extern "C" int tncb_gate_derivative(const char* name, const double* angles, int n_angles, int adjoint, int slot, int slot2,
                                    double* out_re_im, int* rank) {
  if (!name || !out_re_im || (n_angles > 0 && !angles)) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  tncb::cd buf[16];
  int cnt = tncb::gate_matrix(name, angles, n_angles, adjoint != 0, buf);    // the errors of tncb_gate_matrix
  if (cnt < 0) return cnt;
  const int g = tncb::angle_gate(name);
  const int n = g < 0 ? 0 : tncb::ga::n_angles(g);
  if (slot < 0 || slot >= n || slot2 >= n)
    return tncb::fail(TNCB_ERR_GATE, "slot out of range for this gate: '" + std::string(name) + "' takes " + std::to_string(n) +
                                         " angles, slots " + std::to_string(slot) + ", " + std::to_string(slot2));
  cnt = tncb::angle_entries(g, angles, slot, slot2 < 0 ? -1 : slot2, adjoint != 0, buf);
  for (int q = 0; q < cnt; q++) { out_re_im[2 * q] = buf[q].real(); out_re_im[2 * q + 1] = buf[q].imag(); }
  if (rank) *rank = cnt == 4 ? 2 : 4;
  return TNCB_OK;
}
