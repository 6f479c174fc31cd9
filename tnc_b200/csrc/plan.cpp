// Host-side leg algebra: turns one pairwise contraction into its GEMM view.
// Follows Tensor::symmetric_difference (tnc/src/tensornetwork/tensor.rs:463-479) for the
// output legs and the call contract of tetra::contract (contraction.rs:78-84).
#include "internal.h"
#include <algorithm>

namespace tncb {

static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
int fail(int status, const std::string& msg) { g_last_error = msg; return status; }
const std::string& last_error_ref() { return g_last_error; }

struct RawLeg { long long dim, sa, sb; };

// Merge neighbours that are contiguous in every operand they index; drop dim-1 legs.
static void fuse(std::vector<RawLeg>& v, bool use_b) {
  std::vector<RawLeg> out;
  for (const RawLeg& l : v) {
    if (l.dim == 1) continue;
    if (!out.empty()) {
      RawLeg& p = out.back();
      bool ok = p.sa == l.sa * l.dim && (!use_b || p.sb == l.sb * l.dim);
      if (ok) { p.dim *= l.dim; p.sa = l.sa; p.sb = l.sb; continue; }
    }
    out.push_back(l);
  }
  v.swap(out);
}

static int to_list(const std::vector<RawLeg>& v, LegList& L) {
  if ((int)v.size() > kMaxGroups) return fail(TNCB_ERR_INVALID, "too many leg groups");
  L.n = (int)v.size();
  for (int i = 0; i < L.n; i++) { L.dim[i] = v[i].dim; L.sa[i] = v[i].sa; L.sb[i] = v[i].sb; }
  return TNCB_OK;
}

int plan_pair(int n_a, const uint64_t* a_legs, const uint64_t* a_dims,
              int n_b, const uint64_t* b_legs, const uint64_t* b_dims, PairPlan& P) {
  if (n_a < 0 || n_b < 0 || n_a > kMaxLegs || n_b > kMaxLegs)
    return fail(TNCB_ERR_INVALID, "tensor rank out of range");
  std::vector<long long> sa(n_a), sb(n_b);
  long long s = 1;
  for (int i = n_a - 1; i >= 0; i--) { sa[i] = s; s *= (long long)a_dims[i]; }
  s = 1;
  for (int i = n_b - 1; i >= 0; i--) { sb[i] = s; s *= (long long)b_dims[i]; }
  for (int i = 0; i < n_a; i++)
    for (int j = i + 1; j < n_a; j++)
      if (a_legs[i] == a_legs[j]) return fail(TNCB_ERR_INVALID, "duplicate leg id in tensor a");
  for (int i = 0; i < n_b; i++)
    for (int j = i + 1; j < n_b; j++)
      if (b_legs[i] == b_legs[j]) return fail(TNCB_ERR_INVALID, "duplicate leg id in tensor b");

  auto find = [](const uint64_t* legs, int n, uint64_t l) { for (int i = 0; i < n; i++) if (legs[i] == l) return i; return -1; };

  P = PairPlan();
  std::vector<RawLeg> mv, nv, kv_a, kv_b;
  // (b \ a) first, then (a \ b): tensor.rs:466-476 with self = b, other = a (contraction.rs:64)
  for (int j = 0; j < n_b; j++) {
    if (find(a_legs, n_a, b_legs[j]) < 0) {
      P.out_legs.push_back(b_legs[j]); P.out_dims.push_back(b_dims[j]);
      nv.push_back({(long long)b_dims[j], sb[j], 0}); P.N *= (long long)b_dims[j];
    }
  }
  for (int i = 0; i < n_a; i++) {
    int j = find(b_legs, n_b, a_legs[i]);
    if (j < 0) {
      P.out_legs.push_back(a_legs[i]); P.out_dims.push_back(a_dims[i]);
      mv.push_back({(long long)a_dims[i], sa[i], 0}); P.M *= (long long)a_dims[i];
    } else {
      if (a_dims[i] != b_dims[j])
        return fail(TNCB_ERR_SHAPE, "bond dimension mismatch on leg " + std::to_string(a_legs[i]));
      kv_a.push_back({(long long)a_dims[i], sa[i], sb[j]}); P.K *= (long long)a_dims[i];
    }
  }
  // The order in which the shared legs are enumerated is free (a sum); try a's order and
  // b's order and keep the one that fuses into fewer groups (longer contiguous runs).
  for (int j = 0; j < n_b; j++) {
    int i = find(a_legs, n_a, b_legs[j]);
    if (i >= 0) kv_b.push_back({(long long)a_dims[i], sa[i], sb[j]});
  }
  fuse(mv, false); fuse(nv, false); fuse(kv_a, true); fuse(kv_b, true);
  const std::vector<RawLeg>& kv = (kv_b.size() < kv_a.size()) ? kv_b : kv_a;
  int rc;
  if ((rc = to_list(mv, P.m)) || (rc = to_list(nv, P.n)) || (rc = to_list(kv, P.k))) return rc;

  long long a_k_in = P.k.n ? P.k.sa[P.k.n - 1] : (1LL << 62);
  long long b_k_in = P.k.n ? P.k.sb[P.k.n - 1] : (1LL << 62);
  long long a_m_in = P.m.n ? P.m.sa[P.m.n - 1] : (1LL << 62);
  long long b_n_in = P.n.n ? P.n.sa[P.n.n - 1] : (1LL << 62);
  P.a_kfast = a_k_in < a_m_in;
  P.b_kfast = b_k_in < b_n_in;

  // K1 (gather + DMMA ZGEMM) pays off once the tile is reasonably full and there is
  // enough arithmetic to amortise the offset tables; everything else goes to K0.
  bool gemm_like = P.M >= 16 && P.N >= 16 && P.K >= 4 &&
                   (double)P.M * (double)P.N * (double)P.K >= (double)(1 << 17);
  P.kernel_class = gemm_like ? 1 : 0;
  // K2: "gate application" shapes -- a big tensor against a tiny one (low arithmetic intensity,
  // HBM-bound).  One thread owns one index of the big free side and produces all outputs of the
  // small side, so the big operand is read exactly once.
  if (P.K <= 64) {
    if (P.N <= 16 && P.N * P.K <= 256 && P.M >= 4096) { P.kernel_class = 2; P.k2_big_is_a = true; }
    else if (P.M <= 16 && P.M * P.K <= 256 && P.N >= 4096) { P.kernel_class = 2; P.k2_big_is_a = false; }
  }
  return TNCB_OK;
}

} // namespace tncb

extern "C" {

const char* tncb_last_error(void) { return tncb::last_error_ref().c_str(); }

const char* tncb_strerror(int status) {
  switch (status) {
    case TNCB_OK: return "ok";
    case TNCB_ERR_INVALID: return "invalid argument";
    case TNCB_ERR_SHAPE: return "bond dimension mismatch";
    case TNCB_ERR_UNCONTRACTED: return "Cannot convert uncontracted tensor to data";
    case TNCB_ERR_NOT_CONTRACTED: return "Not fully contracted";
    case TNCB_ERR_OOM: return "device arena exhausted";
    case TNCB_ERR_CUDA: return "CUDA error";
    case TNCB_ERR_GATE: return "gate error";
    case TNCB_ERR_NCCL: return "NCCL error";
    case TNCB_ERR_UNSUPPORTED: return "unsupported";
    case TNCB_ERR_IO: return "file error";
    default: return "unknown status";
  }
}

const char* tncb_version(void) { return "libtncb200 0.3 (sm_90a; K0 strided/split-K, K1 gather+DMMA ZGEMM, K1' wgmma int8 modular / digit slicing, K2 streaming)"; }

int tncb_pair_out_legs(int n_a, const uint64_t* a_legs, const uint64_t* a_dims,
                       int n_b, const uint64_t* b_legs, const uint64_t* b_dims,
                       int* n_out, uint64_t* out_legs, uint64_t* out_dims,
                       uint64_t* m, uint64_t* n, uint64_t* k) {
  tncb::PairPlan P;
  int rc = tncb::plan_pair(n_a, a_legs, a_dims, n_b, b_legs, b_dims, P);
  if (rc) return rc;
  if (n_out) *n_out = (int)P.out_legs.size();
  for (size_t i = 0; i < P.out_legs.size(); i++) {
    if (out_legs) out_legs[i] = P.out_legs[i];
    if (out_dims) out_dims[i] = P.out_dims[i];
  }
  if (m) *m = (uint64_t)P.M;
  if (n) *n = (uint64_t)P.N;
  if (k) *k = (uint64_t)P.K;
  return TNCB_OK;
}

int tncb_pair_kernel_class(int n_a, const uint64_t* a_legs, const uint64_t* a_dims,
                           int n_b, const uint64_t* b_legs, const uint64_t* b_dims) {
  tncb::PairPlan P;
  int rc = tncb::plan_pair(n_a, a_legs, a_dims, n_b, b_legs, b_dims, P);
  if (rc) return rc;
  return P.kernel_class;
}

} // extern "C"
