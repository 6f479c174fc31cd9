// K1' -- the dense contraction on the int8 tensor cores (Hopper wgmma) through an integer modular
// (Chinese-remainder) emulation of the complex128 GEMM.
//
// The tensor cores have no f64 wgmma.  The FP64 contraction C[n,m] = sum_k Bt[n,k] * At[m,k] reaches the int8
// tensor pipe like this (all arithmetic below is exact until the last conversion):
//   1. every row of the K-major operands is scaled by a power of two and truncated to an integer,
//        X' = trunc(x * 2^(a - e_row)),   |X'| < 2^a,  a <= 53   (e_row: max(|re|,|im|) of the row < 2^e_row)
//   2. for N pairwise coprime moduli m_i <= 256 the residues X' mod m_i (symmetric, int8) are written as
//      K-major planes -- the leg permutation of the reference's TTGT is fused into this pass (gather
//      through the plan's offset tables);
//   3. per modulus ONE int8 GEMM on wgmma.mma_async.s32.s8.s8 (int32 accumulators in registers) gives
//      C' mod m_i for the exact integer product C' = sum_k B'[n,k] A'[m,k]; the GEMM epilogue reduces the
//      accumulator mod m_i and stores one int8 per real output;
//   4. a reconstruction pass evaluates the CRT in split double precision,
//        C'/P = frac( sum_i y_i * rho_i ),  rho_i = ((P/m_i)^-1 mod m_i) / m_i,  P = prod m_i,
//      and scales by P * 2^(e_n + e_m - 2a).
// P > 8 K 2^(2a) makes |C'| < P/4, so the representative in (-P/2, P/2) is C' itself.  With a = 53 (the
// default) that needs N = 16 moduli for K <= 2^13: 16 int8 GEMM sweeps instead of the 36 digit-pair sweeps of
// the 7-bit slicing it replaces (csrc/ozaki.cu, kept for A/B), at a provable bound
//      |C - C_exact|[n,m] <= 2^(4-a) * K * max|B[n,:]| * max|A[m,:]|      (max over re/im parts)
// (each element is truncated by < 2^(e-a); 4K products per real output; 2^e <= 2 max).  The scheme is the
// published "Ozaki scheme II" (integer modular technique for GEMM emulation); this is an independent
// implementation for complex operands with the TTGT gather fused in.
//
// GEMM kernel (crt_gemm_kernel, main loop in sm90.h): persistent CTAs of three warpgroups, work item = (modulus, K chunk,
// 128 x 128 complex tile; three products: 128 x 256 of one product), items ordered modulus-major with a banded tile
// raster so that the Bt tiles of a band of ONE modulus stay in L2 while its At tiles stream from HBM once.
#include "internal.h"
#include "sm90.h"
#include <cuda.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>

namespace tncb {

constexpr int CRT_MAX_MOD = 20;
// pairwise coprime, descending; 255 is left out on purpose: with every odd modulus <= 253 the residue
// |r| <= 127 falls out of the FMA reduction without a range fix (see crt_residue_kernel)
static const int kModuli[CRT_MAX_MOD] = {256, 253, 251, 249, 247, 245, 241, 239, 233, 229,
                                         227, 223, 211, 199, 197, 193, 191, 181, 179, 173};
constexpr int CRT_BT = 128;        // tile rows per CTA (n) = tile cols (m)
constexpr int CRT_BKB = WG_BKB;    // K padding of the operand planes (one 128-byte swizzle row); a K block is 128 / BK stages
// Stage ring of the GEMM kernel (stage layouts in sm90.h), one configuration per form: STAGES slots of BK K bytes each.
// Chosen from tools/crt_gemm_sweep.py at the benchmark network's pairs (profiles/h100_crt_ring.jsonl, H100 80GB HBM3 at a
// 400 W power limit): three products keep 3 x 48 KB (2 slots: ~10 % slower; 4 x 48 KB: no faster; 8 x 24 KB, two wgmmas
// per stage: 25-35 % slower); four products take 5 x 40 KB of 64-byte stages (3-6 % faster than 2 x 80 KB).
// The -D overrides exist for that sweep, which builds each ring variant as a separate copy of the library.
#ifndef CRT_RING3_STAGES
#define CRT_RING3_STAGES 3
#endif
#ifndef CRT_RING3_BK
#define CRT_RING3_BK 128
#endif
#ifndef CRT_RING4_STAGES
#define CRT_RING4_STAGES 5
#endif
#ifndef CRT_RING4_BK
#define CRT_RING4_BK 64
#endif
template <bool KARA> struct CrtRing {
  static constexpr int STAGES = KARA ? CRT_RING3_STAGES : CRT_RING4_STAGES;
  static constexpr int BK = KARA ? CRT_RING3_BK : CRT_RING4_BK;
  using Stage = WgStage<KARA, BK>;
  static constexpr int SMEM = STAGES * Stage::BYTES + 1024;   // + the 1024-byte alignment pad of the dynamic shared memory
  static_assert(SMEM <= 232448 - 1024, "stage ring exceeds the per-block shared memory of sm_90");
};
constexpr int CRT_KCHUNK_MAX = 32768;           // 2 * K * 128 * 128 < 2^31 for K <= 2^15
constexpr int CRT_G = 34;                       // fixed-point bits of the leading CRT weight

struct CrtTables {
  int nmod;
  int a_bits_a, a_bits_b;     // integer bits kept per operand
  int mod[CRT_MAX_MOD];
  int magic[CRT_MAX_MOD];     // round(2^32 / m)
  double inv_mod[CRT_MAX_MOD];
  double rho1[CRT_MAX_MOD];   // floor(rho * 2^G) / 2^G
  double rho2[CRT_MAX_MOD];   // rho - rho1
  double p_scaled;            // P * 2^-(a_bits_a + a_bits_b)
};

// ---- host: moduli / CRT weights ------------------------------------------------------------------
double crt_log2_product(int n) {
  double s = 0;
  for (int i = 0; i < n; i++) s += std::log2((double)kModuli[i]);
  return s;
}

// Number of moduli and operand bits for a pair with contraction length K.
//   want_bits: integer bits per operand asked for (53 = full mantissa); nmod_force > 0 pins the modulus count.
void crt_choose(long long K, int want_bits, int nmod_force, int* nmod, int* bits_a, int* bits_b) {
  const double lk = std::log2((double)std::max<long long>(K, 1));
  auto needed = [&](int bits) {
    int q = 2;
    while (q < CRT_MAX_MOD && crt_log2_product(q) - 1e-9 < 2.0 * bits + lk + 3.0) q++;
    return q;
  };
  // A forced count is clamped to what 53-bit operands need: more moduli add no accuracy (the operands have no more
  // bits) but make C'/P a tiny fraction of 1, where the absolute error of the split CRT sum (~2^-75) would show.
  int n = nmod_force > 0 ? std::min(nmod_force, needed(53)) : needed(want_bits);
  n = std::max(2, std::min(n, CRT_MAX_MOD));
  int tot = (int)std::floor(crt_log2_product(n) - lk - 3.0 - 1e-9);
  tot = std::max(tot, 2);
  int a = std::min(want_bits, tot / 2), b = std::min(want_bits, tot - a);
  *nmod = n; *bits_a = a; *bits_b = b;
}

// Operand bits that guarantee |C - C_exact|[n,m] <= tol * max|B[n,:]| * max|A[m,:]|:  2^(4-a) K <= tol.
int crt_bits_for_tolerance(long long K, double tol) {
  if (!(tol > 0.0)) return 53;
  const int a = (int)std::ceil(std::log2(16.0 * (double)std::max<long long>(K, 1) / tol));
  return std::max(8, std::min(53, a));
}

static void crt_make_tables(int nmod, int bits_a, int bits_b, CrtTables& T) {
  T.nmod = nmod; T.a_bits_a = bits_a; T.a_bits_b = bits_b;
  long double P = 1.0L;
  for (int i = 0; i < nmod; i++) P *= (long double)kModuli[i];
  for (int i = 0; i < CRT_MAX_MOD; i++) { T.mod[i] = 1; T.magic[i] = 0; T.inv_mod[i] = 1.0; T.rho1[i] = T.rho2[i] = 0.0; }
  for (int i = 0; i < nmod; i++) {
    const int m = kModuli[i];
    long long pim = 1;                               // (P / m_i) mod m_i
    for (int j = 0; j < nmod; j++) if (j != i) pim = (pim * (kModuli[j] % m)) % m;
    long long inv = 1;
    while ((pim * inv) % m != 1) inv++;              // m <= 256: brute force
    const unsigned long long num = (unsigned long long)inv << CRT_G;
    const unsigned long long q = num / (unsigned long long)m, rem = num % (unsigned long long)m;
    T.mod[i] = m;
    T.magic[i] = (int)std::llround(4294967296.0 / (double)m);
    T.inv_mod[i] = 1.0 / (double)m;
    T.rho1[i] = std::ldexp((double)q, -CRT_G);
    T.rho2[i] = std::ldexp((double)rem / (double)m, -CRT_G);
  }
  T.p_scaled = (double)std::ldexp(P, -(bits_a + bits_b));
}

int crt_export_tables(int nmod, int* moduli, double* rho1, double* rho2, double* log2_product) {
  CrtTables T;
  crt_make_tables(nmod, 0, 0, T);
  for (int i = 0; i < nmod; i++) {
    if (moduli) moduli[i] = T.mod[i];
    if (rho1) rho1[i] = T.rho1[i];
    if (rho2) rho2[i] = T.rho2[i];
  }
  if (log2_product) *log2_product = crt_log2_product(nmod);
  return TNCB_OK;
}

// ---- operand preparation ---------------------------------------------------------------------------
constexpr int RES_ROWS_C = 32, RES_K_C = 128;   // operand tile of the preparation kernels
constexpr int kExpNonFinite = 0x7fffffff;   // row contains NaN / Inf: its outputs are poisoned with NaN
constexpr int kExpMin = -1000;              // rows below 2^-1000 keep absolute accuracy 2^(-1000-a)

// Row maxima: max over k of max(|re|, |im|) as the BIT PATTERN of a non-negative double (integer max == value
// max for those; NaN / Inf patterns are the largest, so one non-finite element marks the row).  Same 32 x 128
// tiling and lane split as the residue kernel; one shared-memory atomicMax per row and warp, one global per row and CTA.
__device__ __forceinline__ int crt_exp_from_bits(unsigned long long bits) {
  const int field = (int)(bits >> 52) & 0x7ff;        // (sign bit is clear)
  if (field == 0x7ff) return kExpNonFinite;
  if (field == 0) return bits == 0ull ? 0 : kExpMin;   // zero row / denormal row
  return max(field - 1022, kExpMin);                   // ilogb(max) + 1: max * 2^-e in [0.5, 1)
}

// Element -> thread map of the 32 x 128 operand tile (shared by the row-max and the residue kernel): a warp covers
// 2^lk consecutive k times 2^(5-lk) consecutive rows, chosen on the host from the operand's strides so that a warp-wide
// load touches whole contiguous runs (lk = 5: k is the fastest index, lk = 0: the free index is; e.g. lk = 2 when four
// consecutive k are contiguous and the next-fastest index is the row).
__device__ __forceinline__ void crt_tile_coord(int e, int lk, int& r, int& k) {
  const int lane = e & 31, blk = e >> 5;               // blk in [0, 128): 2^(7-lk) k-blocks x 2^lk row-blocks
  const int kb = blk & ((128 >> lk) - 1), rb = blk >> (7 - lk);
  k = (kb << lk) + (lane & ((1 << lk) - 1));
  r = (rb << (5 - lk)) + (lane >> lk);
}

__global__ void __launch_bounds__(256)
crt_rowmax_kernel(const double2* __restrict__ src, const long long* __restrict__ off_row, const long long* __restrict__ off_k,
                  long long rows, long long K, int lk, unsigned long long* __restrict__ rowmax) {
  __shared__ unsigned long long s_max[RES_ROWS_C];
  __shared__ long long s_offr[RES_ROWS_C], s_offk[RES_K_C];
  const long long row0 = (long long)blockIdx.x * RES_ROWS_C, k0 = (long long)blockIdx.y * RES_K_C;
  const int tid = threadIdx.x;
  // the tile's offset tables first (one round trip), then 16 independent element loads per thread (a second one)
  if (tid < RES_ROWS_C) { s_max[tid] = 0ull; s_offr[tid] = row0 + tid < rows ? __ldg(off_row + row0 + tid) : -1; }
  else if (tid >= 128) { const int k = tid - 128; s_offk[k] = k0 + k < K ? __ldg(off_k + k0 + k) : -1; }
  __syncthreads();
  unsigned long long mv[RES_ROWS_C * RES_K_C / 256];
#pragma unroll
  for (int it = 0; it < RES_ROWS_C * RES_K_C / 256; it++) {
    int r, k;
    crt_tile_coord(it * 256 + tid, lk, r, k);
    const long long orow = s_offr[r], ok = s_offk[k];
    mv[it] = 0ull;
    if (orow >= 0 && ok >= 0) {
      const double2 v = __ldg(src + orow + ok);
      mv[it] = max((unsigned long long)__double_as_longlong(fabs(v.x)), (unsigned long long)__double_as_longlong(fabs(v.y)));
    }
  }
  // a thread's row changes at most 2^lk times over the iterations (never for lk = 0), so its running maximum is flushed
  // to shared memory only when the row changes
  int cur_r = -1;
  unsigned long long cur_m = 0ull;
#pragma unroll
  for (int it = 0; it < RES_ROWS_C * RES_K_C / 256; it++) {
    int r, k;
    crt_tile_coord(it * 256 + tid, lk, r, k);
    unsigned long long m = mv[it];
    // lanes with the same row sit next to each other (2^lk of them): reduce over them, lane 0 of the group keeps the result
    for (int d = 1; d < (1 << lk); d <<= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if (r != cur_r) {
      if (cur_m && (tid & ((1 << lk) - 1)) == 0) atomicMax(&s_max[cur_r], cur_m);
      cur_r = r; cur_m = 0ull;
    }
    cur_m = max(cur_m, m);
  }
  if (cur_m && (tid & ((1 << lk) - 1)) == 0) atomicMax(&s_max[cur_r], cur_m);
  __syncthreads();
  if (tid < RES_ROWS_C && row0 + tid < rows && s_max[tid] != 0ull) atomicMax(rowmax + row0 + tid, s_max[tid]);
}

// Tile of 32 rows x 128 k: load (coalesced along whichever index is contiguous in the source), scale +
// truncate to integer-valued doubles in shared memory, then every thread reduces 4 consecutive k of each of four rows
// modulo every m_i and writes 4 bytes per plane and row; the 32 lanes of a warp write a row's 128 bytes of a plane in one
// instruction, so every plane line is written whole.  At 4 k per thread the integers x mod 2^32 stay in registers within
// the 80-register budget of 3 CTAs per SM (at 8 the compiler converted them again for every modulus).
// planes: [((mod * NPL + plane) * rowsP + row) * Kp + k];
//   four-product form:  COMPS == 2 (Bt side): NPL = 2 planes (re, im);  COMPS == 3 (At side): NPL = 3 planes (-im, re, im)
//   three-product form (KARA, see crt_gemm_kernel): NPL = 3 on both sides, (re, im, re + im); plane p of Bt meets plane p
//   of At (Karatsuba: k1 = Br Ar, k2 = Bi Ai, k3 = (Br + Bi)(Ar + Ai); re = k1 - k2, im = k3 - k1 - k2).
//   The sum of two residues is brought back into a byte ([-128, 127], still the same class mod m_i) by crt_fix_byte.
__device__ __forceinline__ int crt_fix_byte(int s, int m) {
  // |s| <= 256: s > 127 -> s - m in [-125, 83], s < -128 -> s + m in [-83, 124] (173 <= m <= 256; for m = 256 the byte is unchanged)
  if (s > 127) s -= m;
  else if (s < -128) s += m;
  return s;
}
constexpr int RES_ROWS = RES_ROWS_C, RES_K = RES_K_C, RES_RS = RES_K + RES_K / 8 + 1;   // padded row stride (elements)
template <int COMPS, bool KARA>
__global__ void __launch_bounds__(256, 3)
crt_residue_kernel(const double2* __restrict__ src, const long long* __restrict__ off_row, const long long* __restrict__ off_k,
                   long long rows, long long K, long long rowsP, long long Kp, const unsigned long long* __restrict__ rowmax, int bits, int lk,
                   const __grid_constant__ CrtTables T, int8_t* __restrict__ planes) {
  extern __shared__ __align__(16) unsigned char res_smem_raw[];
  double2* tile = reinterpret_cast<double2*>(res_smem_raw);
  __shared__ double s_scale[RES_ROWS];
  __shared__ long long s_offr[RES_ROWS], s_offk[RES_K];
  __shared__ double s_inv[CRT_MAX_MOD];      // the moduli tables out of the constant bank: an LDC with a register index
  __shared__ int s_mod[CRT_MAX_MOD];         // per loop trip was 35 % of this kernel's stall samples (ncu r02)
  const long long row0 = (long long)blockIdx.x * RES_ROWS, k0 = (long long)blockIdx.y * RES_K;
  const int tid = threadIdx.x;
  const double two_a = scalbn(1.0, bits);
  if (tid >= 64 && tid < 64 + CRT_MAX_MOD) { s_inv[tid - 64] = T.inv_mod[tid - 64]; s_mod[tid - 64] = T.mod[tid - 64]; }
  // the tile's offset tables and row scales first (one round trip), then 16 independent element loads per thread
  if (tid < RES_ROWS) {
    const long long r = row0 + tid;
    const int e = r < rows ? crt_exp_from_bits(rowmax[r]) : 0;
    s_scale[tid] = (e == kExpNonFinite) ? 0.0 : scalbn(1.0, -e);   // non-finite rows contribute zeros (outputs are poisoned later)
    s_offr[tid] = r < rows ? __ldg(off_row + r) : -1;
  } else if (tid >= 128) {
    const int k = tid - 128;
    s_offk[k] = k0 + k < K ? __ldg(off_k + k0 + k) : -1;
  }
  __syncthreads();
  double2 vv[RES_ROWS * RES_K / 256];
#pragma unroll
  for (int it = 0; it < RES_ROWS * RES_K / 256; it++) {
    int r, k;
    crt_tile_coord(it * 256 + tid, lk, r, k);
    const long long orow = s_offr[r], ok = s_offk[k];
    vv[it] = make_double2(0.0, 0.0);
    if (orow >= 0 && ok >= 0) vv[it] = __ldg(src + orow + ok);
  }
#pragma unroll
  for (int it = 0; it < RES_ROWS * RES_K / 256; it++) {
    int r, k;
    crt_tile_coord(it * 256 + tid, lk, r, k);
    const double sc = s_scale[r];
    double2 v = vv[it];
    v.x = trunc(v.x * sc * two_a);    // (x * 2^-e) is exact, * 2^a is exact, |.| < 2^a <= 2^53
    v.y = trunc(v.y * sc * two_a);
    if (sc == 0.0) { v.x = 0.0; v.y = 0.0; }   // (Inf * 0 = NaN)
    tile[r * RES_RS + k + (k >> 3)] = v;
  }
  __syncthreads();
  const double RMAGIC = 6755399441055744.0;   // 1.5 * 2^52: the low word of (x + RMAGIC) is rint(x) mod 2^32
  const long long plane_stride = rowsP * Kp;
  const int g = tid & 31;                      // group of 4 consecutive k: a warp stores a whole 128-byte row of a plane
  const int nmod = T.nmod;
#pragma unroll 1
  for (int pass = 0; pass < RES_ROWS / 8; pass++) {
    const int r = (tid >> 5) + 8 * pass;
    if (row0 + r >= rows) return;
    double xr[4], xi[4];
    int lr[4], li[4];                           // the integers x mod 2^32
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const double2 v = tile[r * RES_RS + g * 4 + j + (g >> 1)];
      xr[j] = v.x; xi[j] = v.y;
      lr[j] = (int)__double2ll_rn(v.x); li[j] = (int)__double2ll_rn(v.y);
    }
    int8_t* dst = planes + (row0 + r) * Kp + k0 + g * 4;
#pragma unroll 1
    for (int i = 0; i < nmod; i++) {
      const int m = s_mod[i];
      const double inv = s_inv[i];
      uint32_t wr = 0, wi = 0, ws = 0;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        // q = rint(x / m): ONE rounding (the product is exact inside the FMA, the sum has ulp 1); its low 32 bits are
        // the low word of the sum.  r = x - q m is tiny, so computing it modulo 2^32 in int32 is exact.
        // |x inv - x/m| <= 2^53/m * 2^-53 < 0.006  =>  |r| <= 0.506 m: <= 127 for every odd m <= 253, and for
        // m = 256 the byte wrap (128 -> -128) is itself a valid representative.
        const int qr = __double2loint(fma(xr[j], inv, RMAGIC));
        const int qi = __double2loint(fma(xi[j], inv, RMAGIC));
        const int rr = lr[j] - qr * m, ri = li[j] - qi * m;
        constexpr uint32_t sel[4] = {0x3214u, 0x3240u, 0x3410u, 0x4210u};   // low byte of the 2nd operand into byte j
        wr = __byte_perm(wr, (uint32_t)rr, sel[j]);
        wi = __byte_perm(wi, (uint32_t)ri, sel[j]);
        if (KARA) ws = __byte_perm(ws, (uint32_t)crt_fix_byte(rr + ri, m), sel[j]);
      }
      uint32_t* d = reinterpret_cast<uint32_t*>(dst + (long long)i * (KARA ? 3 : COMPS) * plane_stride);
      const long long ps = plane_stride / 4;
      if (KARA) {
        d[0] = wr; d[ps] = wi; d[2 * ps] = ws;
      } else if (COMPS == 2) {
        d[0] = wr; d[ps] = wi;
      } else {
        // byte-wise negation: |ri| <= 127 for odd m; for m = 256 the wrap -(-128) = -128 is again == 128 (mod 256)
        d[0] = __vneg4(wi); d[ps] = wr; d[2 * ps] = wi;
      }
    }
  }
}

// ---- GEMM kernel -----------------------------------------------------------------------------------
struct CrtGemmArgs {
  int8_t* R;          // residues + 128 as bytes: [((mod * nkc + kc) * NPL + plane) * Np + n] * Mp + m
                      //   four products: NPL = 2 (re, im);  three products: NPL = 3 (k1, k2, k3; re = k1 + k3, im = k1 + k2)
  int Np, Mp;         // padded plane rows of this panel (Np % 128 == 0, Mp % tile_m == 0)
  int tiles_n, tiles_m, tile_m;   // tile_m: 128 (four products: 128 re + 128 im columns) or 256 (three products)
  int nmod, nkc, kb_per_chunk, num_kb;
  int total_items;
  int group;          // n-tiles per raster band
  int negmod[CRT_MAX_MOD];   // -m_i (kept as data so that the epilogue's a - q m is ONE multiply-add)
  int magic[CRT_MAX_MOD];
};

struct CrtItem { int mod_i, prod, kc, n0, m0; };
template <bool KARA>
__device__ __forceinline__ CrtItem crt_decode(const CrtGemmArgs& p, int item) {
  const int tiles = p.tiles_n * p.tiles_m;
  const int mk = item / tiles, t = item - mk * tiles;
  CrtItem it;
  const int mp = mk / p.nkc;            // (modulus, product) major, K chunk minor
  it.kc = mk - mp * p.nkc;
  it.mod_i = KARA ? mp / 3 : mp; it.prod = KARA ? mp - it.mod_i * 3 : 0;
  // banded raster: bands of `group` n-tiles x all m-tiles; concurrently running CTAs (consecutive items)
  // share `group` Bt row bands and ~(#CTAs / group) At tiles
  const int per_band = p.group * p.tiles_m;
  const int band = t / per_band, first = band * p.group;
  const int gsize = min(p.group, p.tiles_n - first);
  const int r = t - band * per_band;
  it.n0 = (first + r % gsize) * CRT_BT;
  it.m0 = (r / gsize) * p.tile_m;
  return it;
}

// Persistent CTAs, work item = (modulus, K chunk, 128 x 128 complex tile), items ordered modulus-major with a banded tile
// raster.  Warpgroup 0 streams the operand tiles (TMA), warpgroups 1-2 run the wgmma main loop (sm90.h) on 64 Bt rows each
// and then their epilogue: accumulator mod m_i -> one offset byte -> a transpose of 32-bit words inside each lane quad
// (shuffles, no shared memory) -> 16-byte stores.  The producer runs ahead into the next item, up to the ring's depth,
// while the consumers are in their epilogue.
template <bool KARA>
__global__ void __launch_bounds__(WG_THREADS, 1)
crt_gemm_kernel(const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapA,
                const __grid_constant__ CrtGemmArgs p) {
  constexpr int STAGES = CrtRing<KARA>::STAGES, BK = CrtRing<KARA>::BK, SUB = CRT_BKB / BK;
  using Stage = typename CrtRing<KARA>::Stage;
  extern __shared__ __align__(1024) uint8_t crt_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(crt_smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t full_bar[STAGES], empty_bar[STAGES];
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) { wg_mbar_init(&full_bar[s], 1); wg_mbar_init(&empty_bar[s], 2); }   // 2 consumer warpgroups
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ================= TMA producer =================
    wg_setmaxnreg_producer();
    if (tid != 0) return;
    int it = 0;
    for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
      const CrtItem w = crt_decode<KARA>(p, item);
      const int kb0 = w.kc * p.kb_per_chunk, kb1 = min(p.num_kb, kb0 + p.kb_per_chunk);
      // three products: plane `prod` of both operands (256 At rows); four: Br, Bi and the three At planes (-Ai, Ar, Ai)
      const int rowB = (KARA ? w.mod_i * 3 + w.prod : w.mod_i * 2) * p.Np + w.n0;
      const int rowA = (KARA ? w.mod_i * 3 + w.prod : w.mod_i * 3) * p.Mp + w.m0;
      for (int ks = kb0 * SUB; ks < kb1 * SUB; ks++, it++) {
        uint8_t* st = wg_produce_begin<STAGES, KARA, BK>(smem, full_bar, empty_bar, it);
        uint64_t* bar = &full_bar[it % STAGES];
        const int kx = ks * BK;
        uint8_t* a = st + Stage::A;
        wg_tma_2d(&mapB, bar, st, kx, rowB);
        if (KARA) {
          wg_tma_2d(&mapA, bar, a, kx, rowA);
          wg_tma_2d(&mapA, bar, a + Stage::TILE, kx, rowA + WG_ROWS);
        } else {
          wg_tma_2d(&mapB, bar, st + Stage::B1, kx, rowB + p.Np);
          wg_tma_2d(&mapA, bar, a, kx, rowA);
          wg_tma_2d(&mapA, bar, a + Stage::TILE, kx, rowA + p.Mp);
          wg_tma_2d(&mapA, bar, a + 2 * Stage::TILE, kx, rowA + 2 * p.Mp);
        }
      }
    }
  } else {
    // ================= consumers: wgmma main loop + epilogue (own 64 Bt rows) =================
    wg_setmaxnreg_consumer();
    const int c = wg - 1, wq = tid >> 5, lane = tid & 31;
    const int q = lane & 3;
    const bool q0 = q & 1, q1 = q & 2;
    WgRing<STAGES, KARA, BK> ring{smem, full_bar, empty_bar};
    uint32_t acc[128];
#pragma unroll
    for (int i = 0; i < 128; i++) acc[i] = 0u;
    for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
      const CrtItem w = crt_decode<KARA>(p, item);
      const int kb0 = w.kc * p.kb_per_chunk, kb1 = min(p.num_kb, kb0 + p.kb_per_chunk);
      bool first = true;
      for (int ks = kb0 * SUB; ks < kb1 * SUB; ks++) ring.mma_stage(acc, c, first, tid == 0);
      ring.drain(tid == 0);
      const int negm = p.negmod[w.mod_i], magic = p.magic[w.mod_i];
      // A lane quad (same lane / 4) holds 256 consecutive residue bytes of each of its two rows h: lane q has the two bytes at
      // columns 8 j + 2 q (+1) for every j.  Per 16-byte chunk c (columns 16 c .. 16 c + 15) lane q packs its four bytes into
      // one word u = (j = 2c: 2 bytes | j = 2c + 1: 2 bytes).  Chunk c is made of word c of all four lanes; per group of four
      // chunks (i), a 4 x 4 transpose of words inside the quad (two butterfly rounds of shuffles) gives lane q the four words
      // of chunk 4 i + q, so the quad stores 64 contiguous bytes of its row per instruction.
      int8_t* row_base[2];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const long long n = (long long)w.n0 + c * 64 + wq * 16 + (lane >> 2) + 8 * h;
        row_base[h] = KARA ? p.R + ((long long)((w.mod_i * p.nkc + w.kc) * 3 + w.prod) * p.Np + n) * p.Mp + w.m0
                           : p.R + ((long long)((w.mod_i * p.nkc + w.kc) * 2) * p.Np + n) * p.Mp + w.m0;
      }
#pragma unroll
      for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          uint32_t x[4];            // x[k]: this lane's word of chunk 4 i + k
#pragma unroll
          for (int k = 0; k < 4; k++) {
            uint32_t u = 0;
#pragma unroll
            for (int jj = 0; jj < 2; jj++) {
#pragma unroll
              for (int e = 0; e < 2; e++) {
                const int a = (int)acc[4 * (8 * i + 2 * k + jj) + 2 * h + e];
                // q = floor(a * magic / 2^32) in [a/m - 1.25, a/m + 0.25] (|a| < 2^31, |magic / 2^32 - 1/m| <= 2^-33), so
                // t = a - q m lies in [-0.25 m, 1.25 m] = [-64, 320]: one conditional subtraction of m leaves a representative
                // in [-128, 127]; its low byte with the top bit flipped is the OFFSET byte residue + 128.
                int t = __mulhi(a, magic) * negm + a;
                if (t > 127) t += negm;
                u |= (((uint32_t)t & 0xffu) ^ 0x80u) << (8 * (2 * jj + e));
              }
            }
            x[k] = u;
          }
          // round 1 (lanes q, q ^ 1): keep the words for lanes with bit 0 = q0, hand over the others
          const uint32_t r0 = __shfl_xor_sync(0xffffffffu, q0 ? x[0] : x[1], 1);
          const uint32_t r1 = __shfl_xor_sync(0xffffffffu, q0 ? x[2] : x[3], 1);
          // words for lane q0 (a) and lane q0 + 2 (b) from the lanes 2 q1 + 0 and 2 q1 + 1
          const uint32_t a0 = q0 ? r0 : x[0], a1 = q0 ? x[1] : r0;
          const uint32_t b0 = q0 ? r1 : x[2], b1 = q0 ? x[3] : r1;
          // round 2 (lanes q, q ^ 2): keep the pair for lane q, hand over the other
          const uint32_t g0 = __shfl_xor_sync(0xffffffffu, q1 ? a0 : b0, 2);
          const uint32_t g1 = __shfl_xor_sync(0xffffffffu, q1 ? a1 : b1, 2);
          const uint32_t k0 = q1 ? b0 : a0, k1 = q1 ? b1 : a1;
          const uint32_t y0 = q1 ? g0 : k0, y1 = q1 ? g1 : k1, y2 = q1 ? k0 : g0, y3 = q1 ? k1 : g1;   // y[s]: word of lane s
          // columns 16 c + 4 v .. + 3 of chunk c = 4 i + q: lanes (0, 1) for v = 0, 2 and lanes (2, 3) for v = 1, 3
          const uint4 v = make_uint4(__byte_perm(y0, y1, 0x5410), __byte_perm(y2, y3, 0x5410),
                                     __byte_perm(y0, y1, 0x7632), __byte_perm(y2, y3, 0x7632));
          // three products: 256 columns of one plane; four products: chunks 0-7 real plane, 8-15 imaginary plane
          const int cc = 4 * i + q;
          int8_t* dst = KARA ? row_base[h] + cc * 16
                             : row_base[h] + (i >= 2 ? (long long)p.Np * p.Mp : 0LL) + (cc & 7) * 16;
          *reinterpret_cast<uint4*>(dst) = v;
        }
      }
    }
  }
}

// ---- CRT reconstruction -------------------------------------------------------------------------------
struct CrtReconArgs {
  const int8_t* R;
  double2* C;          // &C[n_begin * ldc + m_begin]
  const unsigned long long* max_n;   // row maxima (bit patterns) of this panel's Bt rows
  const unsigned long long* max_m;   // ... of this panel's At rows
  long long rows, cols, ldc;   // valid panel extent, row stride of C
  long long Np, Mp;
  int nkc;
};

// one thread: 4 consecutive m of one row n.  The kernel is bound by the latency of its residue loads, so with one K chunk the
// words of RB moduli (RB x 3 or RB x 2 independent loads) are all in flight before the first is used: 3 (three products) or
// 4 resident CTAs per SM keep 24 x 24 or 32 x 16 loads of 128 bytes per warp outstanding.
// No conversion-pipe instruction in the inner loop: a residue byte u = y + 128 becomes the double 2^52 + u by a byte
// permute into the low mantissa word, one DADD removes 2^52 + 128 nkc.
// KARA (three products): the planes hold k1, k2, k3 (+128 each); re = k1 - k2 and im = k3 - k1 - k2 are formed here from the
// bytes (the CRT sum is linear, no reduction mod m_i needed: |y| <= 3 * 128 * 32 < 2^13.6 keeps S1 exact, 13.6 + 34 + 4.4 bits).
template <bool ONE_CHUNK, bool KARA>
__global__ void __launch_bounds__(256, KARA ? 3 : 4)
crt_reconstruct_kernel(const __grid_constant__ CrtReconArgs a, const __grid_constant__ CrtTables T) {
  constexpr int NPR = KARA ? 3 : 2, RB = 8;
  const long long cols4 = a.Mp >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = idx / cols4, m4 = (idx - n * cols4) * 4;
  if (n >= a.rows || m4 >= a.cols) return;
  double s1r[4], s2r[4], s1i[4], s2i[4];
#pragma unroll
  for (int j = 0; j < 4; j++) { s1r[j] = s2r[j] = s1i[j] = s2i[j] = 0.0; }
  const long long plane = a.Np * a.Mp;
  const int8_t* base = a.R + n * a.Mp + m4;
  // a byte is u = y + 128; four products: sum of u over chunks - 128 nkc.  Three: re = (u1 - u2 + 256) - 256 per chunk,
  // im = (u3 - u1 - u2 + 512) - 384 per chunk (the +256 / +512 keep the running sums non-negative for the conversion below)
  const double bias = 4503599627370496.0 + (KARA ? 256.0 : 128.0) * (double)a.nkc;   // 2^52 + ...
  const double bias_i = 4503599627370496.0 + (KARA ? 384.0 : 128.0) * (double)a.nkc;
  const int nmod = T.nmod;
#pragma unroll 1
  for (int i0 = 0; i0 < nmod; i0 += RB) {
    uint32_t w[RB][NPR];       // one K chunk: the residue words of moduli i0 .. i0 + RB - 1
    if (ONE_CHUNK) {
#pragma unroll
      for (int u = 0; u < RB; u++) {
        if (i0 + u < nmod) {
#pragma unroll
          for (int p = 0; p < NPR; p++) w[u][p] = __ldg(reinterpret_cast<const uint32_t*>(base + (long long)((i0 + u) * NPR + p) * plane));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < RB; u++) {
      const int i = i0 + u;
      if (i >= nmod) break;
      uint32_t ur[4], ui[4];     // byte sums over the K chunks (still == C' + 128 nkc mod m_i)
#pragma unroll
      for (int j = 0; j < 4; j++) { ur[j] = 0; ui[j] = 0; }
      for (int c = 0; c < (ONE_CHUNK ? 1 : a.nkc); c++) {
        uint32_t x[NPR];
        if (ONE_CHUNK) {
#pragma unroll
          for (int p = 0; p < NPR; p++) x[p] = w[u][p];
        } else {
          const int8_t* pk = base + (long long)((i * a.nkc + c) * NPR) * plane;
#pragma unroll
          for (int p = 0; p < NPR; p++) x[p] = __ldg(reinterpret_cast<const uint32_t*>(pk + p * plane));
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const uint32_t k1 = __byte_perm(x[0], 0, 0x4440 + j), k2 = __byte_perm(x[1], 0, 0x4440 + j);
          if (KARA) {
            ur[j] += 256u + k1 - k2;
            ui[j] += 512u + __byte_perm(x[NPR - 1], 0, 0x4440 + j) - k1 - k2;
          } else {
            ur[j] += k1; ui[j] += k2;
          }
        }
      }
      const double r1 = T.rho1[i], r2 = T.rho2[i];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        // y * rho1 is exact (|y| <= 2^13, rho1 on a 2^-34 grid) and so is the sum over <= 20 moduli (|S1| < 2^18)
        const double dr = __hiloint2double(0x43300000, (int)ur[j]) - bias;
        const double di = __hiloint2double(0x43300000, (int)ui[j]) - bias_i;
        s1r[j] = fma(dr, r1, s1r[j]); s2r[j] = fma(dr, r2, s2r[j]);
        s1i[j] = fma(di, r1, s1i[j]); s2i[j] = fma(di, r2, s2i[j]);
      }
    }
  }
  const int en = crt_exp_from_bits(a.max_n[n]);
  double2* dst = a.C + n * a.ldc + m4;
  const double RMAGIC = 6755399441055744.0;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    if (m4 + j >= a.cols) break;
    const int em = crt_exp_from_bits(a.max_m[m4 + j]);
    double2 out;
    if (en == kExpNonFinite || em == kExpNonFinite) {
      out = make_double2(__longlong_as_double(0x7ff8000000000000LL), __longlong_as_double(0x7ff8000000000000LL));
    } else {
      // C'/P = S - round(S), |C'/P| <= 1/4; (S1 - Q) is exact, the rest rounds relative to the result itself
      const double qr = ((s1r[j] + s2r[j]) + RMAGIC) - RMAGIC;
      const double qi = ((s1i[j] + s2i[j]) + RMAGIC) - RMAGIC;
      const double fr = (s1r[j] - qr) + s2r[j], fi = (s1i[j] - qi) + s2i[j];
      out = make_double2(scalbn(fr * T.p_scaled, en + em), scalbn(fi * T.p_scaled, en + em));
    }
    __stcs(dst + j, out);   // C is not read again by this pair: stream it past the L2
  }
}

// ---- host side ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    cudaDriverEntryPointQueryResult q;
    void* p = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess) fn = (EncodeTiledFn)p;
  }
  return fn;
}
template <int BK>
int wg_make_map(CUtensorMap* m, void* ptr, uint64_t rows, uint64_t kbytes) {
  static_assert(BK == 128 || BK == 64, "SWIZZLE_128B or SWIZZLE_64B");
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(TNCB_ERR_CUDA, "cuTensorMapEncodeTiled is not available");
  cuuint64_t dims[2] = {kbytes, rows};
  cuuint64_t strides[1] = {kbytes};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)WG_ROWS};   // the inner box extent must not exceed the swizzle span
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   BK == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(TNCB_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  return TNCB_OK;
}
template int wg_make_map<128>(CUtensorMap*, void*, uint64_t, uint64_t);
template int wg_make_map<64>(CUtensorMap*, void*, uint64_t, uint64_t);

static inline long long round_up_ll(long long x, long long a) { return (x + a - 1) / a * a; }


// tables: offAm[M], offBn[N], offAk[K], offBk[K] (built by the caller, see kernels.cu)
int launch_k1_crt(tncb_ctx* ctx, const PairPlan& P, const double2* A, const double2* B, double2* C,
                  const long long* offAm, const long long* offBn, const long long* offAk, const long long* offBk) {
  int nmod, bits_a, bits_b;
  const int want = ctx->crt_tol > 0.0 ? crt_bits_for_tolerance(P.K, ctx->crt_tol) : ctx->crt_bits;
  crt_choose(P.K, want, ctx->crt_nmod_force, &nmod, &bits_a, &bits_b);
  CrtTables T;
  crt_make_tables(nmod, bits_a, bits_b, T);
  cudaStream_t st = ctx->stream;
  const long long Kp = round_up_ll(P.K, CRT_BKB);
  const int num_kb = (int)(Kp / CRT_BKB);
  const int ctas_max = std::max(1, ctx->sm_count);
  // three real products per complex product (Karatsuba; sums of residues are exact mod m_i) instead of four: 25 % fewer int8
  // operations for one more operand plane per side and one more residue plane.  An item then carries half the MMA work per
  // accumulator, so short K (where the epilogue paces the item) keeps the four-product form.  Measured on an H100
  // (profiles/h100_engine_sweep.jsonl, 4096 x 4096 x K): three products win by 18 % at K = 2048 and by ~2 % (noise) at K = 1024.
  const bool kara = ctx->crt_products == 3 || (ctx->crt_products == 0 && Kp >= ctx->crt_kara_min_k);
  const int TM = kara ? 2 * CRT_BT : CRT_BT;        // At rows per tile
  const int NPB = kara ? 3 : 2, NPR = kara ? 3 : 2;  // Bt operand planes, residue planes per modulus
  // K chunks: int32-safe length, and more chunks when there are too few tiles to fill the machine (split-K:
  // the reconstruction adds the chunk residues)
  const long long tiles_total = round_up_ll(P.N, CRT_BT) / CRT_BT * (round_up_ll(P.M, TM) / TM);
  int nkc = (int)((Kp + CRT_KCHUNK_MAX - 1) / CRT_KCHUNK_MAX);
  {
    const long long items = tiles_total * nmod * (kara ? 3 : 1);
    const long long want = ctas_max;
    if (items * nkc < want) nkc = (int)std::min<long long>((want + items - 1) / items, std::max(1, num_kb / 8));
    nkc = std::max(1, std::min(nkc, 32));      // exactness of the reconstruction: sum of <= 32 chunk residues
  }
  int kb_per_chunk = (num_kb + nkc - 1) / nkc;
  nkc = (num_kb + kb_per_chunk - 1) / kb_per_chunk;
  if ((long long)kb_per_chunk * CRT_BKB > CRT_KCHUNK_MAX) return fail(TNCB_ERR_UNSUPPORTED, "K too long for the int8 engine");

  // ---- panels: bound the workspace (planes + residues) ----
  const size_t budget = ctx->crt_ws_bytes;
  long long pn = round_up_ll(P.N, CRT_BT), pm = round_up_ll(P.M, TM);   // panel extents (padded)
  auto ws_bytes = [&](long long n_, long long m_) {
    return (size_t)nmod * (size_t)Kp * (size_t)(NPB * n_ + 3 * m_) + (size_t)nmod * nkc * NPR * (size_t)n_ * (size_t)m_;
  };
  while (ws_bytes(pn, pm) > budget && (pm > TM || pn > CRT_BT)) {
    if (pm >= pn && pm > TM) pm = round_up_ll(pm / 2, TM);
    else if (pn > CRT_BT) pn = round_up_ll(pn / 2, CRT_BT);
    else pm = round_up_ll(pm / 2, TM);
  }
  const size_t bytesB = (size_t)nmod * NPB * pn * Kp, bytesA = (size_t)nmod * 3 * pm * Kp;
  const size_t bytesR = (size_t)nmod * nkc * NPR * pn * pm;
  const size_t bytesE = (size_t)(pn + pm) * sizeof(unsigned long long);
  void *pb = nullptr, *pa = nullptr, *pr = nullptr, *pe = nullptr;
  int rc;
  if ((rc = ctx->arena.alloc(bytesB, &pb))) return rc;
  if ((rc = ctx->arena.alloc(bytesA, &pa))) { ctx->arena.free(pb, bytesB); return rc; }
  if ((rc = ctx->arena.alloc(bytesR, &pr))) { ctx->arena.free(pb, bytesB); ctx->arena.free(pa, bytesA); return rc; }
  if ((rc = ctx->arena.alloc(bytesE, &pe))) { ctx->arena.free(pb, bytesB); ctx->arena.free(pa, bytesA); ctx->arena.free(pr, bytesR); return rc; }
  auto cleanup = [&]() { ctx->arena.free(pb, bytesB); ctx->arena.free(pa, bytesA); ctx->arena.free(pr, bytesR); ctx->arena.free(pe, bytesE); };
  unsigned long long* max_n = (unsigned long long*)pe;
  unsigned long long* max_m = max_n + pn;

  static bool attr_done_dev[64] = {false};          // cudaFuncSetAttribute is per device
  bool& attr_done = attr_done_dev[ctx->device & 63];
  const int smem_gemm4 = CrtRing<false>::SMEM, smem_gemm3 = CrtRing<true>::SMEM;
  const int smem_res = RES_ROWS * RES_RS * (int)sizeof(double2);
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(crt_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_gemm4);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(crt_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_gemm3);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(crt_residue_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_res);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(crt_residue_kernel<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_res);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(crt_residue_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_res);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(crt_residue_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_res);
    if (e != cudaSuccess) { cleanup(); return fail(TNCB_ERR_CUDA, cudaGetErrorString(e)); }
    attr_done = true;
  }
  // lanes of a warp: 2^lk along k, the rest along rows -- as many k lanes as the operand's fastest K leg is long when k is
  // the fastest index (stride 1), otherwise as many row lanes as the fastest free leg is long
  auto lane_split = [](const LegList& kl, bool k_is_b, const LegList& fl) {
    auto p2 = [](long long d) { int b = 0; while ((2LL << b) <= d && b < 5) b++; return b; };
    const long long ks = kl.n ? (k_is_b ? kl.sb[kl.n - 1] : kl.sa[kl.n - 1]) : (1LL << 62);
    const long long fs = fl.n ? fl.sa[fl.n - 1] : (1LL << 62);
    if (ks <= fs) return kl.n ? p2(kl.dim[kl.n - 1]) : 0;          // k fastest: as many k lanes as that leg is long
    return 0;   // rows fastest: all lanes along rows (the K list's last group need not be this operand's fastest K leg,
                // so lanes along k could land on far-apart addresses)
  };
  const int lk_b = lane_split(P.k, true, P.n), lk_a = lane_split(P.k, false, P.m);
  ctx->last_int8_ops = 0.0; ctx->last_nmod = nmod; ctx->last_products = kara ? 3 : 4;
  bool timed = false;

  for (long long n0 = 0; n0 < P.N; n0 += pn) {
    const long long nrows = std::min(pn, P.N - n0);
    const long long Np = round_up_ll(nrows, CRT_BT);
    // ---- Bt panel: exponents + residues (padding rows / K tail must be zero residues) ----
    if (Np != nrows) cudaMemsetAsync(pb, 0, (size_t)nmod * NPB * Np * Kp, st);
    cudaMemsetAsync(max_n, 0, (size_t)nrows * sizeof(unsigned long long), st);
    {
      dim3 g((unsigned)((nrows + RES_ROWS - 1) / RES_ROWS), (unsigned)(Kp / RES_K));
      crt_rowmax_kernel<<<g, 256, 0, st>>>(B, offBn + n0, offBk, nrows, P.K, lk_b, max_n);
      if (kara) crt_residue_kernel<2, true><<<g, 256, smem_res, st>>>(B, offBn + n0, offBk, nrows, P.K, Np, Kp, max_n, bits_b, lk_b, T, (int8_t*)pb);
      else crt_residue_kernel<2, false><<<g, 256, smem_res, st>>>(B, offBn + n0, offBk, nrows, P.K, Np, Kp, max_n, bits_b, lk_b, T, (int8_t*)pb);
    }
    ctx->launches += 2;
    CUtensorMap mapB;
    if ((rc = kara ? wg_make_map<CrtRing<true>::BK>(&mapB, pb, (uint64_t)nmod * NPB * Np, (uint64_t)Kp)
                   : wg_make_map<CrtRing<false>::BK>(&mapB, pb, (uint64_t)nmod * NPB * Np, (uint64_t)Kp))) { cleanup(); return rc; }
    for (long long m0 = 0; m0 < P.M; m0 += pm) {
      const long long mcols = std::min(pm, P.M - m0);
      const long long Mp = round_up_ll(mcols, TM);
      if (Mp != mcols) cudaMemsetAsync(pa, 0, (size_t)nmod * 3 * Mp * Kp, st);
      cudaMemsetAsync(max_m, 0, (size_t)mcols * sizeof(unsigned long long), st);
      {
        dim3 g((unsigned)((mcols + RES_ROWS - 1) / RES_ROWS), (unsigned)(Kp / RES_K));
        crt_rowmax_kernel<<<g, 256, 0, st>>>(A, offAm + m0, offAk, mcols, P.K, lk_a, max_m);
        if (kara) crt_residue_kernel<3, true><<<g, 256, smem_res, st>>>(A, offAm + m0, offAk, mcols, P.K, Mp, Kp, max_m, bits_a, lk_a, T, (int8_t*)pa);
        else crt_residue_kernel<3, false><<<g, 256, smem_res, st>>>(A, offAm + m0, offAk, mcols, P.K, Mp, Kp, max_m, bits_a, lk_a, T, (int8_t*)pa);
      }
      ctx->launches += 2;
      CUtensorMap mapA;
      if ((rc = kara ? wg_make_map<CrtRing<true>::BK>(&mapA, pa, (uint64_t)nmod * 3 * Mp, (uint64_t)Kp)
                     : wg_make_map<CrtRing<false>::BK>(&mapA, pa, (uint64_t)nmod * 3 * Mp, (uint64_t)Kp))) { cleanup(); return rc; }
      CrtGemmArgs g;
      g.R = (int8_t*)pr; g.Np = (int)Np; g.Mp = (int)Mp;
      g.tiles_n = (int)(Np / CRT_BT); g.tiles_m = (int)(Mp / TM); g.tile_m = TM;
      g.nmod = nmod; g.nkc = nkc; g.kb_per_chunk = kb_per_chunk; g.num_kb = num_kb;
      const long long items = (long long)g.tiles_n * g.tiles_m * nmod * nkc * (kara ? 3 : 1);
      if (items > 0x7fffffffLL) { cleanup(); return fail(TNCB_ERR_UNSUPPORTED, "too many work items"); }
      g.total_items = (int)items;
      // raster band (n-tiles): the Bt tiles of a whole band stay in L2 while the At tiles stream past them, so a band over
      // all n-tiles reads every At tile from HBM once per (modulus, product) instead of once per band.  The band takes at
      // most half of the L2, so that the streamed At tiles do not evict it.
      const long long bt_tile_bytes = (long long)CRT_BT * Kp * (kara ? 1 : 2);   // three products: plane `prod`; four: Br, Bi
      g.group = (int)std::max<long long>(1, std::min<long long>(g.tiles_n, ctx->l2_bytes / 2 / bt_tile_bytes));
      for (int i = 0; i < CRT_MAX_MOD; i++) { g.negmod[i] = -T.mod[i]; g.magic[i] = T.magic[i]; }
      const unsigned grid = (unsigned)std::min<long long>(ctas_max, items);
      const double ops = 2.0 * (kara ? 3.0 : 4.0) * (double)nmod * (double)Np * (double)Mp * (double)Kp;
      const bool time_this = ctx->time_gemm == 2 || (ctx->time_gemm == 1 && !timed);
      if (time_this) gemm_timer_begin(ctx);
      if (kara) crt_gemm_kernel<true><<<grid, WG_THREADS, smem_gemm3, st>>>(mapB, mapA, g);
      else crt_gemm_kernel<false><<<grid, WG_THREADS, smem_gemm4, st>>>(mapB, mapA, g);
      cudaError_t e = cudaGetLastError();
      if (time_this) { gemm_timer_end(ctx, ops); timed = true; }
      if (e != cudaSuccess) { cleanup(); return fail(TNCB_ERR_CUDA, std::string("crt_gemm_kernel launch: ") + cudaGetErrorString(e)); }
      ctx->last_int8_ops += ops;
      CrtReconArgs r;
      r.R = (const int8_t*)pr; r.C = C + n0 * P.M + m0; r.max_n = max_n; r.max_m = max_m;
      r.rows = nrows; r.cols = mcols; r.ldc = P.M; r.Np = Np; r.Mp = Mp; r.nkc = nkc;
      const long long threads = nrows * (Mp / 4);
      const unsigned rg = (unsigned)((threads + 255) / 256);
      if (kara) {
        if (nkc == 1) crt_reconstruct_kernel<true, true><<<rg, 256, 0, st>>>(r, T);
        else crt_reconstruct_kernel<false, true><<<rg, 256, 0, st>>>(r, T);
      } else {
        if (nkc == 1) crt_reconstruct_kernel<true, false><<<rg, 256, 0, st>>>(r, T);
        else crt_reconstruct_kernel<false, false><<<rg, 256, 0, st>>>(r, T);
      }
      ctx->launches += 2;
    }
  }
  ctx->engine_count[4]++;
  cudaError_t e = cudaGetLastError();
  cleanup();   // stream-ordered reuse: later allocations are only touched by later kernels
  if (e != cudaSuccess) return fail(TNCB_ERR_CUDA, std::string("K1' (CRT) launch: ") + cudaGetErrorString(e));
  return TNCB_OK;
}

} // namespace tncb
