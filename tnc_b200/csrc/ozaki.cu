// K1' (LEGACY engine, round 1; selectable with tncb_ctx_set_tcgen05_engine(ctx, 1) for A/B measurements -- the default
// engine is the modular / CRT emulation in crt.cu, which needs 16 int8 GEMM sweeps where this one needs 36).
//
// The dense contraction on the int8 tensor cores (Hopper wgmma) by 7-bit digit slicing (Ozaki scheme I): every real operand
// row is scaled by a power of two and cut into S signed 7-bit digit planes,
//     x * 2^-e = sum_{p<S} d_p * 128^-(p+1) + r,   |d_p| <= 127,  |r| < 128^-S,
// and  C ~= sum_{t<S} 128^-(t+2) * sum_{p+q=t} (D^B_p . D^A_q)  with every D.D an exact int8 GEMM (int32 accumulation,
// K chunked so it cannot overflow) and the recombination in FP64.  NOT exact: the digit products with p + q >= S are
// dropped, so |C - C_exact|[n,m] <= (S+1) K 2^(-7S) * 4 max|b[n,:]| max|a[m,:]| (S = 8: measured 1e-15..7e-15 of max|C|),
// with max|.| = max(|re|, |im|) over the row.  The bound holds over the whole double range: a row's scale exponent
// e = ilogb(max) + 1 is clamped below at kOzExpMin = -1000 (rows under 2^-1001, denormal ones included, keep ABSOLUTE
// accuracy: read max|.| as max(max|.|, 2^-1001) in the bound), and e <= 1024 for any finite row, so 2^-e is finite and
// non-zero; the output scale 2^(e_n + e_m - 7(t+2)) is applied as one scalbn, so no partial scale overflows or underflows.
// Rows containing NaN / Inf give unspecified finite values (the CRT engine poisons them with NaN), and there is no
// tolerance control beyond the digit count.  The leg permutation of the reference's TTGT is fused into the slicing pass (gather
// through the plan's offset tables), which writes K-major int8 planes that TMA can stream.
//
// Complex arithmetic without int negation in the MMA: planes Br, Bi for Bt and nAi(=-Ai), Ar, Ai
// for At; in shared memory the At planes sit as [nAi | Ar | Ai] so that
//     Br x [Ar ; Ai]^T  -> (real | imag) columns,    Bi x [nAi ; Ar]^T -> (real | imag) columns
// are two N=256 wgmmas into one 256-column accumulator (cols 0..127 real, 128..255 imag): the four-product stage of sm90.h.
//
// Kernel structure (one CTA per 128x128 complex output tile, three warpgroups, main loop in sm90.h):
//   warpgroup 0    TMA producer
//   warpgroups 1-2 wgmma on 64 Bt rows each, then the epilogue of digit level t and K chunk kc:
//                  scalbn(int32 -> FP64, e_n + e_m - 7(t+2)) -> C (+=)
#include "internal.h"
#include "sm90.h"
#include <cuda.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace tncb {

constexpr int OZ_BT = 128;      // tile rows (n) = tile cols (m)
constexpr int OZ_BKB = 128;     // K bytes per stage row (one 128-byte swizzle row)
constexpr int OZ_STAGES = 2;    // 2 x 80 KB (128-byte stages, sm90.h)
constexpr int OZ_KCHUNK = 8192;                   // int32-safe: 2*(t+1)*K*127^2 < 2^31 for t <= 7
constexpr int OZ_MAX_S = 8;
constexpr int kOzExpMin = -1000;                  // as crt.cu's kExpMin: 2^-e stays finite for every row

// ---- operand preparation --------------------------------------------------------------------
// exponent e (per row of the K-major operand) with max(|re|,|im|) * 2^-e in [0.5, 1), clamped at kOzExpMin (then the
// scaled row is below 0.5); e <= 1024 for a finite maximum
__global__ void oz_rowexp_kernel(const double2* __restrict__ src, const long long* __restrict__ off_row,
                                 const long long* __restrict__ off_k, long long rows, long long K, int* __restrict__ exps) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long long base = off_row[row];
  double m = 0.0;
  for (long long k = lane; k < K; k += 32) {
    const double2 v = __ldg(src + base + __ldg(off_k + k));
    m = fmax(m, fmax(fabs(v.x), fabs(v.y)));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, d));
  if (lane == 0) exps[row] = (m > 0.0 && isfinite(m)) ? max(ilogb(m) + 1, kOzExpMin) : 0;
}

// One thread: 16 consecutive k of one row -> 16 bytes of every digit plane.
// planes layout: [(comp * S + p) * rowsP + row] * Kp + k,  comp order given by COMPS:
//   COMPS == 2: (re, im)          -- Bt side
//   COMPS == 3: (-im, re, im)     -- At side
template <int COMPS>
__global__ void oz_slice_kernel(const double2* __restrict__ src, const long long* __restrict__ off_row,
                                const long long* __restrict__ off_k, long long rows, long long K, long long rowsP,
                                long long Kp, const int* __restrict__ exps, int S, int8_t* __restrict__ planes) {
  const long long kg = (long long)blockIdx.y * blockDim.x + threadIdx.x;   // group of 16 k
  const long long row = blockIdx.x;
  if (kg * 16 >= Kp) return;
  const long long base = off_row[row];
  const double sc = scalbn(1.0, -exps[row]);
  uint32_t re_w[OZ_MAX_S][4], im_w[OZ_MAX_S][4];
#pragma unroll
  for (int p = 0; p < OZ_MAX_S; p++)
#pragma unroll
    for (int w = 0; w < 4; w++) { re_w[p][w] = 0; im_w[p][w] = 0; }
#pragma unroll
  for (int j = 0; j < 16; j++) {
    const long long k = kg * 16 + j;
    double re = 0.0, im = 0.0;
    if (k < K) { const double2 v = __ldg(src + base + __ldg(off_k + k)); re = v.x * sc; im = v.y * sc; }
#pragma unroll
    for (int p = 0; p < OZ_MAX_S; p++) {
      if (p < S) {
        re *= 128.0; im *= 128.0;
        const int dr = (int)re, di = (int)im;     // truncation toward zero, |d| <= 127
        re -= (double)dr; im -= (double)di;        // exact
        re_w[p][j >> 2] |= (uint32_t)(dr & 0xff) << ((j & 3) * 8);
        im_w[p][j >> 2] |= (uint32_t)(di & 0xff) << ((j & 3) * 8);
      }
    }
  }
  const long long plane_stride = rowsP * Kp;
  int8_t* dst = planes + row * Kp + kg * 16;
  for (int p = 0; p < S; p++) {
    const uint4 r4 = make_uint4(re_w[p][0], re_w[p][1], re_w[p][2], re_w[p][3]);
    const uint4 i4 = make_uint4(im_w[p][0], im_w[p][1], im_w[p][2], im_w[p][3]);
    if (COMPS == 2) {
      *reinterpret_cast<uint4*>(dst + (long long)(0 * S + p) * plane_stride) = r4;
      *reinterpret_cast<uint4*>(dst + (long long)(1 * S + p) * plane_stride) = i4;
    } else {
      // byte-wise negation of the imaginary digits (|d| <= 127, so -d is representable)
      uint4 n4;
      uint32_t* nw = reinterpret_cast<uint32_t*>(&n4);
      const uint32_t* iw = reinterpret_cast<const uint32_t*>(&i4);
#pragma unroll
      for (int w = 0; w < 4; w++) nw[w] = __vneg4(iw[w]);
      *reinterpret_cast<uint4*>(dst + (long long)(0 * S + p) * plane_stride) = n4;
      *reinterpret_cast<uint4*>(dst + (long long)(1 * S + p) * plane_stride) = r4;
      *reinterpret_cast<uint4*>(dst + (long long)(2 * S + p) * plane_stride) = i4;
    }
  }
}

struct OzArgs {
  double2* C;
  const int* exp_n;   // per Bt row
  const int* exp_m;   // per At row (= C column)
  long long M, N;     // logical sizes of C [N][M]
  int Np, Mp;         // padded plane rows
  int num_kb;         // Kp / 128
  int S;
};

__global__ void __launch_bounds__(WG_THREADS, 1)
oz_gemm_kernel(const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapA,
               const __grid_constant__ OzArgs p) {
  extern __shared__ __align__(1024) uint8_t oz_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(oz_smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t full_bar[OZ_STAGES], empty_bar[OZ_STAGES];
  __shared__ int col_exp[OZ_BT];
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int n0 = blockIdx.y * OZ_BT, m0 = blockIdx.x * OZ_BT;
  const int S = p.S;
  const int kb_per_chunk = OZ_KCHUNK / OZ_BKB;
  const int nkc = (p.num_kb + kb_per_chunk - 1) / kb_per_chunk;

  if (threadIdx.x == 0) {
    for (int s = 0; s < OZ_STAGES; s++) { wg_mbar_init(&full_bar[s], 1); wg_mbar_init(&empty_bar[s], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < OZ_BT) {
    const long long gm = (long long)m0 + threadIdx.x;
    col_exp[threadIdx.x] = gm < p.M ? p.exp_m[gm] : 0;
  }
  __syncthreads();

  if (wg == 0) {
    // ================= TMA producer =================
    wg_setmaxnreg_producer();
    if (tid != 0) return;
    int it = 0;
    for (int t = 0; t < S; t++)
      for (int kc = 0; kc < nkc; kc++) {
        const int kb0 = kc * kb_per_chunk, kb1 = min(p.num_kb, kb0 + kb_per_chunk);
        for (int pp = 0; pp <= t; pp++) {
          const int qq = t - pp;
          for (int kb = kb0; kb < kb1; kb++, it++) {
            using Stage = WgStage<false, OZ_BKB>;
            uint8_t* st = wg_produce_begin<OZ_STAGES, false, OZ_BKB>(smem, full_bar, empty_bar, it);
            uint64_t* bar = &full_bar[it % OZ_STAGES];
            uint8_t* a = st + Stage::A;
            const int kx = kb * OZ_BKB;
            wg_tma_2d(&mapB, bar, st, kx, (0 * S + pp) * p.Np + n0);                      // Br_p
            wg_tma_2d(&mapB, bar, st + Stage::B1, kx, (1 * S + pp) * p.Np + n0);          // Bi_p
            wg_tma_2d(&mapA, bar, a, kx, (0 * S + qq) * p.Mp + m0);                       // nAi_q
            wg_tma_2d(&mapA, bar, a + Stage::TILE, kx, (1 * S + qq) * p.Mp + m0);         // Ar_q
            wg_tma_2d(&mapA, bar, a + 2 * Stage::TILE, kx, (2 * S + qq) * p.Mp + m0);     // Ai_q
          }
        }
      }
  } else {
    // ================= consumers: wgmma + epilogue (own 64 Bt rows) =================
    wg_setmaxnreg_consumer();
    const int c = wg - 1, wq = tid >> 5, lane = tid & 31;
    WgRing<OZ_STAGES, false, OZ_BKB> ring{smem, full_bar, empty_bar};
    long long gn[2];
    bool row_ok[2];
    int en[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      gn[h] = (long long)n0 + c * 64 + wq * 16 + (lane >> 2) + 8 * h;
      row_ok[h] = gn[h] < p.N;
      en[h] = row_ok[h] ? p.exp_n[gn[h]] : 0;
    }
    uint32_t acc[128];
#pragma unroll
    for (int i = 0; i < 128; i++) acc[i] = 0u;
    int f = 0;
    for (int t = 0; t < S; t++) {
      const int row_exp[2] = {en[0] - 7 * (t + 2), en[1] - 7 * (t + 2)};
      for (int kc = 0; kc < nkc; kc++, f++) {
        const int kb0 = kc * kb_per_chunk, kb1 = min(p.num_kb, kb0 + kb_per_chunk);
        bool first = true;
        for (int pp = 0; pp <= t; pp++)
          for (int kb = kb0; kb < kb1; kb++) ring.mma_stage(acc, c, first, tid == 0);
        ring.drain(tid == 0);
#pragma unroll
        for (int h = 0; h < 2; h++) {
          if (!row_ok[h]) continue;
          double2* crow = p.C + gn[h] * p.M + m0;
#pragma unroll
          for (int j = 0; j < 16; j++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
              const int col = 8 * j + 2 * (lane & 3) + e;
              if ((long long)m0 + col < p.M) {
                const int sc = row_exp[h] + col_exp[col];   // one scalbn: 2^(e_n + e_m - 7(t+2)) may lie outside the double range
                double2 v = make_double2(scalbn((double)(int)acc[4 * j + 2 * h + e], sc), scalbn((double)(int)acc[4 * (j + 16) + 2 * h + e], sc));
                if (f != 0) { const double2 old = crow[col]; v.x += old.x; v.y += old.y; }
                crow[col] = v;
              }
            }
          }
        }
      }
    }
  }
}

// ---- host side --------------------------------------------------------------------------------
// tables: offAm[M], offBn[N], offAk[K], offBk[K] (built by the caller, see kernels.cu)
int launch_k1_ozaki(tncb_ctx* ctx, const PairPlan& P, const double2* A, const double2* B, double2* C, int S,
                    const long long* offAm, const long long* offBn, const long long* offAk, const long long* offBk) {
  if (S < 2) S = 2;
  if (S > OZ_MAX_S) S = OZ_MAX_S;
  const long long Np = (P.N + OZ_BT - 1) / OZ_BT * OZ_BT, Mp = (P.M + OZ_BT - 1) / OZ_BT * OZ_BT;
  const long long Kp = (P.K + OZ_BKB - 1) / OZ_BKB * OZ_BKB;
  const size_t bytesB = (size_t)2 * S * Np * Kp, bytesA = (size_t)3 * S * Mp * Kp;
  const size_t bytesE = (size_t)(Np + Mp) * sizeof(int);
  void *pb = nullptr, *pa = nullptr, *pe = nullptr;
  int rc;
  if ((rc = ctx->arena.alloc(bytesB, &pb))) return rc;
  if ((rc = ctx->arena.alloc(bytesA, &pa))) { ctx->arena.free(pb, bytesB); return rc; }
  if ((rc = ctx->arena.alloc(bytesE, &pe))) { ctx->arena.free(pb, bytesB); ctx->arena.free(pa, bytesA); return rc; }
  auto cleanup = [&]() { ctx->arena.free(pb, bytesB); ctx->arena.free(pa, bytesA); ctx->arena.free(pe, bytesE); };
  int* exp_n = (int*)pe;
  int* exp_m = exp_n + Np;
  cudaStream_t st = ctx->stream;
  // padding rows / K tail must be zero digits
  if (Np != P.N) cudaMemsetAsync(pb, 0, bytesB, st);   // (the K tail is written as zeros by the slicer)
  if (Mp != P.M) cudaMemsetAsync(pa, 0, bytesA, st);
  oz_rowexp_kernel<<<(unsigned)((P.N + 7) / 8), 256, 0, st>>>(B, offBn, offBk, P.N, P.K, exp_n);
  oz_rowexp_kernel<<<(unsigned)((P.M + 7) / 8), 256, 0, st>>>(A, offAm, offAk, P.M, P.K, exp_m);
  {
    const unsigned gx = (unsigned)((Kp / 16 + 127) / 128);
    oz_slice_kernel<2><<<dim3((unsigned)P.N, gx), 128, 0, st>>>(B, offBn, offBk, P.N, P.K, Np, Kp, exp_n, S, (int8_t*)pb);
    oz_slice_kernel<3><<<dim3((unsigned)P.M, gx), 128, 0, st>>>(A, offAm, offAk, P.M, P.K, Mp, Kp, exp_m, S, (int8_t*)pa);
  }
  ctx->launches += 4;
  CUtensorMap mapB, mapA;
  if ((rc = wg_make_map<OZ_BKB>(&mapB, pb, (uint64_t)2 * S * Np, (uint64_t)Kp)) || (rc = wg_make_map<OZ_BKB>(&mapA, pa, (uint64_t)3 * S * Mp, (uint64_t)Kp))) { cleanup(); return rc; }
  OzArgs a;
  a.C = C; a.exp_n = exp_n; a.exp_m = exp_m; a.M = P.M; a.N = P.N; a.Np = (int)Np; a.Mp = (int)Mp;
  a.num_kb = (int)(Kp / OZ_BKB); a.S = S;
  const int smem_bytes = OZ_STAGES * WgStage<false, OZ_BKB>::BYTES + 1024;
  cudaError_t e = cudaFuncSetAttribute(oz_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  if (e != cudaSuccess) { cleanup(); return fail(TNCB_ERR_CUDA, cudaGetErrorString(e)); }
  const double ops = 2.0 * 4.0 * (S * (S + 1) / 2) * (double)Np * (double)Mp * (double)Kp;
  if (ctx->time_gemm) gemm_timer_begin(ctx);
  oz_gemm_kernel<<<dim3((unsigned)(Mp / OZ_BT), (unsigned)(Np / OZ_BT)), WG_THREADS, smem_bytes, st>>>(mapB, mapA, a);
  if (ctx->time_gemm) gemm_timer_end(ctx, ops);
  ctx->last_int8_ops = ops; ctx->last_nmod = 0;
  ctx->launches++;
  e = cudaGetLastError();
  cleanup();  // stream-ordered reuse: later allocations are only touched by later kernels
  if (e != cudaSuccess) return fail(TNCB_ERR_CUDA, std::string("oz_gemm_kernel: ") + cudaGetErrorString(e));
  return TNCB_OK;
}

} // namespace tncb
