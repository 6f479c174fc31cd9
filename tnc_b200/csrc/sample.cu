// Sampling bitstrings from a circuit's output distribution (tncb_plan_sample, tncb_plan_sample_slices): the kernels of one
// pass around the batched contraction of the candidates' networks.  The algorithm and the random stream are described in
// tncb.h and DESIGN §5.  Nothing here uses atomics, so a pass's output repeats bit for bit.
#include "internal.h"
#include "philox.h"

namespace tncb {

constexpr int kCandThreads = 128;
constexpr int kSelectThreads = 256;
constexpr int kCompactThreads = 512;
constexpr int kAccThreads = 256;

// |z|^2 and the prefix sums with explicit roundings: no contraction into FMAs, so that every sum of the selection is
// formed the same way in each loop that forms it (and as numpy forms it)
__device__ __forceinline__ double norm2(double2 z) { return __dadd_rn(__dmul_rn(z.x, z.x), __dmul_rn(z.y, z.y)); }

// ------------------------------------------------------------------------------------------
// Candidates: slot i takes Philox block first + i.  Closed bra j of slot i is the one-hot row vector of bit j of w0, the
// payload the leaf staging kernel copies into slot i's leaf block (consecutive slots write consecutive 32-byte bras).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCandThreads)
sample_candidates_kernel(unsigned long long seed, unsigned long long first, unsigned long long n, unsigned long long c,
                         const __grid_constant__ SampleMap map, double2* __restrict__ bras, double2* __restrict__ uv,
                         unsigned long long* __restrict__ closed_bits) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kCandThreads + threadIdx.x;
  if (i >= n) return;
  const philox::Block b = philox::candidate(seed, first + i);
  unsigned long long bits = 0;
  for (int j = 0; j < map.n_closed; j++) {
    const unsigned long long bit = (b.w[0] >> j) & 1ull;
    bits |= bit << map.closed_qubit[j];
    double2* bra = bras + (j * c + i) * 2;
    bra[0] = make_double2(bit ? 0.0 : 1.0, 0.0);
    bra[1] = make_double2(bit ? 1.0 : 0.0, 0.0);
  }
  closed_bits[i] = bits;
  uv[i] = make_double2(philox::unit53(b.w[1]), philox::unit53(b.w[2]));
}

int launch_sample_candidates(tncb_ctx* ctx, unsigned long long seed, unsigned long long first, size_t n, size_t c,
                             const SampleMap& map, double2* bras, double2* uv, unsigned long long* closed_bits) {
  if (n == 0) return TNCB_OK;
  const unsigned blocks = (unsigned)((n + kCandThreads - 1) / kCandThreads);
  sample_candidates_kernel<<<blocks, kCandThreads, 0, ctx->stream>>>(seed, first, n, c, map, bras, uv, closed_bits);
  ctx->launches++;
  TNCB_CUDA(cudaGetLastError());
  return TNCB_OK;
}

// ------------------------------------------------------------------------------------------
// Selection: block i reads slot i's 2^k amplitudes in place, in its workspace copy's result slot.  The fixed-order prefix
// sum of p = |a|^2: T = min(blockDim, 2^k) chunks of 2^k / T consecutive outcomes; thread t sums its chunk left to right,
// thread 0 scans the chunk sums left to right (excl[t]), and prefix(y) = excl[t] + (the chunk's running sum up to y).
// The last prefix of chunk t is excl[t + 1] exactly, so the prefix never decreases, q = excl[T] is its last value, and
// the first y with prefix(y) > v q lies in the one chunk with excl[t] <= v q < excl[t + 1] and has p(y) > 0.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSelectThreads)
sample_select_kernel(const char* __restrict__ ws, long long stride, long long res_off, double scale, double m,
                     const __grid_constant__ SampleMap map, const double2* __restrict__ uv,
                     const unsigned long long* __restrict__ closed_bits, SampleCand* __restrict__ cand) {
  __shared__ double excl[kSelectThreads + 1];
  const unsigned long long i = blockIdx.x;
  const double2* a = reinterpret_cast<const double2*>(ws + (long long)i * stride + res_off);
  const unsigned long long outcomes = 1ull << map.k;
  const unsigned t = threadIdx.x;
  const unsigned T = (unsigned)(outcomes < blockDim.x ? outcomes : blockDim.x);
  const unsigned long long len = outcomes / T;
  if (t < T) {
    double s = 0.0;
    for (unsigned long long y = t * len; y < (t + 1) * len; y++) s = __dadd_rn(s, norm2(a[y]));
    excl[t + 1] = s;
  }
  __syncthreads();
  if (t == 0) {
    double run = 0.0;
    for (unsigned x = 1; x <= T; x++) { run = __dadd_rn(run, excl[x]); excl[x] = run; }
    excl[0] = 0.0;
  }
  __syncthreads();
  const double q = excl[T];
  const double2 w = uv[i];
  const double target = __dmul_rn(w.y, q);
  const double ratio = __ddiv_rn(__dmul_rn(q, scale), m);
  if (t < T && excl[t] <= target && target < excl[t + 1]) {
    double s = 0.0;
    unsigned long long y = t * len;
    for (; y < (t + 1) * len - 1; y++) {
      s = __dadd_rn(s, norm2(a[y]));
      if (__dadd_rn(excl[t], s) > target) break;
    }
    unsigned long long bits = closed_bits[i];
    for (int r = 0; r < map.k; r++) bits |= ((y >> (map.k - 1 - r)) & 1ull) << map.result_qubit[r];
    SampleCand out;
    out.bits = bits;
    out.p = norm2(a[y]);
    out.ratio = ratio;
    out.accept = w.x < ratio;
    out.clipped = ratio > 1.0;
    cand[i] = out;
  } else if (t == 0 && !(target < q)) {   // q == 0 (or not a number): no outcome carries weight, nothing to pick
    cand[i] = SampleCand{closed_bits[i], 0.0, ratio, 0, ratio > 1.0};
  }
}

int launch_sample_select(tncb_ctx* ctx, const char* ws, long long stride, long long res_off, size_t n, double m,
                         const SampleMap& map, const double2* uv, const unsigned long long* closed_bits, SampleCand* cand) {
  if (n == 0) return TNCB_OK;
  if (n > 0x7fffffffull) return fail(TNCB_ERR_UNSUPPORTED, "too many candidates in one selection launch");
  const double scale = ldexp(1.0, map.n_qubits - map.k);    // 2^(n - k), exact
  sample_select_kernel<<<(unsigned)n, kSelectThreads, 0, ctx->stream>>>(ws, stride, res_off, scale, m, map, uv, closed_bits, cand);
  ctx->launches++;
  TNCB_CUDA(cudaGetLastError());
  return TNCB_OK;
}

// ------------------------------------------------------------------------------------------
// Slice sum (tncb_plan_sample_slices): row i of acc gets slot i's result, the instance blockIdx.y.  The first slice is
// copied, every later one added with add_kernel's arithmetic, so that a row is the left fold tncb_plan_run_slices forms.
// One 16-byte load (and store) per element and operand.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kAccThreads)
sample_accumulate_kernel(const char* __restrict__ ws, long long stride, long long res_off, long long elems, int first,
                         double2* __restrict__ acc) {
  const unsigned long long i = blockIdx.y;
  const double2* r = reinterpret_cast<const double2*>(ws + (long long)i * stride + res_off);
  double2* a = acc + (long long)i * elems;
  for (long long o = (long long)blockIdx.x * kAccThreads + threadIdx.x; o < elems; o += (long long)gridDim.x * kAccThreads) {
    const double2 v = r[o];
    if (first) { a[o] = v; continue; }
    double2 d = a[o];
    d.x += v.x; d.y += v.y; a[o] = d;
  }
}

int launch_sample_accumulate(tncb_ctx* ctx, const char* ws, long long stride, long long res_off, size_t n, size_t elems,
                             bool first, double2* acc) {
  if (n == 0 || elems == 0) return TNCB_OK;
  if (n > 65535) return fail(TNCB_ERR_UNSUPPORTED, "too many candidates in one accumulate launch");
  const unsigned blocks = (unsigned)std::min<long long>(((long long)elems + kAccThreads - 1) / kAccThreads, (long long)ctx->sm_count * 16);
  sample_accumulate_kernel<<<dim3(blocks, (unsigned)n), kAccThreads, 0, ctx->stream>>>(ws, stride, res_off, (long long)elems,
                                                                                      first ? 1 : 0, acc);
  ctx->launches++;
  TNCB_CUDA(cudaGetLastError());
  return TNCB_OK;
}

// ------------------------------------------------------------------------------------------
// Compaction, one block: thread t owns slots [t E, (t + 1) E).  A scan of the per-thread accept counts places every
// accepted candidate at its rank in slot order; the candidate of rank remaining - 1 (if any) is the last one the pass
// consumes, and the counts cover the consumed slots only.  Integer scans and a max: the same bits on every run.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCompactThreads)
sample_compact_kernel(const SampleCand* __restrict__ cand, unsigned long long n, unsigned long long remaining,
                      unsigned long long* __restrict__ bits, double* __restrict__ probs, SampleCounts* __restrict__ counts) {
  __shared__ unsigned long long off[kCompactThreads + 1];
  __shared__ unsigned long long consumed;
  __shared__ unsigned long long clip_part[kCompactThreads / 32];
  __shared__ double max_part[kCompactThreads / 32];
  const unsigned t = threadIdx.x;
  const unsigned long long per = (n + kCompactThreads - 1) / kCompactThreads;
  const unsigned long long lo = min(n, t * per), hi = min(n, lo + per);
  unsigned long long mine = 0;
  for (unsigned long long j = lo; j < hi; j++) mine += cand[j].accept != 0;
  off[t + 1] = mine;
  if (t == 0) { consumed = n; off[0] = 0; }
  __syncthreads();
  for (unsigned d = 1; d < kCompactThreads; d <<= 1) {      // inclusive scan of off[1..T] (Hillis-Steele, integers)
    const unsigned long long add = t + 1 > d ? off[t + 1 - d] : 0;
    __syncthreads();
    off[t + 1] += add;
    __syncthreads();
  }
  const unsigned long long total = off[kCompactThreads];
  const unsigned long long base = off[t];
  if (total >= remaining && base < remaining && remaining <= base + mine) {   // this thread holds the last sample
    unsigned long long r = base;
    for (unsigned long long j = lo; j < hi; j++)
      if (cand[j].accept && ++r == remaining) { consumed = j + 1; break; }
  }
  __syncthreads();
  const unsigned long long end = min(hi, consumed);
  unsigned long long r = base, clipped = 0;
  double mx = 0.0;
  for (unsigned long long j = lo; j < end; j++) {
    const SampleCand& c = cand[j];
    clipped += c.clipped != 0;
    mx = fmax(mx, c.ratio);
    if (c.accept) {
      bits[r] = c.bits;
      if (probs) probs[r] = c.p;
      r++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    clipped += __shfl_down_sync(0xffffffffu, clipped, o);
    mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
  }
  if ((t & 31) == 0) { clip_part[t >> 5] = clipped; max_part[t >> 5] = mx; }
  __syncthreads();
  if (t == 0) {
    unsigned long long cl = 0;
    double m2 = 0.0;
    for (int w = 0; w < kCompactThreads / 32; w++) { cl += clip_part[w]; m2 = fmax(m2, max_part[w]); }
    counts->consumed = consumed;
    counts->accepted = total < remaining ? total : remaining;
    counts->clipped = cl;
    counts->max_ratio = m2;
  }
}

int launch_sample_compact(tncb_ctx* ctx, const SampleCand* cand, size_t n, unsigned long long remaining,
                          unsigned long long* bits, double* probs, SampleCounts* counts) {
  sample_compact_kernel<<<1, kCompactThreads, 0, ctx->stream>>>(cand, n, remaining, bits, probs, counts);
  ctx->launches++;
  TNCB_CUDA(cudaGetLastError());
  return TNCB_OK;
}

}  // namespace tncb
