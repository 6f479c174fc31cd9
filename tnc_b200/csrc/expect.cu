// Expectation values of Pauli sums (tncb_plan_expect): the kernels around the batched contraction of the terms'
// networks.  The contract is described in tncb.h and DESIGN §5.  Nothing here uses atomics, so a call repeats bit for bit.
#include "internal.h"

namespace tncb {

constexpr int kLayerThreads = 128;

// ------------------------------------------------------------------------------------------
// Layer payloads: thread (i, j) writes layer leaf j of slot i, term first + i's Pauli on qubit layer.qubit[j], as the
// 2x2 matrix M with legs [ket, bra].  The network contracts to sum_ab psi_a M[a, b] conj(psi_b), so <psi|P|psi> needs
// M = P^T: Y's payload is [[0, i], [-i, 0]].  pauli_layer_matrix (observables.py) writes the same bits on the host.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLayerThreads)
expect_layer_kernel(const unsigned long long* __restrict__ x_mask, const unsigned long long* __restrict__ z_mask,
                    unsigned long long first, unsigned long long n, unsigned long long c,
                    const __grid_constant__ ExpectLayer layer, double2* __restrict__ out) {
  const unsigned long long i = (unsigned long long)blockIdx.x * kLayerThreads + threadIdx.x;
  if (i >= n) return;
  const unsigned j = blockIdx.y;
  const int q = layer.qubit[j];
  const unsigned x = (unsigned)(x_mask[first + i] >> q) & 1u, z = (unsigned)(z_mask[first + i] >> q) & 1u;
  double2* m = out + (j * c + i) * 4;
  const double2 zero = make_double2(0.0, 0.0), one = make_double2(1.0, 0.0);
  if (!x) {                                                         // I, Z
    m[0] = one; m[1] = zero; m[2] = zero; m[3] = make_double2(z ? -1.0 : 1.0, 0.0);
  } else if (!z) {                                                  // X
    m[0] = zero; m[1] = one; m[2] = one; m[3] = zero;
  } else {                                                          // Y^T
    m[0] = zero; m[1] = make_double2(0.0, 1.0); m[2] = make_double2(0.0, -1.0); m[3] = zero;
  }
}

int launch_expect_layer(tncb_ctx* ctx, const unsigned long long* x_mask, const unsigned long long* z_mask,
                        unsigned long long first, size_t n, size_t c, const ExpectLayer& layer, double2* out) {
  if (n == 0 || layer.n_layer == 0) return TNCB_OK;
  const unsigned blocks = (unsigned)((n + kLayerThreads - 1) / kLayerThreads);
  expect_layer_kernel<<<dim3(blocks, (unsigned)layer.n_layer), kLayerThreads, 0, ctx->stream>>>(x_mask, z_mask, first, n, c,
                                                                                               layer, out);
  ctx->launches++;
  TNCB_CUDA(cudaGetLastError());
  return TNCB_OK;
}

// ------------------------------------------------------------------------------------------
// Energy: thread 0 folds the real parts, thread 1 the imaginary parts, each left to right in term order with explicit
// roundings (no FMA), so that numpy's ((0 + c_0 Re R_0) + c_1 Re R_1) + ... gives the same bits.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
expect_fold_kernel(const double2* __restrict__ values, const double2* __restrict__ seeds, unsigned long long n,
                   double2* __restrict__ energy) {
  const unsigned t = threadIdx.x;
  if (t > 1) return;
  double e = 0.0;
  for (unsigned long long k = 0; k < n; k++) {
    const double2 r = values[k];
    e = __dadd_rn(e, __dmul_rn(seeds[k].x, t ? r.y : r.x));
  }
  if (t) energy->y = e; else energy->x = e;
}

int launch_expect_fold(tncb_ctx* ctx, const double2* values, const double2* seeds, size_t n, double2* energy) {
  expect_fold_kernel<<<1, 32, 0, ctx->stream>>>(values, seeds, n, energy);
  ctx->launches++;
  TNCB_CUDA(cudaGetLastError());
  return TNCB_OK;
}

}  // namespace tncb
