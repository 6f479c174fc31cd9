// Internal definitions shared by the host runtime and the CUDA kernels of libtncb200.
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>
#include <map>
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/tncb.h"

namespace tncb {

constexpr int kMaxLegs = 64;   // max rank of a tensor accepted at the ABI
constexpr int kMaxGroups = 40; // max fused leg groups per list passed to a kernel

// A list of (fused) legs of one index class, outermost first, innermost last.
struct LegList {
  int n;
  int _pad;
  long long dim[kMaxGroups];
  long long sa[kMaxGroups]; // element stride in operand A (or in the only operand)
  long long sb[kMaxGroups]; // element stride in operand B (K-list only)
};

// The GEMM view of one pairwise contraction  C[N,M] = sum_K Bt[N,K] * At[K,M]
// (SURVEY 3.4): M = legs(a)\legs(b) in a's order, N = legs(b)\legs(a) in b's
// order, K = shared legs.  C is plain row-major [N][M], which *is* the
// reference's output layout (b\a)++(a\b) (tensor.rs:463-479).
struct PairPlan {
  std::vector<uint64_t> out_legs, out_dims;
  long long M = 1, N = 1, K = 1;
  LegList m{}, n{}, k{};  // m: strides in A; n: strides in B (stored in .sa); k: sa=A, sb=B
  int kernel_class = 0;   // 0 = K0, 1 = K1 (K1' above a size threshold), 2 = K2 streaming (big x tiny)
  bool k2_big_is_a = true; // K2: which operand is the big one
  // K1 loader modes: true = consecutive threads walk the K index, false = the free index
  bool a_kfast = false, b_kfast = true;
  double flops() const { return 8.0 * (double)M * (double)N * (double)K; }
  double bytes() const { return 16.0 * ((double)M * K + (double)K * N + (double)M * N); }
};

// Returns TNCB_OK or an error; fills plan. Pure host code (no CUDA calls).
int plan_pair(int n_a, const uint64_t* a_legs, const uint64_t* a_dims,
              int n_b, const uint64_t* b_legs, const uint64_t* b_dims, PairPlan& plan);

void set_error(const std::string& msg);
int fail(int status, const std::string& msg);

// ---- device arena -------------------------------------------------------------------
struct Slab { char* base; size_t size; std::map<size_t, size_t> free_by_off; };

struct Arena {
  std::vector<Slab> slabs;
  size_t capacity_limit = 0; // 0 = device free memory
  size_t reserved = 0, live = 0, peak = 0;
  size_t next_slab = (size_t)256 << 20;
  int alloc(size_t bytes, void** out);
  void free(void* p, size_t bytes);
  void release_all();
  size_t trim();             // cudaFree every slab that holds no live block; returns the bytes given back
};

} // namespace tncb

struct tncb_tensor {
  double2* ptr = nullptr;
  int rank = 0;
  uint64_t dims[tncb::kMaxLegs];
  uint64_t elems = 1;
  size_t bytes = 0;      // arena bytes (0 = not owned by the arena)
  bool owned = true;
};

struct NcclApi;

struct tncb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  tncb::Arena arena;
  uint64_t launches = 0;
  int oz_slices = 8;  // 0 = DMMA only; otherwise the int8 tensor-core engine (K1') takes large pairs (digit-slicing engine: #slices)
  int oz_engine = 0;  // 0 = CRT / modular engine (crt.cu, default), 1 = 7-bit digit slicing (ozaki.cu, kept for A/B)
  long long oz_min_tiles = 96, oz_min_k = 1536;   // thresholds of the digit-slicing engine
  // CRT engine: operand bits (53 = full mantissa) or a requested tolerance, forced modulus count, thresholds, workspace
  int crt_bits = 53; double crt_tol = 0.0; int crt_nmod_force = 0;
  long long crt_min_k = 256; double crt_min_mnk = 268435456.0;   // K >= 256 and M*N*K >= 2^28
  size_t crt_ws_bytes = (size_t)12 << 30;
  double last_int8_ops = 0.0; int last_nmod = 0; int last_products = 0;
  int crt_products = 0;            // real int8 products per complex product: 0 = auto (3 when K >= crt_kara_min_k), 3, 4
  long long crt_kara_min_k = 2048;
  uint64_t engine_count[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // K0, K0 split-K, K1 DMMA, K1 DMMA split-K, K1' int8, K2, permute, -
  // dominant-kernel timing: 0 off, 1 keep the last launch (gemm_ev0/1), 2 accumulate every launch (event pool)
  int time_gemm = 0; cudaEvent_t gemm_ev0 = nullptr, gemm_ev1 = nullptr; bool gemm_ev_valid = false;
  std::vector<cudaEvent_t> gemm_pool; size_t gemm_used = 0; std::vector<double> gemm_ops;
  int sm_count = 132;
  long long l2_bytes = 50LL << 20;
  // pinned staging for leaf uploads
  void* stage_host = nullptr; size_t stage_bytes = 0;
  // K1 offset-table workspace (grown on demand, stream-ordered reuse)
  long long* tab = nullptr; size_t tab_elems = 0;
  // signature of the tables currently in `tab` (they depend on the plan only, like a TMA
  // descriptor): an identical consecutive pair re-uses them without a rebuild
  bool tab_valid = false; tncb::LegList tab_m{}, tab_n{}, tab_k{};
  // split-K partial workspace
  double2* partial = nullptr; size_t partial_elems = 0;
  double2* partial_override = nullptr; size_t partial_override_elems = 0;  // set while a plan graph is captured
  // NCCL
  void* nccl_comm = nullptr; int world = 1, rank = 0;
  // host pipeline (tncb_contract_pair_host): 3 in-flight jobs, each with its own device operands/result and events;
  // copies run on their own streams so that H2D of pair j+1, the kernels of pair j and D2H of pair j-1 overlap
  struct HostSlot { void* buf[3] = {nullptr, nullptr, nullptr}; size_t bytes[3] = {0, 0, 0};
                    cudaEvent_t in_done = nullptr, comp_done = nullptr, out_done = nullptr; bool busy = false; };
  HostSlot host_slot[3]; uint64_t host_jobs = 0;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
  // plans that hold device state (graph, workspace) on this context; detached by tncb_ctx_destroy
  std::vector<struct tncb_plan*> plans;
  // structure-keyed cache of plans behind tncb_contract_tensor_network (most recently used last)
  struct CachedPlan { std::vector<uint64_t> key; struct tncb_plan* plan; };
  std::vector<CachedPlan> plan_cache;
  // angle maps whose tables live in this context's arena; detached by tncb_ctx_destroy
  std::vector<struct tncb_angles*> angle_maps;
};

extern "C" void tncb_plan_release_device_state(struct tncb_plan* plan);
namespace tncb { void angles_release(struct tncb_angles* a, tncb_ctx* ctx); }   // angles.cu

namespace tncb {
// ---- kernel launchers (kernels.cu) ---------------------------------------------------
// count > 1: the same pair of `count` networks whose operands and result lie `stride` bytes apart (instance i at
// A + i * stride, ...), as one launch per kernel; every launch decision (tile config, lanes, split-K) is the one a
// single instance gets, so each instance's result is bit-identical to count = 1
int launch_pair(tncb_ctx* ctx, const PairPlan& p, const double2* A, const double2* B, double2* C,
                int count = 1, long long stride = 0);
int launch_permute(tncb_ctx* ctx, const double2* in, double2* out, int rank,
                   const uint64_t* in_dims, const int* perm);
int launch_conj(tncb_ctx* ctx, double2* data, uint64_t elems);
int launch_add(tncb_ctx* ctx, double2* dst, const double2* src, uint64_t elems);
int ensure_tab(tncb_ctx* ctx, size_t elems);
// K1': int8 digit-sliced ZGEMM on wgmma (ozaki.cu); tables as built by launch_k1
int launch_k1_ozaki(tncb_ctx* ctx, const PairPlan& p, const double2* A, const double2* B, double2* C, int S,
                    const long long* offAm, const long long* offBn, const long long* offAk, const long long* offBk);

// K1' default engine: wgmma int8 GEMMs over coprime moduli + CRT reconstruction (crt.cu)
int launch_k1_crt(tncb_ctx* ctx, const PairPlan& p, const double2* A, const double2* B, double2* C,
                  const long long* offAm, const long long* offBn, const long long* offAk, const long long* offBk);
void crt_choose(long long K, int want_bits, int nmod_force, int* nmod, int* bits_a, int* bits_b);
int crt_bits_for_tolerance(long long K, double tol);
int crt_export_tables(int nmod, int* moduli, double* rho1, double* rho2, double* log2_product);

void gemm_timer_begin(tncb_ctx* ctx);              // brackets one launch of the dominant GEMM kernel (K1 / K1')
void gemm_timer_end(tncb_ctx* ctx, double ops);    // ops: executed int8 ops (K1') or flops (K1) of that launch

int ensure_partial(tncb_ctx* ctx, size_t elems);
size_t k0_partial_elems(int sm_count, const PairPlan& p);

// ---- batched tiny pairs: every independent K0 pair of one tree level in ONE launch (plans with a static layout) ----
constexpr int kBatchGroups = 8;
struct CompactLegs { int n; int _pad; long long dim[kBatchGroups]; long long sa[kBatchGroups]; long long sb[kBatchGroups]; };
struct K0BatchItem {
  long long offA, offB, offC;   // byte offsets into the plan workspace
  long long M, N, K;
  int G, _pad;                  // lanes per output element: the value k0_config picks for the single-pair kernel (bit-identical sums)
  CompactLegs m, n, k;
};
bool k0_batch_eligible(int sm_count, const PairPlan& p);
int k0_batch_fill(int sm_count, const PairPlan& p, K0BatchItem* item);   // returns the number of 256-thread blocks of the item
int launch_k0_batch(tncb_ctx* ctx, const K0BatchItem* d_items, const int* d_block_start, int n_items, int total_blocks, char* ws,
                    int count = 1, long long stride = 0);

// ---- leaf gradients of a gradient plan: every requested leaf adjoint, from its workspace slot (pair output order) into
// the packed gradient block (the leaf's own leg order), in ONE launch ----
constexpr int kGradGroups = 8;
struct GradItem {
  long long src;                // byte offset of the adjoint slot in the plan workspace
  long long dst;                // element offset of the leaf's gradient in the output block
  long long elems;
  int n, _pad;                  // fused leg groups in the leaf's order, outermost first
  long long dim[kGradGroups];
  long long st[kGradGroups];    // element stride of each group in the adjoint slot
};
constexpr int kGradThreads = 256;   // outputs per block
int launch_grad_gather(tncb_ctx* ctx, const GradItem* d_items, const long long* d_block_start, int n_items,
                       long long total_blocks, const char* ws, double2* out);
// n instances' workspaces `stride` bytes apart: instance i's gradients into rows + i * row_elems (rows != nullptr) and/or
// added to sum in instance order (sum != nullptr); one launch for the pass
int launch_grad_gather_batch(tncb_ctx* ctx, const GradItem* d_items, const long long* d_block_start, int n_items,
                             long long total_blocks, const char* ws, long long stride, int n, double2* rows,
                             long long row_elems, double2* sum);

// ---- sliced gradient plans: slice q's sub-block of every full leaf <-> the slice leaf in the workspace, in ONE launch
// per direction.  Element o of the slice leaf (row-major in its kept legs, the full leaf's order) decomposes over the
// fused groups; the slot side reads / writes sum_g i_g * st[g], the full side base(q) + sum_g i_g * fst[g] with
// base(q) = sum_k ((q / sdiv[k]) % sdim[k]) * sst[k] over the leaf's sliced legs ----
constexpr int kSliceGroups = 8, kSliceLegs = 8;
struct SliceItem {
  long long slot;               // byte offset in the plan workspace (or in the plan's permute scratch, from_scratch)
  long long full;               // element offset of the full leaf in the full leaf block / the full gradient block
  long long elems;              // elements of the slice leaf
  int n, ns;                    // fused leg groups (outermost first); sliced legs of this leaf
  int from_scratch, _pad;
  long long dim[kSliceGroups];
  long long st[kSliceGroups];   // element stride of each group on the slot side
  long long fst[kSliceGroups];  // element stride of each group in the full leaf
  unsigned long long sdiv[kSliceLegs], sdim[kSliceLegs];   // digit k of slice q: (q / sdiv[k]) % sdim[k]
  long long sst[kSliceLegs];    // element stride of that sliced leg in the full leaf
};
int launch_slice_extract(tncb_ctx* ctx, const SliceItem* d_items, const long long* d_block_start, int n_items,
                         long long total_blocks, const double2* full, char* ws, unsigned long long q);
int launch_grad_accumulate(tncb_ctx* ctx, const SliceItem* d_items, const long long* d_block_start, int n_items,
                           long long total_blocks, const char* ws, const double2* scratch, double2* grad, unsigned long long q);

// ---- device staging of leaf payloads (tncb_plan_set_leaves / tncb_plan_stage_instances): copies from arbitrary device
// addresses into leaf blocks, n instances per launch.  Items never overlap; the table travels as a kernel parameter ----
constexpr int kStageThreads = 256;  // elements per block
constexpr int kStageItems = 512;    // items per launch (table + prefix: 20.5 KB of the 32 KB parameter space)
struct LeafStageItem {
  const double2* src;           // instance i reads src + i * src_stride
  unsigned long long src_stride; // elements between instances, 0 = the same payload for every instance
  long long dst;                // element offset in the leaf block
  long long elems;
};
struct LeafStageBatch {
  int n, _pad;
  long long block_start[kStageItems + 1];   // block-count prefix
  LeafStageItem items[kStageItems];
};
// instance i's leaf block at dst + i * block_elems; any number of items and instances (several launches if needed)
int launch_leaf_stage(tncb_ctx* ctx, const LeafStageItem* items, size_t n_items, double2* dst, long long block_elems,
                      size_t n_instances);
// cuMemGetAddressRange, resolved through the runtime (network.cpp); nullptr when the driver does not offer it
typedef CUresult (*MemRangeFn)(CUdeviceptr*, size_t*, CUdeviceptr);
MemRangeFn get_mem_range();

// the table index (gate_angles.h) of a gate that takes angles, -1 for the others (gates.cpp)
int angle_gate(const char* name);

// ---- tangent sums of a tangent plan: every two-sided forward step of one level, out = t1 + t2, in ONE launch; count
// instances whose workspaces lie `stride` bytes apart (the instance a grid dimension) ----
constexpr int kSumThreads = 256;    // elements per block
struct TangentSumItem { long long t1, t2, out, elems; };   // byte offsets in the plan workspace; elements
int launch_tangent_sum(tncb_ctx* ctx, const TangentSumItem* d_items, const long long* d_block_start, int n_items,
                       long long total_blocks, char* ws, int count, long long stride);

// ---- sampling (tncb_plan_sample, sample.cu): the kernels of one pass of c candidate slots ----
struct SampleMap {
  int n_qubits, n_closed, k, _pad;
  unsigned char closed_qubit[64];   // closed bit j (bit j of w0) is qubit closed_qubit[j]
  unsigned char result_qubit[64];   // result leg r (row-major, leg 0 outermost) is qubit result_qubit[r]
};
struct SampleCand { unsigned long long bits; double p, ratio; int accept, clipped; };   // one candidate after selection
struct SampleCounts { unsigned long long consumed, accepted, clipped; double max_ratio; };   // one pass, after the cut
// candidates first .. first + n - 1: the one-hot bras of the closed bits, closed bra j of slot i at bras + (j c + i) * 2,
// u and v at uv[i], the closed bits deposited on their qubits at closed_bits[i]
int launch_sample_candidates(tncb_ctx* ctx, unsigned long long seed, unsigned long long first, size_t n, size_t c,
                             const SampleMap& map, double2* bras, double2* uv, unsigned long long* closed_bits);
// one block per slot i < n: the 2^k amplitudes at ws + i * stride + res_off, accept / reject, the pick (SampleCand)
int launch_sample_select(tncb_ctx* ctx, const char* ws, long long stride, long long res_off, size_t n, double m,
                         const SampleMap& map, const double2* uv, const unsigned long long* closed_bits, SampleCand* cand);
// tncb_plan_sample_slices: slot i's result (ws + i * stride + res_off, `elems` elements) into row i of acc ([n, elems]),
// copied (first) or added, the arithmetic of launch_add
int launch_sample_accumulate(tncb_ctx* ctx, const char* ws, long long stride, long long res_off, size_t n, size_t elems,
                             bool first, double2* acc);
// the accepted candidates of slots 0 .. n - 1, in slot order, up to `remaining` of them, into bits / probs (NULL: not
// written); the pass's counts into *counts
int launch_sample_compact(tncb_ctx* ctx, const SampleCand* cand, size_t n, unsigned long long remaining,
                          unsigned long long* bits, double* probs, SampleCounts* counts);

// ---- expectation values of Pauli sums (tncb_plan_expect, expect.cu) ----
struct ExpectLayer {
  int n_layer, _pad;
  unsigned char qubit[64];          // layer leaf j (in the caller's order) is qubit qubit[j]
};
// the layer payloads of terms first .. first + n - 1 (bit q of x_mask / z_mask picks qubit q's Pauli): layer leaf j of
// slot i at out + (j c + i) * 4, the 2x2 matrix with legs [ket, bra]
int launch_expect_layer(tncb_ctx* ctx, const unsigned long long* x_mask, const unsigned long long* z_mask,
                        unsigned long long first, size_t n, size_t c, const ExpectLayer& layer, double2* out);
// *energy = the left fold over k < n of (c_k Re R_k, c_k Im R_k), c_k = seeds[k].x, R_k = values[k]; one block
int launch_expect_fold(tncb_ctx* ctx, const double2* values, const double2* seeds, size_t n, double2* energy);

int tensor_new(tncb_ctx* ctx, int rank, const uint64_t* dims, tncb_tensor** out);

// TensorData::File leaf (hdf5io.cpp): first member of /tensors, optionally adjointed, checked against the leaf's dims
namespace h5 { int load_file_leaf(const char* path, bool adjoint, int rank, const uint64_t* dims, double* out_re_im); }
} // namespace tncb

#define TNCB_CUDA(call)                                                                   \
  do {                                                                                    \
    cudaError_t _e = (call);                                                              \
    if (_e != cudaSuccess)                                                                \
      return tncb::fail(TNCB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)
