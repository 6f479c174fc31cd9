/*
 * tncb.h -- C ABI of libtncb200: the H100-native pairwise tensor-contraction hot
 * path of qc-tum/TNC (tnc v1.0.0 @ 5dd62b3).
 *
 * This is the drop-in boundary.  TNC reaches its numeric kernel through plain
 * Rust calls into the un-vendored crate `tetra` (tnc/src/tensornetwork/
 * contraction.rs:3,78-84); a maintainer replaces those calls by the entry
 * points below through an `extern "C"` block (see INTEGRATION.md for the Rust
 * binding).  Every entry point cites the reference interface it replaces
 * (paths relative to the reference checkout).
 *
 * Conventions (identical to the reference, SURVEY.md A.1):
 *   - elements are complex128, passed as interleaved (re, im) doubles;
 *   - data is row-major (C order) over the tensor's leg order;
 *   - the result of contracting a and b has legs (b \ a) ++ (a \ b)
 *     (tnc/src/tensornetwork/tensor.rs:463-479 via contraction.rs:64);
 *   - paths are "replace-left": (i, j) stores the result in slot i
 *     (tnc/src/contractionpath.rs:29-35).
 *
 * Errors: every function returns 0 (TNCB_OK) or a negative tncb_status; nothing
 * aborts.  The reference panics instead (tensordata.rs:42, contraction.rs:50);
 * the language shim maps non-zero to panic!/exception.
 * Threading: a tncb_ctx is single-threaded like the reference's driver loop;
 * distinct contexts (devices) may be driven from distinct threads.
 * There is NO CPU fallback: without a CUDA device tncb_ctx_create fails with
 * TNCB_ERR_CUDA.
 */
#ifndef TNCB_H
#define TNCB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum tncb_status {
  TNCB_OK = 0,
  TNCB_ERR_INVALID = -1,      /* bad argument / malformed network or path            */
  TNCB_ERR_SHAPE = -2,        /* bond dimensions of a shared leg disagree            */
  TNCB_ERR_UNCONTRACTED = -3, /* slot already consumed / no data (tensordata.rs:42)  */
  TNCB_ERR_NOT_CONTRACTED = -4, /* >1 tensor left ("Not fully contracted", contraction.rs:50) */
  TNCB_ERR_OOM = -5,          /* device arena exhausted (peak live bytes > capacity) */
  TNCB_ERR_CUDA = -6,         /* CUDA runtime error (tncb_last_error has the text)   */
  TNCB_ERR_GATE = -7,         /* unknown gate / wrong angle count (gates.rs:54,103)  */
  TNCB_ERR_NCCL = -8,         /* NCCL error or libnccl not loadable                  */
  TNCB_ERR_UNSUPPORTED = -9,  /* e.g. an HDF5 feature outside the supported subset     */
  TNCB_ERR_IO = -10           /* file missing / unreadable / not (well-formed) HDF5    */
} tncb_status;

typedef struct tncb_ctx tncb_ctx;       /* one device + stream + arena              */
typedef struct tncb_tensor tncb_tensor; /* a device-resident complex128 tensor      */
typedef struct tncb_plan tncb_plan;     /* a compiled (network, path) schedule      */
typedef struct tncb_h5file tncb_h5file; /* an opened HDF5 tensor file (host only)   */

const char* tncb_strerror(int status);
/* Text of the last error raised on this thread (CUDA/NCCL message, offending pair). */
const char* tncb_last_error(void);
/* Library version / build info (arch list) -- cheap, needs no GPU. */
const char* tncb_version(void);

/* ---- context ------------------------------------------------------------------ */
/* arena_bytes = 0: grow on demand up to the device's free memory. */
int tncb_ctx_create(int device, size_t arena_bytes, tncb_ctx** out);
void tncb_ctx_destroy(tncb_ctx* ctx);
int tncb_ctx_synchronize(tncb_ctx* ctx);
/* The CUDA stream every kernel of this ctx is enqueued on (a cudaStream_t). */
void* tncb_ctx_stream(tncb_ctx* ctx);
/* Counters since creation / last reset: kernels launched by this library, arena peak. */
/* Give device memory back to the driver: synchronises, then cudaFree's every arena slab that holds no live block (the
 * arena otherwise keeps what it reserved for reuse).  For processes that switch between workloads of very different
 * footprints (e.g. a flat network, then a sliced one with a tens-of-GiB workspace).  The internal plan cache of
 * tncb_contract_tensor_network is dropped as well; plans created with tncb_plan_create keep their workspaces until they
 * are destroyed. */
int tncb_ctx_trim(tncb_ctx* ctx, uint64_t* freed_bytes, uint64_t* reserved_bytes);
int tncb_ctx_stats(tncb_ctx* ctx, uint64_t* kernel_launches, uint64_t* arena_peak_bytes,
                   uint64_t* arena_live_bytes);
int tncb_ctx_reset_stats(tncb_ctx* ctx);
/* Dense-GEMM engine for large GEMM-like pairs (M, N >= 128, K >= 256, M*N*K >= 2^28): K1', the int8
 * tensor cores (wgmma has no f64 kind; the API keeps its historical tcgen05 names).  Default engine = integer modular (CRT) emulation: every operand row
 * is scaled by a power of two and truncated to an `a`-bit integer (a = 53 by default = the whole mantissa of the
 * row's largest element), one int8 GEMM per coprime modulus (16 moduli for a = 53, K <= 2^13), exact CRT
 * reconstruction.  GUARANTEED bound (not "exact"):
 *     |C - C_exact|[n,m] <= 2^(4-a) * K * max|b[n,:]| * max|a[m,:]|     (max over real and imaginary parts)
 * i.e. normwise per output row/column, FP64-GEMM-equivalent for a = 53 (measured 3e-16..1e-15 of max|C|).
 * Elements far below their row maximum lose relative precision; a row whose maximum is below 2^-1000 keeps absolute
 * accuracy 2^(-1000-a); a row containing NaN/Inf poisons its outputs with NaN.
 * slices = 0 -> FP64 tensor pipe (DMMA) for every pair; non-zero -> K1' enabled (the value is the digit count of the
 * legacy 7-bit digit-slicing engine, see tncb_ctx_set_tcgen05_engine).  Smaller pairs always use DMMA / K0 / K2.
 * Environment: TNCB_OZAKI_SLICES, TNCB_TCGEN05_ENGINE, TNCB_CRT_MODULI override the defaults. */
int tncb_ctx_set_tcgen05_slices(tncb_ctx* ctx, int slices);
/* 0 = modular / CRT engine (default), 1 = 7-bit digit slicing of round 1 (S(S+1)/2 int8 GEMMs, drops digit
 * products p+q >= S: error <= (S+1) K 2^(-7S) of the same scale; kept for A/B measurements). */
int tncb_ctx_set_tcgen05_engine(tncb_ctx* ctx, int engine);
/* Requested normwise tolerance of K1': the engine keeps a = min(53, ceil(log2(16 K / rel))) bits per operand so that
 * |C - C_exact|[n,m] <= rel * max|b[n,:]| * max|a[m,:]| holds for every pair; rel = 0 (default) = full mantissa.
 * Fewer bits need fewer moduli (= int8 GEMM sweeps): see tncb_tcgen05_bound. */
int tncb_ctx_set_tolerance(tncb_ctx* ctx, double rel);
/* Pin the number of moduli (2..20; 0 = derive from the tolerance).  The operand bits then follow from
 * log2(prod m_i) >= a + b + log2(K) + 3; counts above what 53-bit operands need for the pair's K are clamped to that
 * (more moduli cannot add accuracy).  Measurement / test aid. */
int tncb_ctx_set_tcgen05_moduli(tncb_ctx* ctx, int n_moduli);
/* Real int8 GEMMs per modulus behind one complex product: 4 (re = ArBr - AiBi, im = ArBi + AiBr) or 3 (Karatsuba:
 * k1 = ArBr, k2 = AiBi, k3 = (Ar+Ai)(Br+Bi); re = k1 - k2, im = k3 - k1 - k2 -- the operand sums are taken on the residues,
 * i.e. exactly, so both forms reconstruct the same integers and differ only in the last rounding of the reconstruction).
 * 25 % fewer int8 operations for one more operand plane per side and one more residue plane, which pays for long K.
 * 0 (default) = 3 when K >= min_k3 (default 2048), else 4; min_k3 <= 0 keeps the
 * current threshold. */
int tncb_ctx_set_tcgen05_products(tncb_ctx* ctx, int products, long long min_k3);
/* What K1' would do for contraction length k (no GPU): modulus count, operand bits and the guaranteed factor
 * `bound` with |C - C_exact|[n,m] <= bound * max|b[n,:]| * max|a[m,:]|. */
int tncb_tcgen05_bound(uint64_t k, double rel, int n_moduli_force, int* n_moduli, int* bits_a, int* bits_b, double* bound);
/* The moduli and the split CRT weights rho_i = rho1_i + rho2_i = ((P/m_i)^-1 mod m_i) / m_i the engine uses for
 * `n_moduli` moduli (host-only; arrays of n_moduli entries): C'/P = frac(sum_i y_i rho_i) for residues y_i. */
int tncb_tcgen05_tables(int n_moduli, int* moduli, double* rho1, double* rho2, double* log2_product);
/* Workspace budget of K1' (residue planes + residues, default 12 GiB): larger pairs are processed in panels. */
int tncb_ctx_set_tcgen05_workspace(tncb_ctx* ctx, size_t bytes);
/* Size thresholds: (min_tiles, min_k) of the digit-slicing engine; for the modular engine min_k is the K threshold
 * and min_tiles == 1 drops the M*N*K >= 2^28 requirement (used by the parity tests). */
int tncb_ctx_set_tcgen05_threshold(tncb_ctx* ctx, long long min_tiles, long long min_k);
/* Pairs executed per engine since the last tncb_ctx_reset_stats: [0] K0, [1] K0 split-K, [2] K1 (DMMA),
 * [3] K1 split-K, [4] K1' (int8 tensor cores), [5] K2, [6] permute, [7] reserved. */
int tncb_ctx_engine_counts(tncb_ctx* ctx, uint64_t counts[8]);
/* int8 operations (2 x MAC) executed by the GEMM kernels of the last K1' pair and its modulus count. */
int tncb_ctx_last_tcgen05_info(tncb_ctx* ctx, double* int8_ops, int* n_moduli);
/* ... and whether it used the 3- or the 4-product form. */
int tncb_ctx_last_tcgen05_products(tncb_ctx* ctx, int* products);
/* Measurement aid: bracket the dominant GEMM kernel of every large pair (k1_kernel / oz_gemm_kernel)
 * with CUDA events on the ctx stream; tncb_ctx_last_gemm_ms synchronises and returns the last one. */
int tncb_ctx_time_gemm(tncb_ctx* ctx, int enable);
int tncb_ctx_last_gemm_ms(tncb_ctx* ctx, float* ms);
/* enable = 2: every launch of the int8 GEMM kernel is bracketed; tncb_ctx_gemm_totals synchronises, returns the
 * summed device time, the executed int8 operations (2 x MAC, padded tiles) and the launch count, and resets. */
int tncb_ctx_gemm_totals(tncb_ctx* ctx, double* ms, double* int8_ops, uint64_t* launches);

/* ---- tensors: replaces tetra::Tensor::{new_from_flat, elements, shape, ndim}
 *      (tnc/src/tensornetwork/tensordata.rs:31-37, tnc/src/io/hdf5.rs:105-106) ---- */
int tncb_tensor_upload(tncb_ctx* ctx, int rank, const uint64_t* dims,
                       const double* host_re_im, tncb_tensor** out);
int tncb_tensor_alloc(tncb_ctx* ctx, int rank, const uint64_t* dims, tncb_tensor** out);
int tncb_tensor_download(tncb_ctx* ctx, const tncb_tensor* t, double* host_re_im);
/* Asynchronous variants on the ctx stream (host buffer should be pinned; the caller
 * synchronises with tncb_ctx_synchronize before touching it). */
int tncb_tensor_write(tncb_ctx* ctx, tncb_tensor* t, const double* host_re_im);
int tncb_tensor_read(tncb_ctx* ctx, const tncb_tensor* t, double* host_re_im);
int tncb_tensor_free(tncb_ctx* ctx, tncb_tensor* t);
int tncb_tensor_rank(const tncb_tensor* t);
int tncb_tensor_dims(const tncb_tensor* t, uint64_t* dims_out);
uint64_t tncb_tensor_elements(const tncb_tensor* t);
void* tncb_tensor_device_ptr(const tncb_tensor* t); /* double2*, row-major */

/* ---- one pairwise contraction: replaces
 *      tetra::contract(out_legs, a_legs, a, b_legs, b) as called at
 *      tnc/src/tensornetwork/contraction.rs:78-84.  Consumes a and b (the Rust
 *      call moves them), returns a new tensor whose legs are out_legs, which must
 *      equal (b \ a) ++ (a \ b).  Pass out_legs = NULL to skip that check and
 *      read the legs back with tncb_pair_out_legs. ---- */
int tncb_contract_pair(tncb_ctx* ctx, int n_out, const uint64_t* out_legs,
                       int n_a, const uint64_t* a_legs, tncb_tensor* a,
                       int n_b, const uint64_t* b_legs, tncb_tensor* b,
                       tncb_tensor** out);
/* Same, but a and b stay alive (for benchmarking a single pair repeatedly). */
int tncb_contract_pair_keep(tncb_ctx* ctx, int n_a, const uint64_t* a_legs, const tncb_tensor* a,
                            int n_b, const uint64_t* b_legs, const tncb_tensor* b,
                            tncb_tensor** out);
/* Into a caller-provided output tensor (no allocation inside the timed region). */
int tncb_contract_pair_into(tncb_ctx* ctx, int n_a, const uint64_t* a_legs, const tncb_tensor* a,
                            int n_b, const uint64_t* b_legs, const tncb_tensor* b,
                            tncb_tensor* out);
/* tetra::contract for HOST operands (interleaved complex128, row-major), pipelined and asynchronous: the call enqueues
 * H2D(a, b) on a copy stream, the pair kernels on the ctx stream and D2H(result) on a second copy stream, then
 * returns.  Back-to-back calls overlap the upload of pair j+1, the kernels of pair j and the download of pair j-1
 * (three private sets of device buffers).  host_c receives (b \ a) ++ (a \ b) in row-major order
 * (tncb_pair_out_legs gives legs and dims).  Pinned host memory is required for the overlap; buffers are valid /
 * reusable after tncb_ctx_synchronize. */
int tncb_contract_pair_host(tncb_ctx* ctx, int n_a, const uint64_t* a_legs, const uint64_t* a_dims, const double* host_a,
                            int n_b, const uint64_t* b_legs, const uint64_t* b_dims, const double* host_b, double* host_c);
/* Leg algebra only (no GPU): Tensor::symmetric_difference, tensor.rs:463-479.
 * Writes (b\a)++(a\b) and the GEMM view M=|a\b|, N=|b\a|, K=|a&b|. */
int tncb_pair_out_legs(int n_a, const uint64_t* a_legs, const uint64_t* a_dims,
                       int n_b, const uint64_t* b_legs, const uint64_t* b_dims,
                       int* n_out, uint64_t* out_legs, uint64_t* out_dims,
                       uint64_t* m, uint64_t* n, uint64_t* k);
/* Which kernel class the planner would pick for that pair (no GPU):
 * 0 = K0 strided/warp-reduce kernel, 1 = K1 fused gather ZGEMM (DMMA, or the int8 K1' above the size
 * threshold), 2 = K2 streaming kernel (big tensor x tiny tensor, HBM-bound). */
int tncb_pair_kernel_class(int n_a, const uint64_t* a_legs, const uint64_t* a_dims,
                           int n_b, const uint64_t* b_legs, const uint64_t* b_dims);

/* ---- tetra::Tensor::transpose / conjugate
 *      (tnc/src/builders/circuit_builder.rs:106 Permutor::apply; gates.rs:87,98) ---- */
/* out dims[i] = in dims[perm[i]] (numpy.transpose semantics); consumes `t`. */
int tncb_permute(tncb_ctx* ctx, tncb_tensor* t, const int* perm, tncb_tensor** out);
int tncb_conjugate(tncb_ctx* ctx, tncb_tensor* t); /* in place */
/* dst += src (same element count): accumulation of sliced contractions (the reference's declared
 * future work, book/src/future_work.md:9-11). */
int tncb_tensor_add(tncb_ctx* ctx, tncb_tensor* dst, const tncb_tensor* src);

/* ---- gate table: replaces load_gate / load_gate_adjoint (tnc/src/gates.rs:50-66).
 *      Host-side; writes 4 or 16 interleaved complex values, *rank = 2 or 4. ---- */
int tncb_gate_matrix(const char* name, const double* angles, int n_angles, int adjoint,
                     double* out_re_im, int* rank);
/* The derivative of that matrix with respect to its angles, for the six gates that take angles (u, rx, ry, rz, cp,
 * fsim): dU/da_slot (slot2 < 0) or d²U/da_slot da_slot2, in the same element order, adjointed when adjoint != 0 (the
 * angles are real, so d(U†) = (dU)†).  The errors of tncb_gate_matrix, plus TNCB_ERR_GATE "slot out of range for this
 * gate" for a slot (or slot2 >= 0) at or past the gate's angle count -- every slot of a gate without angles. */
int tncb_gate_derivative(const char* name, const double* angles, int n_angles, int adjoint, int slot, int slot2,
                         double* out_re_im, int* rank);

/* ---- networks: mirrors tnc::tensornetwork::tensor::Tensor (tensor.rs:21-37) and
 *      tnc::contractionpath::ContractionPath (contractionpath.rs:29-35) as plain
 *      C trees so that cgo / Rust repr(C) / ctypes can build them. ---- */
typedef enum tncb_data_kind {
  TNCB_DATA_UNCONTRACTED = 0, /* TensorData::Uncontracted (composite or empty slot) */
  TNCB_DATA_MATRIX = 1,       /* TensorData::Matrix: host_re_im, row-major          */
  TNCB_DATA_GATE = 2,         /* TensorData::Gate((name, angles, adjoint))          */
  TNCB_DATA_DEVICE = 3,       /* already on the device (consumed by the call)       */
  TNCB_DATA_FILE = 4          /* TensorData::File((path, adjoint)): HDF5, see below */
} tncb_data_kind;

typedef struct tncb_tn {
  /* composite: n_children > 0, legs ignored.  leaf: n_children == 0. */
  size_t n_children;
  const struct tncb_tn* children;
  int rank;
  const uint64_t* legs;
  const uint64_t* dims;
  int kind; /* tncb_data_kind */
  const double* host_re_im;
  const char* gate_name;
  const double* gate_angles;
  int n_gate_angles;
  int gate_adjoint;
  tncb_tensor* device;
  /* TNCB_DATA_FILE (tensordata.rs:43-49): the first member of the file's /tensors group is loaded while the leaves are
   * staged (load_data, io/hdf5.rs:37-43), adjointed when file_adjoint != 0 (halves of the dims swapped + conjugated,
   * gates.rs:82-99; the rank must then be a power of two) and must have exactly this leaf's dims -> TNCB_ERR_SHAPE. */
  const char* file_path;
  int file_adjoint;
} tncb_tn;

typedef struct tncb_path {
  size_t n_pairs;
  const uint64_t* pairs; /* i0, j0, i1, j1, ... replace-left */
  size_t n_nested;
  const uint64_t* nested_index; /* child indices that have their own path */
  const struct tncb_path* nested;
} tncb_path;

/* contract_tensor_network(tn, path) (tnc/src/tensornetwork/contraction.rs:30-52):
 * nested paths first (ascending child index), then the top-level pairs in order.
 * Leaves are materialised (gates.rs tables) and uploaded in ONE host->device
 * copy, every pair runs on the device without host round trips, and the result
 * stays on the device.  out_legs must have room for *n_out legs (<= 64).
 * TNCB_DATA_DEVICE leaves are consumed atomically: on TNCB_OK every one of them has been freed
 * (the Rust call moves them); on ANY error none has been touched and the caller still owns all of
 * them.  Their storage stays allocated until the whole schedule has been enqueued.
 * The second and later calls with the same STRUCTURE (tree, legs, dims, payload kinds, path -- payload values are free)
 * run through a compiled plan kept in a small per-context cache (at most 4 plans / a quarter of the device memory,
 * least recently used evicted; TNCB_PLAN_CACHE=0 disables): no schedule construction, tiny pairs batched per level. */
int tncb_contract_tensor_network(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path,
                                 tncb_tensor** out, int* n_out, uint64_t* out_legs);

/* Legs and bond dimensions of the result of tncb_contract_tensor_network(tn, path), from metadata alone (host only, no
 * GPU work; the same validation and the same errors as the real call).  The fan-in needs it: only the raw buffer of a
 * contracted partition travels (tncb_comm_send), so the receiver derives the leg order of what arrives from the sender's
 * partition and local path (the reference ships legs inside the serialised tensor, serialization.rs:43-67).
 * out_legs / out_dims need room for 64 entries; either may be NULL. */
int tncb_network_out_legs(const tncb_tn* tn, const tncb_path* path, int* n_out, uint64_t* out_legs, uint64_t* out_dims);

/* Compile once / execute many: the same circuit with different payloads
 * (e.g. other bitstrings or angles) re-uses the schedule, arena layout and the
 * captured CUDA graph.
 * A plan has one of seven kinds: plain (tncb_plan_create), vjp, jvp, hvp (tncb_plan_create_vjp / _jvp / _hvp) and sliced
 * vjp, jvp, hvp (the _sliced creators).  Every call that takes a plan checks its kind first, right after its null
 * checks: "." takes it; U (TNCB_ERR_UNSUPPORTED) and I (TNCB_ERR_INVALID) refuse it with a message that names the call
 * that runs the plan, or the creator the call wants.  tncb_plan_info and tncb_plan_destroy take every kind.
 *                        plain  vjp  jvp  hvp  sliced vjp  sliced jvp  sliced hvp
 *   stage                  .     .    .    .       .           .           .
 *   run, execute           .     .    U    U       U           U           U
 *   stage_slices           .     U    U    U       U           U           U
 *   run_slices             .     U    U    U       .           .           .
 *   run_batch              .     U    U    U       U           U           U
 *   vjp                    I     .    U    U       U           U           U
 *   vjp_sliced             I     I    U    U       .           U           U
 *   stage_batch            I     .    .    U       U           U           U
 *   vjp_batch              I     .    U    U       U           U           U
 *   jvp, jvp_batch         I     I    .    U       I           U           U
 *   jvp_sliced             I     I    I    I       I           .           I
 *   hvp, hvp_batch         I     I    I    .       I           U           U
 *   hvp_sliced             I     I    I    I       I           I           .
 *   stage_instances        .     .    .    U       U           U           U
 *   set_leaves             .     .    .    .       .           U           U
 *   grad_offsets           I     .    .    .       .           .           .
 *   sample                 .     U    U    U       U           U           U
 *   sample_slices          .     U    U    U       U           U           U
 *   expect                 .     .    U    U       U           U           U          */
int tncb_plan_create(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, tncb_plan** out);
/* `tn` must have the structure the plan was compiled from: every leaf is re-validated (kind, rank,
 * dims, non-null payload, live device handle) -> TNCB_ERR_INVALID / TNCB_ERR_SHAPE /
 * TNCB_ERR_UNCONTRACTED before any copy.  Device leaves: same atomic rule as above.  A plan may be
 * destroyed before or after its context. */
int tncb_plan_execute(tncb_ctx* ctx, tncb_plan* plan, const tncb_tn* tn,
                      tncb_tensor** out, int* n_out, uint64_t* out_legs);
/* Keep the materialised leaves of `tn` on the device (one H2D), then execute the schedule any number of times with no
 * host work besides the kernel launches: the "inputs already resident in HBM" mode.  Not for plans with
 * TNCB_DATA_DEVICE leaves (consumed per call) -> TNCB_ERR_UNSUPPORTED. */
int tncb_plan_stage(tncb_ctx* ctx, tncb_plan* plan, const tncb_tn* tn);
int tncb_plan_run(tncb_ctx* ctx, tncb_plan* plan, tncb_tensor** out, int* n_out, uint64_t* out_legs);
/* Many networks of the plan's structure: the leaf payloads of all n_slices networks are materialised and uploaded ONCE.
 * They may be slices (fixing the value of summed legs splits one contraction into independent contractions whose results
 * add up; the reference's declared future work, book/src/future_work.md:9-11), other bitstrings, other angle sets or any
 * other payloads.  tncb_plan_run_slices contracts networks first, first + stride, ... with no host work per network and
 * returns their sum (zeros if the range is empty) -- ranks of a multi-GPU job pass (rank, world) and combine with
 * tncb_comm_allreduce_sum.  tncb_plan_run_batch returns them one by one instead. */
int tncb_plan_stage_slices(tncb_ctx* ctx, tncb_plan* plan, size_t n_slices, const tncb_tn* const* slice_tns);
int tncb_plan_run_slices(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride,
                         tncb_tensor** out_sum, int* n_out, uint64_t* out_legs);
/* Contract the networks first .. first+count-1 staged by tncb_plan_stage_slices, each on its own (NOT summed), and
 * return them as ONE tensor of rank r+1 and dims [count, d_0 .. d_{r-1}].  *n_out / out_legs describe one instance
 * (r legs); instance i is the i-th row-major block.  Results are bit-identical to tncb_plan_run_slices(i, n_slices) of
 * each instance.  The instances are a grid dimension of every kernel: one walk over the schedule per pass, each pass
 * holding as many copies of the plan's workspace as fit the static-workspace limit (TNCB_PLAN_WS_GB) and the free
 * device memory.  The plan's staged leaves (tncb_plan_stage) are untouched.  Needs a static plan (else
 * TNCB_ERR_UNSUPPORTED); count == 0, first + count > n_slices, a result rank of 64, or no staged networks on this
 * context -> TNCB_ERR_INVALID; not even one workspace copy fits -> TNCB_ERR_OOM. */
int tncb_plan_run_batch(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t count,
                        tncb_tensor** out, int* n_out, uint64_t* out_legs);
/* Schedule facts: #pairs, sum 8MNK, sum 16(MK+KN+MN), peak arena bytes, #kernels.  For a gradient plan they cover the
 * whole pass (forward + backward pairs, leaf-gradient gather) and peak_bytes is its static workspace. */
int tncb_plan_info(const tncb_plan* plan, uint64_t* n_pairs, double* flops, double* bytes,
                   uint64_t* peak_bytes, uint64_t* n_kernels);
/* ---- gradients with respect to the leaves (reverse mode) ----
 * For a plan of (tn, path) with result R and a seed S shaped like R, the holomorphic vector-Jacobian product of every
 * requested leaf X_l:   G_l[e] = sum_r S[r] * dR[r]/dX_l[e]   (plain contraction, no conjugation anywhere).  For a
 * scalar R and S = 1, G_l is the environment of leaf l: the network contracted without it.  G_l is row-major in the
 * leaf's OWN leg order (it has the leaf's shape).  The backward pass contracts, for every forward pair C = A.B, the
 * adjoint of C with B (giving A's adjoint) and with A (giving B's), each of the forward pair's M*N*K volume, on the same
 * engines; an operand gets its pair only if its subtree holds a requested leaf.  Cost: about two forward passes with
 * every leaf requested, whatever the number of leaves.
 * wrt: one flag per leaf (collect order: depth first, children in order); NULL = every leaf that has a payload.
 * ctx may be NULL (host-only compile: tncb_plan_info / tncb_plan_grad_offsets).  Refused with TNCB_ERR_UNSUPPORTED:
 * device leaves, networks without pairs, legs joining more than two tensors, and a static workspace (forward operands
 * kept until the backward pair that reads them + adjoints) above the static-workspace limit (0.62 of the device,
 * TNCB_PLAN_WS_GB; the message states the bytes needed).  wrt selecting no leaf, or a leaf without a payload ->
 * TNCB_ERR_INVALID.  Gradient plans always run on their static layout (also under TNCB_TRACE), are never captured into
 * a CUDA graph and have no pair-by-pair fallback: a workspace that does not fit at run time -> TNCB_ERR_OOM. */
int tncb_plan_create_vjp(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, const uint8_t* wrt, tncb_plan** out);
/* After tncb_plan_stage + tncb_plan_run (or tncb_plan_execute) of this plan -- which run the forward levels only and
 * return the result a plain plan returns, bit for bit -- the backward levels + the gather.
 * seed: device tensor with the result's dims (else TNCB_ERR_SHAPE); NULL only for a rank-0 result (seed 1).
 * *grads: new rank-1 device tensor holding every requested G_l back to back (tncb_plan_grad_offsets).
 * TNCB_ERR_INVALID without such a forward run on the currently staged leaves, and for a second call after one (the
 * backward slots reuse freed forward memory).  Errors leave the arena as they found it. */
int tncb_plan_vjp(tncb_ctx* ctx, tncb_plan* plan, const tncb_tensor* seed, tncb_tensor** grads);
/* Element offset of each leaf's gradient inside *grads, -1 for leaves not requested (n_leaves entries); host only.
 * For a sliced gradient plan the offsets pack the FULL leaves' shapes; for a tangent plan they place each requested
 * leaf's tangent in a tangent row (tncb_plan_jvp). */
int tncb_plan_grad_offsets(const tncb_plan* plan, int64_t* offsets);
/* ---- sliced gradients: networks whose gradient workspace does not fit unsliced ----
 * Fixing the sliced legs splits R into slices, R = sum_q R_q, so dR/dX_l = sum_q dR_q/dX_l; a slice leaf is a
 * fixed-index sub-block of the full leaf, so its adjoint adds into that sub-block of the full gradient.
 * tn is the FULL network and `path` the path every slice uses (slicing removes legs, not leaves).  The slice structure
 * (every leaf without the sliced legs; a leaf may become rank 0) is compiled exactly as tncb_plan_create_vjp compiles the
 * host-sliced slice network: the same pairs, backward schedule, static layout and refusals; tncb_plan_info covers one
 * slice's pass (with its leaf extraction and gradient accumulation launches) and peak_bytes is the per-slice workspace.
 * Slice q is the row-major mixed-radix digit vector of q over sliced_legs in the order given, last leg fastest.  wrt
 * indexes the full network's leaves (collect order).  ctx may be NULL (host-only compile).  A sliced leg that does not
 * occur, occurs once (an open leg), has dimension 0 or is listed twice, and a slice count above 2^64 - 1 ->
 * TNCB_ERR_INVALID; a leaf carrying more than 8 sliced legs, or needing more than 8 leg groups to address its slices ->
 * TNCB_ERR_UNSUPPORTED.
 * Use: tncb_plan_stage(ctx, plan, full tn) validates against the full structure and uploads the full leaf block once
 * into a plan-owned block outside the workspace (re-staging replaces it); tncb_plan_run_slices(ctx, plan, first,
 * stride, ...) runs the forward levels of slices first, first+stride, ... and returns their sum, bit-identical to a
 * plain plan of the host-sliced networks staged with tncb_plan_stage_slices; tncb_plan_vjp_sliced adds the backward. */
int tncb_plan_create_vjp_sliced(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, size_t n_sliced,
                                const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out);
/* Per slice q = first, first+stride, ...: extract q's sub-blocks of the leaves that carry a sliced leg (one launch),
 * forward levels, seed copy, backward levels, accumulate every requested leaf adjoint into q's sub-block of its
 * full-shape gradient (one launch).  No host work per slice; slices run in stream order, so results repeat bit for bit.
 * seed: device tensor with the result's dims, NULL only for a rank-0 result (seed 1); the same seed for every slice.
 * *value: new tensor, the sum of the slices' results, bit-identical to tncb_plan_run_slices(first, stride).
 * *grads: new rank-1 tensor, every requested full-shape G_l back to back (tncb_plan_grad_offsets).  An empty range
 * (more ranks than slices) gives zeros for both; partial ranges add up, so ranks of a multi-GPU job pass (rank, world)
 * and run tncb_comm_allreduce_sum on both tensors.  Not staged on this context / stride 0
 * -> TNCB_ERR_INVALID; seed errors as tncb_plan_vjp.  Errors leave the arena as they found it. */
int tncb_plan_vjp_sliced(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, const tncb_tensor* seed,
                         tncb_tensor** value, tncb_tensor** grads);
/* ---- batched gradients: many networks of one gradient plan's structure (sampled bitstrings, angle sets, input states)
 * Stage n networks of a (non-sliced) gradient plan's structure for tncb_plan_vjp_batch: every leaf validated and
 * materialised, one H2D; the structure-validation errors are those of tncb_plan_stage_slices.  The plan's own staged
 * leaves (tncb_plan_stage) and forward state are untouched.  Tangent plans take it as well (for tncb_plan_jvp_batch). */
int tncb_plan_stage_batch(tncb_ctx* ctx, tncb_plan* plan, size_t n, const tncb_tn* const* tns);
/* Instances first .. first+count-1, each contracted forward and backward on its own with the instance as a grid
 * dimension of every kernel, in passes of as many workspace copies as fit (as tncb_plan_run_batch; a gradient workspace
 * is about twice a forward one).  Each output may be NULL (not produced); at least one must be non-NULL.
 *   seeds:      [count, result dims..] device tensor; NULL only for a rank-0 result (seed 1 for every instance) or
 *               when no gradient is requested
 *   *values:    new [count, result dims..]; row i bit-identical to stage(net_i) + run
 *   *grad_rows: new [count, grad_elems]; row i bit-identical to stage(net_i) + run + tncb_plan_vjp(seed_i), leaves at
 *               tncb_plan_grad_offsets inside each row
 *   *grad_sum:  new [grad_elems]; the left fold 0 + row_0 + row_1 + ... in instance order, bit for bit
 * grad_rows == grad_sum == NULL: forward levels only.  The plan's workspace, staged leaves and forward state are left
 * alone, so stage + run + tncb_plan_vjp_batch + tncb_plan_vjp works.  Ranks of a multi-GPU job may split [first, count)
 * and combine their grad_sum with tncb_comm_allreduce_sum.
 * Nothing staged by tncb_plan_stage_batch on this context, count == 0, a range past the staged networks, every output
 * NULL, NULL seeds for a non-scalar result with gradients requested, a result of rank 64 -> TNCB_ERR_INVALID; seed dims
 * other than [count, result dims] ->
 * TNCB_ERR_SHAPE; not even one workspace copy fits -> TNCB_ERR_OOM.  Errors leave the arena as they found it. */
int tncb_plan_vjp_batch(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t count, const tncb_tensor* seeds,
                        tncb_tensor** values, tncb_tensor** grad_rows, tncb_tensor** grad_sum);
/* ---- leaf payloads from device memory (e.g. torch CUDA tensors): no host round trip ----
 * A source is row-major complex128 (re, im) in the leaf's own leg order, 16-byte aligned, in device (or managed) memory of
 * the ctx's device.  The library copies it (one launch of leaf_stage_kernel on the ctx stream, asynchronous); the caller
 * orders its writes before the call and keeps the memory alive until the ctx stream has passed the call.
 * Validation is complete before any copy, and a failure leaves every staged state untouched: a leaf index out of range,
 * listed twice or naming a leaf without a payload, a null / misaligned source, one that is not device memory of the ctx's
 * device, or whose bytes run past the end of the allocation that holds it (cuMemGetAddressRange) -> TNCB_ERR_INVALID;
 * plans with TNCB_DATA_DEVICE leaves -> TNCB_ERR_UNSUPPORTED.
 *
 * Overwrite the payloads of leaves leaf_index[0..n) of a STAGED plan with device memory: src[k] points to the leaf's
 * elements.  The payloads go where the next run reads them: a static plan's leaf block (also replayed by its graph), a
 * non-static plan's resident block, a sliced gradient plan's full leaf block (leaf indices and shapes of the full
 * network).  A gradient plan then needs a new forward run before tncb_plan_vjp.  They stay in place across runs,
 * tncb_plan_vjp and tncb_plan_vjp_sliced, as staged leaves do.  Not staged on this ctx (tncb_plan_stage) ->
 * TNCB_ERR_INVALID. */
int tncb_plan_set_leaves(tncb_ctx* ctx, tncb_plan* plan, size_t n, const uint64_t* leaf_index, const void* const* src);
/* Stage n_instances networks of the plan's structure: every leaf from the host template `tmpl` (validated as
 * tncb_plan_stage validates a network; materialised and uploaded ONCE, whatever n_instances is), except leaves
 * leaf_index[0..n), whose instance i reads src[k] + i * instance_stride[k] elements (stride 0 = the same device payload
 * in every instance; a non-zero stride below the leaf's element count -> TNCB_ERR_INVALID).  Plain plans: replaces
 * tncb_plan_stage_slices (feeds run_slices / run_batch; needs a static plan, else TNCB_ERR_UNSUPPORTED).  Gradient plans:
 * replaces tncb_plan_stage_batch (feeds vjp_batch; the plan's own workspace is not allocated); tangent plans likewise
 * (feeds jvp_batch).  Staged instances are
 * bit-identical to the host-staged networks with the same payloads.  n_instances == 0 -> TNCB_ERR_INVALID. */
int tncb_plan_stage_instances(tncb_ctx* ctx, tncb_plan* plan, const tncb_tn* tmpl, size_t n_instances,
                              size_t n, const uint64_t* leaf_index, const void* const* src, const uint64_t* instance_stride);
/* ---- directional derivatives with respect to the leaves (forward mode) ----
 * For a plan of (tn, path) with result R and tangents Ẋ_l of the requested leaves, the holomorphic Jacobian-vector product
 *   Ṙ[r] = sum_l sum_e dR[r]/dX_l[e] * Ẋ_l[e]      (plain contraction, no conjugation anywhere)
 * the transpose of tncb_plan_vjp: sum_r S[r] Ṙ[r] = sum_l sum_e G_l[e] Ẋ_l[e] with G = vjp(S).  Leaves not requested have
 * zero tangent.  The tangents are one packed rank-1 block: every requested leaf's Ẋ_l row-major in the leaf's OWN leg
 * order at tncb_plan_grad_offsets, the layout tncb_plan_vjp returns, so a gradient block and a tangent block are
 * interchangeable.  For every forward pair C = A.B with a requested leaf below it, the tangent pass contracts Ȧ with B
 * and/or A with Ḃ, each with the forward pair's legs and GEMM view on the same engines, on the forward pair's own tree
 * level, and adds the two when both exist (one launch per level).  Cost: about three forward passes with every leaf
 * requested, in ONE walk over the forward levels.
 * wrt: one flag per leaf (collect order); NULL = every leaf that has a payload.  ctx may be NULL (host-only compile:
 * tncb_plan_info, which then covers forward pairs, tangent pairs and sums, and tncb_plan_grad_offsets).  Refused with
 * TNCB_ERR_UNSUPPORTED: device leaves, networks without pairs, and a static workspace above the static-workspace limit
 * (TNCB_PLAN_WS_GB; the message states the bytes needed).  wrt selecting no leaf, or a leaf without a payload ->
 * TNCB_ERR_INVALID.  Tangent plans always run on their static layout, are never captured into a CUDA graph and have no
 * pair-by-pair fallback. */
int tncb_plan_create_jvp(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, const uint8_t* wrt, tncb_plan** out);
/* One forward-mode pass on the leaves staged by tncb_plan_stage (and overwritten by tncb_plan_set_leaves).
 * tangents: [tangent_elems] device tensor (tangent_elems = the sum of the requested leaves' sizes).
 * *value: new tensor with the result's dims, bit-identical to a plain plan's tncb_plan_run on the same leaves.
 * *tangent_out: new tensor with the result's dims, Ṙ.  Either may be NULL, not both.  Each call is self-contained and
 * repeats bit for bit.  Not staged on this context, both outputs NULL, NULL tangents ->
 * TNCB_ERR_INVALID; tangent dims other than [tangent_elems] -> TNCB_ERR_SHAPE.  Errors leave the arena as they found it. */
int tncb_plan_jvp(tncb_ctx* ctx, tncb_plan* plan, const tncb_tensor* tangents, tncb_tensor** value, tncb_tensor** tangent_out);
/* Instances first .. first+count-1 staged by tncb_plan_stage_batch or tncb_plan_stage_instances, each with its own
 * tangent row, in passes of as many workspace copies as fit (as tncb_plan_run_batch).
 *   tangents:      [count, tangent_elems] device tensor, row i for instance first + i
 *   *values:       new [count, result dims..]; row i bit-identical to tncb_plan_jvp of instance i
 *   *tangent_rows: new [count, result dims..]; row i bit-identical to tncb_plan_jvp of instance i with tangent row i
 * Either output may be NULL, not both.  Many directions of one network: stage count instances of it with
 * tncb_plan_stage_instances (every device source at stride 0, or the host template alone) and pass one tangent row per
 * direction.  Nothing staged on this context, count == 0, a range past the staged networks, both
 * outputs NULL, NULL tangents, a result of rank 64 -> TNCB_ERR_INVALID; tangent dims other than [count, tangent_elems]
 * -> TNCB_ERR_SHAPE; not even one workspace copy fits -> TNCB_ERR_OOM.  Errors leave the arena as they found it. */
int tncb_plan_jvp_batch(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t count, const tncb_tensor* tangents,
                        tncb_tensor** values, tncb_tensor** tangent_rows);
/* ---- Hessian-vector products (forward over reverse) ----
 * For a plan of (tn, path) with result R, seed S, leaf tangents Ẋ_l of the requested leaves and a seed tangent Ṡ, one
 * pass gives (holomorphic, no conjugation anywhere)
 *   R;   Ṙ = sum_l sum_e dR/dX_l[e] Ẋ_l[e]                                   (as tncb_plan_jvp)
 *   G_l  = sum_r S[r] dR[r]/dX_l                                             (as tncb_plan_vjp)
 *   Ġ_l  = sum_r Ṡ[r] dR[r]/dX_l + sum_r S[r] sum_m sum_e' d²R[r]/dX_l dX_m[e'] Ẋ_m[e']
 * the forward derivative of G in the direction (Ẋ, Ṡ).  Second derivatives are symmetric, so the vjp of (X, S) -> G
 * with cotangent W is (Ġ with Ẋ = W and Ṡ = 0, Ṙ with Ẋ = W): one call serves double backward and forward-over-reverse.
 * Every leaf occurs once, so R is multilinear and the diagonal blocks (l = m) of the Hessian are zero.  The plan holds
 * the forward pairs, the tangent pairs of tncb_plan_create_jvp, the backward pairs of tncb_plan_create_vjp and, for
 * every backward pair x̄ = C̄.O, its tangent dx̄ = dC̄.O + C̄.dO: pairs with the backward pair's legs and GEMM view on
 * the same engines and backward level, summed in that order when both exist.  Cost: about nine forward passes with
 * every leaf requested, in one walk over the levels.  Arguments and refusals as tncb_plan_create_jvp (the message of
 * a workspace above the limit states the bytes needed); ctx may be NULL (host-only compile: tncb_plan_info and
 * tncb_plan_grad_offsets).  Always static, never graphed, no pair-by-pair fallback. */
int tncb_plan_create_hvp(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, const uint8_t* wrt, tncb_plan** out);
/* One forward-over-reverse pass on the leaves staged by tncb_plan_stage (and overwritten by tncb_plan_set_leaves).
 * tangents:     [tangent_elems] device tensor at tncb_plan_grad_offsets (the gradient block's layout)
 * seed:         the result's dims; NULL only for a rank-0 result (seed 1)
 * seed_tangent: the result's dims; NULL = zero
 * *value, *tangent_out: new tensors with the result's dims, R (bit-identical to a plain plan's tncb_plan_run) and Ṙ
 *   (bit-identical to tncb_plan_jvp with the same tangents)
 * *grads, *grad_tangents: new [tangent_elems] tensors at tncb_plan_grad_offsets, G (bit-identical to tncb_plan_vjp(seed)
 *   of a gradient plan after a run) and Ġ
 * Each output may be NULL, not all four.  Each call is self-contained and repeats bit for bit.  Not staged on this
 * context, no output, NULL tangents, a NULL seed for a result of rank > 0 ->
 * TNCB_ERR_INVALID; tangent, seed or seed-tangent dims that do not match -> TNCB_ERR_SHAPE.  Errors leave the arena as
 * they found it. */
int tncb_plan_hvp(tncb_ctx* ctx, tncb_plan* plan, const tncb_tensor* tangents, const tncb_tensor* seed,
                  const tncb_tensor* seed_tangent, tncb_tensor** value, tncb_tensor** tangent_out, tncb_tensor** grads,
                  tncb_tensor** grad_tangents);
/* count forward-over-reverse passes in one walk over the levels, in passes of as many workspace copies as fit beside
 * the plan's own (as tncb_plan_run_batch): many directions of one network (a Hessian block, block Lanczos), or one
 * direction per sampled network (a loss over bitstrings or input states).  Instance i < count is the network staged
 * by tncb_plan_stage (and tncb_plan_set_leaves), except leaves leaf_index[0..n): instance i reads src[k] +
 * i * instance_stride[k] elements (stride 0 = the same device payload in every instance), validated as
 * tncb_plan_stage_instances validates its sources, before any launch.  n == 0: count copies of the staged network.
 *   tangents:      [count, tangent_elems], row i for instance i at tncb_plan_grad_offsets
 *   seeds:         [count, result dims..]; NULL only for a rank-0 result (every seed 1)
 *   seed_tangents: [count, result dims..]; NULL = zero
 *   *values, *tangent_rows:           new [count, result dims..], R and Ṙ of every instance
 *   *grad_rows, *grad_tangent_rows:   new [count, tangent_elems], G and Ġ of every instance
 *   *grad_sum, *grad_tangent_sum:     new [tangent_elems], the left fold 0 + row 0 + row 1 + ... in instance order
 * Each output may be NULL, not all six; the backward levels run only if one of the four G / Ġ outputs is wanted.  Row i
 * of every output is bit-identical to tncb_plan_set_leaves(instance i's payloads) + tncb_plan_hvp(tangent row i, seed
 * i, seed tangent i): every launch decision is the single-network one, and int8-engine steps run instance by instance.
 * The plan's staged leaves and workspace are left as they are, so tncb_plan_hvp before and after gives the same bits.
 * The sums can be combined across ranks with tncb_comm_allreduce_sum.  Not staged on this context, count == 0, no output, NULL tangents, a NULL seed for a result of rank > 0, a result of rank 64 ->
 * TNCB_ERR_INVALID; device-source errors as
 * tncb_plan_stage_instances; tangent, seed or seed-tangent dims that do not match -> TNCB_ERR_SHAPE; not even one
 * workspace copy fits beside the plan's -> TNCB_ERR_OOM.  Errors leave the arena and the staged plan as they found them. */
int tncb_plan_hvp_batch(tncb_ctx* ctx, tncb_plan* plan, size_t count, size_t n, const uint64_t* leaf_index,
                        const void* const* src, const uint64_t* instance_stride, const tncb_tensor* tangents,
                        const tncb_tensor* seeds, const tncb_tensor* seed_tangents, tncb_tensor** values,
                        tncb_tensor** tangent_rows, tncb_tensor** grad_rows, tncb_tensor** grad_sum,
                        tncb_tensor** grad_tangent_rows, tncb_tensor** grad_tangent_sum);
/* ---- sampling bitstrings from a circuit's output distribution ----
 * A circuit on n <= 64 qubits, its amplitude network with the bras of the closed qubits Q (n - k of them) as leaves and
 * the k open qubits O as the plan's result legs: for a closed assignment c the plan contracts to the 2^k amplitudes
 * a_c(y) = <c, y| C |init>.  With p(c, y) = |a_c(y)|^2 and the exact marginal q(c) = sum_y p(c, y), candidate i carries
 * (c_i, u_i, v_i) from the random stream below and is accepted iff u_i < r_i = q(c_i) 2^(n-k) / m.  An accepted candidate's
 * open bits y_i are the first y, in the row-major order of the result, whose inclusive prefix sum of p exceeds v_i q(c_i),
 * q being the last value of that same fixed-order prefix sum (so such a y exists and p(c_i, y_i) > 0).  The sample is
 * (c_i, y_i) with its p(c_i, y_i).  The prefix sum runs over T = min(256, 2^k) chunks of consecutive outcomes, left to
 * right inside a chunk and over the chunk sums.
 *   Exact when nothing is clipped: if r <= 1 for every c, the samples are i.i.d. with law p / sum p, because a candidate
 *     is accepted with value x with probability p(x) / m (the network need not be normalised).
 *   Clipping biases the result: where r > 1 the assignment c is under-sampled; stats report how many consumed candidates
 *     were clipped and the largest ratio seen, so that m can be raised.
 *   Limiting cases: k = 0 is frugal rejection sampling (Markov et al.); k = n with m = 1 samples the state vector directly.
 *   Open qubits help: q(c) 2^(n-k) is a mean over 2^k outcomes and concentrates near 1, so a larger k allows m close to 1
 *     (nearly every contraction yields a sample) at a higher cost per contraction.  Which qubits are open changes the
 *     contraction's cost a great deal: choose them, or the path, with the open legs in mind (tncb_plan_info).
 * Random stream: candidate i of seed s is the Philox4x64-10 block (Random123 constants) of key (s, 0) and counter
 * (i, 0, 0, 0), words w0..w3; bit j of w0 is the value of closed qubit closed_qubit[j]; u = (w1 >> 11) 2^-53 and
 * v = (w2 >> 11) 2^-53.  Samples come out in candidate order, and a call's output depends only on (seed, first, the
 * candidates consumed): not on the pass size, nor on how the work is split into calls.  Ranks of a multi-GPU job take
 * disjoint candidate ranges through `first`. */
typedef struct tncb_sample_spec {
  int n_qubits;                 /* 1..64 */
  size_t n_closed;
  const uint64_t* closed_leaf;  /* leaf index (collect order) of the bra of closed qubit closed_qubit[j] */
  const int* closed_qubit;
  const int* result_qubit;      /* the qubit of each result leg of the plan, in result-leg order */
} tncb_sample_spec;
typedef struct tncb_sample_stats { uint64_t candidates, samples, clipped, passes; double max_ratio; } tncb_sample_stats;
/* Candidates first, first + 1, ... in passes of `batch` (0: as many workspace copies as fit, as tncb_plan_run_batch)
 * until max_samples are accepted or max_candidates are consumed.  The plan is a static plain plan staged on ctx
 * (tncb_plan_stage): its staged block supplies every leaf except the closed bras, which the device writes per candidate,
 * and it is left untouched.  Per pass: one kernel writes the candidates' bras, u and v; the batched forward levels
 * (tncb_plan_run_batch's launches); one kernel per candidate reads its amplitudes in place and decides; one kernel writes
 * the accepted samples in candidate order; one small device-to-host copy of the pass's counts.  When the target is
 * reached inside a pass, its later candidates are not consumed and do not count, so a call resumed at
 * first + stats->candidates continues the same stream.
 *   bits:  device, max_samples words; sample s at bits[s], bit q = qubit q
 *   probs: device, max_samples doubles, p of each sample; NULL = not written
 *   stats: candidates consumed, samples written, clipped candidates among those consumed, passes, the largest ratio r
 * Every refusal happens before any device work and leaves the arena as it found it.  TNCB_ERR_INVALID: a null argument;
 * n_qubits outside 1..64; a closed leaf out of range, listed twice, or not a rank-1, dimension-2 leaf with a payload; a
 * qubit missing from, or listed twice across, closed_qubit and result_qubit; a result leg whose dimension is not 2; m
 * not finite or not > 0; max_samples == 0; bits / probs not 8-byte aligned device memory of the ctx's device, or running
 * past the end of their allocation (cuMemGetAddressRange); not staged on this context.  TNCB_ERR_UNSUPPORTED: a plan of
 * another kind or without a static layout.  TNCB_ERR_OOM: not even one workspace copy fits. */
int tncb_plan_sample(tncb_ctx* ctx, tncb_plan* plan, const tncb_sample_spec* spec, uint64_t seed, uint64_t first,
                     uint64_t max_candidates, uint64_t max_samples, double m, size_t batch, uint64_t* bits, double* probs,
                     tncb_sample_stats* stats);
/* Sampling a circuit whose amplitude network only contracts sliced: the networks staged by tncb_plan_stage_slices on
 * ctx are the S slices of one open amplitude network, each with the closed bras at the same leaf indices (their staged
 * payloads are ignored), and candidate c's amplitudes are a_c(y) = sum_q R_q(c, y) over q = 0 .. S-1, formed as
 * tncb_plan_run_slices(0, 1) forms its sum: R_0 copied, then R_1, R_2, ... added in slice order, so that a_c is
 * bit-identical to that call on c's sliced networks.  Everything else -- the random stream, acceptance, the pick, the
 * clipping stats, candidate order, resuming at first + stats->candidates -- is tncb_plan_sample's contract.  Ranks of a
 * multi-GPU job split candidates through `first`, never slices: a candidate needs every slice.
 * Per pass: the candidate kernel once; for each slice, one leaf staging launch from that slice's staged block, the
 * batched forward levels and one launch that folds every candidate's result into its row of a [c, 2^k] accumulator;
 * then the select and compact kernels on the accumulator and the counts read-back, as tncb_plan_sample.
 * Memory: `batch` (0: as many as fit) workspace copies beside the plan's own, leaving 1 GiB and the int8 engine's plane
 * budget free, as tncb_plan_run_batch.  When the device has no room for even one copy, the call does not fail: it runs
 * one candidate per pass in the plan's own workspace and clears the leaves tncb_plan_stage put there, so a later
 * tncb_plan_run or tncb_plan_sample needs tncb_plan_stage again (until then they return TNCB_ERR_INVALID).  tncb_plan_run_slices and
 * tncb_plan_run_batch stage their leaves on every call and are unaffected; the staged slices are never written.  The
 * stats do not say which way a call ran, and the bits are the same either way.
 * Refusals: every refusal of tncb_plan_sample, with the same messages, except that "not staged" means nothing staged by
 * tncb_plan_stage_slices on ctx (TNCB_ERR_INVALID).  A slice whose closed bra is not a rank-1, dimension-2 leaf (a
 * sliced leg on a closed bra makes one) is refused as a closed leaf of the wrong shape. */
int tncb_plan_sample_slices(tncb_ctx* ctx, tncb_plan* plan, const tncb_sample_spec* spec, uint64_t seed, uint64_t first,
                            uint64_t max_candidates, uint64_t max_samples, double m, size_t batch, uint64_t* bits,
                            double* probs, tncb_sample_stats* stats);
/* ---- expectation values of Pauli sums: E = sum_k c_k <psi|P_k|psi> and its leaf gradient, every term in one pass ----
 * The plan's network is <psi|L|psi> with one observable ("layer") leaf L_q per qubit q of the layer, legs [ket leg, bra
 * leg]: the circuit's kept tensors, their adjoint mirror images, and the layer (Circuit.into_pauli_expectation_network
 * builds it, light cone pruned).  Term k is P_k = (x) over q of sigma(bit q of x_mask[k], bit q of z_mask[k]), sigma(0,0) = I,
 * (1,0) = X, (0,1) = Z, (1,1) = Y, with a real coefficient c_k.  Its layer payload on qubit q is the 2x2 matrix M = sigma^T
 * (row-major, [ket, bra]): the network contracts to sum_ab psi_a M[a,b] conj(psi_b), so R_k = <psi|P_k|psi>; only Y
 * differs from its transpose, and the transpose fixes the sign of every term with an odd number of Y's.  The payload
 * staged with the plan (the identity, say) is ignored by this call. */
typedef struct tncb_pauli_layer {
  int n_qubits;                 /* 1..64: bit q of a term's masks is qubit q */
  size_t n_layer;
  const uint64_t* layer_leaf;   /* leaf index (collect order) of the observable leaf of qubit layer_qubit[j] */
  const int* layer_qubit;
} tncb_pauli_layer;
/* Terms 0 .. n_terms - 1 (x_mask, z_mask, coeff: host arrays) in passes of `batch` terms (0: as many workspace copies
 * as fit, as tncb_plan_run_batch).  The plan is a static plain or gradient plan staged on ctx (tncb_plan_stage, and
 * tncb_plan_set_leaves for angles): its staged block supplies every leaf except the layer leaves, and it is left
 * untouched, so tncb_plan_run before and after gives the same bits.  The term table goes to the device in one small
 * host-to-device copy per call.  Per pass: one kernel writes the terms' layer payloads, the batched forward levels, the
 * value rows out; with grad_sum the seeds (c_k, 0), the backward levels and the gather that folds sum_k c_k G_k.  One
 * one-block kernel then forms the energy.  No atomics: results do not depend on `batch`, and calls repeat bit for bit.
 *   values:   new [n_terms]; row k bit-identical to tncb_plan_run on the network with term k's layer payloads staged
 *             from the host (for a gradient plan: to tncb_plan_vjp_batch's value row)
 *   energy:   new rank-0; the left fold ((0 + c_0 R_0) + c_1 R_1) + ... in term order, c R formed as (c Re R, c Im R),
 *             every operation rounded on its own (no FMA)
 *   grad_sum: gradient plans only; new [grad_elems] at tncb_plan_grad_offsets, bit-identical to tncb_plan_vjp_batch
 *             (seeds = c_k) over the per-term networks.  Requested layer leaves get sum_k c_k of their environments.
 * Any output may be NULL, not all three.  Ranks of a multi-GPU job pass disjoint subsets of the terms and add their
 * energy and grad_sum with tncb_comm_allreduce_sum.
 * Every refusal happens before any device work and leaves the arena as it found it.  TNCB_ERR_INVALID: a null argument
 * or n_terms == 0; n_qubits outside 1..64; a layer leaf out of range, listed twice, without a payload, or not rank 2 with
 * dims [2, 2]; a layer qubit out of range or listed twice; a term acting on a qubit without a layer leaf (named); a
 * non-finite coefficient (named); a result that is not a scalar; no output; grad_sum on a plain plan; not staged on this
 * context.  TNCB_ERR_UNSUPPORTED: a plan of another kind or without a static layout.  TNCB_ERR_OOM: not even one
 * workspace copy fits. */
int tncb_plan_expect(tncb_ctx* ctx, tncb_plan* plan, const tncb_pauli_layer* layer, size_t n_terms,
                     const uint64_t* x_mask, const uint64_t* z_mask, const double* coeff, size_t batch,
                     tncb_tensor** values, tncb_tensor** energy, tncb_tensor** grad_sum);
/* ---- sliced tangents and Hessian-vector products: networks whose tangent or Hessian-vector workspace does not fit ----
 * By linearity, as for sliced gradients: R = sum_q R_q, so Ṙ = sum_q Ṙ_q; slice q's leaf (and its tangent) is q's
 * fixed-index sub-block of the full leaf (and of its full-shape tangent), and q's G_l and Ġ_l add into q's sub-block of
 * the full-shape blocks.  R_q depends on q's sub-blocks only, so there are no cross-slice Hessian terms.
 * Creation as tncb_plan_create_vjp_sliced (the same sliced-leg checks and messages, ctx may be NULL), with the slice
 * structure compiled exactly as tncb_plan_create_jvp / tncb_plan_create_hvp compile the host-sliced slice network:
 * tncb_plan_info covers one slice's pass (with the leaf and tangent extraction and the accumulation launches) and
 * peak_bytes is the per-slice workspace; a per-slice workspace above the static-workspace limit -> TNCB_ERR_UNSUPPORTED
 * naming the bytes.  tncb_plan_grad_offsets packs the FULL leaves' shapes, for the tangents, G and Ġ alike.
 * Use: tncb_plan_stage(ctx, plan, full tn) uploads the full leaves once; tncb_plan_run_slices runs the forward levels
 * (with zero tangents) and returns a sum bit-identical to the plain sliced run. */
int tncb_plan_create_jvp_sliced(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, size_t n_sliced,
                                const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out);
/* Per slice q = first, first+stride, ...: extract q's sub-blocks of the leaves that carry a sliced leg and of every
 * requested leaf's tangent (one launch each), the forward levels with their tangent pairs, R += and Ṙ +=.  tangents:
 * [tangent_elems] device tensor, every requested leaf's FULL-shape tangent at tncb_plan_grad_offsets.  *value (the
 * sum of R_q, bit-identical to tncb_plan_run_slices) and *tangent_out (the sum of Ṙ_q) are new tensors with the result's
 * dims; either may be NULL, not both.  An empty range (first >= slices) gives zeros; partial ranges add up, for ranks
 * that all-reduce.  Not staged on this context, stride 0, no output, NULL tangents ->
 * TNCB_ERR_INVALID; tangent dims other than [tangent_elems] -> TNCB_ERR_SHAPE.  Errors leave the arena as they found it. */
int tncb_plan_jvp_sliced(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, const tncb_tensor* tangents,
                         tncb_tensor** value, tncb_tensor** tangent_out);
int tncb_plan_create_hvp_sliced(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, size_t n_sliced,
                                const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out);
/* As tncb_plan_jvp_sliced, then per slice: the seed (NULL only for a rank-0 result: 1) and the seed tangent (NULL: zero)
 * written after the forward levels, the backward levels with their tangent pairs, K3 of the adjoints (and adjoint
 * tangents) that need more than 8 leg groups, and the accumulation of G_l and then Ġ_l into q's sub-blocks of the
 * full-shape [tangent_elems] blocks *grads and *grad_tangents (zeroed once per call).  The same seed and seed tangent
 * serve every slice.  Each output may be NULL, not all four; the backward levels run only if *grads or *grad_tangents
 * is wanted.  Errors as tncb_plan_jvp_sliced, seed errors as tncb_plan_hvp. */
int tncb_plan_hvp_sliced(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, const tncb_tensor* tangents,
                         const tncb_tensor* seed, const tncb_tensor* seed_tangent, tncb_tensor** value,
                         tncb_tensor** tangent_out, tncb_tensor** grads, tncb_tensor** grad_tangents);
void tncb_plan_destroy(tncb_plan* plan);

/* ---- angle maps: derivatives with respect to the angles of Gate leaves ----
 * A circuit's gates are functions of real angles; these calls turn a parameter vector θ into Gate-leaf payloads, leaf
 * tangents and, from the leaf gradients of a plan, the gradient with respect to θ, all on the device.  They add no plan
 * kind: they produce and read blocks that the plan calls above take.
 * A ref fixes angle slot `slot` of Gate leaf `leaf` (collect order, as wrt) to scale * θ[param].  Slots no ref names keep
 * the leaf's own angle, captured at creation.  Several refs may share a param (tied angles: rx(2β) on every qubit, the
 * ket and bra copies of a gate in an expectation network).
 * offsets (one per network leaf, -1 = not in the block) place each leaf's elements in a block of block_elems complex
 * elements; every block the calls below read or write has this layout.  The intended source is tncb_plan_grad_offsets
 * with block_elems = the plan's tangent / gradient block size: then gate rows, tangent blocks, G and Ġ share the plan's
 * layout.  offsets NULL: the referenced leaves packed in leaf order (block_elems 0 = their total).
 * Creation is host-only and refuses, naming the offending ref: a leaf out of range or not a Gate leaf; a gate without
 * angles, with the wrong angle count or shape, or a slot past its angle count (TNCB_ERR_GATE / TNCB_ERR_SHAPE); param >=
 * n_params; the same (leaf, slot) twice; a non-finite scale; a referenced leaf at offset -1, whose elements run past
 * block_elems or overlap another's (TNCB_ERR_INVALID).  n_params == 0 or n_refs == 0 -> TNCB_ERR_INVALID.
 * A map may be destroyed before or after the contexts it was used on, as plans may. */
typedef struct { uint64_t leaf; uint32_t slot; uint32_t param; double scale; } tncb_angle_ref;
typedef struct tncb_angles tncb_angles;
int tncb_angles_create(const tncb_tn* tn, size_t n_params, size_t n_refs, const tncb_angle_ref* refs,
                       const int64_t* offsets, size_t block_elems, tncb_angles** out);
int tncb_angles_destroy(tncb_angles* a);
/* n_params, block_elems and the offsets of every network leaf (any may be NULL). */
int tncb_angles_layout(const tncb_angles* a, size_t* n_params, size_t* block_elems, int64_t* offsets);
/* The device calls.  theta, theta_dot and direction are device double rows: row i at p + i * stride (stride 0 = one row
 * shared by all count rows), validated as tncb_plan_set_leaves validates its sources (non-null, 8-byte aligned, device
 * memory of the ctx's device, every byte inside its allocation; a non-zero stride below n_params) -> TNCB_ERR_INVALID.
 * The map's tables are uploaded once per context.  Every call is asynchronous on the ctx stream; count == 0 ->
 * TNCB_ERR_INVALID.  Non-finite angles give non-finite rows and are not refused.  Errors leave the arena as they found it.
 * <A, B> = sum_e A[e] B[e] (no conjugation); r runs over refs, l_r, s_r, p_r, c_r are its leaf, slot, param and scale.
 *   gates:     *rows = new [count, block_elems]; row i holds X_l(θ_i) of every referenced leaf at its offset, zeros elsewhere
 *   tangents:  *rows = new [count, block_elems]; Ẋ_l = sum_{r on l} c_r θ̇[p_r] dU_l/da_{s_r}, zeros elsewhere
 *   pullback:  g[p] = sum_{r: p_r = p} c_r <G_l, dU_l/da_{s_r}>; with G = vjp(S) this is sum_r S[r] dR[r]/dθ_p (complex:
 *              θ is real).  With grad_tangents Ġ and direction v (both or neither) it gives instead the derivative of g
 *              along v:  ġ[p] = sum_{r: p_r = p} c_r ( <Ġ_l, dU_l/da_{s_r}> + sum_{r' on l_r} c_r' v[p_r'] <G_l, d²U_l/da_{s_r} da_{s_r'}> );
 *              with G and Ġ from tncb_plan_hvp on tangents(θ, v) and a zero seed tangent, that is (H_θ v)[p] of S·R.
 *              grads (and grad_tangents) are [block_elems] (shared) or [count, block_elems].  *rows = new [count,
 *              n_params], *sum = new [n_params]; either may be NULL, not both.  Shape errors -> TNCB_ERR_SHAPE.
 * Determinism: no atomics; each param folds its refs in (param, leaf, slot) order; row i of any call is bit-identical to
 * the same call on row i alone; sum is the left fold 0 + row_0 + row_1 + ... bit for bit; calls repeat bit for bit.
 * How the calls compose with plans (no route is added to the table above):
 *   R(θ) without the host:      gates -> tncb_plan_set_leaves(src = row + offset) -> run / run_slices
 *   d(S·R)/dθ:                   gates -> set_leaves -> run -> tncb_plan_vjp(S) -> pullback(G)
 *   sliced:                      gates -> set_leaves on a sliced gradient plan -> vjp_sliced -> pullback of the full G
 *   B angle sets:                gates(B rows) -> stage_instances(src = rows + offset, stride = block_elems) ->
 *                                vjp_batch(seeds) -> pullback(grad rows) with the θ rows
 *   one θ for all instances:     vjp_batch grad_sum -> pullback with count = 1
 *   Ṙ along θ̇; the Jacobian:     tangents -> jvp; tangents(θ, eye(P)) -> jvp_batch over P instances at stride 0
 *   H_θ v, many v:               tangents(θ, v) -> hvp -> pullback(G, Ġ, v); hvp_batch with rows
 *   sliced tangent / Hessian-vector plans take no device payloads, so the angles arrive by staging the Gate network;
 *   then tangents -> jvp_sliced / hvp_sliced -> pullback. */
int tncb_angles_gates(tncb_ctx* ctx, const tncb_angles* a, const double* theta, size_t theta_stride, size_t count,
                      tncb_tensor** rows);
int tncb_angles_tangents(tncb_ctx* ctx, const tncb_angles* a, const double* theta, size_t theta_stride,
                         const double* theta_dot, size_t dot_stride, size_t count, tncb_tensor** rows);
int tncb_angles_pullback(tncb_ctx* ctx, const tncb_angles* a, const double* theta, size_t theta_stride, size_t count,
                         const tncb_tensor* grads, const tncb_tensor* grad_tangents,
                         const double* direction, size_t direction_stride,
                         tncb_tensor** rows, tncb_tensor** sum);

/* ---- HDF5 tensor files: replaces tnc::io::hdf5 (tnc/src/io/hdf5.rs), which binds libhdf5 through hdf5-metno.
 *      Neither is available here; csrc/hdf5io.cpp restates the published file format for the subset those calls produce
 *      and read (old- and new-style groups, object headers 1/2, contiguous / compact / chunked data with deflate and
 *      shuffle, Complex = compound of two floats, integer attributes).  Host only, no GPU needed.  Layout (hdf5.rs:1-15):
 *      one group `tensors`, one dataset per tensor (its shape = the bond dimensions), integer attribute `bids` = the
 *      bond ids; the dataset named "-1" carries the network's open bonds in `bids` and no data. ---- */
/* File::open + group(`group`), NULL = "/tensors".  Members are listed in ascending name order (strcmp), the order of
 * Group::member_names (H5Literate by name), so "-1" < "0" < "1" < "10" < "2". */
int tncb_hdf5_open(const char* path, const char* group, tncb_h5file** out);
void tncb_hdf5_close(tncb_h5file* file);
size_t tncb_hdf5_count(const tncb_h5file* file);
const char* tncb_hdf5_name(const tncb_h5file* file, size_t i);      /* NULL when i is out of range */
/* Shape of member i (dims needs room for 32 entries); any of rank / dims / elems may be NULL. */
int tncb_hdf5_shape(const tncb_h5file* file, size_t i, int* rank, uint64_t* dims, uint64_t* elems);
/* Integer attribute (`bids`, `tids`) of member i, widened to int64 (Attribute::read_1d, hdf5.rs:61,70).
 * out == NULL: only *n is set. */
int tncb_hdf5_attr(const tncb_h5file* file, size_t i, const char* name, size_t cap, int64_t* out, size_t* n);
/* read_dyn::<Complex64> (hdf5.rs:71,96): row-major interleaved re/im doubles.  Compounds of two f32 / big-endian floats
 * are converted; a real floating-point dataset is widened with zero imaginary parts (extension). */
int tncb_hdf5_read(const tncb_h5file* file, size_t i, double* out_re_im);
/* TensorData::File((path, adjoint)).into_data() (tensordata.rs:43-49) on the host: load_data(path) = the first member of
 * /tensors, then matrix_adjoint_inplace when adjoint != 0; the result must have exactly rank / dims (-> TNCB_ERR_SHAPE).
 * This is the routine the network executors call for TNCB_DATA_FILE leaves. */
int tncb_hdf5_load_leaf(const char* path, int adjoint, int rank, const uint64_t* dims, double* out_re_im);
/* store_data (hdf5.rs:46-52,105-113): a new file with /tensors/-1 = the tensor. */
int tncb_hdf5_store_data(const char* path, int rank, const uint64_t* dims, const double* data_re_im);
/* A whole network file in the layout read_tensor expects (the reference builds such files only in its tests,
 * hdf5.rs:141-170): n datasets, data_re_im[i] == NULL declares a dataset without data, n_bids[i] < 0 (or n_bids == NULL)
 * omits the attribute. */
int tncb_hdf5_store(const char* path, size_t n, const char* const* names, const int* ranks, const uint64_t* const* dims,
                    const double* const* data_re_im, const int64_t* n_bids, const uint64_t* const* bids);

/* ---- partitioned fan-in: replaces tnc::mpi::communication
 *      (scatter_tensor_network :125-195, intermediate_reduce_tensor_network :199-249).
 *      One process per GPU; boundary tensors move GPU->GPU with ncclSend/ncclRecv
 *      on the ctx stream (no serialisation: legs/dims are derived on every rank). ---- */
/* 128-byte NCCL unique id; create on rank 0, broadcast out of band. */
int tncb_comm_unique_id(uint8_t id_out[128]);
int tncb_comm_init(tncb_ctx* ctx, int world_size, int rank, const uint8_t id[128]);
int tncb_comm_send(tncb_ctx* ctx, const tncb_tensor* t, int peer);
int tncb_comm_recv(tncb_ctx* ctx, int rank_dims, const uint64_t* dims, int peer, tncb_tensor** out);
/* In-place sum over all ranks (ncclAllReduce on the ctx stream): combines sliced contractions. */
int tncb_comm_allreduce_sum(tncb_ctx* ctx, tncb_tensor* t);
int tncb_comm_destroy(tncb_ctx* ctx);
/* get_tensor_mapping (mpi/communication.rs:89-115): partition -> rank, the
 * partition on the left of the last top-level pair goes to rank 0, the others
 * to 1, 2, ... in the order the reference walks `path.nested.keys()`: the
 * iteration order of FxHashMap<usize,_>::from_iter(partition_index) (rustc-hash
 * 2.1.1 on hashbrown), reproduced bit-exactly and pinned by the reference KAT
 * communication.rs:257-279 (0 -> 0, 1 -> 2, 2 -> 1).  rank_of[p] for p < n_partitions. */
int tncb_fanin_mapping(size_t n_partitions, const uint64_t* partition_index,
                       size_t n_pairs, const uint64_t* toplevel_pairs, int world_size,
                       int* rank_of_partition);

/* ---- planning aids (host only, no GPU work) ---------------------------------------------------------------
 * Subtree reconfiguration of a contraction tree -- what the reference gets from cotengra via rustengra
 * (tnc/src/contractionpath/paths/tree_reconfiguration.rs:54-58).  Legs are relabelled by the caller to bit positions
 * 0 .. 64*n_words-1; leaf_legs holds n_leaves bitsets of n_words words; leg_log2[l] = log2(dim of leg l); a leg joins at
 * most two leaves (the reference's tensor model).  ssa_pairs (n_leaves-1 pairs, SSA ids) is refined in place:
 * pieces of the tree with at most subtree_size (2..15) frontier nodes are re-ordered optimally (subset DP) while that lowers
 *   sum over pair steps of  prod dims(legs(a) | legs(b)) + size_weight * prod dims(legs(a) ^ legs(b)),
 * for at most max_sweeps sweeps.  With time_model != NULL (8 doubles: int8-engine flop/s, its K half-rate constant, FP64
 * flop/s, HBM byte/s, seconds per launch, the FP64 kernels' K half-rate constant, the int8 engine's largest K, its operand
 * conversion bytes per element -- contraction_cost.GPU_RATES) the objective is the modelled device time
 *   sum over pair steps of  max(8 mnk / rate(m, n, k), 16 (mk + nk + mn) / hbm) + launch       (gpu_time_mnk)
 * instead.  flops = sum of prod dims(legs(a) | legs(b)), max_size = the largest tensor, objective = the minimised sum. */
int tncb_path_reconfigure(int n_leaves, int n_words, const uint64_t* leaf_legs, const double* leg_log2, int32_t* ssa_pairs,
                          int subtree_size, int max_sweeps, double size_weight, const double* time_model, uint64_t seed,
                          double* flops, double* max_size, double* objective);
/* Slicing scores of a tree, per leg l (arrays of 64*n_words): cost_without[l] = the objective of ONE slice once l is fixed,
 * size_without[l] = the largest tensor then; cost / max_size = the unsliced tree's. */
int tncb_path_leg_scores(int n_leaves, int n_words, const uint64_t* leaf_legs, const double* leg_log2, const int32_t* ssa_pairs,
                         double size_weight, const double* time_model,
                         double* cost_without, double* size_without, double* cost, double* max_size);

#ifdef __cplusplus
}
#endif
#endif /* TNCB_H */
