// contract_tensor_network on the device: replaces tnc/src/tensornetwork/contraction.rs:30-88.
//
// The reference walks the path sequentially and, per pair, materialises the payloads
// (tensordata.rs:40-59), allocates a result and calls tetra::contract.  Here the (nested)
// path is first compiled from metadata alone into a flat schedule of pair plans (leg algebra
// of tensor.rs:463-479); execution stages every leaf payload (gate tables, host matrices)
// into pinned memory, ships them in ONE host->device copy and then enqueues all pair kernels
// on the context stream without host round trips.  Arena memory of consumed operands is
// recycled in stream order.
#include "internal.h"
#include <cuda.h>
#include <algorithm>
#include <complex>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <memory>

namespace tncb {

int gate_matrix(const char* name, const double* ang, int n_ang, bool adjoint, std::complex<double>* out);

struct SlotMeta {
  std::vector<uint64_t> legs, dims;
  uint64_t elems = 1;
  int leaf_index = -1;      // >= 0: payload comes from the leaf block / a device handle
};

// bw_level > 0: a backward pair of a gradient plan, on that level of the backward pass (1 = the root's backward)
struct Step { int a, b, out; PairPlan plan; int bw_level = 0; };

struct Schedule {
  std::vector<SlotMeta> slots;
  std::vector<size_t> leaf_offset; // element offset of leaf i in the leaf block
  std::vector<int> leaf_kind;
  size_t leaf_block_elems = 0;
  std::vector<Step> steps;
  int result_slot = -1;
  double flops = 0, bytes = 0;
  size_t n_leaves_total = 0;
};

static const tncb_path* find_nested(const tncb_path* path, size_t idx) {
  if (!path) return nullptr;
  for (size_t q = 0; q < path->n_nested; q++)
    if (path->nested_index[q] == idx) return &path->nested[q];
  return nullptr;
}

static size_t count_leaves(const tncb_tn* tn) {
  if (tn->n_children == 0) return 1;
  size_t c = 0;
  for (size_t i = 0; i < tn->n_children; i++) c += count_leaves(&tn->children[i]);
  return c;
}

static int add_leaf(const tncb_tn* leaf, Schedule& S, size_t leaf_idx, int* slot_out) {
  S.leaf_kind[leaf_idx] = leaf->kind;
  if (leaf->kind == TNCB_DATA_UNCONTRACTED) { *slot_out = -1; return TNCB_OK; }
  if (leaf->rank < 0 || leaf->rank > kMaxLegs) return fail(TNCB_ERR_INVALID, "leaf rank out of range");
  SlotMeta m;
  m.legs.assign(leaf->legs, leaf->legs + leaf->rank);
  m.dims.assign(leaf->dims, leaf->dims + leaf->rank);
  for (int i = 0; i < leaf->rank; i++) m.elems *= leaf->dims[i];
  m.leaf_index = (int)leaf_idx;
  if (leaf->kind == TNCB_DATA_GATE) {
    if (!leaf->gate_name) return fail(TNCB_ERR_GATE, "gate leaf without a name");
    std::complex<double> tmp[16];
    int cnt = gate_matrix(leaf->gate_name, leaf->gate_angles, leaf->n_gate_angles, leaf->gate_adjoint != 0, tmp);
    if (cnt < 0) return cnt;
    if ((uint64_t)cnt != m.elems) return fail(TNCB_ERR_SHAPE, std::string("gate '") + leaf->gate_name + "' does not match the leaf's bond dimensions");
  } else if (leaf->kind == TNCB_DATA_MATRIX) {
    if (!leaf->host_re_im) return fail(TNCB_ERR_INVALID, "matrix leaf without host data");
  } else if (leaf->kind == TNCB_DATA_DEVICE) {
    if (!leaf->device) return fail(TNCB_ERR_INVALID, "device leaf without a tensor handle");
    if (leaf->device->elems != m.elems) return fail(TNCB_ERR_SHAPE, "device leaf: element count mismatch");
  } else if (leaf->kind == TNCB_DATA_FILE) {
    if (!leaf->file_path) return fail(TNCB_ERR_INVALID, "file leaf without a path");
  } else {
    return fail(TNCB_ERR_INVALID, "unknown TensorData kind " + std::to_string(leaf->kind));
  }
  if (leaf->kind != TNCB_DATA_DEVICE) {
    S.leaf_offset[leaf_idx] = S.leaf_block_elems;
    S.leaf_block_elems += std::max<uint64_t>(m.elems, 1);
  }
  S.slots.push_back(std::move(m));
  *slot_out = (int)S.slots.size() - 1;
  return TNCB_OK;
}

// Returns the slot id that holds the contraction result of `tn` (-1: nothing / empty tensor).
static int build(const tncb_tn* tn, const tncb_path* path, Schedule& S, size_t& leaf_counter, int* result) {
  if (tn->n_children == 0) { // a leaf handed to contract_tensor_network: only an empty path is legal
    if (path && (path->n_pairs || path->n_nested)) return fail(TNCB_ERR_INVALID, "path given for a leaf tensor");
    return add_leaf(tn, S, leaf_counter++, result);
  }
  const size_t nc = tn->n_children;
  std::vector<int> slot(nc, -1);
  std::vector<char> uncontracted_composite(nc, 0);
  if (path) for (size_t q = 0; q < path->n_nested; q++)
    if (path->nested_index[q] >= nc) return fail(TNCB_ERR_INVALID, "nested path index out of range");
  // nested paths first (contraction.rs:34-38); ascending child order
  for (size_t i = 0; i < nc; i++) {
    const tncb_tn* c = &tn->children[i];
    const tncb_path* np = find_nested(path, i);
    int rc;
    if (c->n_children == 0) {
      if (np && (np->n_pairs || np->n_nested)) return fail(TNCB_ERR_INVALID, "nested path given for a leaf child");
      if ((rc = add_leaf(c, S, leaf_counter++, &slot[i]))) return rc;
    } else if (np) {
      if ((rc = build(c, np, S, leaf_counter, &slot[i]))) return rc;
    } else {
      uncontracted_composite[i] = 1; // stays TensorData::Uncontracted
      size_t n = count_leaves(c);
      for (size_t q = 0; q < n; q++) S.leaf_kind[leaf_counter + q] = TNCB_DATA_UNCONTRACTED;
      leaf_counter += n;
    }
  }
  const size_t np_ = path ? path->n_pairs : 0;
  for (size_t q = 0; q < np_; q++) {
    const uint64_t i = path->pairs[2 * q], j = path->pairs[2 * q + 1];
    if (i >= nc || j >= nc) return fail(TNCB_ERR_INVALID, "pair (" + std::to_string(i) + "," + std::to_string(j) + ") indexes past the tensor list");
    if (i == j || slot[i] < 0 || slot[j] < 0)
      return fail(TNCB_ERR_UNCONTRACTED, "pair (" + std::to_string(i) + "," + std::to_string(j) + "): Cannot convert uncontracted tensor to data");
    const SlotMeta& a = S.slots[slot[i]];
    const SlotMeta& b = S.slots[slot[j]];
    Step st; st.a = slot[i]; st.b = slot[j];
    int rc = plan_pair((int)a.legs.size(), a.legs.data(), a.dims.data(), (int)b.legs.size(), b.legs.data(), b.dims.data(), st.plan);
    if (rc) return rc;
    SlotMeta o; o.legs = st.plan.out_legs; o.dims = st.plan.out_dims;
    for (uint64_t d : o.dims) o.elems *= d;
    S.slots.push_back(std::move(o));
    st.out = (int)S.slots.size() - 1;
    S.flops += st.plan.flops(); S.bytes += st.plan.bytes();
    S.steps.push_back(std::move(st));
    slot[i] = S.steps.back().out; slot[j] = -1; uncontracted_composite[j] = 0;
  }
  // retain(non-empty leaf or composite); at most one may remain (contraction.rs:48-51)
  int remaining = 0, last = -1;
  for (size_t i = 0; i < nc; i++) {
    if (slot[i] >= 0) { remaining++; last = slot[i]; }
    else if (uncontracted_composite[i]) { remaining++; last = -2; }
  }
  if (remaining > 1 || last == -2) return fail(TNCB_ERR_NOT_CONTRACTED, "Not fully contracted");
  *result = last;
  return TNCB_OK;
}

static int build_schedule(const tncb_tn* tn, const tncb_path* path, Schedule& S) {
  if (!tn) return fail(TNCB_ERR_INVALID, "tn is null");
  S.n_leaves_total = count_leaves(tn);
  S.leaf_offset.assign(S.n_leaves_total, 0);
  S.leaf_kind.assign(S.n_leaves_total, TNCB_DATA_UNCONTRACTED);
  size_t counter = 0;
  return build(tn, path, S, counter, &S.result_slot);
}

static void collect_leaf_nodes(const tncb_tn* tn, std::vector<const tncb_tn*>& v) {
  if (tn->n_children == 0) { v.push_back(tn); return; }
  for (size_t i = 0; i < tn->n_children; i++) collect_leaf_nodes(&tn->children[i], v);
}

// A schedule may be executed on a network other than the one it was compiled from (tncb_plan_execute):
// every leaf must still have the kind, rank, dims and a payload that the plan's offsets were sized for.
static int validate_leaves(const Schedule& S, const std::vector<const tncb_tn*>& leaves) {
  if (leaves.size() != S.n_leaves_total) return fail(TNCB_ERR_INVALID, "network does not match the plan (leaf count)");
  std::vector<const SlotMeta*> meta(leaves.size(), nullptr);
  for (const SlotMeta& m : S.slots) if (m.leaf_index >= 0) meta[m.leaf_index] = &m;
  for (size_t li = 0; li < leaves.size(); li++) {
    const tncb_tn* lf = leaves[li];
    if (S.leaf_kind[li] != lf->kind) return fail(TNCB_ERR_INVALID, "network payload kinds do not match the plan (leaf " + std::to_string(li) + ")");
    if (lf->kind == TNCB_DATA_UNCONTRACTED) continue;
    const SlotMeta* m = meta[li];
    if (!m) return fail(TNCB_ERR_INVALID, "plan has no slot for leaf " + std::to_string(li));
    if (lf->rank != (int)m->dims.size() || (lf->rank > 0 && !lf->dims))
      return fail(TNCB_ERR_SHAPE, "leaf " + std::to_string(li) + ": rank differs from the plan");
    for (int i = 0; i < lf->rank; i++)
      if (lf->dims[i] != m->dims[i]) return fail(TNCB_ERR_SHAPE, "leaf " + std::to_string(li) + ": bond dimensions differ from the plan");
    if (lf->kind == TNCB_DATA_MATRIX && !lf->host_re_im) return fail(TNCB_ERR_INVALID, "matrix leaf " + std::to_string(li) + " without host data");
    if (lf->kind == TNCB_DATA_GATE && !lf->gate_name) return fail(TNCB_ERR_GATE, "gate leaf " + std::to_string(li) + " without a name");
    if (lf->kind == TNCB_DATA_FILE && !lf->file_path) return fail(TNCB_ERR_INVALID, "file leaf " + std::to_string(li) + " without a path");
    if (lf->kind == TNCB_DATA_DEVICE) {
      if (!lf->device || !lf->device->ptr) return fail(TNCB_ERR_UNCONTRACTED, "device leaf " + std::to_string(li) + " without a tensor handle (already consumed?)");
      if (lf->device->elems != m->elems) return fail(TNCB_ERR_SHAPE, "device leaf " + std::to_string(li) + ": element count mismatch");
    }
  }
  for (size_t x = 0; x < leaves.size(); x++)       // the same device handle twice would be freed twice
    if (leaves[x]->kind == TNCB_DATA_DEVICE)
      for (size_t y = x + 1; y < leaves.size(); y++)
        if (leaves[y]->kind == TNCB_DATA_DEVICE && leaves[y]->device == leaves[x]->device)
          return fail(TNCB_ERR_INVALID, "the same device tensor is passed as two leaves");
  return TNCB_OK;
}

static int stage_leaves(const Schedule& S, const std::vector<const tncb_tn*>& leaves, std::complex<double>* stage);

// `resident` != nullptr: the leaf block already sits on the device (tncb_plan_stage); `tn` may then be null.
static int execute(tncb_ctx* ctx, const Schedule& S, const tncb_tn* tn, tncb_tensor** out, int* n_out, uint64_t* out_legs,
                   const double2* resident = nullptr) {
  TNCB_CUDA(cudaSetDevice(ctx->device));
  std::vector<const tncb_tn*> leaves;
  if (tn) collect_leaf_nodes(tn, leaves);
  if (!resident) { int vrc = validate_leaves(S, leaves); if (vrc) return vrc; }
  // ---- stage all host payloads, one H2D copy ----
  const size_t block_bytes = resident ? 0 : S.leaf_block_elems * sizeof(double2);
  void* leaf_block = nullptr;
  if (block_bytes) {
    if (ctx->stage_bytes < block_bytes) {
      if (ctx->stage_host) { TNCB_CUDA(cudaStreamSynchronize(ctx->stream)); cudaFreeHost(ctx->stage_host); ctx->stage_host = nullptr; }
      size_t want = std::max(block_bytes, (size_t)1 << 20);
      TNCB_CUDA(cudaMallocHost(&ctx->stage_host, want));
      ctx->stage_bytes = want;
    } else {
      // the previous network's upload may still be reading the staging buffer
      TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    { int src = stage_leaves(S, leaves, (std::complex<double>*)ctx->stage_host); if (src) return src; }
    int rc = ctx->arena.alloc(block_bytes, &leaf_block);
    if (rc) return rc;
    TNCB_CUDA(cudaMemcpyAsync(leaf_block, ctx->stage_host, block_bytes, cudaMemcpyHostToDevice, ctx->stream));
  }
  // ---- run the schedule ----
  struct Live { double2* ptr = nullptr; size_t bytes = 0; tncb_tensor* handle = nullptr; };
  std::vector<Live> live(S.slots.size());
  for (size_t s = 0; s < S.slots.size(); s++) {
    const int li = S.slots[s].leaf_index;
    if (li < 0) continue;
    if (S.leaf_kind[li] == TNCB_DATA_DEVICE) { live[s].ptr = leaves[li]->device->ptr; live[s].handle = leaves[li]->device; }
    else live[s].ptr = (resident ? const_cast<double2*>(resident) : (double2*)leaf_block) + S.leaf_offset[li];
  }
  int rc = TNCB_OK;
  std::vector<tncb_tensor*> consumed;
  // TNCB_TRACE=1: per-step device times on stderr (tuning aid; adds two events per pair)
  const bool trace = std::getenv("TNCB_TRACE") != nullptr;
  std::vector<cudaEvent_t> tev;
  if (trace) { tev.resize(S.steps.size() + 1); for (auto& e : tev) cudaEventCreate(&e); cudaEventRecord(tev[0], ctx->stream); }
  size_t step_no = 0;
  for (const Step& st : S.steps) {
    const SlotMeta& om = S.slots[st.out];
    size_t bytes = std::max<size_t>(om.elems * sizeof(double2), 16);
    void* p = nullptr;
    if ((rc = ctx->arena.alloc(bytes, &p))) break;
    live[st.out].ptr = (double2*)p; live[st.out].bytes = bytes;
    if ((rc = launch_pair(ctx, st.plan, live[st.a].ptr, live[st.b].ptr, live[st.out].ptr))) break;
    for (int s : {st.a, st.b}) { // operands are consumed (mem::take, contraction.rs:61-62)
      // caller-owned device leaves are released only after the WHOLE schedule was enqueued (atomic consumption:
      // on any error every device input is still alive and owned by the caller, see tncb.h)
      if (live[s].handle) consumed.push_back(live[s].handle);
      else if (live[s].bytes) ctx->arena.free(live[s].ptr, live[s].bytes);
      live[s].ptr = nullptr; live[s].bytes = 0; live[s].handle = nullptr;
    }
    if (trace) cudaEventRecord(tev[++step_no], ctx->stream);
  }
  if (trace) {
    cudaStreamSynchronize(ctx->stream);
    for (size_t q = 0; q < step_no; q++) {
      float ms = 0; cudaEventElapsedTime(&ms, tev[q], tev[q + 1]);
      const PairPlan& P = S.steps[q].plan;
      fprintf(stderr, "TNCB_TRACE step %zu class K%d M %lld N %lld K %lld groups m%d n%d k%d akf %d bkf %d ms %.4f tflops %.2f gbs %.1f\n",
              q, P.kernel_class, P.M, P.N, P.K, P.m.n, P.n.n, P.k.n, (int)P.a_kfast, (int)P.b_kfast, ms,
              P.flops() / (ms * 1e-3) * 1e-12, P.bytes() / (ms * 1e-3) * 1e-9);
    }
    for (auto& e : tev) cudaEventDestroy(e);
  }
  tncb_tensor* result = nullptr;
  if (!rc && S.result_slot >= 0) {
    const SlotMeta& rm = S.slots[S.result_slot];
    Live& rl = live[S.result_slot];
    result = new tncb_tensor();
    result->rank = (int)rm.dims.size(); result->elems = rm.elems;
    for (size_t i = 0; i < rm.dims.size(); i++) result->dims[i] = rm.dims[i];
    if (rl.bytes) { // produced by a pair: hand the arena block over
      result->ptr = rl.ptr; result->bytes = rl.bytes; rl.bytes = 0;
    } else if (rl.handle) { // a device leaf that was never contracted: the result takes its storage over
      *result = *rl.handle; rl.handle->ptr = nullptr; rl.handle->bytes = 0; consumed.push_back(rl.handle); rl.handle = nullptr;
    } else { // an uploaded leaf that was never contracted: copy it out of the leaf block
      result->bytes = std::max<size_t>(rm.elems * sizeof(double2), 16);
      void* p = nullptr;
      rc = ctx->arena.alloc(result->bytes, &p);
      if (!rc) {
        result->ptr = (double2*)p;
        cudaMemcpyAsync(p, rl.ptr, rm.elems * sizeof(double2), cudaMemcpyDeviceToDevice, ctx->stream);
      } else { delete result; result = nullptr; }
    }
  }
  // anything still live was not consumed because of an error
  for (size_t s = 0; s < live.size(); s++)
    if (live[s].bytes) ctx->arena.free(live[s].ptr, live[s].bytes);
  if (leaf_block) ctx->arena.free(leaf_block, block_bytes);
  if (rc) return rc;                                 // nothing in `consumed` was touched
  for (tncb_tensor* h : consumed) tncb_tensor_free(ctx, h);
  if (out) *out = result; else if (result) tncb_tensor_free(ctx, result);
  if (n_out) *n_out = S.result_slot >= 0 ? (int)S.slots[S.result_slot].legs.size() : 0;
  if (out_legs && S.result_slot >= 0)
    for (size_t i = 0; i < S.slots[S.result_slot].legs.size(); i++) out_legs[i] = S.slots[S.result_slot].legs[i];
  return TNCB_OK;
}

} // namespace tncb

// Compile once / execute many.  A plan gets a STATIC memory layout (every slot at a fixed offset of one workspace,
// blocks recycled level by level) unless it has caller-owned device leaves.  Its steps are re-ordered by the level of
// the contraction tree; all independent tiny (K0) pairs of a level run as ONE batched launch (k0_batch_kernel), the
// other pairs one by one.  Plans without K1 steps (the launch-bound regime) are additionally captured into a CUDA
// graph (H2D of the staged leaves + every kernel) and replayed.
struct tncb_plan {
  tncb::Schedule S;
  bool is_static = false;            // static layout + level batches available
  bool graphable = false;
  std::vector<size_t> slot_off;      // byte offset of every slot in the workspace
  size_t ws_bytes = 0, scratch_off = 0, scratch_elems = 0, leaf_off = 0;
  // level structure: steps [level_begin[l], level_begin[l+1]) of S.steps form level l; the batched ones come first
  std::vector<int> level_begin, level_batched;
  std::vector<tncb::K0BatchItem> items;            // batched steps of all levels, level by level
  std::vector<int> block_start;                    // per level: n_batched + 1 prefix entries
  std::vector<size_t> item_first, bs_first;        // per level: first index into items / block_start
  void* batch_dev = nullptr; size_t batch_bytes = 0;   // device copy of items + block_start
  tncb_ctx* ctx = nullptr;           // device state is tied to this context (stream, device)
  void* ws = nullptr;                // arena block
  void* stage = nullptr;             // plan-owned pinned staging of the leaf block
  cudaEvent_t stage_ev = nullptr;    // recorded after the last eager upload out of `stage` (re-staging waits for it)
  bool stage_busy = false;
  bool leaves_resident = false;      // tncb_plan_stage put the leaf block into ws
  cudaGraphExec_t exec[2] = {nullptr, nullptr};    // [0]: with the H2D of the staged leaves, [1]: leaves resident
  uint64_t kernels_per_run = 0;
  void* resident = nullptr;          // non-static plans: device copy of the leaf block (tncb_plan_stage)
  size_t resident_bytes = 0;
  void* slices_dev = nullptr;        // tncb_plan_stage_slices: n_slices leaf blocks, back to back
  size_t n_slices = 0, slices_bytes = 0;
  // the plan kind (tncb_plan_create / _vjp / _jvp / _hvp), sliced or not (the _sliced creators; never plain).  Only the
  // routing table asks which kind a plan is; everything else asks what it has: backward levels and leaf adjoints
  // (grad), tangent pairs (tangent)
  enum class Kind { plain, vjp, jvp, hvp };
  Kind kind = Kind::plain;
  bool sliced = false;
  bool grad() const { return kind == Kind::vjp || kind == Kind::hvp; }
  bool tangent() const { return kind == Kind::jvp || kind == Kind::hvp; }
  // gradient plans (tncb_plan_create_vjp): the backward pairs follow the forward ones in S.steps and occupy the levels
  // from n_fwd_levels on; always static, never graphed
  int n_fwd_levels = 0;              // levels [0, n_fwd_levels) are the forward pass (all levels of a plain plan)
  int seed_slot = -1;
  std::vector<int64_t> grad_offset;  // per leaf (collect order): element offset in the gradient block, -1 = not requested
  uint64_t grad_elems = 0;
  std::vector<tncb::GradItem> grad_items;           // leaves the gather kernel permutes
  std::vector<long long> grad_block_start;          // n_items + 1 prefix entries
  struct GradPermute { int slot; int64_t dst; std::vector<int> perm; };
  std::vector<GradPermute> grad_permutes;           // leaves with more fused groups than a GradItem holds: K3
  void* grad_dev = nullptr; size_t grad_dev_bytes = 0;   // device copy of grad_items + grad_block_start
  bool fwd_ready = false;            // a forward run left its state in the workspace for one tncb_plan_vjp
  // sliced gradient plans (tncb_plan_create_vjp_sliced): S is the structure of one slice, `full` holds the full
  // network's leaves; tncb_plan_stage uploads the full leaf block once and every slice is extracted from it on the device
  uint64_t n_sl = 1;                                // slices: the product of the sliced legs' dims
  tncb::Schedule full;                              // leaves only: kinds, dims, offsets in the full leaf block
  std::vector<tncb::SliceItem> sl_items, const_items, acc_items;   // extract (leaves with / without a sliced leg), accumulate
  std::vector<long long> sl_bs, const_bs, acc_bs;   // their block-count prefixes (n_items + 1 entries each)
  // sliced tangent / Hessian-vector plans (sliced && tangent): extract of every requested leaf's tangent from the caller's
  // full-shape tangent block, accumulate of the adjoints' tangents (Ġ)
  std::vector<tncb::SliceItem> tan_items, dacc_items;
  std::vector<long long> tan_bs, dacc_bs;
  size_t acc_scratch_elems = 0;                     // permute scratch of the leaves that take K3 before the accumulate
  void* sl_dev = nullptr; size_t sl_dev_bytes = 0;  // device copy of the items + prefixes, the seed 1, the permute scratch
  size_t sl_off[11] = {};                           // byte offsets inside sl_dev: 5 item arrays, 5 prefixes, seed 1 (+ scratch)
  void* full_dev = nullptr; size_t full_bytes = 0;  // the staged full leaf block (outside the workspace)
  bool full_staged = false;
  // tncb_plan_stage_instances: the template's leaves that take no device payload, packed, in plan-owned pinned memory
  // (re-used once tmpl_ev says its last upload ran) and on the device
  void* tmpl_host = nullptr; void* tmpl_dev = nullptr; size_t tmpl_bytes = 0;
  cudaEvent_t tmpl_ev = nullptr;
  bool tmpl_busy = false;
  // tangent plans (tncb_plan_create_jvp): the tangent pairs follow the forward ones in S.steps, each on its forward
  // step's level; grad_offset / grad_elems give the packing of the leaf tangents.  Always static, never graphed.
  int tan_result = -1;                              // the slot of the result's tangent
  struct TanLeaf { int slot; int64_t off; };        // a requested leaf's tangent slot and its offset in a tangent row
  std::vector<TanLeaf> tan_leaves;
  struct TanSum { int t1, t2; };                    // a two-sided step: t1 += t2 (t1 becomes the output's tangent)
  std::vector<TanSum> tan_sums;
  std::vector<tncb::TangentSumItem> sum_items;      // the sums of all levels, level by level
  std::vector<long long> sum_bs;                    // per level with sums: n + 1 block-count prefix entries
  std::vector<int> sum_first, sum_count;            // per level: first index into sum_items, number of sums
  std::vector<size_t> sum_bs_first;                 // per level: first index into sum_bs
  void* sum_dev = nullptr; size_t sum_dev_bytes = 0;  // device copy of sum_items + sum_bs
  // Hessian-vector plans (tncb_plan_create_hvp) are gradient and tangent plans at once: S.steps holds the forward,
  // tangent, backward and backward-tangent pairs; tan_sums holds the sums of both tangent passes.  grad_* gathers the
  // leaf adjoints (G), dgrad_* their tangents (Ġ), both at grad_offset.
  int seed_tan_slot = -1;                           // Ṡ, written (or zeroed) by tncb_plan_hvp before the backward levels
  std::vector<tncb::GradItem> dgrad_items;
  std::vector<long long> dgrad_block_start;
  std::vector<GradPermute> dgrad_permutes;
  void* dgrad_dev = nullptr; size_t dgrad_dev_bytes = 0;   // device copy of dgrad_items + dgrad_block_start
};

namespace tncb {

// first-fit offset allocator with coalescing (same policy as the arena) for the static layout
struct OffsetAlloc {
  std::map<size_t, size_t> free_by_off; size_t top = 0;
  static size_t up(size_t b) { return (std::max<size_t>(b, 256) + 255) / 256 * 256; }
  size_t alloc(size_t bytes) {
    bytes = up(bytes);
    for (auto it = free_by_off.begin(); it != free_by_off.end(); ++it)
      if (it->second >= bytes) {
        size_t off = it->first, sz = it->second;
        free_by_off.erase(it);
        if (sz > bytes) free_by_off[off + bytes] = sz - bytes;
        return off;
      }
    size_t off = top; top += bytes; return off;
  }
  void free(size_t off, size_t bytes) {
    bytes = up(bytes);
    auto it = free_by_off.emplace(off, bytes).first;
    auto nx = std::next(it);
    if (nx != free_by_off.end() && it->first + it->second == nx->first) { it->second += nx->second; free_by_off.erase(nx); }
    if (it != free_by_off.begin()) { auto pv = std::prev(it); if (pv->first + pv->second == it->first) { pv->second += it->second; free_by_off.erase(it); } }
  }
};

// one workspace for all intermediates of a run: at most 0.62 of the device (H100 80 GB: ~46 GiB; leaves room for the
// int8 engine's 12 GiB of planes and the staged leaves), 46 GiB when the device size is unknown (plan created without a
// context); TNCB_PLAN_WS_GB overrides.  Read on every call.
static size_t static_ws_limit(size_t device_bytes) {
  size_t limit = device_bytes ? (size_t)(0.62 * (double)device_bytes) : (size_t)46 << 30;
  if (const char* e = std::getenv("TNCB_PLAN_WS_GB")) limit = (size_t)std::max(1, atoi(e)) << 30;
  return limit;
}

// the size of ctx's device (0: no context, or the device does not answer), which scales the static-workspace limit
static size_t device_bytes(tncb_ctx* ctx) {
  size_t dev_free = 0, dev_total = 0;
  if (ctx) { cudaSetDevice(ctx->device); if (cudaMemGetInfo(&dev_free, &dev_total) != cudaSuccess) { dev_total = 0; cudaGetLastError(); } }
  return dev_total;
}

// ---- which call takes which plan kind (the table in tncb.h) ----
// The calls that take a plan, in the order of kRoutes' rows
enum class Call { stage, run, execute, stage_slices, run_slices, run_batch, vjp, vjp_sliced, stage_batch, vjp_batch, jvp,
                  jvp_batch, jvp_sliced, hvp, hvp_batch, hvp_sliced, stage_instances, set_leaves, grad_offsets, sample, sample_slices,
                  expect, count };
struct Refusal { int status; const char* msg; };
static const Refusal
    kHvpRuns{TNCB_ERR_UNSUPPORTED, "a Hessian-vector plan runs through tncb_plan_hvp"},
    kSlJvpRuns{TNCB_ERR_UNSUPPORTED, "a sliced tangent plan runs through tncb_plan_jvp_sliced / tncb_plan_run_slices"},
    kSlHvpRuns{TNCB_ERR_UNSUPPORTED, "a sliced Hessian-vector plan runs through tncb_plan_hvp_sliced / tncb_plan_run_slices"},
    kSlVjpRuns{TNCB_ERR_UNSUPPORTED, "a sliced gradient plan runs through tncb_plan_run_slices / tncb_plan_vjp_sliced"},
    kSlVjpGrads{TNCB_ERR_UNSUPPORTED, "a sliced gradient plan runs through tncb_plan_vjp_sliced"},
    kSlVjpStage{TNCB_ERR_UNSUPPORTED, "a sliced gradient plan stages its full network once (tncb_plan_stage)"},
    kSlVjpNoBatch{TNCB_ERR_UNSUPPORTED, "a sliced gradient plan has no batched gradients"},
    kSlVjpLeaves{TNCB_ERR_UNSUPPORTED, "a sliced gradient plan takes device payloads through tncb_plan_set_leaves"},
    kVjpOne{TNCB_ERR_UNSUPPORTED, "gradient plans run one staged network at a time"},
    kJvpRuns{TNCB_ERR_UNSUPPORTED, "a tangent plan runs through tncb_plan_jvp"},
    kJvpBatch{TNCB_ERR_UNSUPPORTED, "a tangent plan runs through tncb_plan_jvp_batch"},
    kJvpEither{TNCB_ERR_UNSUPPORTED, "a tangent plan runs through tncb_plan_jvp / tncb_plan_jvp_batch"},
    kJvpStage{TNCB_ERR_UNSUPPORTED, "tangent plans stage many networks with tncb_plan_stage_batch"},
    kNotVjp{TNCB_ERR_INVALID, "not a gradient plan (tncb_plan_create_vjp)"},
    kNotJvp{TNCB_ERR_INVALID, "not a tangent plan (tncb_plan_create_jvp)"},
    kNotHvp{TNCB_ERR_INVALID, "not a Hessian-vector plan (tncb_plan_create_hvp)"},
    kNotSlVjp{TNCB_ERR_INVALID, "not a sliced gradient plan (tncb_plan_create_vjp_sliced)"},
    kNotSlJvp{TNCB_ERR_INVALID, "not a sliced tangent plan (tncb_plan_create_jvp_sliced)"},
    kNotSlHvp{TNCB_ERR_INVALID, "not a sliced Hessian-vector plan (tncb_plan_create_hvp_sliced)"},
    kNotDerivStage{TNCB_ERR_INVALID, "not a gradient or tangent plan (plain plans stage many networks with tncb_plan_stage_slices)"},
    kNotDeriv{TNCB_ERR_INVALID, "not a gradient or tangent plan (tncb_plan_create_vjp / _jvp)"},
    kSamplePlain{TNCB_ERR_UNSUPPORTED, "tncb_plan_sample takes a plain plan (tncb_plan_create)"},
    kSampleSlPlain{TNCB_ERR_UNSUPPORTED, "tncb_plan_sample_slices takes a plain plan (tncb_plan_create)"},
    kExpectPlain{TNCB_ERR_UNSUPPORTED, "tncb_plan_expect takes a plain or a gradient plan (tncb_plan_create / _vjp)"};
static const Refusal* const kTakes = nullptr;
static const Refusal* const kRoutes[(int)Call::count][7] = {
  //                    plain            vjp             jvp           hvp          sliced vjp      sliced jvp    sliced hvp
  /* stage */           {kTakes,          kTakes,         kTakes,       kTakes,      kTakes,         kTakes,       kTakes},
  /* run */             {kTakes,          kTakes,         &kJvpRuns,    &kHvpRuns,   &kSlVjpRuns,    &kSlJvpRuns,  &kSlHvpRuns},
  /* execute */         {kTakes,          kTakes,         &kJvpRuns,    &kHvpRuns,   &kSlVjpRuns,    &kSlJvpRuns,  &kSlHvpRuns},
  /* stage_slices */    {kTakes,          &kVjpOne,       &kJvpStage,   &kHvpRuns,   &kSlVjpStage,   &kSlJvpRuns,  &kSlHvpRuns},
  /* run_slices */      {kTakes,          &kVjpOne,       &kJvpEither,  &kHvpRuns,   kTakes,         kTakes,       kTakes},
  /* run_batch */       {kTakes,          &kVjpOne,       &kJvpBatch,   &kHvpRuns,   &kSlVjpRuns,    &kSlJvpRuns,  &kSlHvpRuns},
  /* vjp */             {&kNotVjp,        kTakes,         &kJvpRuns,    &kHvpRuns,   &kSlVjpGrads,   &kSlJvpRuns,  &kSlHvpRuns},
  /* vjp_sliced */      {&kNotSlVjp,      &kNotSlVjp,     &kJvpRuns,    &kHvpRuns,   kTakes,         &kSlJvpRuns,  &kSlHvpRuns},
  /* stage_batch */     {&kNotDerivStage, kTakes,         kTakes,       &kHvpRuns,   &kSlVjpNoBatch, &kSlJvpRuns,  &kSlHvpRuns},
  /* vjp_batch */       {&kNotVjp,        kTakes,         &kJvpBatch,   &kHvpRuns,   &kSlVjpNoBatch, &kSlJvpRuns,  &kSlHvpRuns},
  /* jvp */             {&kNotJvp,        &kNotJvp,       kTakes,       &kHvpRuns,   &kNotJvp,       &kSlJvpRuns,  &kSlHvpRuns},
  /* jvp_batch */       {&kNotJvp,        &kNotJvp,       kTakes,       &kHvpRuns,   &kNotJvp,       &kSlJvpRuns,  &kSlHvpRuns},
  /* jvp_sliced */      {&kNotSlJvp,      &kNotSlJvp,     &kNotSlJvp,   &kNotSlJvp,  &kNotSlJvp,     kTakes,       &kNotSlJvp},
  /* hvp */             {&kNotHvp,        &kNotHvp,       &kNotHvp,     kTakes,      &kNotHvp,       &kSlJvpRuns,  &kSlHvpRuns},
  /* hvp_batch */       {&kNotHvp,        &kNotHvp,       &kNotHvp,     kTakes,      &kNotHvp,       &kSlJvpRuns,  &kSlHvpRuns},
  /* hvp_sliced */      {&kNotSlHvp,      &kNotSlHvp,     &kNotSlHvp,   &kNotSlHvp,  &kNotSlHvp,     &kNotSlHvp,   kTakes},
  /* stage_instances */ {kTakes,          kTakes,         kTakes,       &kHvpRuns,   &kSlVjpLeaves,  &kSlJvpRuns,  &kSlHvpRuns},
  /* set_leaves */      {kTakes,          kTakes,         kTakes,       kTakes,      kTakes,         &kSlJvpRuns,  &kSlHvpRuns},
  /* grad_offsets */    {&kNotDeriv,      kTakes,         kTakes,       kTakes,      kTakes,         kTakes,       kTakes},
  /* sample */          {kTakes,          &kSamplePlain,  &kSamplePlain, &kSamplePlain, &kSamplePlain, &kSamplePlain, &kSamplePlain},
  /* sample_slices */   {kTakes,          &kSampleSlPlain, &kSampleSlPlain, &kSampleSlPlain, &kSampleSlPlain, &kSampleSlPlain,
                         &kSampleSlPlain},
  /* expect */          {kTakes,          kTakes,         &kExpectPlain, &kExpectPlain, &kExpectPlain, &kExpectPlain, &kExpectPlain},
};

// TNCB_OK if `c` takes P's kind, else the cell's refusal.  Every plan-taking call asks first, right after its null checks.
static int route(const tncb_plan* P, Call c) {
  const Refusal* r = kRoutes[(int)c][(int)P->kind + (P->sliced ? 3 : 0)];
  return r ? fail(r->status, r->msg) : TNCB_OK;
}

// the item sets of a sliced plan, in their sl_dev order: extract of the leaves with / without a sliced leg, accumulate of
// the adjoints, extract of the leaf tangents, accumulate of the adjoints' tangents
enum { kSlExtract, kSlConst, kSlAcc, kSlTan, kSlDacc, kSliceSets };

static void plan_static_layout(tncb_plan* P, int sm_count, size_t device_bytes) {
  Schedule& S = P->S;
  P->is_static = !S.steps.empty() && (P->grad() || P->tangent() || std::getenv("TNCB_NO_STATIC") == nullptr);
  for (int k : S.leaf_kind) if (k == TNCB_DATA_DEVICE) P->is_static = false;   // addresses change per call
  if (!P->is_static) return;
  // ---- levels: a step's level is 1 + the deepest level among its operands' producers (leaves: 0); backward pairs
  // follow the whole forward pass on their backward level.  A tangent pair reads a tangent of its forward step's operand
  // (on that operand's level) and the other forward operand, so it lands on its forward step's level; a backward-tangent
  // pair carries its backward pair's bw_level ----
  std::vector<int> slot_level(S.slots.size(), 0), step_level(S.steps.size(), 0);
  int n_levels = 0;
  for (size_t q = 0; q < S.steps.size(); q++) {
    const Step& st = S.steps[q];
    if (st.bw_level) continue;
    step_level[q] = std::max(slot_level[st.a], slot_level[st.b]) + 1;
    slot_level[st.out] = step_level[q];
    n_levels = std::max(n_levels, step_level[q]);
  }
  P->n_fwd_levels = n_levels;
  for (size_t q = 0; q < S.steps.size(); q++)
    if (S.steps[q].bw_level) {
      step_level[q] = P->n_fwd_levels + S.steps[q].bw_level;
      slot_level[S.steps[q].out] = step_level[q];
      n_levels = std::max(n_levels, step_level[q]);
    }
  static const bool no_batch = std::getenv("TNCB_NO_BATCH") != nullptr;
  std::vector<size_t> order(S.steps.size());
  for (size_t q = 0; q < order.size(); q++) order[q] = q;
  std::vector<char> batchable(S.steps.size(), 0);
  for (size_t q = 0; q < S.steps.size(); q++) batchable[q] = !no_batch && k0_batch_eligible(sm_count, S.steps[q].plan);
  std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) {
    if (step_level[x] != step_level[y]) return step_level[x] < step_level[y];
    return batchable[x] > batchable[y];                  // batched pairs first inside a level
  });
  std::vector<Step> sorted; sorted.reserve(S.steps.size());
  std::vector<int> lv; std::vector<char> bt;
  for (size_t q : order) { sorted.push_back(std::move(S.steps[q])); lv.push_back(step_level[q]); bt.push_back(batchable[q]); }
  S.steps.swap(sorted);
  // steps [level_begin[l], level_begin[l+1]) form level l (0-based); step_level counts from 1
  P->level_begin.assign(n_levels + 1, 0); P->level_batched.assign(n_levels, 0);
  for (size_t q = 0; q < S.steps.size(); q++) { P->level_begin[lv[q]]++; if (bt[q]) P->level_batched[lv[q] - 1]++; }
  for (int l = 1; l <= n_levels; l++) P->level_begin[l] += P->level_begin[l - 1];
  for (int l = 0; l < n_levels; l++) if (P->level_batched[l] < 2) P->level_batched[l] = 0;   // a batch of one is just a launch
  // ---- layout: outputs of a level are allocated before any operand of that level is released ----
  size_t scratch = 0;
  for (const Step& st : S.steps) if (st.plan.kernel_class == 0) scratch = std::max(scratch, k0_partial_elems(sm_count, st.plan));
  OffsetAlloc A;
  P->leaf_off = A.alloc(std::max<size_t>(S.leaf_block_elems * sizeof(double2), 16));
  P->scratch_elems = scratch;
  P->scratch_off = scratch ? A.alloc(scratch * sizeof(double2)) : 0;
  P->slot_off.assign(S.slots.size(), 0);
  std::vector<size_t> sz(S.slots.size(), 0);
  for (size_t s2 = 0; s2 < S.slots.size(); s2++)
    if (S.slots[s2].leaf_index >= 0) P->slot_off[s2] = P->leaf_off + S.leaf_offset[S.slots[s2].leaf_index] * sizeof(double2);
  // a slot is released after the last level that reads it: for a plain plan that is its consumer's level; a gradient
  // plan keeps each forward operand alive until the backward pair that reads it
  std::vector<int> last_read(S.slots.size(), -1);
  for (int l = 0; l < n_levels; l++)
    for (int q = P->level_begin[l]; q < P->level_begin[l + 1]; q++) last_read[S.steps[q].a] = last_read[S.steps[q].b] = l;
  // a tangent plan: the sums run after the pairs of the level that produced t1 and release the second tangent pair's
  // output; the leaf tangents are written before the first level
  std::vector<int> sum_level(P->tan_sums.size());
  for (size_t k = 0; k < P->tan_sums.size(); k++) {
    sum_level[k] = slot_level[P->tan_sums[k].t1] - 1;
    last_read[P->tan_sums[k].t2] = sum_level[k];
  }
  for (const auto& tl : P->tan_leaves) {
    sz[tl.slot] = std::max<size_t>(S.slots[tl.slot].elems * sizeof(double2), 16);
    P->slot_off[tl.slot] = A.alloc(sz[tl.slot]);
  }
  for (int l = 0; l < n_levels; l++) {
    if (P->grad() && l == P->n_fwd_levels) {       // the seed, written by tncb_plan_vjp before the backward levels
      sz[P->seed_slot] = std::max<size_t>(S.slots[P->seed_slot].elems * sizeof(double2), 16);
      P->slot_off[P->seed_slot] = A.alloc(sz[P->seed_slot]);
      if (P->seed_tan_slot >= 0) {                 // a Hessian-vector plan's seed tangent, written with the seed
        sz[P->seed_tan_slot] = sz[P->seed_slot];
        P->slot_off[P->seed_tan_slot] = A.alloc(sz[P->seed_tan_slot]);
      }
    }
    for (int q = P->level_begin[l]; q < P->level_begin[l + 1]; q++) {
      const Step& st = S.steps[q];
      sz[st.out] = std::max<size_t>(S.slots[st.out].elems * sizeof(double2), 16);
      P->slot_off[st.out] = A.alloc(sz[st.out]);
    }
    for (int q = P->level_begin[l]; q < P->level_begin[l + 1]; q++) {
      const Step& st = S.steps[q];
      for (int s2 : {st.a, st.b}) if (sz[s2] && last_read[s2] == l) { A.free(P->slot_off[s2], sz[s2]); sz[s2] = 0; }
    }
    for (size_t k = 0; k < P->tan_sums.size(); k++) {
      const int t2 = P->tan_sums[k].t2;
      if (sum_level[k] == l && sz[t2]) { A.free(P->slot_off[t2], sz[t2]); sz[t2] = 0; }
    }
  }
  P->ws_bytes = A.top;
  if (P->ws_bytes > static_ws_limit(device_bytes)) { P->is_static = false; return; }
  // ---- batch descriptors ----
  P->item_first.assign(n_levels, 0); P->bs_first.assign(n_levels, 0);
  for (int l = 0; l < n_levels; l++) {
    P->item_first[l] = P->items.size(); P->bs_first[l] = P->block_start.size();
    const int nb = P->level_batched[l];
    if (!nb) continue;
    int blocks = 0;
    for (int q = P->level_begin[l]; q < P->level_begin[l] + nb; q++) {
      const Step& st = S.steps[q];
      K0BatchItem it{};
      const int nblk = k0_batch_fill(sm_count, st.plan, &it);
      it.offA = (long long)P->slot_off[st.a]; it.offB = (long long)P->slot_off[st.b]; it.offC = (long long)P->slot_off[st.out];
      P->items.push_back(it);
      P->block_start.push_back(blocks);
      blocks += nblk;
    }
    P->block_start.push_back(blocks);
  }
  if (P->tangent()) {
    P->sum_first.assign(n_levels, 0); P->sum_count.assign(n_levels, 0); P->sum_bs_first.assign(n_levels, 0);
    for (int l = 0; l < n_levels; l++) {
      P->sum_first[l] = (int)P->sum_items.size(); P->sum_bs_first[l] = P->sum_bs.size();
      long long blocks = 0;
      for (size_t k = 0; k < P->tan_sums.size(); k++) {
        if (sum_level[k] != l) continue;
        const auto& ts = P->tan_sums[k];
        const long long e = (long long)S.slots[ts.t1].elems;
        P->sum_items.push_back({(long long)P->slot_off[ts.t1], (long long)P->slot_off[ts.t2], (long long)P->slot_off[ts.t1], e});
        P->sum_bs.push_back(blocks);
        blocks += (e + kSumThreads - 1) / kSumThreads;
      }
      P->sum_count[l] = (int)P->sum_items.size() - P->sum_first[l];
      if (P->sum_count[l]) P->sum_bs.push_back(blocks);
    }
  }
  P->graphable = !P->grad() && !P->tangent() && std::getenv("TNCB_NO_GRAPH") == nullptr && P->ws_bytes <= ((size_t)1 << 30);   // graphs are for small networks
  for (const Step& st : S.steps) if (st.plan.kernel_class == 1) { P->graphable = false; break; }   // K1/K1' use ctx-owned tables / arena scratch
}

// the payload of one leaf into `dst`
static int stage_leaf(const tncb_tn* lf, std::complex<double>* dst) {
  if (lf->kind == TNCB_DATA_GATE) {
    int cnt = gate_matrix(lf->gate_name, lf->gate_angles, lf->n_gate_angles, lf->gate_adjoint != 0, dst);
    if (cnt < 0) return cnt;
  } else if (lf->kind == TNCB_DATA_MATRIX) {
    uint64_t e = 1; for (int i = 0; i < lf->rank; i++) e *= lf->dims[i];
    std::memcpy(dst, lf->host_re_im, e * sizeof(double2));
  } else if (lf->kind == TNCB_DATA_FILE) {      // into_data for TensorData::File (tensordata.rs:43-49)
    int rc = h5::load_file_leaf(lf->file_path, lf->file_adjoint != 0, lf->rank, lf->dims, (double*)dst);
    if (rc) return rc;
  }
  return TNCB_OK;
}

static int stage_leaves(const Schedule& S, const std::vector<const tncb_tn*>& leaves, std::complex<double>* stage) {
  for (size_t li = 0; li < leaves.size(); li++) {
    if (S.leaf_kind[li] != leaves[li]->kind) return fail(TNCB_ERR_INVALID, "network payload kinds do not match the plan");
    int rc = stage_leaf(leaves[li], stage + S.leaf_offset[li]);
    if (rc) return rc;
  }
  return TNCB_OK;
}

// one descriptor set on the device, once: `items` followed by its block-count prefixes `bs`
template <class Item, class Prefix>
static int upload(tncb_ctx* ctx, const std::vector<Item>& items, const std::vector<Prefix>& bs, void** dev, size_t* bytes) {
  if (*dev || items.empty()) return TNCB_OK;
  const size_t ib = items.size() * sizeof(Item), bb = bs.size() * sizeof(Prefix);
  int rc = ctx->arena.alloc(ib + bb, dev);
  if (rc) return rc;
  *bytes = ib + bb;
  TNCB_CUDA(cudaMemcpyAsync(*dev, items.data(), ib, cudaMemcpyHostToDevice, ctx->stream));
  TNCB_CUDA(cudaMemcpyAsync((char*)*dev + ib, bs.data(), bb, cudaMemcpyHostToDevice, ctx->stream));
  TNCB_CUDA(cudaStreamSynchronize(ctx->stream));   // (pageable sources)
  return TNCB_OK;
}

// workspace, pinned staging and the device copy of the batch descriptors (once per plan and context).  workspace =
// false: the descriptors only (a gradient plan's batched pass runs on workspace copies of its own)
static int plan_device_state(tncb_ctx* ctx, tncb_plan* P, bool workspace = true) {
  if (P->ctx && P->ctx != ctx) return fail(TNCB_ERR_INVALID, "plan belongs to another context");
  if (!P->ctx) { P->ctx = ctx; ctx->plans.push_back(P); }
  int rc;
  if (workspace && !P->ws && (rc = ctx->arena.alloc(P->ws_bytes, &P->ws))) return rc;
  const size_t block_bytes = std::max<size_t>(P->S.leaf_block_elems * sizeof(double2), 16);
  if (workspace && !P->stage) TNCB_CUDA(cudaMallocHost(&P->stage, block_bytes));
  if ((rc = upload(ctx, P->items, P->block_start, &P->batch_dev, &P->batch_bytes)) ||
      (rc = upload(ctx, P->grad_items, P->grad_block_start, &P->grad_dev, &P->grad_dev_bytes)) ||
      (rc = upload(ctx, P->dgrad_items, P->dgrad_block_start, &P->dgrad_dev, &P->dgrad_dev_bytes)) ||
      (rc = upload(ctx, P->sum_items, P->sum_bs, &P->sum_dev, &P->sum_dev_bytes)))
    return rc;
  if (P->sliced && !P->sl_dev) {
    auto up16 = [](size_t b) { return (b + 15) / 16 * 16; };
    const std::vector<SliceItem>* iv[kSliceSets] = {&P->sl_items, &P->const_items, &P->acc_items, &P->tan_items, &P->dacc_items};
    const std::vector<long long>* bv[kSliceSets] = {&P->sl_bs, &P->const_bs, &P->acc_bs, &P->tan_bs, &P->dacc_bs};
    size_t off = 0;
    for (int i = 0; i < kSliceSets; i++) { P->sl_off[i] = off; off = up16(off + iv[i]->size() * sizeof(SliceItem)); }
    for (int i = 0; i < kSliceSets; i++) { P->sl_off[kSliceSets + i] = off; off = up16(off + bv[i]->size() * sizeof(long long)); }
    P->sl_off[2 * kSliceSets] = off; off += sizeof(double2);
    std::vector<char> host(off, 0);
    for (int i = 0; i < kSliceSets; i++) {
      if (!iv[i]->empty()) std::memcpy(host.data() + P->sl_off[i], iv[i]->data(), iv[i]->size() * sizeof(SliceItem));
      if (!bv[i]->empty()) std::memcpy(host.data() + P->sl_off[kSliceSets + i], bv[i]->data(), bv[i]->size() * sizeof(long long));
    }
    const double2 one = {1.0, 0.0};
    std::memcpy(host.data() + P->sl_off[2 * kSliceSets], &one, sizeof(one));
    const size_t bytes = off + P->acc_scratch_elems * sizeof(double2);
    if ((rc = ctx->arena.alloc(bytes, &P->sl_dev))) return rc;
    P->sl_dev_bytes = bytes;
    TNCB_CUDA(cudaMemcpyAsync(P->sl_dev, host.data(), off, cudaMemcpyHostToDevice, ctx->stream));
    TNCB_CUDA(cudaStreamSynchronize(ctx->stream));   // (pageable source)
  }
  return TNCB_OK;
}

// the kernels of levels [l_begin, l_end) on the ctx stream, level by level, on the workspace `ws`.  count > 1: `count`
// instances whose workspaces (each laid out like the plan's) lie `stride` bytes apart run in every launch
static int enqueue_static(tncb_ctx* ctx, tncb_plan* P, char* ws, int count, long long stride, int l_begin, int l_end) {
  const Schedule& S = P->S;
  ctx->partial_override = P->scratch_elems ? (double2*)(ws + P->scratch_off) : nullptr;
  ctx->partial_override_elems = P->scratch_elems;
  int rc = TNCB_OK;
  const K0BatchItem* d_items = (const K0BatchItem*)P->batch_dev;
  const int* d_bs = (const int*)((char*)P->batch_dev + P->items.size() * sizeof(K0BatchItem));
  for (int l = l_begin; l < l_end && !rc; l++) {
    const int nb = P->level_batched[l];
    if (nb) {
      const int total_blocks = P->block_start[P->bs_first[l] + nb];
      rc = launch_k0_batch(ctx, d_items + P->item_first[l], d_bs + P->bs_first[l], nb, total_blocks, ws, count, stride);
    }
    for (int q = P->level_begin[l] + nb; q < P->level_begin[l + 1] && !rc; q++) {
      const Step& st = S.steps[q];
      rc = launch_pair(ctx, st.plan, (const double2*)(ws + P->slot_off[st.a]), (const double2*)(ws + P->slot_off[st.b]),
                       (double2*)(ws + P->slot_off[st.out]), count, stride);
    }
    if (!rc && P->tangent() && P->sum_count[l]) {  // a tangent plan: the level's tangent sums, after its pairs
      const TangentSumItem* d_sum = (const TangentSumItem*)P->sum_dev;
      const long long* d_sbs = (const long long*)((char*)P->sum_dev + P->sum_items.size() * sizeof(TangentSumItem));
      const int ns = P->sum_count[l];
      rc = launch_tangent_sum(ctx, d_sum + P->sum_first[l], d_sbs + P->sum_bs_first[l], ns, P->sum_bs[P->sum_bs_first[l] + ns],
                              ws, count, stride);
    }
  }
  ctx->partial_override = nullptr; ctx->partial_override_elems = 0;
  return rc;
}

// `tn` == nullptr: run on the leaves that tncb_plan_stage left in the workspace
static int execute_static(tncb_ctx* ctx, tncb_plan* P, const tncb_tn* tn, tncb_tensor** out, int* n_out, uint64_t* out_legs) {
  const Schedule& S = P->S;
  TNCB_CUDA(cudaSetDevice(ctx->device));
  int rc;
  std::vector<const tncb_tn*> leaves;
  if (tn) {
    collect_leaf_nodes(tn, leaves);
    if ((rc = validate_leaves(S, leaves))) return rc;
  } else if (!P->leaves_resident) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan");
  if ((rc = plan_device_state(ctx, P))) return rc;
  P->fwd_ready = false;
  const size_t block_bytes = std::max<size_t>(S.leaf_block_elems * sizeof(double2), 16);
  char* ws = (char*)P->ws;
  const int which = tn ? 0 : 1;
  if (tn) {
    // an earlier upload may still read the staging buffer (it waits behind the previous network's kernels on the stream)
    if (P->exec[0] || P->leaves_resident) TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
    else if (P->stage_busy) TNCB_CUDA(cudaEventSynchronize(P->stage_ev));
    if ((rc = stage_leaves(S, leaves, (std::complex<double>*)P->stage))) return rc;
    P->leaves_resident = false;     // the workspace copy is about to be overwritten with this call's payloads
  }
  if (P->graphable) {
    if (!P->exec[which]) {
      cudaGraph_t graph = nullptr;
      const uint64_t launches_before = ctx->launches;
      uint64_t ec_before[8]; for (int i = 0; i < 8; i++) ec_before[i] = ctx->engine_count[i];
      TNCB_CUDA(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
      if (tn) cudaMemcpyAsync(ws + P->leaf_off, P->stage, block_bytes, cudaMemcpyHostToDevice, ctx->stream);
      rc = enqueue_static(ctx, P, ws, 1, 0, 0, P->n_fwd_levels);
      cudaError_t ce = cudaStreamEndCapture(ctx->stream, &graph);
      P->kernels_per_run = ctx->launches - launches_before;
      ctx->launches = launches_before;
      for (int i = 0; i < 8; i++) ctx->engine_count[i] = ec_before[i];
      if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
      if (ce != cudaSuccess) { P->graphable = false; return fail(TNCB_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(ce)); }
      ce = cudaGraphInstantiate(&P->exec[which], graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) {   // the plan runs eagerly from now on
        P->exec[which] = nullptr; P->graphable = false;
        return fail(TNCB_ERR_CUDA, std::string("graph instantiate: ") + cudaGetErrorString(ce));
      }
    }
    TNCB_CUDA(cudaGraphLaunch(P->exec[which], ctx->stream));
    ctx->launches += P->kernels_per_run;
    ctx->engine_count[0] += S.steps.size();   // (graphable plans hold K0 / K2 pairs only; counted as tiny pairs)
  } else {
    if (tn) {
      TNCB_CUDA(cudaMemcpyAsync(ws + P->leaf_off, P->stage, block_bytes, cudaMemcpyHostToDevice, ctx->stream));
      if (!P->stage_ev) TNCB_CUDA(cudaEventCreateWithFlags(&P->stage_ev, cudaEventDisableTiming));
      TNCB_CUDA(cudaEventRecord(P->stage_ev, ctx->stream));
      P->stage_busy = true;
    }
    if ((rc = enqueue_static(ctx, P, ws, 1, 0, 0, P->n_fwd_levels))) return rc;
  }
  P->fwd_ready = P->grad();    // the forward operands the backward levels read are in the workspace now
  tncb_tensor* result = nullptr;
  if (S.result_slot >= 0) {
    const SlotMeta& rm = S.slots[S.result_slot];
    if ((rc = tensor_new(ctx, (int)rm.dims.size(), rm.dims.data(), &result))) return rc;
    TNCB_CUDA(cudaMemcpyAsync(result->ptr, ws + P->slot_off[S.result_slot], rm.elems * sizeof(double2), cudaMemcpyDeviceToDevice, ctx->stream));
  }
  if (out) *out = result; else if (result) tncb_tensor_free(ctx, result);
  if (n_out) *n_out = S.result_slot >= 0 ? (int)S.slots[S.result_slot].legs.size() : 0;
  if (out_legs && S.result_slot >= 0)
    for (size_t i = 0; i < S.slots[S.result_slot].legs.size(); i++) out_legs[i] = S.slots[S.result_slot].legs[i];
  return TNCB_OK;
}

// Appends the backward pairs of a gradient plan to its forward schedule.  For C = contract(A, B) with seed-weighted
// adjoint C̄, the adjoints are Ā = contract(C̄, B) and B̄ = contract(C̄, A): plain pairwise contractions of the forward
// pair's M·N·K volume, planned like any other pair.  An operand gets its pair only if its subtree holds a requested
// leaf.  build() consumes every slot exactly once, so the contraction is a tree, every adjoint is produced exactly once
// and nothing is accumulated.  leaf_adj[l] = the slot holding leaf l's adjoint (in its pair's output leg order), -1 if
// not requested.  The forward steps are S.steps[0, n_fwd): a Hessian-vector plan has appended its tangent pairs after them.
static int build_backward(tncb_plan* P, const uint8_t* wrt, std::vector<int>& leaf_adj, size_t n_fwd) {
  Schedule& S = P->S;
  const size_t nl = S.n_leaves_total;
  if (S.steps.empty() || S.result_slot < 0) return fail(TNCB_ERR_UNSUPPORTED, "a gradient plan needs a network with at least one pair");
  std::vector<int> leaf_slot(nl, -1);
  for (size_t s = 0; s < S.slots.size(); s++) if (S.slots[s].leaf_index >= 0) leaf_slot[S.slots[s].leaf_index] = (int)s;
  std::vector<char> want(S.slots.size(), 0);        // the slot's subtree holds a requested leaf
  bool any = false;
  for (size_t li = 0; li < nl; li++) {
    if (wrt ? !wrt[li] : leaf_slot[li] < 0) continue;
    if (leaf_slot[li] < 0) return fail(TNCB_ERR_INVALID, "leaf " + std::to_string(li) + " has no payload to differentiate");
    want[leaf_slot[li]] = 1; any = true;
  }
  if (!any) return fail(TNCB_ERR_INVALID, "wrt selects no leaf");
  std::vector<int> consumer(S.slots.size(), -1);
  for (size_t q = 0; q < n_fwd; q++) {
    const Step& st = S.steps[q];
    want[st.out] = want[st.a] || want[st.b];
    consumer[st.a] = consumer[st.b] = (int)q;
  }
  {
    SlotMeta seed;
    seed.legs = S.slots[S.result_slot].legs; seed.dims = S.slots[S.result_slot].dims; seed.elems = S.slots[S.result_slot].elems;
    S.slots.push_back(std::move(seed));
    P->seed_slot = (int)S.slots.size() - 1;
  }
  std::vector<int> adj(S.slots.size(), -1), bw_level(n_fwd, 0);
  adj[S.result_slot] = P->seed_slot;
  for (size_t q = n_fwd; q-- > 0;) {               // consumers come after their producers: walk the tree from the root
    const int a = S.steps[q].a, b = S.steps[q].b, out = S.steps[q].out;
    if (!want[out]) continue;
    bw_level[q] = out == S.result_slot ? 1 : bw_level[consumer[out]] + 1;
    for (int x : {a, b}) {
      if (!want[x]) continue;
      const int other = x == a ? b : a;
      Step bs; bs.a = adj[out]; bs.b = other; bs.bw_level = bw_level[q];
      const SlotMeta& g = S.slots[bs.a];
      const SlotMeta& o = S.slots[other];
      int rc = plan_pair((int)g.legs.size(), g.legs.data(), g.dims.data(), (int)o.legs.size(), o.legs.data(), o.dims.data(), bs.plan);
      if (rc) return rc;
      std::vector<uint64_t> got = bs.plan.out_legs, exp = S.slots[x].legs;
      std::sort(got.begin(), got.end()); std::sort(exp.begin(), exp.end());
      if (got != exp) return fail(TNCB_ERR_UNSUPPORTED, "gradient plans need every leg to join at most two tensors");
      SlotMeta m; m.legs = bs.plan.out_legs; m.dims = bs.plan.out_dims;
      for (uint64_t d : m.dims) m.elems *= d;
      S.slots.push_back(std::move(m));
      bs.out = (int)S.slots.size() - 1;
      adj[x] = bs.out;
      S.flops += bs.plan.flops(); S.bytes += bs.plan.bytes();
      S.steps.push_back(std::move(bs));
    }
  }
  leaf_adj.assign(nl, -1);
  P->grad_offset.assign(nl, -1);
  P->grad_elems = 0;
  for (size_t li = 0; li < nl; li++)
    if (leaf_slot[li] >= 0 && want[leaf_slot[li]]) {
      leaf_adj[li] = adj[leaf_slot[li]];
      P->grad_offset[li] = (int64_t)P->grad_elems;
      P->grad_elems += S.slots[leaf_slot[li]].elems;
    }
  return TNCB_OK;
}

// The gather items of the leaf adjoints (after the layout fixed their slots): fused leg groups in the leaf's order with
// the adjoint slot's strides.  A leaf that needs more groups than a GradItem holds goes through launch_permute (K3).
// items / block_start / permutes: the plan's grad_* set, or a Hessian-vector plan's dgrad_* set for the adjoints' tangents.
static int build_gather(tncb_plan* P, const std::vector<int>& leaf_adj, std::vector<GradItem>& items,
                        std::vector<long long>& block_start, std::vector<tncb_plan::GradPermute>& permutes) {
  const Schedule& S = P->S;
  long long blocks = 0;
  for (const SlotMeta& leaf : S.slots) {
    if (leaf.leaf_index < 0 || leaf_adj[leaf.leaf_index] < 0 || leaf.elems == 0) continue;
    const int gs = leaf_adj[leaf.leaf_index];
    const SlotMeta& g = S.slots[gs];
    const int r = (int)leaf.legs.size();
    std::vector<long long> gst(r);
    { long long s = 1; for (int j = r - 1; j >= 0; j--) { gst[j] = s; s *= (long long)g.dims[j]; } }
    std::vector<int> perm(r);
    for (int i = 0; i < r; i++) perm[i] = (int)(std::find(g.legs.begin(), g.legs.end(), leaf.legs[i]) - g.legs.begin());
    GradItem it{};
    it.src = (long long)P->slot_off[gs]; it.dst = P->grad_offset[leaf.leaf_index]; it.elems = (long long)leaf.elems;
    bool fits = true;
    for (int i = 0; i < r && fits; i++) {
      const long long d = (long long)leaf.dims[i], st = gst[perm[i]];
      if (d == 1) continue;
      if (it.n > 0 && it.st[it.n - 1] == st * d) { it.dim[it.n - 1] *= d; it.st[it.n - 1] = st; continue; }
      if (it.n == kGradGroups) { fits = false; break; }
      it.dim[it.n] = d; it.st[it.n] = st; it.n++;
    }
    if (!fits) { permutes.push_back({gs, it.dst, perm}); continue; }
    for (int k = it.n; k < kGradGroups; k++) { it.dim[k] = 1; it.st[k] = 0; }
    items.push_back(it);
    block_start.push_back(blocks);
    blocks += (it.elems + kGradThreads - 1) / kGradThreads;
  }
  block_start.push_back(blocks);
  if (blocks > 0x7fffffffLL) return fail(TNCB_ERR_UNSUPPORTED, "leaf gradients too large for one gather launch");
  return TNCB_OK;
}

// Appends the tangent pairs of a tangent plan to its forward schedule.  For C = contract(A, B) the tangent is
// Ċ = contract(Ȧ, B) + contract(A, Ḃ); each term has the forward pair's legs, shapes and GEMM view, so it takes the
// forward step's PairPlan unchanged.  A slot has a tangent only if its subtree holds a requested leaf; a step with one
// such operand gets one tangent pair, a step with two gets two and a sum (t1 += t2, always in that order).  The requested
// leaves' tangents get slots of their own (written from the caller's tangent row before the first level), packed in a
// row at grad_offset like a gradient plan's gradients.  tan_of (optional): the tangent slot of every forward slot, -1 =
// zero tangent.
static int build_tangent(tncb_plan* P, const uint8_t* wrt, std::vector<int>* tan_of = nullptr) {
  Schedule& S = P->S;
  const size_t nl = S.n_leaves_total;
  if (S.steps.empty() || S.result_slot < 0) return fail(TNCB_ERR_UNSUPPORTED, "a tangent plan needs a network with at least one pair");
  std::vector<int> leaf_slot(nl, -1);
  for (size_t s = 0; s < S.slots.size(); s++) if (S.slots[s].leaf_index >= 0) leaf_slot[S.slots[s].leaf_index] = (int)s;
  const size_t n_slots = S.slots.size();
  std::vector<int> tan(n_slots, -1);                // the tangent slot of a forward slot, -1 = zero tangent
  P->grad_offset.assign(nl, -1);
  P->grad_elems = 0;
  bool any = false;
  for (size_t li = 0; li < nl; li++) {
    if (wrt ? !wrt[li] : leaf_slot[li] < 0) continue;
    if (leaf_slot[li] < 0) return fail(TNCB_ERR_INVALID, "leaf " + std::to_string(li) + " has no payload to differentiate");
    any = true;
  }
  if (!any) return fail(TNCB_ERR_INVALID, "wrt selects no leaf");
  for (size_t li = 0; li < nl; li++) {
    if (leaf_slot[li] < 0 || (wrt && !wrt[li])) continue;
    SlotMeta m;
    const SlotMeta& leaf = S.slots[leaf_slot[li]];
    m.legs = leaf.legs; m.dims = leaf.dims; m.elems = leaf.elems;
    S.slots.push_back(std::move(m));
    tan[leaf_slot[li]] = (int)S.slots.size() - 1;
    P->grad_offset[li] = (int64_t)P->grad_elems;
    P->tan_leaves.push_back({tan[leaf_slot[li]], (int64_t)P->grad_elems});
    P->grad_elems += S.slots[tan[leaf_slot[li]]].elems;
  }
  const size_t n_fwd = S.steps.size();
  for (size_t q = 0; q < n_fwd; q++) {             // producers come before their consumers
    const int a = S.steps[q].a, b = S.steps[q].b, out = S.steps[q].out;
    int first = -1;
    for (int x : {a, b}) {
      if (tan[x] < 0) continue;
      Step ts; ts.a = x == a ? tan[a] : a; ts.b = x == b ? tan[b] : b;
      ts.plan = S.steps[q].plan;
      SlotMeta m; m.legs = S.slots[out].legs; m.dims = S.slots[out].dims; m.elems = S.slots[out].elems;
      S.slots.push_back(std::move(m));
      ts.out = (int)S.slots.size() - 1;
      S.flops += ts.plan.flops(); S.bytes += ts.plan.bytes();
      S.steps.push_back(std::move(ts));
      if (first < 0) first = S.steps.back().out;
      else P->tan_sums.push_back({first, S.steps.back().out});
    }
    tan[out] = first;
  }
  P->tan_result = tan[S.result_slot];
  if (P->tan_result < 0) return fail(TNCB_ERR_INVALID, "no requested leaf reaches the result");
  if (tan_of) tan_of->swap(tan);
  return TNCB_OK;
}

// Appends the backward-tangent pairs of a Hessian-vector plan: the forward derivative of every backward pair
// x̄ = contract(C̄, O) (S.steps[b0, end), appended by build_backward) in the direction of the leaf tangents and the seed
// tangent, dx̄ = contract(dC̄, O) + contract(C̄, dO).  Each term has the backward pair's legs and GEMM view, so it takes
// the backward pair's PairPlan and bw_level; with both terms a sum follows (first term += second term, in that order).
// The seed tangent always has a slot, so every adjoint gets a tangent.  tan: the forward slots' tangents
// (build_tangent); leaf_dadj[l] = the slot holding the tangent of leaf l's adjoint, -1 if not requested.
static int build_backward_tangent(tncb_plan* P, size_t b0, const std::vector<int>& tan, const std::vector<int>& leaf_adj,
                                  std::vector<int>& leaf_dadj) {
  Schedule& S = P->S;
  {
    const SlotMeta& seed = S.slots[P->seed_slot];
    SlotMeta m; m.legs = seed.legs; m.dims = seed.dims; m.elems = seed.elems;
    S.slots.push_back(std::move(m));
    P->seed_tan_slot = (int)S.slots.size() - 1;
  }
  std::vector<int> dadj(S.slots.size(), -1);        // the tangent slot of an adjoint slot
  dadj[P->seed_slot] = P->seed_tan_slot;
  const size_t b1 = S.steps.size();
  for (size_t q = b0; q < b1; q++) {               // a consumer's adjoint is produced before its operands' adjoints
    const Step bs = S.steps[q];                    // (a copy: push_back below may move the steps)
    int first = -1;
    for (int side = 0; side < 2; side++) {
      const int a = side == 0 ? dadj[bs.a] : bs.a;
      const int b = side == 0 ? bs.b : (bs.b < (int)tan.size() ? tan[bs.b] : -1);
      if (a < 0 || b < 0) continue;
      Step ts; ts.a = a; ts.b = b; ts.plan = bs.plan; ts.bw_level = bs.bw_level;
      const SlotMeta& o = S.slots[bs.out];
      SlotMeta m; m.legs = o.legs; m.dims = o.dims; m.elems = o.elems;
      S.slots.push_back(std::move(m));
      ts.out = (int)S.slots.size() - 1;
      S.flops += ts.plan.flops(); S.bytes += ts.plan.bytes();
      S.steps.push_back(std::move(ts));
      if (first < 0) first = S.steps.back().out;
      else P->tan_sums.push_back({first, S.steps.back().out});
    }
    dadj[bs.out] = first;
  }
  leaf_dadj.assign(leaf_adj.size(), -1);
  for (size_t li = 0; li < leaf_adj.size(); li++)
    if (leaf_adj[li] >= 0) leaf_dadj[li] = dadj[leaf_adj[li]];
  return TNCB_OK;
}

// ---- sliced gradient plans ----
// `tn` with the sliced legs dropped from every leaf: the structure every slice shares.  A leaf may lose all its legs.
// Payload leaves become MATRIX stand-ins (the schedule reads no payload, and a gate's table would not match its sliced
// dims); the full leaves are validated and staged through the plan's `full` schedule instead.
struct SliceTree { std::vector<std::unique_ptr<tncb_tn[]>> nodes; std::vector<std::unique_ptr<uint64_t[]>> arrs; };
static void slice_tree(const tncb_tn* src, tncb_tn* dst, const std::vector<uint64_t>& sl, SliceTree& keep) {
  static const double stand_in[2] = {0.0, 0.0};
  *dst = *src;
  if (src->n_children) {
    keep.nodes.emplace_back(new tncb_tn[src->n_children]);
    tncb_tn* ch = keep.nodes.back().get();
    for (size_t i = 0; i < src->n_children; i++) slice_tree(&src->children[i], &ch[i], sl, keep);
    dst->children = ch;
    return;
  }
  if (src->kind == TNCB_DATA_UNCONTRACTED) return;
  if (src->rank > 0 && src->rank <= kMaxLegs && src->legs && src->dims) {
    keep.arrs.emplace_back(new uint64_t[2 * src->rank]);
    uint64_t* a = keep.arrs.back().get();
    int r = 0;
    for (int i = 0; i < src->rank; i++)
      if (std::find(sl.begin(), sl.end(), src->legs[i]) == sl.end()) { a[r] = src->legs[i]; a[src->rank + r] = src->dims[i]; r++; }
    dst->rank = r; dst->legs = a; dst->dims = a + src->rank;
  }
  dst->kind = TNCB_DATA_MATRIX; dst->host_re_im = stand_in;
  dst->gate_name = nullptr; dst->gate_angles = nullptr; dst->n_gate_angles = 0; dst->gate_adjoint = 0;
  dst->device = nullptr; dst->file_path = nullptr; dst->file_adjoint = 0;
}

// fuses neighbouring groups that are contiguous on both sides; false if more than kSliceGroups remain
static bool fuse_slice_groups(SliceItem& it, const std::vector<long long>& d, const std::vector<long long>& st, const std::vector<long long>& fst) {
  it.n = 0;
  for (size_t i = 0; i < d.size(); i++) {
    if (d[i] == 1) continue;
    if (it.n > 0 && it.st[it.n - 1] == st[i] * d[i] && it.fst[it.n - 1] == fst[i] * d[i]) {
      it.dim[it.n - 1] *= d[i]; it.st[it.n - 1] = st[i]; it.fst[it.n - 1] = fst[i]; continue;
    }
    if (it.n == kSliceGroups) return false;
    it.dim[it.n] = d[i]; it.st[it.n] = st[i]; it.fst[it.n] = fst[i]; it.n++;
  }
  for (int k = it.n; k < kSliceGroups; k++) { it.dim[k] = 1; it.st[k] = 0; it.fst[k] = 0; }
  return true;
}

static void push_item(std::vector<SliceItem>& items, std::vector<long long>& bs, const SliceItem& it) {
  if (bs.empty()) bs.push_back(0);
  items.push_back(it);
  bs.push_back(bs.back() + (it.elems + kGradThreads - 1) / kGradThreads);
}

// The full leaves (P->full), the gradient offsets in full-leaf shapes, the extract items (after the layout fixed the leaf
// slots) and the accumulate items of the leaf adjoints.  An accumulate item whose adjoint order needs more groups than an
// item holds reads a K3-permuted copy of the adjoint (slice-leaf order) from the plan's permute scratch instead.  A
// tangent plan (leaf_adj empty) also gets the extract items of the requested leaves' tangents (full-shape tangent block
// at the gradient offsets -> the tangent slots); a Hessian-vector plan also gets the accumulate items of the adjoints'
// tangents (leaf_dadj), their K3 copies after the adjoints' in the same scratch.
static int build_slice_items(tncb_plan* P, const std::vector<const tncb_tn*>& lv, const std::vector<uint64_t>& sl,
                             const std::vector<uint64_t>& sdim, const std::vector<int>& leaf_adj,
                             const std::vector<int>& leaf_dadj = {}) {
  const Schedule& S = P->S;
  Schedule& F = P->full;
  const size_t nl = S.n_leaves_total;
  std::vector<int> sslot(nl, -1), fslot(nl, -1), leaf_tan(nl, -1);
  for (size_t s = 0; s < S.slots.size(); s++) if (S.slots[s].leaf_index >= 0) sslot[S.slots[s].leaf_index] = (int)s;
  if (P->tangent()) {                              // build_tangent: tan_leaves in leaf order, one per offset >= 0
    size_t k = 0;
    for (size_t li = 0; li < nl; li++) if (P->grad_offset[li] >= 0) leaf_tan[li] = P->tan_leaves[k++].slot;
  }
  auto wanted = [&](size_t li) { return leaf_adj.empty() ? leaf_tan[li] >= 0 : leaf_adj[li] >= 0; };
  F.n_leaves_total = nl;
  F.leaf_offset.assign(nl, 0);
  F.leaf_kind.assign(nl, TNCB_DATA_UNCONTRACTED);
  for (size_t li = 0; li < nl; li++) {             // collect order, as build() adds them
    if (sslot[li] < 0) continue;
    int rc = add_leaf(lv[li], F, li, &fslot[li]);
    if (rc) return rc;
  }
  const size_t ns = sl.size();
  std::vector<unsigned long long> div(ns);
  { unsigned long long d = 1; for (size_t k = ns; k-- > 0;) { div[k] = d; d *= sdim[k]; } }   // last leg fastest
  P->grad_offset.assign(nl, -1);
  P->grad_elems = 0;
  for (size_t li = 0; li < nl; li++)
    if (wanted(li)) { P->grad_offset[li] = (int64_t)P->grad_elems; P->grad_elems += F.slots[fslot[li]].elems; }
  size_t scratch = 0;
  for (size_t li = 0; li < nl; li++) {
    if (sslot[li] < 0) continue;
    const SlotMeta& sm = S.slots[sslot[li]];
    const SlotMeta& fm = F.slots[fslot[li]];
    if (sm.elems == 0) continue;
    const int fr = (int)fm.legs.size();
    std::vector<long long> fstr(fr);
    { long long s = 1; for (int j = fr - 1; j >= 0; j--) { fstr[j] = s; s *= (long long)fm.dims[j]; } }
    SliceItem it{};
    std::vector<long long> d, fst;                  // the kept legs, in the leaf's order = the slice leaf's legs
    for (int j = 0; j < fr; j++) {
      const size_t k = std::find(sl.begin(), sl.end(), fm.legs[j]) - sl.begin();
      if (k == ns) { d.push_back((long long)fm.dims[j]); fst.push_back(fstr[j]); continue; }
      if (it.ns == kSliceLegs) return fail(TNCB_ERR_UNSUPPORTED, "leaf " + std::to_string(li) + " carries more than " + std::to_string(kSliceLegs) + " sliced legs");
      it.sdiv[it.ns] = div[k]; it.sdim[it.ns] = sdim[k]; it.sst[it.ns] = fstr[j]; it.ns++;
    }
    std::vector<long long> rm(d.size());
    { long long s = 1; for (size_t j = d.size(); j-- > 0;) { rm[j] = s; s *= d[j]; } }
    it.elems = (long long)sm.elems;
    // extract: full leaf block -> the leaf's slot in the workspace (row-major slice leaf)
    SliceItem ex = it;
    ex.slot = (long long)P->slot_off[sslot[li]]; ex.full = (long long)F.leaf_offset[li];
    if (!fuse_slice_groups(ex, d, rm, fst))
      return fail(TNCB_ERR_UNSUPPORTED, "leaf " + std::to_string(li) + " needs more than " + std::to_string(kSliceGroups) + " leg groups to address its slices");
    if (ex.ns) push_item(P->sl_items, P->sl_bs, ex); else push_item(P->const_items, P->const_bs, ex);
    if (!wanted(li)) continue;
    if (leaf_tan[li] >= 0) {                         // the leaf's tangent: caller's full-shape block -> its tangent slot
      SliceItem tx = ex;
      tx.slot = (long long)P->slot_off[leaf_tan[li]]; tx.full = (long long)P->grad_offset[li];
      push_item(P->tan_items, P->tan_bs, tx);
    }
    if (leaf_adj.empty()) continue;
    // accumulate: the adjoint slot (pair output order) -> q's sub-block of the full-shape gradient; the same for the
    // adjoint's tangent, which has the adjoint's legs
    auto accumulate = [&](int gs, std::vector<SliceItem>& items, std::vector<long long>& bs,
                          std::vector<tncb_plan::GradPermute>& permutes) {
      const SlotMeta& g = S.slots[gs];
      std::vector<long long> gst(g.legs.size());
      { long long s = 1; for (size_t j = g.legs.size(); j-- > 0;) { gst[j] = s; s *= (long long)g.dims[j]; } }
      std::vector<int> perm(sm.legs.size());
      std::vector<long long> ast(sm.legs.size());
      for (size_t i = 0; i < sm.legs.size(); i++) {
        perm[i] = (int)(std::find(g.legs.begin(), g.legs.end(), sm.legs[i]) - g.legs.begin());
        ast[i] = gst[perm[i]];
      }
      SliceItem ac = it;
      ac.full = (long long)P->grad_offset[li];
      ac.slot = (long long)P->slot_off[gs];
      if (!fuse_slice_groups(ac, d, ast, fst)) {     // many groups: K3 into the scratch, then the same kernel
        ac.from_scratch = 1; ac.slot = (long long)scratch;
        fuse_slice_groups(ac, d, rm, fst);          // (the extract item fitted with the same groups)
        permutes.push_back({gs, (int64_t)scratch, perm});
        scratch += sm.elems;
      }
      push_item(items, bs, ac);
    };
    accumulate(leaf_adj[li], P->acc_items, P->acc_bs, P->grad_permutes);
    if (!leaf_dadj.empty()) accumulate(leaf_dadj[li], P->dacc_items, P->dacc_bs, P->dgrad_permutes);
  }
  P->acc_scratch_elems = scratch;
  for (const auto* bs : {&P->sl_bs, &P->const_bs, &P->acc_bs, &P->tan_bs, &P->dacc_bs})
    if (!bs->empty() && bs->back() > 0x7fffffffLL) return fail(TNCB_ERR_UNSUPPORTED, "slice leaves too large for one launch");
  return TNCB_OK;
}

// Per slice q of [first, n_sl) step stride: extract, forward levels, value accumulation and, with `grad`, the seed copy,
// backward levels, K3 of the many-group adjoints and the accumulation into the full-shape gradient (zeroed here).  The
// leaves without a sliced leg are the same in every slice: they are copied once per call (the leaf block is never
// released by the layout, so they stay in place across slices).
// A sliced tangent / Hessian-vector plan also extracts slice q's sub-block of every requested leaf's tangent (tangents:
// the caller's full-shape block) before the forward levels, adds the result's tangent into tan_value, writes the seed
// tangent with the seed (NULL: zero) and accumulates the adjoints' tangents into dgrad after the adjoints.  The tangent
// slots are released by the layout after their last read, so every tangent is extracted per slice.  Any output may be
// NULL; the backward levels run only if grad or dgrad is wanted.
struct SliceRun {
  const double2 *seed = nullptr, *seed_tan = nullptr, *tangents = nullptr;
  double2 *value = nullptr, *tan_value = nullptr, *grad = nullptr, *dgrad = nullptr;
};
static int run_sliced(tncb_ctx* ctx, tncb_plan* P, size_t first, size_t stride, const SliceRun& io) {
  const Schedule& S = P->S;
  char* ws = (char*)P->ws;
  char* dev = (char*)P->sl_dev;
  const SlotMeta& rm = S.slots[S.result_slot];
  const size_t vbytes = std::max<size_t>(rm.elems, 1) * sizeof(double2), rbytes = rm.elems * sizeof(double2);
  auto items = [&](int i) { return (const SliceItem*)(dev + P->sl_off[i]); };
  auto bs = [&](int i) { return (const long long*)(dev + P->sl_off[kSliceSets + i]); };
  const double2* one = (const double2*)(dev + P->sl_off[2 * kSliceSets]);
  double2* scratch = (double2*)(dev + P->sl_off[2 * kSliceSets] + sizeof(double2));
  const double2* full = (const double2*)P->full_dev;
  const size_t gbytes = std::max<uint64_t>(P->grad_elems, 1) * sizeof(double2);
  P->fwd_ready = false;
  for (double2* g : {io.grad, io.dgrad}) if (g) TNCB_CUDA(cudaMemsetAsync(g, 0, gbytes, ctx->stream));
  if (first >= P->n_sl) {                          // more ranks than slices
    for (double2* v : {io.value, io.tan_value}) if (v) TNCB_CUDA(cudaMemsetAsync(v, 0, vbytes, ctx->stream));
    return TNCB_OK;
  }
  const bool backward = io.grad || io.dgrad;
  auto accumulate = [&](const std::vector<tncb_plan::GradPermute>& permutes) {
    int rc = TNCB_OK;
    for (size_t i = 0; i < permutes.size() && !rc; i++) {
      const auto& gp = permutes[i];
      const SlotMeta& sm = S.slots[gp.slot];
      rc = launch_permute(ctx, (const double2*)(ws + P->slot_off[gp.slot]), scratch + gp.dst, (int)sm.dims.size(), sm.dims.data(), gp.perm.data());
    }
    return rc;
  };
  int rc = launch_slice_extract(ctx, items(kSlConst), bs(kSlConst), (int)P->const_items.size(), P->const_items.empty() ? 0 : P->const_bs.back(), full, ws, 0);
  for (size_t q = first; q < P->n_sl && !rc; q += stride) {
    if (!P->sl_items.empty() && (rc = launch_slice_extract(ctx, items(kSlExtract), bs(kSlExtract), (int)P->sl_items.size(), P->sl_bs.back(), full, ws, q))) break;
    if (!P->tan_items.empty() &&
        (rc = launch_slice_extract(ctx, items(kSlTan), bs(kSlTan), (int)P->tan_items.size(), P->tan_bs.back(), io.tangents, ws, q))) break;
    if ((rc = enqueue_static(ctx, P, ws, 1, 0, 0, P->n_fwd_levels))) break;
    for (auto [sum, slot] : {std::pair<double2*, int>{io.value, S.result_slot}, {io.tan_value, P->tan_result}}) {
      if (!sum || rc) continue;
      const double2* r = (const double2*)(ws + P->slot_off[slot]);
      if (q != first) rc = launch_add(ctx, sum, r, rm.elems);
      else if (cudaMemcpyAsync(sum, r, rbytes, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess)
        rc = fail(TNCB_ERR_CUDA, "result copy failed");
    }
    if (rc || !backward) continue;
    // the seed slots may reuse memory the forward levels freed: written after them, on the stream
    TNCB_CUDA(cudaMemcpyAsync(ws + P->slot_off[P->seed_slot], io.seed ? io.seed : one, rbytes, cudaMemcpyDeviceToDevice, ctx->stream));
    if (P->seed_tan_slot >= 0) {
      char* ds = ws + P->slot_off[P->seed_tan_slot];
      TNCB_CUDA(io.seed_tan ? cudaMemcpyAsync(ds, io.seed_tan, rbytes, cudaMemcpyDeviceToDevice, ctx->stream)
                            : cudaMemsetAsync(ds, 0, rbytes, ctx->stream));
    }
    if ((rc = enqueue_static(ctx, P, ws, 1, 0, P->n_fwd_levels, (int)P->level_batched.size()))) break;
    if ((io.grad && (rc = accumulate(P->grad_permutes))) || (io.dgrad && (rc = accumulate(P->dgrad_permutes)))) break;
    if (io.grad && !P->acc_items.empty())
      rc = launch_grad_accumulate(ctx, items(kSlAcc), bs(kSlAcc), (int)P->acc_items.size(), P->acc_bs.back(), ws, scratch, io.grad, q);
    if (!rc && io.dgrad && !P->dacc_items.empty())
      rc = launch_grad_accumulate(ctx, items(kSlDacc), bs(kSlDacc), (int)P->dacc_items.size(), P->dacc_bs.back(), ws, scratch, io.dgrad, q);
  }
  return rc;
}

// ---- many networks of one structure (tncb_plan_stage_slices / tncb_plan_stage_batch, tncb_plan_run_batch /
// tncb_plan_vjp_batch) ----
// Validates and materialises the leaves of n networks of the plan's structure, then uploads them in one H2D copy into
// slices_dev: n leaf blocks back to back.  workspace = false: the plan's own workspace is not needed (gradient plans).
static int stage_networks(tncb_ctx* ctx, tncb_plan* P, size_t n, const tncb_tn* const* tns, bool workspace) {
  const Schedule& S = P->S;
  TNCB_CUDA(cudaSetDevice(ctx->device));
  int rc;
  if ((rc = plan_device_state(ctx, P, workspace))) return rc;
  const size_t block = std::max<size_t>(S.leaf_block_elems, 1);
  std::vector<std::complex<double>> host(block * n);
  for (size_t q = 0; q < n; q++) {
    if (!tns[q]) return fail(TNCB_ERR_INVALID, "slice network is null");
    std::vector<const tncb_tn*> leaves;
    collect_leaf_nodes(tns[q], leaves);
    if ((rc = validate_leaves(S, leaves))) return rc;
    if ((rc = stage_leaves(S, leaves, host.data() + q * block))) return rc;
  }
  TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
  if (P->slices_dev) { ctx->arena.free(P->slices_dev, P->slices_bytes); P->slices_dev = nullptr; }
  P->slices_bytes = host.size() * sizeof(double2);
  if ((rc = ctx->arena.alloc(P->slices_bytes, &P->slices_dev))) return rc;
  TNCB_CUDA(cudaMemcpyAsync(P->slices_dev, host.data(), P->slices_bytes, cudaMemcpyHostToDevice, ctx->stream));
  TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
  P->n_slices = n;
  return TNCB_OK;
}

// A batched pass runs c instances on c copies of the plan's workspace, ws_bytes apart (a multiple of 256: every instance
// base stays aligned) in one arena block that lives for one call.
struct BatchBlock {
  size_t ws = 0, c = 0;         // bytes per copy, copies per pass
  bool strided = true;          // the copies fit the device's largest copy pitch (2 GiB): one 2D copy per pass
  bool no_room = false;         // batch_size refused because the device had no room for one copy
  void* blk = nullptr;
};

// c = min(count, static-workspace limit / ws, 65535 (grid.y / grid.z limit), what the device can give): the copies must
// also leave what the arena keeps in reserve (1 GiB) and the int8 engine's plane budget, because an engine that found
// no room would fall back to DMMA and change the bits.
static int batch_size(tncb_ctx* ctx, const tncb_plan* P, size_t count, BatchBlock* B) {
  size_t dev_free = 0, dev_total = 0;
  TNCB_CUDA(cudaMemGetInfo(&dev_free, &dev_total));
  int max_pitch = 0;
  TNCB_CUDA(cudaDeviceGetAttribute(&max_pitch, cudaDevAttrMaxPitch, ctx->device));
  B->ws = P->ws_bytes;
  B->strided = B->ws <= (size_t)max_pitch;
  B->c = std::min<size_t>({static_ws_limit(dev_total) / B->ws, count, (size_t)65535});
  if (B->c == 0) return fail(TNCB_ERR_OOM, "the workspace of one instance exceeds the static-workspace limit (TNCB_PLAN_WS_GB)");
  bool int8 = false;
  for (const Step& st : P->S.steps) int8 |= st.plan.kernel_class == 1 && ctx->oz_slices > 0;
  const size_t keep = ((size_t)1 << 30) + (int8 ? ctx->crt_ws_bytes : 0);
  const size_t room = dev_free + (ctx->arena.reserved - ctx->arena.live);
  B->c = std::min(B->c, room > keep ? (room - keep) / B->ws : 0);
  B->no_room = B->c == 0;
  if (B->c == 0) return fail(TNCB_ERR_OOM, "no room on the device for the workspace of one instance");
  return TNCB_OK;
}

// the block of c copies; c halves until it fits (a fragmented arena)
static int batch_alloc(tncb_ctx* ctx, BatchBlock* B) {
  int rc;
  while ((rc = ctx->arena.alloc(B->c * B->ws, &B->blk)) == TNCB_ERR_OOM && B->c > 1) B->c = (B->c + 1) / 2;
  return rc;
}

static void batch_free(tncb_ctx* ctx, BatchBlock* B) {
  if (B->blk) ctx->arena.free(B->blk, B->c * B->ws);   // stream-ordered: the next user of the block queues behind the pass
  B->blk = nullptr;
}

// n rows of `width` bytes, pitches dpitch / spitch, device to device: one strided copy, or one copy per row above the
// largest copy pitch
static int batch_copy(tncb_ctx* ctx, const BatchBlock& B, char* dst, size_t dpitch, const char* src, size_t spitch,
                      size_t width, size_t n) {
  cudaError_t e = cudaSuccess;
  if (B.strided) e = cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, n, cudaMemcpyDeviceToDevice, ctx->stream);
  else for (size_t i = 0; i < n && e == cudaSuccess; i++)
    e = cudaMemcpyAsync(dst + i * dpitch, src + i * spitch, width, cudaMemcpyDeviceToDevice, ctx->stream);
  return e == cudaSuccess ? TNCB_OK : fail(TNCB_ERR_CUDA, std::string("batched copy: ") + cudaGetErrorString(e));
}

// One gather set (grad_* or dgrad_*) of a pass of n instances whose workspaces lie `stride` bytes apart: instance i's
// leaf blocks into rows + i * row_elems (rows != nullptr) and/or added to `sum` in instance order, in one launch; the
// leaves with more fused groups than a GradItem holds take K3 per instance, in instance order, the sum through `scratch`
static int gather_set_batch(tncb_ctx* ctx, const tncb_plan* P, const std::vector<GradItem>& items, const std::vector<long long>& bs,
                            const std::vector<tncb_plan::GradPermute>& permutes, const void* dev, const char* base, size_t stride,
                            size_t n, double2* rows, uint64_t row_elems, double2* sum, double2* scratch) {
  int rc = TNCB_OK;
  if (!items.empty())
    rc = launch_grad_gather_batch(ctx, (const GradItem*)dev, (const long long*)((const char*)dev + items.size() * sizeof(GradItem)),
                                  (int)items.size(), bs.back(), base, (long long)stride, (int)n, rows, (long long)row_elems, sum);
  for (size_t i = 0; i < n && !rc; i++)
    for (size_t k = 0; k < permutes.size() && !rc; k++) {
      const auto& gp = permutes[k];
      const SlotMeta& sm = P->S.slots[gp.slot];
      const double2* adj = (const double2*)(base + i * stride + P->slot_off[gp.slot]);
      if (rows) rc = launch_permute(ctx, adj, rows + i * row_elems + gp.dst, (int)sm.dims.size(), sm.dims.data(), gp.perm.data());
      if (!rc && sum) rc = launch_permute(ctx, adj, scratch, (int)sm.dims.size(), sm.dims.data(), gp.perm.data());
      if (!rc && sum) rc = launch_add(ctx, sum + gp.dst, scratch, sm.elems);
    }
  return rc;
}

// ---- leaf payloads from device memory (tncb_plan_set_leaves / tncb_plan_stage_instances) ----
// cuMemGetAddressRange, resolved through the runtime as crt.cu resolves cuTensorMapEncodeTiled: the allocation that holds
// a device address, so that a source range running past its end is refused before anything is launched
MemRangeFn get_mem_range() {
  static const MemRangeFn fn = [] {
    cudaDriverEntryPointQueryResult q;
    void* p = nullptr;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      return (MemRangeFn)p;
    cudaGetLastError();
    return (MemRangeFn) nullptr;
  }();
  return fn;
}

// payload elements of every leaf of S, -1 = no payload
static std::vector<long long> leaf_elems(const Schedule& S) {
  std::vector<long long> elems(S.n_leaves_total, -1);
  for (const SlotMeta& m : S.slots) if (m.leaf_index >= 0) elems[m.leaf_index] = (long long)m.elems;
  return elems;
}
// leaf li of a caller's list (`seen`: the leaves listed so far): in range, listed once, with a payload
static int listed_leaf(const std::vector<long long>& elems, std::vector<char>& seen, uint64_t li, const std::string& name) {
  if (li >= elems.size()) return fail(TNCB_ERR_INVALID, name + " is out of range (" + std::to_string(elems.size()) + " leaves)");
  if (seen[li]) return fail(TNCB_ERR_INVALID, name + " is listed twice");
  seen[li] = 1;
  if (elems[li] < 0) return fail(TNCB_ERR_INVALID, name + " has no payload");
  return TNCB_OK;
}

// Memory a launch will read or write at p, named `noun` in the messages after `name`: device or managed memory of the
// ctx's device (device_memory), and its `bytes` inside the allocation that holds p (in_allocation)
static int device_memory(const tncb_ctx* ctx, const void* p, const std::string& name, const char* noun) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return fail(TNCB_ERR_INVALID, name + ": " + noun + " is not device memory"); }
  if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) return fail(TNCB_ERR_INVALID, name + ": " + noun + " is not device memory");
  if (a.device != ctx->device)
    return fail(TNCB_ERR_INVALID, name + ": " + noun + " is on device " + std::to_string(a.device) + ", the context on device " + std::to_string(ctx->device));
  return TNCB_OK;
}
static int in_allocation(const void* p, unsigned long long bytes, const std::string& name, const char* noun) {
  const MemRangeFn range = get_mem_range();
  if (!range) return fail(TNCB_ERR_CUDA, "cuMemGetAddressRange is not available");
  CUdeviceptr base = 0;
  size_t size = 0;
  if (range(&base, &size, (CUdeviceptr)p) != CUDA_SUCCESS) return fail(TNCB_ERR_INVALID, name + ": no device allocation holds " + noun);
  if ((unsigned long long)((CUdeviceptr)p - base) + bytes > size)
    return fail(TNCB_ERR_INVALID, name + ": " + noun + "'s " + std::to_string(bytes) + " bytes run past the end of its allocation");
  return TNCB_OK;
}

// The stage items of the leaves leaf_index[0..n) of S, leaf k read from src[k] + i * stride[k] elements for instance
// i < n_inst (stride == NULL: one instance).  Everything a launch could trip over is checked here, on the host, before
// any copy: the leaf (in range, listed once, with a payload), the stride, and the source (non-null, 16-byte aligned,
// device or managed memory of the ctx's device, every byte it reads inside one allocation).
static int device_items(const tncb_ctx* ctx, const Schedule& S, size_t n_inst, size_t n, const uint64_t* leaf_index,
                        const void* const* src, const uint64_t* stride, std::vector<LeafStageItem>& items) {
  const std::vector<long long> elems = leaf_elems(S);
  std::vector<char> seen(elems.size(), 0);
  items.clear();
  for (size_t k = 0; k < n; k++) {
    const uint64_t li = leaf_index[k];
    const std::string name = "leaf " + std::to_string(li);
    if (int rc = listed_leaf(elems, seen, li, name)) return rc;
    const unsigned long long e = (unsigned long long)elems[li], st = stride ? stride[k] : 0;
    if (st != 0 && st < e)
      return fail(TNCB_ERR_INVALID, name + ": instance stride " + std::to_string(st) + " is below its " + std::to_string(e) + " elements");
    const void* p = src[k];
    if (!p) return fail(TNCB_ERR_INVALID, name + ": the source is null");
    if ((uintptr_t)p % 16) return fail(TNCB_ERR_INVALID, name + ": the source is not 16-byte aligned");
    if (int rc = device_memory(ctx, p, name, "the source")) return rc;
    unsigned long long span = 0, bytes = 0;        // [p, p + ((n_inst - 1) * stride + elems) * 16)
    if (__builtin_mul_overflow((unsigned long long)(n_inst - 1), st, &span) || __builtin_add_overflow(span, e, &span) ||
        __builtin_mul_overflow(span, 16ull, &bytes))
      return fail(TNCB_ERR_INVALID, name + ": the source range overflows 64 bits");
    if (int rc = in_allocation(p, bytes, name, "the source")) return rc;
    items.push_back({(const double2*)p, st, (long long)S.leaf_offset[li], (long long)e});
  }
  return TNCB_OK;
}

// The runs of a leaf block of `block` elements that the device items do not cover (sorted by dst here): run r covers
// block elements [start, start + len) and sits at `packed` once the runs are packed back to back
struct LeafRun { long long start, len, packed; };
static std::vector<LeafRun> leaf_runs(std::vector<LeafStageItem>& items, long long block) {
  std::vector<LeafRun> runs;
  std::sort(items.begin(), items.end(), [](const LeafStageItem& x, const LeafStageItem& y) { return x.dst < y.dst; });
  long long pos = 0, packed = 0;
  auto gap = [&](long long end) { if (end > pos) { runs.push_back({pos, end - pos, packed}); packed += end - pos; } };
  for (const LeafStageItem& it : items) { gap(it.dst); pos = std::max(pos, it.dst + it.elems); }
  gap(block);
  return runs;
}

// ---- the arguments and outputs of the derivative calls ----
// the checks every call of a tangent plan makes: an output, tangents shaped `want` with storage
static int jvp_args(const tncb_tensor* tangents, bool any_out, const std::vector<uint64_t>& want) {
  if (!any_out) return fail(TNCB_ERR_INVALID, "no output requested");
  if (!tangents) return fail(TNCB_ERR_INVALID, "tangents are needed");
  bool same = tangents->rank == (int)want.size();
  for (size_t i = 0; same && i < want.size(); i++) same = tangents->dims[i] == want[i];
  if (!same) {
    std::string w;
    for (uint64_t d : want) w += (w.empty() ? "" : ", ") + std::to_string(d);
    return fail(TNCB_ERR_SHAPE, "the tangents' dims differ from [" + w + "]");
  }
  if (!tangents->ptr) return fail(TNCB_ERR_UNCONTRACTED, "the tangent tensor has no storage");
  return TNCB_OK;
}

// a seed or seed tangent: the result's dims, with storage.  NULL: needed (a seed) unless the result is a scalar
static int seed_args(const SlotMeta& rm, const tncb_tensor* t, const char* what, bool needed = false) {
  if (!t) {
    if (needed && !rm.dims.empty()) return fail(TNCB_ERR_INVALID, "a seed is needed for a result of rank " + std::to_string(rm.dims.size()));
    return TNCB_OK;
  }
  bool same = t->rank == (int)rm.dims.size();
  for (int i = 0; same && i < t->rank; i++) same = t->dims[i] == rm.dims[i];
  if (!same) return fail(TNCB_ERR_SHAPE, std::string("the ") + what + "'s dims differ from the result's");
  if (!t->ptr) return fail(TNCB_ERR_UNCONTRACTED, std::string("the ") + what + " tensor has no storage");
  return TNCB_OK;
}

// the instances [first, first + count) of a batched call: within the staged networks
static int instance_range(const tncb_plan* P, size_t first, size_t count) {
  if (count == 0 || first > P->n_slices || count > P->n_slices - first)
    return fail(TNCB_ERR_INVALID, "instances [" + std::to_string(first) + ", " + std::to_string(first + count) + ") are not within the " +
                                  std::to_string(P->n_slices) + " staged networks");
  return TNCB_OK;
}

// the dims of a batched call's value rows: [count, result dims]
static int result_rows(const tncb_plan* P, size_t count, std::vector<uint64_t>& dims) {
  const SlotMeta& rm = P->S.slots[P->S.result_slot];
  if (rm.dims.size() + 1 > (size_t)kMaxLegs) return fail(TNCB_ERR_INVALID, "a result of rank 64 leaves no room for the instance dimension");
  dims.assign(1, count);
  dims.insert(dims.end(), rm.dims.begin(), rm.dims.end());
  return TNCB_OK;
}

// seed or seed-tangent rows of a batched call: shaped `rows` (result_rows), with storage
static int seed_rows(const tncb_tensor* t, const std::vector<uint64_t>& rows, const char* what, const char* noun) {
  bool same = t->rank == (int)rows.size();
  for (size_t i = 0; same && i < rows.size(); i++) same = t->dims[i] == rows[i];
  if (!same) return fail(TNCB_ERR_SHAPE, std::string("the ") + what + "' dims differ from [count, result dims]");
  if (!t->ptr) return fail(TNCB_ERR_UNCONTRACTED, std::string("the ") + noun + " tensor has no storage");
  return TNCB_OK;
}

// The output tensors of a call: one per requested (non-null) destination, handed out together on success and all freed
// on an error, so that a failed call leaves the caller's pointers as they were.  After a failed allocation add() makes
// nothing more and rc holds the error.
struct Outputs {
  tncb_ctx* ctx;
  int rc = TNCB_OK;
  std::vector<std::pair<tncb_tensor**, tncb_tensor*>> made;
  tncb_tensor* add(tncb_tensor** dst, int rank, const uint64_t* dims) {
    tncb_tensor* t = nullptr;
    if (dst && !rc && !(rc = tensor_new(ctx, rank, dims, &t))) made.push_back({dst, t});
    return t;
  }
  int finish(int status) {
    for (auto [dst, t] : made) if (status) tncb_tensor_free(ctx, t); else *dst = t;
    return status;
  }
};

// the leaf tangents of n instances (rows of `row_elems` elements from `tangents` on) into the workspaces at `ws`,
// `stride` bytes apart: one leaf_stage_kernel launch, the instance a grid dimension
static int stage_tangents(tncb_ctx* ctx, const tncb_plan* P, const double2* tangents, unsigned long long row_elems,
                          char* ws, long long stride, size_t n) {
  std::vector<LeafStageItem> items;
  for (const auto& tl : P->tan_leaves)
    items.push_back({tangents + tl.off, n > 1 ? row_elems : 0, (long long)(P->slot_off[tl.slot] / sizeof(double2)),
                     (long long)P->S.slots[tl.slot].elems});
  return launch_leaf_stage(ctx, items.data(), items.size(), (double2*)ws, stride / (long long)sizeof(double2), n);
}

// the result and its tangent (either may be null) out of the workspace `ws`
static int copy_results(tncb_ctx* ctx, const tncb_plan* P, const char* ws, tncb_tensor* value, tncb_tensor* tangent) {
  const size_t res_bytes = P->S.slots[P->S.result_slot].elems * sizeof(double2);
  for (auto [dst, slot] : {std::pair<tncb_tensor*, int>{value, P->S.result_slot}, {tangent, P->tan_result}}) {
    if (!dst || !res_bytes) continue;
    cudaError_t e = cudaMemcpyAsync(dst->ptr, ws + P->slot_off[slot], res_bytes, cudaMemcpyDeviceToDevice, ctx->stream);
    if (e != cudaSuccess) return fail(TNCB_ERR_CUDA, std::string("result copy: ") + cudaGetErrorString(e));
  }
  return TNCB_OK;
}

// the seed (NULL: the 1 of a scalar result) and a Hessian-vector plan's seed tangent (NULL: zero) into the workspace `ws`.
// The seed slots may reuse memory the forward levels freed: written after them, on the stream.
static int write_seed(tncb_ctx* ctx, const tncb_plan* P, char* ws, const tncb_tensor* seed, const tncb_tensor* seed_tangent) {
  static const double2 one = {1.0, 0.0};
  const size_t res_bytes = P->S.slots[P->S.result_slot].elems * sizeof(double2);
  char* s = ws + P->slot_off[P->seed_slot];
  cudaError_t e = seed ? cudaMemcpyAsync(s, seed->ptr, res_bytes, cudaMemcpyDeviceToDevice, ctx->stream)
                       : cudaMemcpyAsync(s, &one, sizeof(double2), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess && P->seed_tan_slot >= 0) {
    char* ds = ws + P->slot_off[P->seed_tan_slot];
    e = seed_tangent ? cudaMemcpyAsync(ds, seed_tangent->ptr, res_bytes, cudaMemcpyDeviceToDevice, ctx->stream)
                     : cudaMemsetAsync(ds, 0, res_bytes, ctx->stream);
  }
  return e == cudaSuccess ? TNCB_OK : fail(TNCB_ERR_CUDA, std::string("seed copy: ") + cudaGetErrorString(e));
}

// one gather set (grad_* or dgrad_*) from the workspace into the packed block `out`: one grad_gather_kernel launch, K3
// for the leaves with more fused groups than a GradItem holds
static int gather_set(tncb_ctx* ctx, const tncb_plan* P, const std::vector<GradItem>& items, const std::vector<long long>& bs,
                      const std::vector<tncb_plan::GradPermute>& permutes, const void* dev, const char* ws, double2* out) {
  int rc = TNCB_OK;
  if (!items.empty())
    rc = launch_grad_gather(ctx, (const GradItem*)dev, (const long long*)((const char*)dev + items.size() * sizeof(GradItem)),
                            (int)items.size(), bs.back(), ws, out);
  for (size_t i = 0; i < permutes.size() && !rc; i++) {
    const auto& gp = permutes[i];
    const SlotMeta& sm = P->S.slots[gp.slot];
    rc = launch_permute(ctx, (const double2*)(ws + P->slot_off[gp.slot]), out + gp.dst, (int)sm.dims.size(), sm.dims.data(), gp.perm.data());
  }
  return rc;
}

// ---- instance-batched passes (tncb_plan_run_batch / _vjp_batch / _jvp_batch / _hvp_batch) ----
// Where a pass's leaf blocks come from: the staged instance blocks from `first` on (dev == nullptr), or the device
// payloads `dev` (sorted by leaf_runs) with the `runs` between them from the plan's staged leaf block, at stride 0
// (slices > 0, with dev: the runs come from the first `slices` staged instance blocks in turn, and every pass contracts
// once per block, PassHook::fold after each)
struct InstanceFill {
  size_t first = 0;
  const std::vector<LeafStageItem>* dev = nullptr;
  const std::vector<LeafRun>* runs = nullptr;
  size_t slices = 0;
};
// The inputs (rows of the instances: a tangent plan's tangents, seeds, seed tangents; NULL seeds: 1, NULL seed tangents:
// zero) and the outputs, each made if its destination is non-null
// A caller's work around every pass (tncb_plan_sample): at most `width` instances per pass (0: as many as fit); begin(c)
// once the pass size c is known; fill(done, n) before the leaf blocks of instances done .. done + n - 1 are filled, to
// write their device payloads (InstanceFill::dev then holds one pass: instance i of a pass reads src + i * src_stride);
// end(base, ws, n, &stop) after the forward levels, to read the pass's workspaces; stop = true ends the call.
// fold(q, base, ws, n) after the forward levels of staged block q (InstanceFill::slices).  in_place: when the device has
// no room for one copy beside the plan's workspace, run one instance per pass in that workspace instead; its staged
// leaves are then gone (leaves_resident is cleared before the first launch).  Only for fills whose runs do not come
// from the plan's own staged block.
struct PassHook {
  size_t width = 0;
  bool in_place = false;
  std::function<int(size_t c)> begin;
  std::function<int(size_t done, size_t n)> fill;
  std::function<int(size_t q, const char* base, size_t ws, size_t n)> fold;
  std::function<int(const char* base, size_t ws, size_t n, bool* stop)> end;
};
struct InstanceIO {
  const tncb_tensor *tangents = nullptr, *seeds = nullptr, *seed_tangents = nullptr;
  tncb_tensor **values = nullptr, **tangent_rows = nullptr, **grad_rows = nullptr, **grad_sum = nullptr,
              **grad_tangent_rows = nullptr, **grad_tangent_sum = nullptr;
  const PassHook* hook = nullptr;
};

// rows[0] instances with value rows of dims `rows` (result_rows), in passes of c instances on c copies of the plan's
// workspace (BatchBlock).  Per pass: the leaf blocks, a tangent plan's leaf tangents, the forward levels, values and
// tangent rows out; if a G or Ġ output is wanted, the seeds and seed tangents, the backward levels and the gathers of G,
// then Ġ, into rows and/or sums.  Every launch decision is the single-network one, so row i is bit-identical to the
// single-network call on instance i; passes run in stream order, so a sum is the left fold of its rows in instance order.
static int run_instances(tncb_ctx* ctx, tncb_plan* P, const std::vector<uint64_t>& rows, const InstanceFill& fill,
                         const InstanceIO& io) {
  const Schedule& S = P->S;
  const size_t count = rows[0];
  const uint64_t ge = P->grad_elems, row_dims[2] = {(uint64_t)count, ge};
  const bool backward = io.grad_rows || io.grad_sum || io.grad_tangent_rows || io.grad_tangent_sum;
  TNCB_CUDA(cudaSetDevice(ctx->device));
  BatchBlock B;
  int rc = batch_size(ctx, P, io.hook && io.hook->width ? std::min(count, io.hook->width) : count, &B);
  const bool may_borrow = io.hook && io.hook->in_place;
  bool in_place = rc == TNCB_ERR_OOM && B.no_room && may_borrow;
  if (in_place) rc = TNCB_OK;
  if (rc) return rc;
  Outputs out{ctx};
  tncb_tensor* v = out.add(io.values, (int)rows.size(), rows.data());
  tncb_tensor* t = out.add(io.tangent_rows, (int)rows.size(), rows.data());
  tncb_tensor* gr = out.add(io.grad_rows, 2, row_dims);
  tncb_tensor* gs = out.add(io.grad_sum, 1, &ge);
  tncb_tensor* dgr = out.add(io.grad_tangent_rows, 2, row_dims);
  tncb_tensor* dgs = out.add(io.grad_tangent_sum, 1, &ge);
  if (!(rc = out.rc) && !in_place && (rc = batch_alloc(ctx, &B)) == TNCB_ERR_OOM && may_borrow) { in_place = true; rc = TNCB_OK; }
  if (!rc && in_place) {         // the plan's own workspace is the one copy
    B.c = 1; B.blk = nullptr;
    P->leaves_resident = false; P->fwd_ready = false;
  }
  const size_t ws = B.ws, c = B.c;
  if (!rc && io.hook) rc = io.hook->begin(c);
  void* aux = nullptr;                 // the seed 1 of every copy (scalar result, NULL seeds), the K3 scratch of the sums
  const size_t ones = backward && !io.seeds ? c : 0;
  size_t scratch = 0;
  if (gs) for (const auto& gp : P->grad_permutes) scratch = std::max<size_t>(scratch, S.slots[gp.slot].elems);
  if (dgs) for (const auto& gp : P->dgrad_permutes) scratch = std::max<size_t>(scratch, S.slots[gp.slot].elems);
  const size_t aux_bytes = (ones + scratch) * sizeof(double2);
  if (!rc && aux_bytes) {
    rc = ctx->arena.alloc(aux_bytes, &aux);
    if (!rc && ones) {
      const std::vector<double2> one(ones, double2{1.0, 0.0});
      cudaError_t e = cudaMemcpyAsync(aux, one.data(), ones * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);      // `one` dies with this scope
      if (e != cudaSuccess) rc = fail(TNCB_ERR_CUDA, std::string("seed copy: ") + cudaGetErrorString(e));
    }
  }
  for (tncb_tensor* x : {gs, dgs}) {
    if (rc || !x) continue;
    cudaError_t e = cudaMemsetAsync(x->ptr, 0, std::max<uint64_t>(ge, 1) * sizeof(double2), ctx->stream);
    if (e != cudaSuccess) rc = fail(TNCB_ERR_CUDA, std::string("gradient sum: ") + cudaGetErrorString(e));
  }
  char* base = in_place ? (char*)P->ws : (char*)B.blk;
  const double2* d_one = (const double2*)aux;
  double2* d_scratch = (double2*)aux + ones;
  const size_t block_bytes = std::max<size_t>(S.leaf_block_elems, 1) * sizeof(double2);
  const size_t res_bytes = S.slots[S.result_slot].elems * sizeof(double2);
  std::vector<LeafStageItem> items;
  bool stop = false;
  for (size_t done = 0; done < count && !rc && !stop; done += c) {
    const size_t n = std::min(c, count - done);
    if (io.hook && (rc = io.hook->fill(done, n))) break;
    for (size_t q = 0; q < std::max<size_t>(fill.slices, 1) && !rc; q++) {
      if (!fill.dev) {
        const char* src = (const char*)P->slices_dev + (fill.first + done) * block_bytes;
        rc = batch_copy(ctx, B, base + P->leaf_off, ws, src, block_bytes, block_bytes, n);
      } else {        // every copy's leaf block: the device payloads of instances done .. done+n-1, the staged block between
        const char* block = fill.slices ? (const char*)P->slices_dev + q * block_bytes : (const char*)P->ws + P->leaf_off;
        const double2* staged = (const double2*)block;
        items.clear();
        const size_t at = io.hook ? 0 : done;
        for (const LeafStageItem& it : *fill.dev) items.push_back({it.src + at * it.src_stride, it.src_stride, it.dst, it.elems});
        for (const LeafRun& lr : *fill.runs) items.push_back({staged + lr.start, 0, lr.start, lr.len});
        rc = launch_leaf_stage(ctx, items.data(), items.size(), (double2*)(base + P->leaf_off), (long long)(ws / sizeof(double2)), n);
      }
      if (!rc && P->tangent()) rc = stage_tangents(ctx, P, io.tangents->ptr + done * ge, ge, base, (long long)ws, n);
      if (!rc) rc = enqueue_static(ctx, P, base, (int)n, (long long)ws, 0, P->n_fwd_levels);
      if (!rc && fill.slices) rc = io.hook->fold(q, base, ws, n);
    }
    if (rc) break;
    for (auto [x, slot] : {std::pair<tncb_tensor*, int>{v, S.result_slot}, {t, P->tan_result}})
      if (!rc && x && res_bytes) rc = batch_copy(ctx, B, (char*)x->ptr + done * res_bytes, res_bytes, base + P->slot_off[slot], ws, res_bytes, n);
    if (!rc && io.hook) rc = io.hook->end(base, ws, n, &stop);
    if (rc || !backward) continue;
    // the seed slots may reuse memory the forward levels freed: written after them, on the stream
    char* seed_dst = base + P->slot_off[P->seed_slot];
    if (io.seeds) { if (res_bytes && (rc = batch_copy(ctx, B, seed_dst, ws, (const char*)io.seeds->ptr + done * res_bytes, res_bytes, res_bytes, n))) break; }
    else if ((rc = batch_copy(ctx, B, seed_dst, ws, (const char*)d_one, sizeof(double2), sizeof(double2), n))) break;
    if (P->seed_tan_slot >= 0) {
      char* seed_tan_dst = base + P->slot_off[P->seed_tan_slot];
      if (io.seed_tangents) {
        if (res_bytes && (rc = batch_copy(ctx, B, seed_tan_dst, ws, (const char*)io.seed_tangents->ptr + done * res_bytes, res_bytes, res_bytes, n))) break;
      } else if (res_bytes) {
        cudaError_t e = cudaSuccess;
        if (B.strided) e = cudaMemset2DAsync(seed_tan_dst, ws, 0, res_bytes, n, ctx->stream);
        else for (size_t i = 0; i < n && e == cudaSuccess; i++) e = cudaMemsetAsync(seed_tan_dst + i * ws, 0, res_bytes, ctx->stream);
        if (e != cudaSuccess) { rc = fail(TNCB_ERR_CUDA, std::string("seed tangent: ") + cudaGetErrorString(e)); break; }
      }
    }
    if ((rc = enqueue_static(ctx, P, base, (int)n, (long long)ws, P->n_fwd_levels, (int)P->level_batched.size()))) break;
    if ((gr || gs) &&
        (rc = gather_set_batch(ctx, P, P->grad_items, P->grad_block_start, P->grad_permutes, P->grad_dev, base, ws, n,
                               gr ? gr->ptr + done * ge : nullptr, ge, gs ? gs->ptr : nullptr, d_scratch))) break;
    if (dgr || dgs)
      rc = gather_set_batch(ctx, P, P->dgrad_items, P->dgrad_block_start, P->dgrad_permutes, P->dgrad_dev, base, ws, n,
                            dgr ? dgr->ptr + done * ge : nullptr, ge, dgs ? dgs->ptr : nullptr, d_scratch);
  }
  batch_free(ctx, &B);
  if (aux) ctx->arena.free(aux, aux_bytes);
  return out.finish(rc);
}

} // namespace tncb

extern "C" {

// Structure key of a (network, path): everything the schedule depends on (tree shape, legs, dims, payload kinds, pairs)
// and nothing it does not (payload values).  Two calls with equal keys share one compiled plan.
static void key_tn(const tncb_tn* t, std::vector<uint64_t>& k, bool* cacheable) {
  k.push_back(0x7e00000000000000ull | (uint64_t)t->n_children);
  if (t->n_children == 0) {
    k.push_back(((uint64_t)(uint32_t)t->kind << 32) | (uint32_t)t->rank);
    if (t->kind == TNCB_DATA_DEVICE) *cacheable = false;       // consumed per call, addresses differ
    if (t->rank < 0 || t->rank > tncb::kMaxLegs || (t->rank > 0 && (!t->legs || !t->dims))) { *cacheable = false; return; }
    for (int i = 0; i < t->rank; i++) { k.push_back(t->legs[i]); k.push_back(t->dims[i]); }
    return;
  }
  for (size_t i = 0; i < t->n_children; i++) key_tn(&t->children[i], k, cacheable);
}
static void key_path(const tncb_path* p, std::vector<uint64_t>& k) {
  if (!p) { k.push_back(0x7f00000000000000ull); return; }
  k.push_back(0x7d00000000000000ull | (uint64_t)p->n_pairs);
  for (size_t i = 0; i < 2 * p->n_pairs; i++) k.push_back(p->pairs[i]);
  k.push_back(0x7c00000000000000ull | (uint64_t)p->n_nested);
  for (size_t i = 0; i < p->n_nested; i++) { k.push_back(p->nested_index[i]); key_path(&p->nested[i], k); }
}

int tncb_contract_tensor_network(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path,
                                 tncb_tensor** out, int* n_out, uint64_t* out_legs) {
  if (!ctx || !tn) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  // Repeated contractions of the same circuit (other bitstrings, angles, or simply again) hit a small per-context cache
  // of compiled plans: no schedule construction, static layout, batched tiny pairs.  TNCB_PLAN_CACHE=0 disables it.
  static const bool cache_on = !(std::getenv("TNCB_PLAN_CACHE") && atoi(std::getenv("TNCB_PLAN_CACHE")) == 0) && std::getenv("TNCB_TRACE") == nullptr;
  if (cache_on) {
    std::vector<uint64_t> key;
    bool cacheable = true;
    key_tn(tn, key, &cacheable);
    key_path(path, key);
    if (cacheable) {
      auto& cache = ctx->plan_cache;
      for (size_t i = 0; i < cache.size(); i++)
        if (cache[i].key == key) {
          tncb_ctx::CachedPlan hit = std::move(cache[i]);
          cache.erase(cache.begin() + i);
          cache.push_back(std::move(hit));                       // most recently used last
          tncb_plan* pl = cache.back().plan;
          int rc = tncb::execute_static(ctx, pl, tn, out, n_out, out_legs);
          if (rc != TNCB_ERR_OOM) return rc;
          tncb_plan_destroy(pl); cache.pop_back();               // no room for its workspace any more: pair-by-pair path
          break;
        }
      // a second sighting is what earns a plan: remember the key of a miss, compile on the next call with the same key
      static thread_local std::vector<uint64_t> last_miss;
      if (last_miss == key) {
        tncb_plan* pl = nullptr;
        if (tncb_plan_create(ctx, tn, path, &pl) == TNCB_OK && pl->is_static) {
          size_t total = 0, free_b = 0, total_b = 0;
          for (auto& c : cache) total += c.plan->ws_bytes;
          cudaMemGetInfo(&free_b, &total_b);
          while (!cache.empty() && (cache.size() >= 4 || total + pl->ws_bytes > total_b / 4)) {   // at most 4 plans / a quarter of the device
            total -= cache.front().plan->ws_bytes;
            tncb_plan_destroy(cache.front().plan); cache.erase(cache.begin());
          }
          if (pl->ws_bytes <= total_b / 4) {
            int rc = tncb::execute_static(ctx, pl, tn, out, n_out, out_legs);
            if (rc == TNCB_OK) { cache.push_back({std::move(key), pl}); last_miss.clear(); return rc; }
            tncb_plan_destroy(pl);
            if (rc != TNCB_ERR_OOM) return rc;
          } else tncb_plan_destroy(pl);
        } else if (pl) tncb_plan_destroy(pl);
      } else last_miss = key;
    }
  }
  tncb::Schedule S;
  int rc = tncb::build_schedule(tn, path, S);
  if (rc) return rc;
  return tncb::execute(ctx, S, tn, out, n_out, out_legs);
}

int tncb_plan_create(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, tncb_plan** out) {
  (void)ctx;
  if (!tn || !out) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  tncb_plan* p = new tncb_plan();
  int rc = tncb::build_schedule(tn, path, p->S);
  if (rc) { delete p; return rc; }
  tncb::plan_static_layout(p, ctx ? ctx->sm_count : 132, tncb::device_bytes(ctx));
  *out = p;
  return TNCB_OK;
}

namespace tncb {
// The checks every sliced creator makes on the sliced legs: every sliced leg listed once, joining two tensors, of
// non-zero dimension, and a slice count that fits 64 bits.  Fills the legs' dims and the slice count.
static int check_sliced_legs(const std::vector<const tncb_tn*>& lv, size_t n_sliced, const uint64_t* sliced_legs,
                             std::vector<uint64_t>& sl, std::vector<uint64_t>& sdim, uint64_t* n_slices) {
  sl.assign(sliced_legs, sliced_legs + n_sliced);
  sdim.assign(n_sliced, 0);
  uint64_t n_sl = 1;
  bool overflow = false;
  for (size_t k = 0; k < n_sliced; k++) {
    const std::string name = "sliced leg " + std::to_string(sl[k]);
    if (std::find(sl.begin(), sl.begin() + k, sl[k]) != sl.begin() + k) return fail(TNCB_ERR_INVALID, name + " is listed twice");
    int count = 0;
    for (const tncb_tn* l : lv)
      if (l->rank > 0 && l->rank <= kMaxLegs && l->legs && l->dims)
        for (int i = 0; i < l->rank; i++)
          if (l->legs[i] == sl[k]) { count++; sdim[k] = l->dims[i]; }
    if (count == 0) return fail(TNCB_ERR_INVALID, name + " does not occur in the network");
    if (count == 1) return fail(TNCB_ERR_INVALID, name + " occurs once: it is an open leg of the result");
    if (sdim[k] == 0) return fail(TNCB_ERR_INVALID, name + " has dimension 0");
    if (n_sl > UINT64_MAX / sdim[k]) overflow = true;
    else n_sl *= sdim[k];
  }
  if (overflow) return fail(TNCB_ERR_INVALID, "the slice count overflows 64 bits");
  *n_slices = n_sl;
  return TNCB_OK;
}

// A derivative plan of a kind other than plain, in one static layout: the forward schedule plus the tangent pairs
// (build_tangent), backward pairs (build_backward) and backward-tangent pairs (build_backward_tangent) the kind has, and
// the gathers of G (and Ġ).  Sliced (n_sliced legs, possibly none): the plan of one slice's structure, compiled exactly
// so on the host-sliced slice network, plus the slice items instead of the gathers.  There is no pair-by-pair fallback:
// a layout above the static-workspace limit is refused here.
static int create(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, tncb_plan::Kind kind, bool sliced, size_t n_sliced,
                  const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out) {
  if (!tn || !out || (n_sliced && !sliced_legs)) return fail(TNCB_ERR_INVALID, "null argument");
  static const char* const noun[4] = {nullptr, "gradient", "tangent", "Hessian-vector"};
  const std::string what = noun[(int)kind];
  std::vector<const tncb_tn*> lv;
  collect_leaf_nodes(tn, lv);
  for (const tncb_tn* l : lv)
    if (l->kind == TNCB_DATA_DEVICE) return fail(TNCB_ERR_UNSUPPORTED, what + " plans do not take device leaves (they are consumed per call)");
  std::vector<uint64_t> sl, sdim;
  uint64_t n_sl = 1;
  SliceTree keep;
  tncb_tn st;
  if (sliced) {
    int rc = check_sliced_legs(lv, n_sliced, sliced_legs, sl, sdim, &n_sl);
    if (rc) return rc;
    slice_tree(tn, &st, sl, keep);
  }
  tncb_plan* p = new tncb_plan();
  p->kind = kind;
  p->sliced = sliced;
  p->n_sl = n_sl;
  std::vector<int> tan, leaf_adj, leaf_dadj;
  int rc = build_schedule(sliced ? &st : tn, path, p->S);
  const size_t n_fwd = p->S.steps.size();
  size_t b0 = n_fwd;
  if (!rc && p->tangent()) { rc = build_tangent(p, wrt, &tan); b0 = p->S.steps.size(); }
  if (!rc && p->grad()) rc = build_backward(p, wrt, leaf_adj, n_fwd);
  if (!rc && kind == tncb_plan::Kind::hvp) rc = build_backward_tangent(p, b0, tan, leaf_adj, leaf_dadj);
  if (rc) { delete p; return rc; }
  const size_t dev_total = device_bytes(ctx);
  plan_static_layout(p, ctx ? ctx->sm_count : 132, dev_total);
  if (!p->is_static) {
    const size_t need = p->ws_bytes, limit = static_ws_limit(dev_total);
    delete p;
    return fail(TNCB_ERR_UNSUPPORTED, "the " + what + (sliced ? " workspace of one slice needs " : " workspace needs ") + std::to_string(need) +
                                      " bytes, above the static-workspace limit of " + std::to_string(limit) + " bytes (TNCB_PLAN_WS_GB)");
  }
  if (sliced) rc = build_slice_items(p, lv, sl, sdim, leaf_adj, leaf_dadj);
  else {
    if (p->grad()) rc = build_gather(p, leaf_adj, p->grad_items, p->grad_block_start, p->grad_permutes);
    if (!rc && kind == tncb_plan::Kind::hvp) rc = build_gather(p, leaf_dadj, p->dgrad_items, p->dgrad_block_start, p->dgrad_permutes);
  }
  if (rc) { delete p; return rc; }
  *out = p;
  return TNCB_OK;
}
} // namespace tncb

// A gradient plan: the forward schedule, the backward pairs of the `wrt` leaves and the leaf-gradient gather.
int tncb_plan_create_vjp(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, const uint8_t* wrt, tncb_plan** out) {
  return tncb::create(ctx, tn, path, tncb_plan::Kind::vjp, false, 0, nullptr, wrt, out);
}

// A tangent plan: the forward schedule and the tangent pairs of the `wrt` leaves, on the forward levels.
int tncb_plan_create_jvp(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, const uint8_t* wrt, tncb_plan** out) {
  return tncb::create(ctx, tn, path, tncb_plan::Kind::jvp, false, 0, nullptr, wrt, out);
}

// A Hessian-vector plan: the forward schedule, the tangent pairs, the backward pairs and the backward-tangent pairs of
// the `wrt` leaves, plus the gathers of G and Ġ.
int tncb_plan_create_hvp(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, const uint8_t* wrt, tncb_plan** out) {
  return tncb::create(ctx, tn, path, tncb_plan::Kind::hvp, false, 0, nullptr, wrt, out);
}

// A sliced gradient plan: the gradient plan of one slice's structure plus the extract / accumulate items that move slice
// q's sub-blocks between the full leaves and the workspace.
int tncb_plan_create_vjp_sliced(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, size_t n_sliced,
                                const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out) {
  return tncb::create(ctx, tn, path, tncb_plan::Kind::vjp, true, n_sliced, sliced_legs, wrt, out);
}

// Sliced tangent and Hessian-vector plans: the tangent / Hessian-vector plan of one slice's structure plus the items that
// also move the leaf tangents in and the adjoints' tangents out per slice.
int tncb_plan_create_jvp_sliced(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, size_t n_sliced,
                                const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out) {
  return tncb::create(ctx, tn, path, tncb_plan::Kind::jvp, true, n_sliced, sliced_legs, wrt, out);
}

int tncb_plan_create_hvp_sliced(tncb_ctx* ctx, const tncb_tn* tn, const tncb_path* path, size_t n_sliced,
                                const uint64_t* sliced_legs, const uint8_t* wrt, tncb_plan** out) {
  return tncb::create(ctx, tn, path, tncb_plan::Kind::hvp, true, n_sliced, sliced_legs, wrt, out);
}

int tncb_plan_grad_offsets(const tncb_plan* plan, int64_t* offsets) {
  if (!plan || !offsets) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = tncb::route(plan, tncb::Call::grad_offsets)) return rc;
  for (size_t i = 0; i < plan->grad_offset.size(); i++) offsets[i] = plan->grad_offset[i];
  return TNCB_OK;
}

// The backward levels and the leaf-gradient gather of a gradient plan, on the forward state its last run left in the
// workspace.  The backward slots reuse freed forward memory, so one forward run serves one call.
int tncb_plan_vjp(tncb_ctx* ctx, tncb_plan* plan, const tncb_tensor* seed, tncb_tensor** grads) {
  using namespace tncb;
  if (!ctx || !plan || !grads) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::vjp);
  if (rc) return rc;
  if (plan->ctx != ctx || !plan->fwd_ready)
    return fail(TNCB_ERR_INVALID, "tncb_plan_vjp needs a forward run (tncb_plan_run / tncb_plan_execute) of the plan on this context "
                                  "since its leaves were staged or its last tncb_plan_vjp");
  if ((rc = seed_args(plan->S.slots[plan->S.result_slot], seed, "seed", true))) return rc;
  TNCB_CUDA(cudaSetDevice(ctx->device));
  Outputs out{ctx};
  tncb_tensor* g = out.add(grads, 1, &plan->grad_elems);
  if (out.rc) return out.rc;
  char* ws = (char*)plan->ws;
  rc = write_seed(ctx, plan, ws, seed, nullptr);
  plan->fwd_ready = false;
  if (!rc) rc = enqueue_static(ctx, plan, ws, 1, 0, plan->n_fwd_levels, (int)plan->level_batched.size());
  if (!rc) rc = gather_set(ctx, plan, plan->grad_items, plan->grad_block_start, plan->grad_permutes, plan->grad_dev, ws, g->ptr);
  return out.finish(rc);
}

// Per slice first, first+stride, ...: extract, forward levels, seed copy, backward levels, accumulate into the
// full-shape gradients.  No host work per slice; the slices are stream-ordered, so the sums repeat bit for bit.
int tncb_plan_vjp_sliced(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, const tncb_tensor* seed,
                         tncb_tensor** value, tncb_tensor** grads) {
  using namespace tncb;
  if (!ctx || !plan || !value || !grads || stride == 0) return fail(TNCB_ERR_INVALID, "bad argument");
  int rc = route(plan, Call::vjp_sliced);
  if (rc) return rc;
  if (plan->ctx != ctx || !plan->full_staged) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this context");
  const SlotMeta& rm = plan->S.slots[plan->S.result_slot];
  if ((rc = seed_args(rm, seed, "seed", true))) return rc;
  TNCB_CUDA(cudaSetDevice(ctx->device));
  Outputs out{ctx};
  tncb_tensor* v = out.add(value, (int)rm.dims.size(), rm.dims.data());
  tncb_tensor* g = out.add(grads, 1, &plan->grad_elems);
  if (!(rc = out.rc)) {
    SliceRun io;
    io.seed = seed ? seed->ptr : nullptr; io.value = v->ptr; io.grad = g->ptr;
    rc = run_sliced(ctx, plan, first, stride, io);
  }
  return out.finish(rc);
}

int tncb_plan_execute(tncb_ctx* ctx, tncb_plan* plan, const tncb_tn* tn, tncb_tensor** out, int* n_out, uint64_t* out_legs) {
  if (!ctx || !plan || !tn) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = tncb::route(plan, tncb::Call::execute)) return rc;
  if (plan->grad()) return tncb::execute_static(ctx, plan, tn, out, n_out, out_legs);   // forward levels only, no fallback
  static const bool trace = std::getenv("TNCB_TRACE") != nullptr;   // per-step times come from the pair-by-pair executor
  if (plan->is_static && !trace && (plan->ctx == nullptr || plan->ctx == ctx)) {
    int rc = tncb::execute_static(ctx, plan, tn, out, n_out, out_legs);
    if (rc != TNCB_ERR_OOM || plan->ws) return rc;
    plan->is_static = false;        // no room for the static workspace (it keeps a whole tree level alive): pair-by-pair executor
  }
  return tncb::execute(ctx, plan->S, tn, out, n_out, out_legs);
}

// Materialise the leaves of `tn` once and keep them on the device; tncb_plan_run then executes the schedule without
// any host work besides the kernel launches (the "inputs already resident in HBM" measurement, and the shared leaf
// block of sliced execution).
int tncb_plan_stage(tncb_ctx* ctx, tncb_plan* plan, const tncb_tn* tn) {
  if (!ctx || !plan || !tn) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = tncb::route(plan, tncb::Call::stage)) return rc;
  const tncb::Schedule& S = plan->S;
  for (int k : S.leaf_kind) if (k == TNCB_DATA_DEVICE) return tncb::fail(TNCB_ERR_UNSUPPORTED, "plans with device leaves cannot be staged (they are consumed per call)");
  if (plan->ctx && plan->ctx != ctx) return tncb::fail(TNCB_ERR_INVALID, "plan belongs to another context");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  std::vector<const tncb_tn*> leaves;
  tncb::collect_leaf_nodes(tn, leaves);
  if (plan->sliced) {         // the FULL leaves, once, into a plan-owned block outside the workspace
    const tncb::Schedule& F = plan->full;
    int rc = tncb::validate_leaves(F, leaves);
    if (rc) return rc;
    std::vector<std::complex<double>> host(std::max<size_t>(F.leaf_block_elems, 1));
    if ((rc = tncb::stage_leaves(F, leaves, host.data()))) return rc;
    if ((rc = tncb::plan_device_state(ctx, plan))) return rc;
    if (!plan->full_dev) {
      if ((rc = ctx->arena.alloc(host.size() * sizeof(double2), &plan->full_dev))) return rc;
      plan->full_bytes = host.size() * sizeof(double2);
    }
    plan->full_staged = false;
    TNCB_CUDA(cudaMemcpyAsync(plan->full_dev, host.data(), plan->full_bytes, cudaMemcpyHostToDevice, ctx->stream));
    TNCB_CUDA(cudaStreamSynchronize(ctx->stream));   // `host` dies with this frame
    plan->full_staged = true;
    return TNCB_OK;
  }
  int rc = tncb::validate_leaves(S, leaves);
  if (rc) return rc;
  const size_t bytes = std::max<size_t>(S.leaf_block_elems * sizeof(double2), 16);
  std::vector<std::complex<double>> host(std::max<size_t>(S.leaf_block_elems, 1));
  if (plan->is_static && (rc = tncb::plan_device_state(ctx, plan))) {
    if (rc != TNCB_ERR_OOM || plan->ws || plan->grad() || plan->tangent()) return rc;
    plan->is_static = false;    // the static workspace does not fit: resident leaf block + pair-by-pair executor
  }
  if (plan->is_static) {      // the leaf block lives inside the plan workspace
    plan->fwd_ready = false;
    TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
    if ((rc = tncb::stage_leaves(S, leaves, (std::complex<double>*)plan->stage))) return rc;
    TNCB_CUDA(cudaMemcpyAsync((char*)plan->ws + plan->leaf_off, plan->stage, bytes, cudaMemcpyHostToDevice, ctx->stream));
    TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
    plan->leaves_resident = true;
    return TNCB_OK;
  }
  if ((rc = tncb::stage_leaves(S, leaves, host.data()))) return rc;
  if (!plan->ctx) { plan->ctx = ctx; ctx->plans.push_back(plan); }
  if (!plan->resident) {
    if ((rc = ctx->arena.alloc(bytes, &plan->resident))) return rc;
    plan->resident_bytes = bytes;
  }
  TNCB_CUDA(cudaMemcpyAsync(plan->resident, host.data(), S.leaf_block_elems * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream));
  TNCB_CUDA(cudaStreamSynchronize(ctx->stream));   // `host` dies with this frame
  return TNCB_OK;
}

int tncb_plan_run(tncb_ctx* ctx, tncb_plan* plan, tncb_tensor** out, int* n_out, uint64_t* out_legs) {
  if (!ctx || !plan) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = tncb::route(plan, tncb::Call::run)) return rc;
  static const bool trace = std::getenv("TNCB_TRACE") != nullptr;
  if (plan->is_static && plan->leaves_resident && plan->ctx == ctx) {
    if (!trace || plan->grad()) return tncb::execute_static(ctx, plan, nullptr, out, n_out, out_legs);
    return tncb::execute(ctx, plan->S, nullptr, out, n_out, out_legs, (const double2*)((char*)plan->ws + plan->leaf_off));
  }
  if (!plan->resident || plan->ctx != ctx) return tncb::fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this context");
  return tncb::execute(ctx, plan->S, nullptr, out, n_out, out_legs, (const double2*)plan->resident);
}

// Sliced execution (the reference's declared future work, book/src/future_work.md:9-11) without host work per slice:
// `plan` is compiled for the SLICED structure; the leaf blocks of all slice networks are materialised and uploaded
// once, then tncb_plan_run_slices walks slices first, first+stride, ... : one device-to-device copy of the slice's leaf
// block (KBs), the plan's kernels (batched / graph as usual), one accumulation kernel.
int tncb_plan_stage_slices(tncb_ctx* ctx, tncb_plan* plan, size_t n_slices, const tncb_tn* const* slice_tns) {
  if (!ctx || !plan || !slice_tns || n_slices == 0) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = tncb::route(plan, tncb::Call::stage_slices)) return rc;
  if (!plan->is_static) return tncb::fail(TNCB_ERR_UNSUPPORTED, "sliced execution needs a plan with a static layout (no device leaves)");
  return tncb::stage_networks(ctx, plan, n_slices, slice_tns, true);
}

int tncb_plan_run_slices(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, tncb_tensor** out, int* n_out, uint64_t* out_legs) {
  if (!ctx || !plan || stride == 0) return tncb::fail(TNCB_ERR_INVALID, "bad argument");
  if (int rc = tncb::route(plan, tncb::Call::run_slices)) return rc;
  if (plan->sliced) {         // forward levels only, slices extracted on the device from the staged full leaves
    if (plan->ctx != ctx || !plan->full_staged) return tncb::fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this context");
    const tncb::SlotMeta& rm = plan->S.slots[plan->S.result_slot];
    TNCB_CUDA(cudaSetDevice(ctx->device));
    tncb_tensor *sum = nullptr, *zero = nullptr;
    int rc = tncb::tensor_new(ctx, (int)rm.dims.size(), rm.dims.data(), &sum);
    tncb::SliceRun io;
    io.value = sum ? sum->ptr : nullptr;
    if (!rc && plan->tangent()) {   // the tangent pairs share the forward levels: they read zero tangents
      rc = tncb::tensor_new(ctx, 1, &plan->grad_elems, &zero);
      if (!rc && cudaMemsetAsync(zero->ptr, 0, zero->elems * sizeof(double2), ctx->stream) != cudaSuccess)
        rc = tncb::fail(TNCB_ERR_CUDA, "tangent block: memset failed");
      if (!rc) io.tangents = zero->ptr;
    }
    if (!rc) rc = tncb::run_sliced(ctx, plan, first, stride, io);
    if (zero) tncb_tensor_free(ctx, zero);      // (stream-ordered: the arena hands it out behind this call's kernels)
    if (rc) { if (sum) tncb_tensor_free(ctx, sum); return rc; }
    if (out) *out = sum; else tncb_tensor_free(ctx, sum);
    if (n_out) *n_out = (int)rm.legs.size();
    if (out_legs) for (size_t i = 0; i < rm.legs.size(); i++) out_legs[i] = rm.legs[i];
    return TNCB_OK;
  }
  if (!plan->slices_dev || plan->ctx != ctx) return tncb::fail(TNCB_ERR_INVALID, "tncb_plan_stage_slices has not been called on this context");
  const tncb::Schedule& S = plan->S;
  if (S.result_slot < 0) return tncb::fail(TNCB_ERR_INVALID, "plan has no result");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  const tncb::SlotMeta& rm = S.slots[S.result_slot];
  tncb_tensor* sum = nullptr;
  int rc = tncb::tensor_new(ctx, (int)rm.dims.size(), rm.dims.data(), &sum);
  if (rc) return rc;
  const size_t block_bytes = std::max<size_t>(S.leaf_block_elems, 1) * sizeof(double2);
  char* ws = (char*)plan->ws;
  bool any = false;
  for (size_t q = first; q < plan->n_slices; q += stride) {
    TNCB_CUDA(cudaMemcpyAsync(ws + plan->leaf_off, (char*)plan->slices_dev + q * block_bytes, block_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    plan->leaves_resident = true;
    tncb_tensor* part = nullptr;
    if ((rc = tncb::execute_static(ctx, plan, nullptr, &part, nullptr, nullptr))) { tncb_tensor_free(ctx, sum); return rc; }
    if (!any) {
      TNCB_CUDA(cudaMemcpyAsync(sum->ptr, part->ptr, rm.elems * sizeof(double2), cudaMemcpyDeviceToDevice, ctx->stream));
      any = true;
    } else if ((rc = tncb::launch_add(ctx, sum->ptr, part->ptr, rm.elems))) { tncb_tensor_free(ctx, part); tncb_tensor_free(ctx, sum); return rc; }
    tncb_tensor_free(ctx, part);
  }
  if (!any) TNCB_CUDA(cudaMemsetAsync(sum->ptr, 0, std::max<size_t>(rm.elems, 1) * sizeof(double2), ctx->stream));   // more ranks than slices
  if (out) *out = sum; else tncb_tensor_free(ctx, sum);
  if (n_out) *n_out = (int)rm.legs.size();
  if (out_legs) for (size_t i = 0; i < rm.legs.size(); i++) out_legs[i] = rm.legs[i];
  return TNCB_OK;
}

// Instance-batched execution: the staged networks first .. first+count-1 (slices, bitstrings, angle sets of one
// structure) are contracted each on its own, with the instance as a grid dimension of every kernel, so that one walk over
// the schedule does the work of many networks.  A pass of c instances runs on c copies of the plan's workspace, ws_bytes
// apart in one arena block that lives for this call only; the plan's own workspace and resident leaves stay untouched.
// Every launch decision is the single-network one, so instance i is bit-identical to tncb_plan_run_slices(i, n_slices).
int tncb_plan_run_batch(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t count,
                        tncb_tensor** out, int* n_out, uint64_t* out_legs) {
  using namespace tncb;
  if (!ctx || !plan) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::run_batch);
  if (rc) return rc;
  if (!plan->is_static) return fail(TNCB_ERR_UNSUPPORTED, "batched execution needs a plan with a static layout (no device leaves)");
  if (!plan->slices_dev || plan->ctx != ctx) return fail(TNCB_ERR_INVALID, "tncb_plan_stage_slices has not been called on this context");
  if ((rc = instance_range(plan, first, count))) return rc;
  if (plan->S.result_slot < 0) return fail(TNCB_ERR_INVALID, "plan has no result");
  std::vector<uint64_t> rows;
  if ((rc = result_rows(plan, count, rows))) return rc;
  tncb_tensor* res = nullptr;
  InstanceIO io;
  io.values = &res;
  if ((rc = run_instances(ctx, plan, rows, {first}, io))) return rc;
  const SlotMeta& rm = plan->S.slots[plan->S.result_slot];
  if (out) *out = res; else tncb_tensor_free(ctx, res);
  if (n_out) *n_out = (int)rm.legs.size();
  if (out_legs) for (size_t i = 0; i < rm.legs.size(); i++) out_legs[i] = rm.legs[i];
  return TNCB_OK;
}

// Instances of a gradient plan's structure for tncb_plan_vjp_batch: staged like tncb_plan_stage_slices stages them, but
// without the plan's own workspace, which a batched pass does not use.
int tncb_plan_stage_batch(tncb_ctx* ctx, tncb_plan* plan, size_t n, const tncb_tn* const* tns) {
  using namespace tncb;
  if (!ctx || !plan || !tns || n == 0) return fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = route(plan, Call::stage_batch)) return rc;
  return stage_networks(ctx, plan, n, tns, false);
}

// Instance-batched reverse mode (run_instances): leaf blocks in, forward levels, values out, seeds in, backward levels,
// one gather launch that writes gradient rows and/or folds them into the sum.  Each instance is bit-identical to
// stage + run + tncb_plan_vjp.
int tncb_plan_vjp_batch(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t count, const tncb_tensor* seeds,
                        tncb_tensor** values, tncb_tensor** grad_rows, tncb_tensor** grad_sum) {
  using namespace tncb;
  if (!ctx || !plan) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::vjp_batch);
  if (rc) return rc;
  if (!plan->slices_dev || plan->ctx != ctx) return fail(TNCB_ERR_INVALID, "tncb_plan_stage_batch has not been called on this context");
  if ((rc = instance_range(plan, first, count))) return rc;
  if (!values && !grad_rows && !grad_sum) return fail(TNCB_ERR_INVALID, "no output requested");
  std::vector<uint64_t> rows;
  if ((rc = result_rows(plan, count, rows))) return rc;
  if (seeds) { if ((rc = seed_rows(seeds, rows, "seeds", "seed"))) return rc; }
  else if ((grad_rows || grad_sum) && rows.size() > 1)
    return fail(TNCB_ERR_INVALID, "seeds are needed for a result of rank " + std::to_string(rows.size() - 1));
  InstanceIO io;
  io.seeds = seeds;
  io.values = values; io.grad_rows = grad_rows; io.grad_sum = grad_sum;
  return run_instances(ctx, plan, rows, {first}, io);
}

// One forward-mode pass on the staged leaves: leaf tangents in, every level (forward pairs, tangent pairs, sums), the
// result and its tangent out.  Nothing is kept between calls, so a call can be repeated and gives the same bits.
int tncb_plan_jvp(tncb_ctx* ctx, tncb_plan* plan, const tncb_tensor* tangents, tncb_tensor** value, tncb_tensor** tangent_out) {
  using namespace tncb;
  if (!ctx || !plan) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::jvp);
  if (rc || (rc = jvp_args(tangents, value || tangent_out, {plan->grad_elems}))) return rc;
  if (plan->ctx != ctx || !plan->leaves_resident) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan and context");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  const SlotMeta& rm = plan->S.slots[plan->S.result_slot];
  Outputs out{ctx};
  tncb_tensor* v = out.add(value, (int)rm.dims.size(), rm.dims.data());
  tncb_tensor* t = out.add(tangent_out, (int)rm.dims.size(), rm.dims.data());
  char* ws = (char*)plan->ws;
  if (!(rc = out.rc)) rc = stage_tangents(ctx, plan, tangents->ptr, plan->grad_elems, ws, 0, 1);
  if (!rc) rc = enqueue_static(ctx, plan, ws, 1, 0, 0, (int)plan->level_batched.size());
  if (!rc) rc = copy_results(ctx, plan, ws, v, t);
  return out.finish(rc);
}

// Instance-batched forward mode (run_instances) over the networks staged by tncb_plan_stage_batch /
// tncb_plan_stage_instances: leaf blocks in, leaf tangents in (row i of `tangents` for instance i), every level, values
// and tangents out.  Row i is bit-identical to tncb_plan_jvp of instance i with tangent row i.
int tncb_plan_jvp_batch(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t count, const tncb_tensor* tangents,
                        tncb_tensor** values, tncb_tensor** tangent_rows) {
  using namespace tncb;
  if (!ctx || !plan) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::jvp_batch);
  if (rc) return rc;
  if (!plan->slices_dev || plan->ctx != ctx)
    return fail(TNCB_ERR_INVALID, "tncb_plan_stage_batch / tncb_plan_stage_instances has not been called on this context");
  std::vector<uint64_t> rows;
  if ((rc = instance_range(plan, first, count)) || (rc = result_rows(plan, count, rows)) ||
      (rc = jvp_args(tangents, values || tangent_rows, {(uint64_t)count, plan->grad_elems})))
    return rc;
  InstanceIO io;
  io.tangents = tangents;
  io.values = values; io.tangent_rows = tangent_rows;
  return run_instances(ctx, plan, rows, {first}, io);
}

// One forward-over-reverse pass on the staged leaves: leaf tangents in, the forward levels (forward pairs, tangent pairs,
// sums), R and Ṙ out, the seed and its tangent in, the backward levels (backward pairs, backward-tangent pairs, sums),
// the gathers of G and Ġ.  Nothing is kept between calls, so a call can be repeated and gives the same bits.
int tncb_plan_hvp(tncb_ctx* ctx, tncb_plan* plan, const tncb_tensor* tangents, const tncb_tensor* seed,
                  const tncb_tensor* seed_tangent, tncb_tensor** value, tncb_tensor** tangent_out, tncb_tensor** grads,
                  tncb_tensor** grad_tangents) {
  using namespace tncb;
  if (!ctx || !plan) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::hvp);
  if (rc || (rc = jvp_args(tangents, value || tangent_out || grads || grad_tangents, {plan->grad_elems}))) return rc;
  const SlotMeta& rm = plan->S.slots[plan->S.result_slot];
  if ((rc = seed_args(rm, seed, "seed", true)) || (rc = seed_args(rm, seed_tangent, "seed tangent"))) return rc;
  if (plan->ctx != ctx || !plan->leaves_resident) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan and context");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  const uint64_t ge = plan->grad_elems;
  Outputs out{ctx};
  tncb_tensor* v = out.add(value, (int)rm.dims.size(), rm.dims.data());
  tncb_tensor* t = out.add(tangent_out, (int)rm.dims.size(), rm.dims.data());
  tncb_tensor* g = out.add(grads, 1, &ge);
  tncb_tensor* dg = out.add(grad_tangents, 1, &ge);
  char* ws = (char*)plan->ws;
  if (!(rc = out.rc)) rc = stage_tangents(ctx, plan, tangents->ptr, ge, ws, 0, 1);
  if (!rc) rc = enqueue_static(ctx, plan, ws, 1, 0, 0, plan->n_fwd_levels);
  if (!rc) rc = copy_results(ctx, plan, ws, v, t);
  if (!rc) rc = write_seed(ctx, plan, ws, seed, seed_tangent);
  if (!rc) rc = enqueue_static(ctx, plan, ws, 1, 0, plan->n_fwd_levels, (int)plan->level_batched.size());
  if (!rc && g) rc = gather_set(ctx, plan, plan->grad_items, plan->grad_block_start, plan->grad_permutes, plan->grad_dev, ws, g->ptr);
  if (!rc && dg) rc = gather_set(ctx, plan, plan->dgrad_items, plan->dgrad_block_start, plan->dgrad_permutes, plan->dgrad_dev, ws, dg->ptr);
  return out.finish(rc);
}

// Instance-batched forward over reverse (run_instances) on c workspace copies beside the plan's own: one launch fills
// every copy's leaf block (the device payloads, and the staged block's runs between them at stride 0), the leaf tangents,
// the forward levels, R and Ṙ out, seeds and seed tangents in, the backward levels, the gathers of G and Ġ into rows
// and/or sums.  Row i is bit-identical to set_leaves + tncb_plan_hvp of instance i.
int tncb_plan_hvp_batch(tncb_ctx* ctx, tncb_plan* plan, size_t count, size_t n, const uint64_t* leaf_index,
                        const void* const* src, const uint64_t* instance_stride, const tncb_tensor* tangents,
                        const tncb_tensor* seeds, const tncb_tensor* seed_tangents, tncb_tensor** values,
                        tncb_tensor** tangent_rows, tncb_tensor** grad_rows, tncb_tensor** grad_sum,
                        tncb_tensor** grad_tangent_rows, tncb_tensor** grad_tangent_sum) {
  using namespace tncb;
  if (!ctx || !plan || (n && (!leaf_index || !src || !instance_stride))) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::hvp_batch);
  if (rc) return rc;
  if (count == 0) return fail(TNCB_ERR_INVALID, "count is 0");
  const bool any_out = values || tangent_rows || grad_rows || grad_sum || grad_tangent_rows || grad_tangent_sum;
  std::vector<uint64_t> rows;
  if ((rc = jvp_args(tangents, any_out, {(uint64_t)count, plan->grad_elems})) || (rc = result_rows(plan, count, rows)) ||
      (seeds && (rc = seed_rows(seeds, rows, "seeds", "seeds"))) ||
      (seed_tangents && (rc = seed_rows(seed_tangents, rows, "seed tangents", "seed tangents"))))
    return rc;
  if (!seeds && rows.size() > 1) return fail(TNCB_ERR_INVALID, "seeds are needed for a result of rank " + std::to_string(rows.size() - 1));
  if (plan->ctx != ctx || !plan->leaves_resident) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan and context");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  std::vector<LeafStageItem> dev_items;
  if ((rc = device_items(ctx, plan->S, count, n, leaf_index, src, instance_stride, dev_items))) return rc;
  const std::vector<LeafRun> runs = leaf_runs(dev_items, (long long)std::max<size_t>(plan->S.leaf_block_elems, 1));
  InstanceIO io;
  io.tangents = tangents; io.seeds = seeds; io.seed_tangents = seed_tangents;
  io.values = values; io.tangent_rows = tangent_rows; io.grad_rows = grad_rows; io.grad_sum = grad_sum;
  io.grad_tangent_rows = grad_tangent_rows; io.grad_tangent_sum = grad_tangent_sum;
  return run_instances(ctx, plan, rows, {0, &dev_items, &runs}, io);
}

namespace tncb {
// The qubits of a sampling spec against the plan: every closed leaf a listed, rank-1, dimension-2 leaf with a payload, every
// result leg of dimension 2, and the closed qubits and result legs' qubits together each qubit 0 .. n_qubits - 1 once
static int sample_map(const Schedule& S, const tncb_sample_spec& sp, SampleMap* map) {
  if (sp.n_qubits < 1 || sp.n_qubits > 64) return fail(TNCB_ERR_INVALID, "n_qubits " + std::to_string(sp.n_qubits) + " is outside 1..64");
  const SlotMeta& rm = S.slots[S.result_slot];
  const size_t k = rm.dims.size();
  if ((sp.n_closed && (!sp.closed_leaf || !sp.closed_qubit)) || (k && !sp.result_qubit)) return fail(TNCB_ERR_INVALID, "null argument");
  for (size_t r = 0; r < k; r++)
    if (rm.dims[r] != 2) return fail(TNCB_ERR_INVALID, "result leg " + std::to_string(r) + " has dimension " + std::to_string(rm.dims[r]) + ", not 2");
  const std::vector<long long> elems = leaf_elems(S);
  std::vector<const SlotMeta*> meta(elems.size(), nullptr);
  for (const SlotMeta& m : S.slots) if (m.leaf_index >= 0) meta[m.leaf_index] = &m;
  std::vector<char> seen(elems.size(), 0), taken(sp.n_qubits, 0);
  auto qubit = [&](int q, const std::string& what) -> int {
    if (q < 0 || q >= sp.n_qubits) return fail(TNCB_ERR_INVALID, what + " is qubit " + std::to_string(q) + ", outside 0.." + std::to_string(sp.n_qubits - 1));
    if (taken[q]) return fail(TNCB_ERR_INVALID, "qubit " + std::to_string(q) + " is listed twice (" + what + ")");
    taken[q] = 1;
    return TNCB_OK;
  };
  for (size_t j = 0; j < sp.n_closed; j++) {
    const uint64_t li = sp.closed_leaf[j];
    const std::string name = "closed leaf " + std::to_string(li);
    if (int rc = listed_leaf(elems, seen, li, name)) return rc;
    if (meta[li]->dims.size() != 1 || meta[li]->dims[0] != 2) return fail(TNCB_ERR_INVALID, name + " is not a rank-1 leaf of dimension 2");
    if (int rc = qubit(sp.closed_qubit[j], "closed qubit " + std::to_string(j))) return rc;
    map->closed_qubit[j] = (unsigned char)sp.closed_qubit[j];
  }
  for (size_t r = 0; r < k; r++) {
    if (int rc = qubit(sp.result_qubit[r], "result leg " + std::to_string(r))) return rc;
    map->result_qubit[r] = (unsigned char)sp.result_qubit[r];
  }
  for (int q = 0; q < sp.n_qubits; q++)
    if (!taken[q]) return fail(TNCB_ERR_INVALID, "qubit " + std::to_string(q) + " is neither closed nor on a result leg");
  map->n_qubits = sp.n_qubits; map->n_closed = (int)sp.n_closed; map->k = (int)k;
  return TNCB_OK;
}

// the output buffer `name` of tncb_plan_sample: 8-byte aligned device memory of the ctx's device holding max_samples words
static int sample_output(const tncb_ctx* ctx, const void* p, uint64_t max_samples, const char* name) {
  unsigned long long bytes = 0;
  if ((uintptr_t)p % 8) return fail(TNCB_ERR_INVALID, std::string(name) + ": the buffer is not 8-byte aligned");
  if (__builtin_mul_overflow((unsigned long long)max_samples, 8ull, &bytes)) return fail(TNCB_ERR_INVALID, std::string(name) + ": max_samples words overflow 64 bits");
  int rc = device_memory(ctx, p, name, "the buffer");
  return rc ? rc : in_allocation(p, bytes, name, "the buffer");
}

// Sampling (tncb.h, DESIGN §5) on the instance-batched path of tncb_plan_hvp_batch: per pass of c candidates the candidate
// kernel writes the closed bras, run_instances stages them as device payloads (the staged block's other leaves at
// stride 0) and runs the forward levels, the select kernel reads every candidate's amplitudes in place and the compact
// kernel writes the accepted samples in candidate order; one device-to-host copy of the pass's counts decides whether
// another pass runs.  No leaf bytes come from the host.
// sliced (tncb_plan_sample_slices): the other leaves come from each network staged by tncb_plan_stage_slices in turn,
// and after each one's forward levels the accumulate kernel folds every candidate's result into its row of a [c, 2^k]
// block, which the select kernel then reads instead of the workspaces.  When no copy fits beside the plan's workspace
// the pass runs one candidate in that workspace (PassHook::in_place).
static int sample_call(tncb_ctx* ctx, tncb_plan* plan, const tncb_sample_spec* spec, uint64_t seed, uint64_t first,
                       uint64_t max_candidates, uint64_t max_samples, double m, size_t batch, uint64_t* bits, double* probs,
                       tncb_sample_stats* stats, bool sliced) {
  if (!ctx || !plan || !spec || !bits || !stats) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, sliced ? Call::sample_slices : Call::sample);
  if (rc) return rc;
  if (!plan->is_static) return fail(TNCB_ERR_UNSUPPORTED, "sampling needs a plan with a static layout (no device leaves)");
  if (sliced) {
    if (!plan->slices_dev || plan->ctx != ctx) return fail(TNCB_ERR_INVALID, "tncb_plan_stage_slices has not been called on this context");
  } else if (plan->ctx != ctx || !plan->leaves_resident) {
    return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan and context");
  }
  const Schedule& S = plan->S;
  SampleMap map{};
  if ((rc = sample_map(S, *spec, &map))) return rc;
  if (!std::isfinite(m) || !(m > 0)) return fail(TNCB_ERR_INVALID, "m must be finite and > 0, got " + std::to_string(m));
  if (max_samples == 0) return fail(TNCB_ERR_INVALID, "max_samples is 0");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  if ((rc = sample_output(ctx, bits, max_samples, "bits")) || (probs && (rc = sample_output(ctx, probs, max_samples, "probs")))) return rc;
  tncb_sample_stats st{};
  if (max_candidates == 0) { *stats = st; return TNCB_OK; }
  const size_t nc = spec->n_closed;
  const size_t res_elems = std::max<size_t>(S.slots[S.result_slot].elems, 1);
  // the closed bras as device payloads, two elements apart from candidate to candidate; their sources are set once the
  // pass size is known
  std::vector<LeafStageItem> dev_items;
  std::vector<long long> closed_dst(nc);
  for (size_t j = 0; j < nc; j++) {
    closed_dst[j] = (long long)S.leaf_offset[spec->closed_leaf[j]];
    dev_items.push_back({nullptr, 2, closed_dst[j], 2});
  }
  const std::vector<LeafRun> runs = leaf_runs(dev_items, (long long)std::max<size_t>(S.leaf_block_elems, 1));
  void* blk = nullptr;
  size_t blk_bytes = 0, c = 0;
  double2 *bras = nullptr, *uv = nullptr, *acc = nullptr;
  unsigned long long* closed_bits = nullptr;
  SampleCand* cand = nullptr;
  SampleCounts* d_counts = nullptr;
  PassHook hook;
  hook.width = batch;
  hook.in_place = sliced;
  hook.begin = [&](size_t pass) -> int {
    auto up = [](size_t b) { return (b + 255) / 256 * 256; };
    c = pass;
    const size_t o_bras = sliced ? up(c * res_elems * sizeof(double2)) : 0;
    const size_t o_uv = o_bras + up(nc * c * 2 * sizeof(double2)), o_bits = o_uv + up(c * sizeof(double2));
    const size_t o_cand = o_bits + up(c * sizeof(unsigned long long)), o_counts = o_cand + up(c * sizeof(SampleCand));
    blk_bytes = o_counts + sizeof(SampleCounts);
    if (int r = ctx->arena.alloc(blk_bytes, &blk)) return r;
    char* b = (char*)blk;
    if (sliced) acc = (double2*)b;
    bras = (double2*)(b + o_bras); uv = (double2*)(b + o_uv); closed_bits = (unsigned long long*)(b + o_bits);
    cand = (SampleCand*)(b + o_cand); d_counts = (SampleCounts*)(b + o_counts);
    for (LeafStageItem& it : dev_items)
      it.src = bras + (size_t)(std::find(closed_dst.begin(), closed_dst.end(), it.dst) - closed_dst.begin()) * c * 2;
    return TNCB_OK;
  };
  hook.fill = [&](size_t done, size_t n) -> int { return launch_sample_candidates(ctx, seed, first + done, n, c, map, bras, uv, closed_bits); };
  hook.fold = [&](size_t q, const char* base, size_t ws, size_t n) -> int {
    return launch_sample_accumulate(ctx, base, (long long)ws, (long long)plan->slot_off[S.result_slot], n, res_elems, q == 0, acc);
  };
  hook.end = [&](const char* base, size_t ws, size_t n, bool* stop) -> int {
    int r = sliced ? launch_sample_select(ctx, (const char*)acc, (long long)(res_elems * sizeof(double2)), 0, n, m, map, uv, closed_bits, cand)
                   : launch_sample_select(ctx, base, (long long)ws, (long long)plan->slot_off[S.result_slot], n, m, map, uv, closed_bits, cand);
    if (!r) r = launch_sample_compact(ctx, cand, n, max_samples - st.samples, (unsigned long long*)bits + st.samples,
                                      probs ? probs + st.samples : nullptr, d_counts);
    if (r) return r;
    SampleCounts h{};
    TNCB_CUDA(cudaMemcpyAsync(&h, d_counts, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    TNCB_CUDA(cudaStreamSynchronize(ctx->stream));
    st.candidates += h.consumed; st.samples += h.accepted; st.clipped += h.clipped; st.passes++;
    st.max_ratio = std::max(st.max_ratio, h.max_ratio);
    *stop = st.samples == max_samples;
    return TNCB_OK;
  };
  InstanceIO io;
  io.hook = &hook;
  rc = run_instances(ctx, plan, std::vector<uint64_t>{max_candidates}, {0, &dev_items, &runs, sliced ? plan->n_slices : 0}, io);
  if (blk) ctx->arena.free(blk, blk_bytes);
  if (rc) return rc;
  *stats = st;
  return TNCB_OK;
}
} // namespace tncb

int tncb_plan_sample(tncb_ctx* ctx, tncb_plan* plan, const tncb_sample_spec* spec, uint64_t seed, uint64_t first,
                     uint64_t max_candidates, uint64_t max_samples, double m, size_t batch, uint64_t* bits, double* probs,
                     tncb_sample_stats* stats) {
  return tncb::sample_call(ctx, plan, spec, seed, first, max_candidates, max_samples, m, batch, bits, probs, stats, false);
}

// A candidate's amplitudes are the sum over the S staged slices, R_0 copied, then R_1, R_2, ... added: the fold
// tncb_plan_run_slices(0, 1) forms.
int tncb_plan_sample_slices(tncb_ctx* ctx, tncb_plan* plan, const tncb_sample_spec* spec, uint64_t seed, uint64_t first,
                            uint64_t max_candidates, uint64_t max_samples, double m, size_t batch, uint64_t* bits,
                            double* probs, tncb_sample_stats* stats) {
  return tncb::sample_call(ctx, plan, spec, seed, first, max_candidates, max_samples, m, batch, bits, probs, stats, true);
}

namespace tncb {
// The observable layer of tncb_plan_expect against the plan: every layer leaf a listed, rank-2 leaf of dims [2, 2] with a
// payload, on a distinct qubit in 0 .. n_qubits - 1; *mask gets the layer's qubits
static int expect_layer_map(const Schedule& S, const tncb_pauli_layer& L, ExpectLayer* map, uint64_t* mask) {
  if (L.n_qubits < 1 || L.n_qubits > 64) return fail(TNCB_ERR_INVALID, "n_qubits " + std::to_string(L.n_qubits) + " is outside 1..64");
  if (L.n_layer && (!L.layer_leaf || !L.layer_qubit)) return fail(TNCB_ERR_INVALID, "null argument");
  const std::vector<long long> elems = leaf_elems(S);
  std::vector<const SlotMeta*> meta(elems.size(), nullptr);
  for (const SlotMeta& m : S.slots) if (m.leaf_index >= 0) meta[m.leaf_index] = &m;
  std::vector<char> seen(elems.size(), 0);
  *mask = 0;
  for (size_t j = 0; j < L.n_layer; j++) {
    const uint64_t li = L.layer_leaf[j];
    const std::string name = "layer leaf " + std::to_string(li);
    if (int rc = listed_leaf(elems, seen, li, name)) return rc;
    const std::vector<uint64_t>& d = meta[li]->dims;
    if (d.size() != 2 || d[0] != 2 || d[1] != 2) return fail(TNCB_ERR_INVALID, name + " is not a rank-2 leaf with dims [2, 2]");
    const int q = L.layer_qubit[j];
    if (q < 0 || q >= L.n_qubits)
      return fail(TNCB_ERR_INVALID, "layer qubit " + std::to_string(j) + " is qubit " + std::to_string(q) + ", outside 0.." + std::to_string(L.n_qubits - 1));
    if ((*mask >> q) & 1) return fail(TNCB_ERR_INVALID, "qubit " + std::to_string(q) + " is listed twice (layer qubit " + std::to_string(j) + ")");
    *mask |= 1ull << q;
    map->qubit[j] = (unsigned char)q;
  }
  map->n_layer = (int)L.n_layer;
  return TNCB_OK;
}
} // namespace tncb

// Expectation values of a Pauli sum (tncb.h, DESIGN §5) on the instance-batched path of tncb_plan_sample: the term table
// goes to the device in one copy; per pass of c terms the layer kernel writes the terms' layer payloads, run_instances
// stages them as device payloads (the staged block's other leaves at stride 0), runs the forward levels and copies the
// value rows out, and with grad_sum writes the seeds c_k, runs the backward levels and folds Σ_k c_k G_k in term order.
// The fold kernel forms the energy from the value rows after the last pass.  No leaf bytes come from the host.
int tncb_plan_expect(tncb_ctx* ctx, tncb_plan* plan, const tncb_pauli_layer* layer, size_t n_terms, const uint64_t* x_mask,
                     const uint64_t* z_mask, const double* coeff, size_t batch, tncb_tensor** values, tncb_tensor** energy,
                     tncb_tensor** grad_sum) {
  using namespace tncb;
  if (!ctx || !plan || !layer || !x_mask || !z_mask || !coeff) return fail(TNCB_ERR_INVALID, "null argument");
  int rc = route(plan, Call::expect);
  if (rc) return rc;
  if (!plan->is_static) return fail(TNCB_ERR_UNSUPPORTED, "expectation values need a plan with a static layout (no device leaves)");
  if (plan->ctx != ctx || !plan->leaves_resident) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan and context");
  if (n_terms == 0) return fail(TNCB_ERR_INVALID, "n_terms is 0");
  if (!values && !energy && !grad_sum) return fail(TNCB_ERR_INVALID, "no output requested");
  if (grad_sum && !plan->grad()) return fail(TNCB_ERR_INVALID, "grad_sum needs a gradient plan (tncb_plan_create_vjp)");
  const Schedule& S = plan->S;
  if (S.result_slot < 0 || !S.slots[S.result_slot].dims.empty())
    return fail(TNCB_ERR_INVALID, "the network does not contract to a scalar (" + std::to_string(S.result_slot < 0 ? 0 : S.slots[S.result_slot].dims.size()) + " result legs)");
  ExpectLayer map{};
  uint64_t mask = 0;
  if ((rc = expect_layer_map(S, *layer, &map, &mask))) return rc;
  for (size_t k = 0; k < n_terms; k++) {
    const uint64_t off = (x_mask[k] | z_mask[k]) & ~mask;
    if (off) return fail(TNCB_ERR_INVALID, "term " + std::to_string(k) + " acts on qubit " + std::to_string(__builtin_ctzll(off)) + ", which has no layer leaf");
    if (!std::isfinite(coeff[k])) return fail(TNCB_ERR_INVALID, "the coefficient of term " + std::to_string(k) + " is not finite");
  }
  TNCB_CUDA(cudaSetDevice(ctx->device));
  // the term table, [x masks][z masks][seeds (c_k, 0)], in one host-to-device copy
  const size_t o_z = n_terms * sizeof(uint64_t), o_seeds = 2 * o_z, table_bytes = o_seeds + n_terms * sizeof(double2);
  std::vector<char> host(table_bytes);
  std::memcpy(host.data(), x_mask, o_z);
  std::memcpy(host.data() + o_z, z_mask, o_z);
  for (size_t k = 0; k < n_terms; k++) ((double2*)(host.data() + o_seeds))[k] = make_double2(coeff[k], 0.0);
  void* table = nullptr;
  if ((rc = ctx->arena.alloc(table_bytes, &table))) return rc;
  cudaError_t e = cudaMemcpyAsync(table, host.data(), table_bytes, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);      // `host` dies with this scope
  if (e != cudaSuccess) { ctx->arena.free(table, table_bytes); return fail(TNCB_ERR_CUDA, std::string("term table copy: ") + cudaGetErrorString(e)); }
  const unsigned long long* d_x = (const unsigned long long*)table;
  const unsigned long long* d_z = (const unsigned long long*)((char*)table + o_z);
  const double2* d_seeds = (const double2*)((char*)table + o_seeds);
  // the layer payloads as device payloads, four elements apart from term to term; their sources are set once the pass
  // size is known
  std::vector<LeafStageItem> dev_items;
  std::vector<long long> layer_dst(layer->n_layer);
  for (size_t j = 0; j < layer->n_layer; j++) {
    layer_dst[j] = (long long)S.leaf_offset[layer->layer_leaf[j]];
    dev_items.push_back({nullptr, 4, layer_dst[j], 4});
  }
  const std::vector<LeafRun> runs = leaf_runs(dev_items, (long long)std::max<size_t>(S.leaf_block_elems, 1));
  void* blk = nullptr;
  size_t blk_bytes = 0, c = 0;
  PassHook hook;
  hook.width = batch;
  hook.begin = [&](size_t pass) -> int {
    c = pass;
    blk_bytes = std::max<size_t>(layer->n_layer * c * 4 * sizeof(double2), 16);
    if (int r = ctx->arena.alloc(blk_bytes, &blk)) return r;
    for (LeafStageItem& it : dev_items)
      it.src = (const double2*)blk + (size_t)(std::find(layer_dst.begin(), layer_dst.end(), it.dst) - layer_dst.begin()) * c * 4;
    return TNCB_OK;
  };
  hook.fill = [&](size_t done, size_t n) -> int { return launch_expect_layer(ctx, d_x, d_z, done, n, c, map, (double2*)blk); };
  hook.end = [](const char*, size_t, size_t, bool*) -> int { return TNCB_OK; };
  Outputs out{ctx};
  tncb_tensor* en = out.add(energy, 0, nullptr);
  tncb_tensor *vals = nullptr, *gs = nullptr;
  tncb_tensor seeds;
  seeds.ptr = (double2*)d_seeds; seeds.rank = 1; seeds.dims[0] = n_terms; seeds.elems = n_terms; seeds.owned = false;
  InstanceIO io;
  io.hook = &hook;
  io.values = &vals;
  if (grad_sum) { io.grad_sum = &gs; io.seeds = &seeds; }
  if (!(rc = out.rc)) rc = run_instances(ctx, plan, std::vector<uint64_t>{n_terms}, {0, &dev_items, &runs}, io);
  if (blk) ctx->arena.free(blk, blk_bytes);
  if (!rc && en) rc = launch_expect_fold(ctx, vals->ptr, d_seeds, n_terms, en->ptr);
  ctx->arena.free(table, table_bytes);          // stream-ordered: after the passes and the fold
  if (rc) {
    for (tncb_tensor* t : {vals, gs}) if (t) tncb_tensor_free(ctx, t);
    return out.finish(rc);
  }
  if (values) *values = vals; else tncb_tensor_free(ctx, vals);
  if (grad_sum) *grad_sum = gs;
  return out.finish(TNCB_OK);
}

namespace tncb {
// tncb_plan_jvp_sliced / tncb_plan_hvp_sliced: the arguments, the outputs (any may be NULL), one run_sliced
static int sliced_tangent_call(tncb_ctx* ctx, tncb_plan* plan, bool hvp, size_t first, size_t stride, const tncb_tensor* tangents,
                               const tncb_tensor* seed, const tncb_tensor* seed_tangent, tncb_tensor** value,
                               tncb_tensor** tangent_out, tncb_tensor** grads, tncb_tensor** grad_tangents) {
  if (!ctx || !plan || stride == 0) return fail(TNCB_ERR_INVALID, "bad argument");
  int rc = route(plan, hvp ? Call::hvp_sliced : Call::jvp_sliced);
  if (rc || (rc = jvp_args(tangents, value || tangent_out || grads || grad_tangents, {plan->grad_elems}))) return rc;
  const SlotMeta& rm = plan->S.slots[plan->S.result_slot];
  if (hvp && ((rc = seed_args(rm, seed, "seed", true)) || (rc = seed_args(rm, seed_tangent, "seed tangent")))) return rc;
  if (plan->ctx != ctx || !plan->full_staged) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this context");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  const uint64_t ge = plan->grad_elems;
  Outputs out{ctx};
  tncb_tensor* v = out.add(value, (int)rm.dims.size(), rm.dims.data());
  tncb_tensor* t = out.add(tangent_out, (int)rm.dims.size(), rm.dims.data());
  tncb_tensor* g = out.add(grads, 1, &ge);
  tncb_tensor* dg = out.add(grad_tangents, 1, &ge);
  if (!(rc = out.rc)) {
    SliceRun io;
    io.tangents = tangents->ptr;
    io.seed = seed ? seed->ptr : nullptr; io.seed_tan = seed_tangent ? seed_tangent->ptr : nullptr;
    io.value = v ? v->ptr : nullptr; io.tan_value = t ? t->ptr : nullptr;
    io.grad = g ? g->ptr : nullptr; io.dgrad = dg ? dg->ptr : nullptr;
    rc = run_sliced(ctx, plan, first, stride, io);
  }
  return out.finish(rc);
}
} // namespace tncb

// Per slice first, first+stride, ...: extract (sliced leaves, every leaf tangent), forward levels with their tangent
// pairs, R += and Ṙ +=.  No host work per slice; slices run in stream order, so a call repeats bit for bit.
int tncb_plan_jvp_sliced(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, const tncb_tensor* tangents,
                         tncb_tensor** value, tncb_tensor** tangent_out) {
  return tncb::sliced_tangent_call(ctx, plan, false, first, stride, tangents, nullptr, nullptr, value, tangent_out, nullptr, nullptr);
}

// As tncb_plan_jvp_sliced, then per slice the seed and its tangent, the backward levels with their tangent pairs, K3 of the
// many-group adjoints and adjoint tangents, and the accumulation of G and Ġ into the full-shape blocks.
int tncb_plan_hvp_sliced(tncb_ctx* ctx, tncb_plan* plan, size_t first, size_t stride, const tncb_tensor* tangents,
                         const tncb_tensor* seed, const tncb_tensor* seed_tangent, tncb_tensor** value,
                         tncb_tensor** tangent_out, tncb_tensor** grads, tncb_tensor** grad_tangents) {
  return tncb::sliced_tangent_call(ctx, plan, true, first, stride, tangents, seed, seed_tangent, value, tangent_out, grads, grad_tangents);
}

// New payloads for some leaves of the staged network, straight from device memory: one launch on the ctx stream into the
// leaf block the next run reads (a static plan's workspace block, which its graph replays also read; a non-static plan's
// resident block; a sliced gradient plan's full block).  The static layout never releases its leaf block, so the new
// payloads stay in place across runs and tncb_plan_vjp, as staged leaves do.
int tncb_plan_set_leaves(tncb_ctx* ctx, tncb_plan* plan, size_t n, const uint64_t* leaf_index, const void* const* src) {
  using namespace tncb;
  if (!ctx || !plan || (n && (!leaf_index || !src))) return fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = route(plan, Call::set_leaves)) return rc;
  for (int k : plan->S.leaf_kind)
    if (k == TNCB_DATA_DEVICE) return fail(TNCB_ERR_UNSUPPORTED, "plans with device leaves cannot be staged (they are consumed per call)");
  const Schedule* S = &plan->S;
  double2* block = nullptr;
  if (plan->ctx == ctx) {
    if (plan->sliced) { if (plan->full_staged) { S = &plan->full; block = (double2*)plan->full_dev; } }
    else if (plan->is_static) { if (plan->leaves_resident) block = (double2*)((char*)plan->ws + plan->leaf_off); }
    else block = (double2*)plan->resident;
  }
  if (!block) return fail(TNCB_ERR_INVALID, "tncb_plan_stage has not been called on this plan and context");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  std::vector<LeafStageItem> items;
  int rc = device_items(ctx, *S, 1, n, leaf_index, src, nullptr, items);
  if (rc || n == 0) return rc;
  plan->fwd_ready = false;     // a gradient plan's forward state belongs to the old payloads
  return launch_leaf_stage(ctx, items.data(), items.size(), block, 0, 1);
}

// n_instances networks of the plan's structure, for tncb_plan_run_slices / run_batch (plain plans) or
// tncb_plan_vjp_batch (gradient plans).  The host work is O(leaves) whatever n_instances is: the template's other leaves
// are materialised once, packed into plan-owned pinned memory, uploaded in one copy; then one launch per 65535 instances
// (and per kStageItems items) fills every instance's leaf block, the device payloads in place, the template's runs
// between them with stride 0.  No host synchronisation once the arguments are validated.
int tncb_plan_stage_instances(tncb_ctx* ctx, tncb_plan* plan, const tncb_tn* tmpl, size_t n_instances, size_t n,
                              const uint64_t* leaf_index, const void* const* src, const uint64_t* instance_stride) {
  using namespace tncb;
  if (!ctx || !plan || !tmpl || (n && (!leaf_index || !src || !instance_stride))) return fail(TNCB_ERR_INVALID, "null argument");
  if (int rc = route(plan, Call::stage_instances)) return rc;
  const Schedule& S = plan->S;
  for (int k : S.leaf_kind)
    if (k == TNCB_DATA_DEVICE) return fail(TNCB_ERR_UNSUPPORTED, "plans with device leaves cannot be staged (they are consumed per call)");
  if (!plan->grad() && !plan->is_static) return fail(TNCB_ERR_UNSUPPORTED, "many networks need a plan with a static layout");
  if (plan->ctx && plan->ctx != ctx) return fail(TNCB_ERR_INVALID, "plan belongs to another context");
  if (n_instances == 0) return fail(TNCB_ERR_INVALID, "n_instances is 0");
  TNCB_CUDA(cudaSetDevice(ctx->device));
  std::vector<const tncb_tn*> leaves;
  collect_leaf_nodes(tmpl, leaves);
  int rc = validate_leaves(S, leaves);
  if (rc) return rc;
  std::vector<LeafStageItem> items;
  if ((rc = device_items(ctx, S, n_instances, n, leaf_index, src, instance_stride, items))) return rc;
  const size_t block = std::max<size_t>(S.leaf_block_elems, 1);
  size_t bytes = 0;
  if (__builtin_mul_overflow(n_instances, block * sizeof(double2), &bytes)) return fail(TNCB_ERR_OOM, "the instances' leaf blocks overflow 64 bits");
  // the runs of the leaf block between the device payloads come from the template, packed
  const std::vector<LeafRun> runs = leaf_runs(items, (long long)block);
  if ((rc = plan_device_state(ctx, plan, !plan->grad() && !plan->tangent()))) return rc;
  if (!plan->tmpl_host) {
    plan->tmpl_bytes = block * sizeof(double2);
    TNCB_CUDA(cudaMallocHost(&plan->tmpl_host, plan->tmpl_bytes));
    if ((rc = ctx->arena.alloc(plan->tmpl_bytes, &plan->tmpl_dev))) { cudaFreeHost(plan->tmpl_host); plan->tmpl_host = nullptr; return rc; }
    TNCB_CUDA(cudaEventCreateWithFlags(&plan->tmpl_ev, cudaEventDisableTiming));
  } else if (plan->tmpl_busy) {
    TNCB_CUDA(cudaEventSynchronize(plan->tmpl_ev));   // the previous call's upload out of tmpl_host has run
    plan->tmpl_busy = false;
  }
  std::vector<char> device_leaf(leaves.size(), 0);
  for (size_t k = 0; k < n; k++) device_leaf[leaf_index[k]] = 1;
  std::complex<double>* host = (std::complex<double>*)plan->tmpl_host;
  for (size_t li = 0; li < leaves.size(); li++) {
    if (device_leaf[li] || S.leaf_kind[li] == TNCB_DATA_UNCONTRACTED) continue;
    const long long off = (long long)S.leaf_offset[li];
    const LeafRun& r = *(std::upper_bound(runs.begin(), runs.end(), off, [](long long o, const LeafRun& x) { return o < x.start; }) - 1);
    if ((rc = stage_leaf(leaves[li], host + r.packed + (off - r.start)))) return rc;
  }
  void* blk = nullptr;
  if ((rc = ctx->arena.alloc(bytes, &blk))) return rc;
  const long long packed = runs.empty() ? 0 : runs.back().packed + runs.back().len;
  if (packed) {
    cudaError_t e = cudaMemcpyAsync(plan->tmpl_dev, plan->tmpl_host, packed * sizeof(double2), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaEventRecord(plan->tmpl_ev, ctx->stream);
    if (e != cudaSuccess) { ctx->arena.free(blk, bytes); return fail(TNCB_ERR_CUDA, std::string("template upload: ") + cudaGetErrorString(e)); }
    plan->tmpl_busy = true;
  }
  for (const LeafRun& r : runs) items.push_back({(const double2*)plan->tmpl_dev + r.packed, 0, r.start, r.len});
  if ((rc = launch_leaf_stage(ctx, items.data(), items.size(), (double2*)blk, (long long)block, n_instances))) {
    ctx->arena.free(blk, bytes);
    return rc;
  }
  if (plan->slices_dev) ctx->arena.free(plan->slices_dev, plan->slices_bytes);   // stream-ordered
  plan->slices_dev = blk;
  plan->slices_bytes = bytes;
  plan->n_slices = n_instances;
  return TNCB_OK;
}

// Legs and bond dimensions of contract_tensor_network(tn, path) from metadata alone (no GPU work): what a receiver of the
// fan-in needs to know about a raw buffer it is about to get (communication.rs:221-226; the reference ships the legs inside
// the serialised tensor instead).
int tncb_network_out_legs(const tncb_tn* tn, const tncb_path* path, int* n_out, uint64_t* out_legs, uint64_t* out_dims) {
  if (!tn || !n_out) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  tncb::Schedule S;
  int rc = tncb::build_schedule(tn, path, S);
  if (rc) return rc;
  if (S.result_slot < 0) { *n_out = 0; return TNCB_OK; }
  const tncb::SlotMeta& m = S.slots[S.result_slot];
  *n_out = (int)m.legs.size();
  for (size_t i = 0; i < m.legs.size(); i++) {
    if (out_legs) out_legs[i] = m.legs[i];
    if (out_dims) out_dims[i] = m.dims[i];
  }
  return TNCB_OK;
}

int tncb_plan_info(const tncb_plan* plan, uint64_t* n_pairs, double* flops, double* bytes, uint64_t* peak_bytes, uint64_t* n_kernels) {
  if (!plan) return tncb::fail(TNCB_ERR_INVALID, "plan is null");
  const tncb::Schedule& S = plan->S;
  if (n_pairs) *n_pairs = S.steps.size();
  if (flops) *flops = S.flops;
  if (bytes) *bytes = S.bytes;
  if (peak_bytes && (plan->grad() || plan->tangent())) *peak_bytes = plan->ws_bytes;   // the whole pass lives in its static workspace
  else if (peak_bytes) { // replay the liveness: leaves + live intermediates
    size_t live = S.leaf_block_elems * 16, peak = live;
    std::vector<size_t> sz(S.slots.size(), 0);
    for (const tncb::Step& st : S.steps) {
      sz[st.out] = std::max<size_t>(S.slots[st.out].elems * 16, 256);
      live += sz[st.out]; peak = std::max(peak, live);
      live -= sz[st.a] + sz[st.b]; sz[st.a] = sz[st.b] = 0;
    }
    *peak_bytes = peak;
  }
  if (n_kernels) {
    uint64_t k = 0;
    for (const tncb::Step& st : S.steps) k += st.plan.kernel_class == 1 ? 2 : 1;  // (K1: table build + GEMM)
    for (int nb : plan->level_batched) if (nb) k -= (uint64_t)(nb - 1);            // a batch is one launch
    if (!plan->grad_items.empty()) k++;                                            // the leaf-gradient gather
    if (!plan->dgrad_items.empty()) k++;                                           // ... and of the gradients' tangents
    if (!plan->acc_items.empty()) k++;                                            // a slice's gradient accumulation
    if (!plan->sl_items.empty()) k++;                                              // a slice's leaf extraction
    if (!plan->dacc_items.empty()) k++;                                            // ... accumulation of the adjoints' tangents
    if (plan->sliced) k += !plan->tan_items.empty();                               // ... and extraction of the leaf tangents
    else k += (plan->tan_leaves.size() + tncb::kStageItems - 1) / tncb::kStageItems;   // the leaf tangents' staging
    for (int ns : plan->sum_count) if (ns) k++;                                    // a level's tangent sums
    *n_kernels = k + 2 * (plan->grad_permutes.size() + plan->dgrad_permutes.size());   // (K3: tables + transpose)
  }
  return TNCB_OK;
}

// Releases everything a plan holds on its context (graph, workspace, staging) and detaches it.  Called by
// tncb_plan_destroy and by tncb_ctx_destroy for plans that outlive their context (either order is safe).
void tncb_plan_release_device_state(tncb_plan* plan) {
  tncb_ctx* ctx = plan->ctx;
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (int i = 0; i < 2; i++) if (plan->exec[i]) { cudaGraphExecDestroy(plan->exec[i]); plan->exec[i] = nullptr; }
  for (auto [dev, bytes] : {std::pair<void**, size_t>{&plan->batch_dev, plan->batch_bytes}, {&plan->grad_dev, plan->grad_dev_bytes},
                            {&plan->dgrad_dev, plan->dgrad_dev_bytes}, {&plan->sum_dev, plan->sum_dev_bytes},
                            {&plan->sl_dev, plan->sl_dev_bytes}})
    if (*dev) { ctx->arena.free(*dev, bytes); *dev = nullptr; }
  if (plan->full_dev) { ctx->arena.free(plan->full_dev, plan->full_bytes); plan->full_dev = nullptr; }
  plan->full_staged = false;
  plan->fwd_ready = false;
  if (plan->slices_dev) { ctx->arena.free(plan->slices_dev, plan->slices_bytes); plan->slices_dev = nullptr; plan->n_slices = 0; }
  plan->leaves_resident = false;
  if (plan->ws) { ctx->arena.free(plan->ws, plan->ws_bytes); plan->ws = nullptr; }
  if (plan->stage) { cudaFreeHost(plan->stage); plan->stage = nullptr; }
  if (plan->stage_ev) { cudaEventDestroy(plan->stage_ev); plan->stage_ev = nullptr; plan->stage_busy = false; }
  if (plan->resident) { ctx->arena.free(plan->resident, plan->resident_bytes); plan->resident = nullptr; }
  if (plan->tmpl_dev) { ctx->arena.free(plan->tmpl_dev, plan->tmpl_bytes); plan->tmpl_dev = nullptr; }
  if (plan->tmpl_host) { cudaFreeHost(plan->tmpl_host); plan->tmpl_host = nullptr; }
  if (plan->tmpl_ev) { cudaEventDestroy(plan->tmpl_ev); plan->tmpl_ev = nullptr; plan->tmpl_busy = false; }
  for (size_t i = 0; i < ctx->plans.size(); i++)
    if (ctx->plans[i] == plan) { ctx->plans.erase(ctx->plans.begin() + i); break; }
  plan->ctx = nullptr;
}

void tncb_plan_destroy(tncb_plan* plan) {
  if (!plan) return;
  tncb_plan_release_device_state(plan);
  delete plan;
}

} // extern "C"
