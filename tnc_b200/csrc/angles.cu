// Angle maps: the gate leaves of a network as functions of real parameters θ, on the device.
//
// A map ties angle slots of Gate leaves to scale * θ[param] (tncb_angles_create) and places every referenced leaf in a
// block of complex elements (usually a gradient plan's tncb_plan_grad_offsets layout).  Three calls turn θ into the
// leaf payloads (gates), θ and a direction θ̇ into leaf tangents (tangents), and leaf gradients G (and Ġ) into the
// gradient with respect to θ (pullback).  They feed and read the existing plan calls; no plan is involved here.
// The gate formulas are those of gate_angles.h, shared with the host table.
#include "internal.h"
#include "gate_angles.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace tncb {
// one referenced leaf: the element offset in the block, the gate, its own angles and its refs refs[first, first + n)
struct AngleLeaf {
  long long off;
  int gate, adjoint, first, n;
  double a[3];
};
struct AngleRef { int leaf, slot, param, _pad; double scale; };   // leaf: index into the AngleLeaf table

constexpr int kAngleThreads = 128;
}  // namespace tncb

struct tncb_angles {
  size_t n_params = 0, block_elems = 0;
  std::vector<int64_t> offsets;                    // per network leaf (collect order), -1 = not in the block
  std::vector<tncb::AngleLeaf> leaves;             // referenced leaves, in leaf order
  std::vector<tncb::AngleRef> refs;                // grouped by leaf, slots ascending within a leaf
  std::vector<int> order;                          // refs sorted by (param, leaf, slot)
  std::vector<int> pstart;                         // [n_params + 1]: param p folds order[pstart[p] .. pstart[p + 1])
  std::vector<char> table;                         // leaves, refs, order, pstart back to back (the device image)
  size_t off_refs = 0, off_order = 0, off_pstart = 0;
  struct Dev { tncb_ctx* ctx; void* ptr; };        // the image uploaded once per context
  std::vector<Dev> dev;
};

namespace tncb {

// ---- kernels ----
// the trigonometric values of leaf L in row th: its own angles, with every referenced slot replaced by scale * θ[param]
__device__ __forceinline__ ga::Trig leaf_trig(const AngleLeaf& L, const AngleRef* refs, const double* th) {
  double a0 = L.a[0], a1 = L.a[1], a2 = L.a[2];
  for (int k = L.first; k < L.first + L.n; k++) {
    const AngleRef r = refs[k];
    const double v = r.scale * th[r.param];
    if (r.slot == 0) a0 = v; else if (r.slot == 1) a1 = v; else a2 = v;
  }
  return ga::trig(L.gate, a0, a1, a2);
}

// thread (leaf j / 16, element j % 16) of row i: U(θ_i) (dot == nullptr) or sum over the leaf's refs of
// scale * θ̇_i[param] * dU/da_slot into rows[i]
__global__ void __launch_bounds__(kAngleThreads) angle_leaves_kernel(const AngleLeaf* leaves, const AngleRef* refs, int n_leaves,
                                                                     const double* theta, unsigned long long th_stride,
                                                                     const double* dot, unsigned long long dot_stride,
                                                                     unsigned long long count, long long block, double2* rows) {
  const long long j = (long long)blockIdx.x * kAngleThreads + threadIdx.x;
  if (j >= 16LL * n_leaves) return;
  const AngleLeaf L = leaves[j / 16];
  const int e = (int)(j % 16), d = ga::dim(L.gate);
  if (e >= d * d) return;
  for (unsigned long long i = blockIdx.y; i < count; i += gridDim.y) {
    const ga::Trig T = leaf_trig(L, refs, theta + i * th_stride);
    ga::Cplx v;
    if (!dot) {
      v = ga::element(L.gate, T, -1, -1, L.adjoint != 0, e);
    } else {
      const double* td = dot + i * dot_stride;
      v = {0.0, 0.0};
      for (int k = L.first; k < L.first + L.n; k++) {
        const AngleRef r = refs[k];
        const double w = r.scale * td[r.param];
        const ga::Cplx u = ga::element(L.gate, T, r.slot, -1, L.adjoint != 0, e);
        v.re += u.re * w;
        v.im += u.im * w;
      }
    }
    rows[i * block + L.off + e] = make_double2(v.re, v.im);
  }
}

// <A_L, d^k U_L> = sum_e A[e] * dU[e], no conjugation
__device__ __forceinline__ ga::Cplx leaf_dot(const AngleLeaf& L, const double2* A, const ga::Trig& T, int s, int t) {
  const int cnt = ga::dim(L.gate) * ga::dim(L.gate);
  ga::Cplx acc{0.0, 0.0};
  for (int e = 0; e < cnt; e++) {
    const double2 x = A[L.off + e];
    const ga::Cplx u = ga::element(L.gate, T, s, t, L.adjoint != 0, e);
    acc.re += x.x * u.re - x.y * u.im;
    acc.im += x.x * u.im + x.y * u.re;
  }
  return acc;
}

// thread (param p, row i): the sum over p's refs r, in (leaf, slot) order, of
//   scale_r * <G_l, dU/da_s>                                                          (Gdot == nullptr: g[p])
//   scale_r * ( <Ġ_l, dU/da_s> + sum_{r' on l} scale_r' v[p_r'] <G_l, d²U/da_s da_s'> )   (with Ġ and v: ġ[p])
__global__ void __launch_bounds__(kAngleThreads) angle_pullback_kernel(const AngleLeaf* leaves, const AngleRef* refs, const int* order,
                                                                       const int* pstart, int n_params, const double* theta,
                                                                       unsigned long long th_stride, unsigned long long count,
                                                                       const double2* G, const double2* Gdot, long long g_stride,
                                                                       const double* v, unsigned long long v_stride, long long block,
                                                                       double2* rows) {
  const int p = blockIdx.x * kAngleThreads + threadIdx.x;
  if (p >= n_params) return;
  for (unsigned long long i = blockIdx.y; i < count; i += gridDim.y) {
    const double* th = theta + i * th_stride;
    const double2* g = G + i * g_stride * block;
    const double2* gd = Gdot ? Gdot + i * g_stride * block : nullptr;
    const double* vi = v ? v + i * v_stride : nullptr;
    ga::Cplx acc{0.0, 0.0};
    for (int k = pstart[p]; k < pstart[p + 1]; k++) {
      const AngleRef r = refs[order[k]];
      const AngleLeaf L = leaves[r.leaf];
      const ga::Trig T = leaf_trig(L, refs, th);
      ga::Cplx t = leaf_dot(L, gd ? gd : g, T, r.slot, -1);
      if (gd) {
        for (int q = L.first; q < L.first + L.n; q++) {
          const AngleRef r2 = refs[q];
          const double w = r2.scale * vi[r2.param];
          const ga::Cplx h = leaf_dot(L, g, T, r.slot, r2.slot);
          t.re += h.re * w; t.im += h.im * w;
        }
      }
      acc.re += t.re * r.scale;
      acc.im += t.im * r.scale;
    }
    rows[i * n_params + p] = make_double2(acc.re, acc.im);
  }
}

// sum[p] = 0 + rows[0][p] + rows[1][p] + ...  (the left fold in row order)
__global__ void __launch_bounds__(kAngleThreads) angle_fold_kernel(const double2* rows, unsigned long long count, int n_params,
                                                                   double2* sum) {
  const int p = blockIdx.x * kAngleThreads + threadIdx.x;
  if (p >= n_params) return;
  double2 s = make_double2(0.0, 0.0);
  for (unsigned long long i = 0; i < count; i++) { const double2 x = rows[i * n_params + p]; s.x += x.x; s.y += x.y; }
  sum[p] = s;
}

// ---- host side ----
static void collect(const tncb_tn* tn, std::vector<const tncb_tn*>& v) {
  if (tn->n_children == 0) { v.push_back(tn); return; }
  for (size_t i = 0; i < tn->n_children; i++) collect(&tn->children[i], v);
}

template <class T> static size_t put(std::vector<char>& img, const std::vector<T>& v) {
  const size_t off = (img.size() + 15) / 16 * 16;
  img.resize(off + v.size() * sizeof(T));
  if (!v.empty()) std::memcpy(img.data() + off, v.data(), v.size() * sizeof(T));
  return off;
}

// the map's device image on ctx, uploaded on first use; *fresh = it was uploaded by this call
static int tables(tncb_ctx* ctx, tncb_angles* a, const char** dev, bool* fresh) {
  *fresh = false;
  for (const tncb_angles::Dev& d : a->dev) if (d.ctx == ctx) { *dev = (const char*)d.ptr; return TNCB_OK; }
  void* p = nullptr;
  if (int rc = ctx->arena.alloc(a->table.size(), &p)) return rc;
  cudaError_t e = cudaMemcpyAsync(p, a->table.data(), a->table.size(), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);   // (pageable source)
  if (e != cudaSuccess) { ctx->arena.free(p, a->table.size()); return fail(TNCB_ERR_CUDA, std::string("angle table upload: ") + cudaGetErrorString(e)); }
  a->dev.push_back({ctx, p});
  ctx->angle_maps.push_back(a);
  *dev = (const char*)p;
  *fresh = true;
  return TNCB_OK;
}

// drop the device image on ctx (tncb_angles_destroy, tncb_ctx_destroy)
void angles_release(tncb_angles* a, tncb_ctx* ctx) {
  for (size_t i = 0; i < a->dev.size(); i++)
    if (a->dev[i].ctx == ctx) {
      ctx->arena.free(a->dev[i].ptr, a->table.size());
      a->dev.erase(a->dev.begin() + i);
      break;
    }
  for (size_t i = 0; i < ctx->angle_maps.size(); i++)
    if (ctx->angle_maps[i] == a) { ctx->angle_maps.erase(ctx->angle_maps.begin() + i); break; }
}

// rows of count parameter vectors: device memory of ctx's device, 8-byte aligned, every byte read inside one allocation
static int check_rows(const tncb_ctx* ctx, const double* p, size_t stride, size_t count, size_t n_params, const char* what) {
  const std::string name = what;
  if (!p) return fail(TNCB_ERR_INVALID, name + " is null");
  if (stride != 0 && stride < n_params)
    return fail(TNCB_ERR_INVALID, name + ": row stride " + std::to_string(stride) + " is below the " + std::to_string(n_params) + " parameters");
  if ((uintptr_t)p % 8) return fail(TNCB_ERR_INVALID, name + " is not 8-byte aligned");
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return fail(TNCB_ERR_INVALID, name + " is not device memory"); }
  if (at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) return fail(TNCB_ERR_INVALID, name + " is not device memory");
  if (at.device != ctx->device)
    return fail(TNCB_ERR_INVALID, name + " is on device " + std::to_string(at.device) + ", the context on device " + std::to_string(ctx->device));
  unsigned long long span = 0, bytes = 0;
  if (__builtin_mul_overflow((unsigned long long)(count - 1), (unsigned long long)stride, &span) ||
      __builtin_add_overflow(span, (unsigned long long)n_params, &span) || __builtin_mul_overflow(span, 8ull, &bytes))
    return fail(TNCB_ERR_INVALID, name + ": the row range overflows 64 bits");
  const MemRangeFn range = get_mem_range();
  if (!range) return fail(TNCB_ERR_CUDA, "cuMemGetAddressRange is not available");
  CUdeviceptr base = 0;
  size_t size = 0;
  if (range(&base, &size, (CUdeviceptr)p) != CUDA_SUCCESS) return fail(TNCB_ERR_INVALID, name + ": no device allocation holds it");
  if ((unsigned long long)((CUdeviceptr)p - base) + bytes > size)
    return fail(TNCB_ERR_INVALID, name + ": its " + std::to_string(bytes) + " bytes run past the end of its allocation");
  return TNCB_OK;
}

// a block argument: [block_elems] (shared by every row, *stride = 0) or [count, block_elems] (*stride = 1)
static int check_block(const tncb_tensor* t, size_t count, size_t block, const char* what, long long* stride) {
  const std::string name = what;
  if (!t || !t->ptr) return fail(TNCB_ERR_INVALID, name + " is null");
  if (t->rank == 1 && t->dims[0] == block) { *stride = 0; return TNCB_OK; }
  if (t->rank == 2 && t->dims[0] == count && t->dims[1] == block) { *stride = 1; return TNCB_OK; }
  return fail(TNCB_ERR_SHAPE, name + " must be [" + std::to_string(block) + "] or [" + std::to_string(count) + ", " +
                                  std::to_string(block) + "]");
}

static unsigned grid_y(size_t count) { return (unsigned)std::min<size_t>(count, 65535); }

// the gates / tangents calls: validation, then the table, the zeroed rows and one launch
static int leaf_rows(tncb_ctx* ctx, tncb_angles* a, const double* theta, size_t theta_stride, const double* dot, size_t dot_stride,
                     size_t count, bool tangents, tncb_tensor** rows) {
  if (!ctx || !a || !rows) return fail(TNCB_ERR_INVALID, "null argument");
  if (count == 0) return fail(TNCB_ERR_INVALID, "count is 0");
  if (cudaSetDevice(ctx->device) != cudaSuccess) return fail(TNCB_ERR_CUDA, "cudaSetDevice failed");
  if (int rc = check_rows(ctx, theta, theta_stride, count, a->n_params, "theta")) return rc;
  if (tangents)
    if (int rc = check_rows(ctx, dot, dot_stride, count, a->n_params, "theta_dot")) return rc;
  const char* dev = nullptr;
  bool fresh = false;
  if (int rc = tables(ctx, a, &dev, &fresh)) return rc;
  const uint64_t dims[2] = {count, a->block_elems};
  tncb_tensor* out = nullptr;
  int rc = tensor_new(ctx, 2, dims, &out);
  if (!rc) {
    cudaError_t e = cudaMemsetAsync(out->ptr, 0, out->elems * sizeof(double2), ctx->stream);
    if (e == cudaSuccess) {
      const long long threads = 16LL * (long long)a->leaves.size();
      dim3 grid((unsigned)((threads + kAngleThreads - 1) / kAngleThreads), grid_y(count));
      angle_leaves_kernel<<<grid, kAngleThreads, 0, ctx->stream>>>((const AngleLeaf*)dev, (const AngleRef*)(dev + a->off_refs),
                                                                  (int)a->leaves.size(), theta, theta_stride,
                                                                  tangents ? dot : nullptr, dot_stride, count,
                                                                  (long long)a->block_elems, out->ptr);
      ctx->launches++;
      e = cudaGetLastError();
    }
    if (e != cudaSuccess) rc = fail(TNCB_ERR_CUDA, std::string("angle rows: ") + cudaGetErrorString(e));
  }
  if (rc) {
    if (out) tncb_tensor_free(ctx, out);
    if (fresh) angles_release(a, ctx);
    return rc;
  }
  *rows = out;
  return TNCB_OK;
}

}  // namespace tncb

extern "C" {

int tncb_angles_create(const tncb_tn* tn, size_t n_params, size_t n_refs, const tncb_angle_ref* refs, const int64_t* offsets,
                       size_t block_elems, tncb_angles** out) {
  using namespace tncb;
  if (!tn || !out || (n_refs && !refs)) return fail(TNCB_ERR_INVALID, "null argument");
  if (n_params == 0) return fail(TNCB_ERR_INVALID, "n_params is 0");
  if (n_params > 0x7fffffff) return fail(TNCB_ERR_INVALID, "n_params is above 2^31 - 1");
  if (n_refs == 0) return fail(TNCB_ERR_INVALID, "no refs");
  std::vector<const tncb_tn*> lv;
  collect(tn, lv);
  std::vector<int> gate_of(lv.size(), -2);         // -2 = not yet looked at
  std::vector<std::vector<int>> by_leaf(lv.size());
  for (size_t k = 0; k < n_refs; k++) {
    const tncb_angle_ref& r = refs[k];
    const std::string who = "ref " + std::to_string(k) + ": leaf " + std::to_string(r.leaf);
    if (r.leaf >= lv.size()) return fail(TNCB_ERR_INVALID, who + " is out of range (" + std::to_string(lv.size()) + " leaves)");
    const tncb_tn* lf = lv[r.leaf];
    if (lf->kind != TNCB_DATA_GATE || !lf->gate_name) return fail(TNCB_ERR_INVALID, who + " is not a Gate leaf");
    const int g = angle_gate(lf->gate_name);
    if (g < 0) return fail(TNCB_ERR_GATE, who + ": gate '" + lf->gate_name + "' takes no angles");
    if (lf->n_gate_angles != ga::n_angles(g) || !lf->gate_angles)
      return fail(TNCB_ERR_GATE, who + ": gate '" + lf->gate_name + "' expects " + std::to_string(ga::n_angles(g)) + " angles, the leaf has " +
                                     std::to_string(lf->n_gate_angles));
    uint64_t elems = 1;
    for (int i = 0; i < lf->rank; i++) elems *= lf->dims ? lf->dims[i] : 0;
    if (elems != (uint64_t)(ga::dim(g) * ga::dim(g)))
      return fail(TNCB_ERR_SHAPE, who + ": " + std::to_string(elems) + " elements, gate '" + lf->gate_name + "' has " +
                                      std::to_string(ga::dim(g) * ga::dim(g)));
    if (r.slot >= (uint32_t)ga::n_angles(g))
      return fail(TNCB_ERR_GATE, who + ": slot " + std::to_string(r.slot) + " is past the " + std::to_string(ga::n_angles(g)) +
                                     " angles of gate '" + lf->gate_name + "'");
    if (r.param >= n_params) return fail(TNCB_ERR_INVALID, who + ": param " + std::to_string(r.param) + " >= n_params " + std::to_string(n_params));
    if (!std::isfinite(r.scale)) return fail(TNCB_ERR_INVALID, who + ": the scale is not finite");
    for (int j : by_leaf[r.leaf])
      if (refs[j].slot == r.slot)
        return fail(TNCB_ERR_INVALID, who + ", slot " + std::to_string(r.slot) + " is already set by ref " + std::to_string(j));
    gate_of[r.leaf] = g;
    by_leaf[r.leaf].push_back((int)k);
  }
  auto* a = new tncb_angles();
  a->n_params = n_params;
  // the layout: the caller's offsets, or the referenced leaves packed in leaf order
  a->offsets.assign(lv.size(), -1);
  size_t packed = 0;
  for (size_t l = 0; l < lv.size(); l++) {
    if (offsets) a->offsets[l] = offsets[l];
    else if (!by_leaf[l].empty()) { a->offsets[l] = (int64_t)packed; packed += ga::dim(gate_of[l]) * ga::dim(gate_of[l]); }
  }
  a->block_elems = offsets || block_elems ? block_elems : packed;
  std::vector<std::pair<int64_t, size_t>> spans;    // (offset, leaf) of the referenced leaves, for the overlap check
  for (size_t l = 0; l < lv.size(); l++) {
    if (by_leaf[l].empty()) continue;
    const std::string who = "ref " + std::to_string(by_leaf[l][0]) + ": leaf " + std::to_string(l);
    const int64_t off = a->offsets[l];
    const int64_t n = ga::dim(gate_of[l]) * ga::dim(gate_of[l]);
    if (off < 0) { delete a; return fail(TNCB_ERR_INVALID, who + " has offset " + std::to_string(off) + " (not in the block)"); }
    if ((uint64_t)off + (uint64_t)n > a->block_elems) {
      const std::string msg = who + ": its " + std::to_string(n) + " elements at offset " + std::to_string(off) + " run past block_elems " +
                              std::to_string(a->block_elems);
      delete a;
      return fail(TNCB_ERR_INVALID, msg);
    }
    spans.push_back({off, l});
  }
  std::sort(spans.begin(), spans.end());
  for (size_t k = 1; k < spans.size(); k++) {
    const size_t l = spans[k - 1].second;
    if (spans[k - 1].first + ga::dim(gate_of[l]) * ga::dim(gate_of[l]) > spans[k].first) {
      delete a;
      return fail(TNCB_ERR_INVALID, "leaves " + std::to_string(l) + " and " + std::to_string(spans[k].second) + " overlap in the block");
    }
  }
  // the tables: leaves in leaf order, each with its refs in slot order; refs folded per param in (param, leaf, slot) order
  for (size_t l = 0; l < lv.size(); l++) {
    if (by_leaf[l].empty()) continue;
    std::vector<int> ks = by_leaf[l];
    std::sort(ks.begin(), ks.end(), [&](int x, int y) { return refs[x].slot < refs[y].slot; });
    AngleLeaf L{};
    L.off = a->offsets[l];
    L.gate = gate_of[l];
    L.adjoint = lv[l]->gate_adjoint != 0;
    L.first = (int)a->refs.size();
    L.n = (int)ks.size();
    for (int s = 0; s < ga::n_angles(L.gate); s++) L.a[s] = lv[l]->gate_angles[s];
    for (int k : ks) {
      a->refs.push_back({(int)a->leaves.size(), (int)refs[k].slot, (int)refs[k].param, 0, refs[k].scale});
    }
    a->leaves.push_back(L);
  }
  for (size_t k = 0; k < a->refs.size(); k++) a->order.push_back((int)k);
  std::stable_sort(a->order.begin(), a->order.end(), [&](int x, int y) { return a->refs[x].param < a->refs[y].param; });
  a->pstart.assign(n_params + 1, 0);
  for (const AngleRef& r : a->refs) a->pstart[r.param + 1]++;
  for (size_t p = 0; p < n_params; p++) a->pstart[p + 1] += a->pstart[p];
  put(a->table, a->leaves);
  a->off_refs = put(a->table, a->refs);
  a->off_order = put(a->table, a->order);
  a->off_pstart = put(a->table, a->pstart);
  *out = a;
  return TNCB_OK;
}

int tncb_angles_destroy(tncb_angles* a) {
  if (!a) return TNCB_OK;
  while (!a->dev.empty()) {
    tncb_ctx* ctx = a->dev.back().ctx;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);            // calls in flight still read the table
    tncb::angles_release(a, ctx);
  }
  delete a;
  return TNCB_OK;
}

int tncb_angles_layout(const tncb_angles* a, size_t* n_params, size_t* block_elems, int64_t* offsets) {
  if (!a) return tncb::fail(TNCB_ERR_INVALID, "null argument");
  if (n_params) *n_params = a->n_params;
  if (block_elems) *block_elems = a->block_elems;
  if (offsets) std::copy(a->offsets.begin(), a->offsets.end(), offsets);
  return TNCB_OK;
}

int tncb_angles_gates(tncb_ctx* ctx, const tncb_angles* a, const double* theta, size_t theta_stride, size_t count, tncb_tensor** rows) {
  return tncb::leaf_rows(ctx, const_cast<tncb_angles*>(a), theta, theta_stride, nullptr, 0, count, false, rows);
}

int tncb_angles_tangents(tncb_ctx* ctx, const tncb_angles* a, const double* theta, size_t theta_stride, const double* theta_dot,
                         size_t dot_stride, size_t count, tncb_tensor** rows) {
  return tncb::leaf_rows(ctx, const_cast<tncb_angles*>(a), theta, theta_stride, theta_dot, dot_stride, count, true, rows);
}

int tncb_angles_pullback(tncb_ctx* ctx, const tncb_angles* ac, const double* theta, size_t theta_stride, size_t count,
                         const tncb_tensor* grads, const tncb_tensor* grad_tangents, const double* direction,
                         size_t direction_stride, tncb_tensor** rows, tncb_tensor** sum) {
  using namespace tncb;
  tncb_angles* a = const_cast<tncb_angles*>(ac);
  if (!ctx || !a) return fail(TNCB_ERR_INVALID, "null argument");
  if (!rows && !sum) return fail(TNCB_ERR_INVALID, "no output requested");
  if (count == 0) return fail(TNCB_ERR_INVALID, "count is 0");
  if (!grad_tangents != !direction) return fail(TNCB_ERR_INVALID, "grad_tangents and direction come together");
  if (cudaSetDevice(ctx->device) != cudaSuccess) return fail(TNCB_ERR_CUDA, "cudaSetDevice failed");
  if (int rc = check_rows(ctx, theta, theta_stride, count, a->n_params, "theta")) return rc;
  long long gs = 0, gds = 0;
  if (int rc = check_block(grads, count, a->block_elems, "grads", &gs)) return rc;
  if (grad_tangents) {
    if (int rc = check_block(grad_tangents, count, a->block_elems, "grad_tangents", &gds)) return rc;
    if (gds != gs) return fail(TNCB_ERR_SHAPE, "grads and grad_tangents must both be shared or both have a row per parameter row");
    if (int rc = check_rows(ctx, direction, direction_stride, count, a->n_params, "direction")) return rc;
  }
  const char* dev = nullptr;
  bool fresh = false;
  if (int rc = tables(ctx, a, &dev, &fresh)) return rc;
  const uint64_t rdims[2] = {count, a->n_params}, sdims[1] = {a->n_params};
  tncb_tensor *r = nullptr, *s = nullptr;
  int rc = tensor_new(ctx, 2, rdims, &r);          // (the rows are the fold's input when only the sum is wanted)
  if (!rc && sum) rc = tensor_new(ctx, 1, sdims, &s);
  if (!rc) {
    const unsigned gx = (unsigned)((a->n_params + kAngleThreads - 1) / kAngleThreads);
    angle_pullback_kernel<<<dim3(gx, grid_y(count)), kAngleThreads, 0, ctx->stream>>>(
        (const AngleLeaf*)dev, (const AngleRef*)(dev + a->off_refs), (const int*)(dev + a->off_order), (const int*)(dev + a->off_pstart),
        (int)a->n_params, theta, theta_stride, count, grads->ptr, grad_tangents ? grad_tangents->ptr : nullptr, gs, direction,
        direction_stride, (long long)a->block_elems, r->ptr);
    ctx->launches++;
    if (s) {
      angle_fold_kernel<<<gx, kAngleThreads, 0, ctx->stream>>>(r->ptr, count, (int)a->n_params, s->ptr);
      ctx->launches++;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(TNCB_ERR_CUDA, std::string("angle pullback: ") + cudaGetErrorString(e));
  }
  if (rc || !rows) { if (r) tncb_tensor_free(ctx, r); r = nullptr; }
  if (rc) {
    if (s) tncb_tensor_free(ctx, s);
    if (fresh) angles_release(a, ctx);
    return rc;
  }
  if (rows) *rows = r;
  if (sum) *sum = s;
  return TNCB_OK;
}

}  // extern "C"
