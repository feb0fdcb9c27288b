// Plain embedding gather, segmented (deterministic) scatter-add, and the row-wise optimizers
// that consume its SelectedRows-style output.
//
// Reference call sites: paddle.nn.Embedding in models/rank/wide_deep/net.py:47-53,90,
// dcn_v2/net.py:45-54,95, din/net.py:33-82,141-147 (forward = lookup_table_v2, backward =
// lookup_table_v2_grad with sparse=True -> SelectedRows); optimizers: Adam(lazy_mode=True)
// models/rank/deepfm/static_model.py:101-103, SGD models/rank/din/dygraph_model.py:64-73,
// SparseAdaGradSGDRule models/rank/slot_dnn/config_online.yaml:57-79.
//
// All kernels are HBM-bound: algorithmic bytes per looked-up row are 8 (id) + 2*4D.
#pragma once

#include "common.cuh"
#include "segreduce.cuh"

namespace b200rec {

constexpr int kGatherThreads = 256;
constexpr int kGatherRowsPerGroup = 4;  // independent rows in flight per lane group

template <int VEC, int TPR>
__global__ void __launch_bounds__(kGatherThreads)
gather_kernel(const float* __restrict__ W, const int64_t* __restrict__ ids,
              float* __restrict__ out, int64_t n, int D, int64_t V, int64_t pad, int64_t ldw) {
  constexpr int GPB = kGatherThreads / TPR;
  const int g = threadIdx.x / TPR;
  const int r = threadIdx.x % TPR;
  const bool lane_ok = r * VEC < D;
  const int64_t base = ((int64_t)blockIdx.x * GPB + g) * kGatherRowsPerGroup;
  Vec<VEC> e[kGatherRowsPerGroup];
#pragma unroll
  for (int j = 0; j < kGatherRowsPerGroup; ++j) {
    e[j] = vzero<VEC>();
    const int64_t i = base + j;
    if (i < n) {
      const int64_t id = __ldg(ids + i);
      const bool in_range = (uint64_t)id < (uint64_t)V;
      if (in_range && id != pad && lane_ok) e[j] = ld_row<VEC>(W + (size_t)id * ldw + r * VEC);
      if (!in_range && r == 0) atomicAdd(&g_oob_count, 1ull);
    }
  }
#pragma unroll
  for (int j = 0; j < kGatherRowsPerGroup; ++j) {
    const int64_t i = base + j;
    if (i < n && lane_ok) st_stream<VEC>(out + (size_t)i * D + r * VEC, e[j]);
  }
}

static int launch_gather(const float* W, const int64_t* ids, float* out, int64_t n, int D,
                         int64_t V, int64_t pad, int64_t ldw, cudaStream_t st) {
  RowShape rs;
  B200_REQUIRE(pick_row_shape(D, &rs), "gather: unsupported D=%d", D);
  B200_REQUIRE(ldw >= D && ldw % rs.vec == 0, "gather: bad row stride %lld", (long long)ldw);
  const int align = rs.vec * 4;
  B200_REQUIRE(reinterpret_cast<uintptr_t>(W) % align == 0 &&
                   reinterpret_cast<uintptr_t>(out) % align == 0,
               "gather: W/out must be %d-byte aligned", align);
  if (n == 0) return B200REC_OK;
  B200_DISPATCH_ROW_SHAPE(rs, {
    constexpr int rows_per_block = (kGatherThreads / TPR) * kGatherRowsPerGroup;
    const int64_t grid = (n + rows_per_block - 1) / rows_per_block;
    gather_kernel<VEC, TPR><<<(unsigned)grid, kGatherThreads, 0, st>>>(W, ids, out, n, D, V, pad,
                                                                       ldw);
  });
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

// ---- multi-hot slots: gather + sum-pool over variable-length key lists (LoD) -----------------
// Reference: sequence_pool(sum) after sparse_embedding, models/rank/slot_dnn/net.py:63-75, and the
// fused_seqpool_cvm call sites tools/utils/static_ps/model_util.py:411-415,465-469.  One lane
// group per bag; empty bags give zeros (pad_value 0); padding / out-of-range keys are skipped.
template <int VEC, int TPR>
__global__ void __launch_bounds__(kGatherThreads)
gather_pool_kernel(const float* __restrict__ W, const int64_t* __restrict__ keys,
                   const int64_t* __restrict__ offsets, float* __restrict__ out, int64_t n_bags,
                   int D, int64_t V, int64_t pad, int64_t ldw) {
  constexpr int GPB = kGatherThreads / TPR;
  const int r = threadIdx.x % TPR;
  const bool lane_ok = r * VEC < D;
  for (int64_t bag = (int64_t)blockIdx.x * GPB + threadIdx.x / TPR; bag < n_bags;
       bag += (int64_t)gridDim.x * GPB) {
    const int64_t beg = offsets[bag], end = offsets[bag + 1];
    Vec<VEC> acc = vzero<VEC>();
    int64_t i = beg;
    for (; i + 1 < end; i += 2) {  // two rows in flight
      const int64_t k0 = __ldg(keys + i), k1 = __ldg(keys + i + 1);
      const bool ok0 = (uint64_t)k0 < (uint64_t)V && k0 != pad;
      const bool ok1 = (uint64_t)k1 < (uint64_t)V && k1 != pad;
      const Vec<VEC> a = ld_row_pred<VEC, false>(W + (size_t)(ok0 ? k0 : 0) * ldw + r * VEC,
                                                 ok0 && lane_ok);
      const Vec<VEC> b = ld_row_pred<VEC, false>(W + (size_t)(ok1 ? k1 : 0) * ldw + r * VEC,
                                                 ok1 && lane_ok);
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc.v[k] = (acc.v[k] + a.v[k]) + b.v[k];
      if (r == 0 && ((uint64_t)k0 >= (uint64_t)V)) atomicAdd(&g_oob_count, 1ull);
      if (r == 0 && ((uint64_t)k1 >= (uint64_t)V)) atomicAdd(&g_oob_count, 1ull);
    }
    if (i < end) {
      const int64_t k0 = __ldg(keys + i);
      const bool ok0 = (uint64_t)k0 < (uint64_t)V && k0 != pad;
      const Vec<VEC> a = ld_row_pred<VEC, false>(W + (size_t)(ok0 ? k0 : 0) * ldw + r * VEC,
                                                 ok0 && lane_ok);
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc.v[k] += a.v[k];
      if (r == 0 && ((uint64_t)k0 >= (uint64_t)V)) atomicAdd(&g_oob_count, 1ull);
    }
    if (lane_ok) st_stream<VEC>(out + (size_t)bag * D + r * VEC, acc);
  }
}

// bag_of_pos[i] = bag that owns key position i (for the pooled backward)
__global__ void bag_of_positions_kernel(const int64_t* __restrict__ offsets, int64_t n_bags,
                                        int32_t* __restrict__ bag_of_pos) {
  const int64_t bag = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (bag >= n_bags) return;
  for (int64_t i = offsets[bag]; i < offsets[bag + 1]; ++i) bag_of_pos[i] = (int32_t)bag;
}

static int launch_gather_pool(const float* W, const int64_t* keys, const int64_t* offsets,
                              float* out, int32_t* bag_of_pos, int64_t n_bags, int D, int64_t V,
                              int64_t pad, int64_t ldw, cudaStream_t st) {
  RowShape rs;
  B200_REQUIRE(pick_row_shape(D, &rs), "gather_pool: unsupported D=%d", D);
  B200_REQUIRE(ldw >= D && ldw % rs.vec == 0, "gather_pool: bad row stride %lld", (long long)ldw);
  const int align = rs.vec * 4;
  B200_REQUIRE(reinterpret_cast<uintptr_t>(W) % align == 0 &&
                   reinterpret_cast<uintptr_t>(out) % align == 0,
               "gather_pool: W/out must be %d-byte aligned", align);
  if (n_bags == 0) return B200REC_OK;
  B200_DISPATCH_ROW_SHAPE(rs, {
    constexpr int GPB = kGatherThreads / TPR;
    const int64_t want = (n_bags + GPB - 1) / GPB;
    const unsigned grid = (unsigned)min(want, (int64_t)sm_count() * 64);
    gather_pool_kernel<VEC, TPR><<<grid, kGatherThreads, 0, st>>>(W, keys, offsets, out, n_bags, D, V,
                                                                  pad, ldw);
  });
  B200_LAUNCH_CHECK();
  if (bag_of_pos != nullptr) {
    bag_of_positions_kernel<<<(unsigned)((n_bags + 255) / 256), 256, 0, st>>>(offsets, n_bags,
                                                                              bag_of_pos);
    B200_LAUNCH_CHECK();
  }
  return B200REC_OK;
}

// rows[u,:] = sum over the segment of dOut[sorted_pos[i],:], fixed order (segreduce.cuh).
struct PlainRowContrib {
  const float* dOut;
  const int32_t* row_of_pos;  // nullptr: dOut row = position; else dOut row = row_of_pos[position]
  int D;
  template <int VEC>
  __device__ __forceinline__ void add(int p, int r, bool lane_ok, Vec<VEC>& acc, float&) const {
    if (lane_ok) {
      const size_t row = row_of_pos ? (size_t)__ldg(row_of_pos + p) : (size_t)p;
      const Vec<VEC> a = ld_row<VEC>(dOut + row * D + r * VEC);
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc.v[k] += a.v[k];
    }
  }
};

static int launch_segment_reduce(const float* dOut, const int32_t* row_of_pos,
                                 const int32_t* seg_offsets, const int32_t* sorted_pos,
                                 const int32_t* num_unique, float* rows, int64_t n, int D, void* ws,
                                 size_t ws_bytes, cudaStream_t st) {
  RowShape rs;
  B200_REQUIRE(pick_row_shape(D, &rs), "segment_reduce: unsupported D=%d", D);
  const int align = rs.vec * 4;
  B200_REQUIRE(reinterpret_cast<uintptr_t>(dOut) % align == 0 &&
                   reinterpret_cast<uintptr_t>(rows) % align == 0,
               "segment_reduce: dOut/rows must be %d-byte aligned", align);
  if (n == 0) return B200REC_OK;
  if (ws_bytes < seg_workspace_bytes(n, D)) {
    set_error("segment_reduce: workspace %zu < %zu bytes", ws_bytes, seg_workspace_bytes(n, D));
    return B200REC_ERR_WORKSPACE;
  }
  int rc = B200REC_OK;
  B200_DISPATCH_ROW_SHAPE(rs, {
    PlainRowContrib contrib{dOut, row_of_pos, D};
    rc = launch_seg_reduce<VEC, TPR, PlainRowContrib>(seg_offsets, sorted_pos, num_unique, contrib,
                                                      rows, nullptr, SegOut{D, 1, 0}, n, D, ws,
                                                      st);
  });
  return rc;
}

// ---- row-wise update kernels ---------------------------------------------------------------
// Common skeleton: one TPR-lane group per distinct row; Op::apply does the RMW of that row.
struct RowsToDenseOp {
  float* dW;
  template <int VEC>
  __device__ __forceinline__ void apply(size_t row_off, const Vec<VEC>& g, int) const {
    Vec<VEC> w = ld_cached<VEC>(dW + row_off);  // plain load is fine: rows are distinct
#pragma unroll
    for (int k = 0; k < VEC; ++k) w.v[k] += g.v[k];
    st_plain<VEC>(dW + row_off, w);
  }
};

struct SgdOp {
  float* W;
  float lr;
  template <int VEC>
  __device__ __forceinline__ void apply(size_t row_off, const Vec<VEC>& g, int) const {
    Vec<VEC> w = *reinterpret_cast<const Vec<VEC>*>(W + row_off);
#pragma unroll
    for (int k = 0; k < VEC; ++k) w.v[k] = fmaf(-lr, g.v[k], w.v[k]);
    st_plain<VEC>(W + row_off, w);
  }
};

struct AdamOp {
  float* W;
  float* m;
  float* v;
  float beta1, beta2, omb1, omb2;  // omb = 1-beta, rounded from double
  float lr_t, eps_t;  // lr_t = lr*sqrt(1-b2^t)/(1-b1^t), eps_t = eps*sqrt(1-b2^t)
  template <int VEC>
  __device__ __forceinline__ void apply(size_t row_off, const Vec<VEC>& g, int) const {
    Vec<VEC> w = *reinterpret_cast<const Vec<VEC>*>(W + row_off);
    Vec<VEC> mm = *reinterpret_cast<const Vec<VEC>*>(m + row_off);
    Vec<VEC> vv = *reinterpret_cast<const Vec<VEC>*>(v + row_off);
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      mm.v[k] = beta1 * mm.v[k] + omb1 * g.v[k];
      vv.v[k] = beta2 * vv.v[k] + omb2 * g.v[k] * g.v[k];
      w.v[k] -= lr_t * (mm.v[k] / (sqrtf(vv.v[k]) + eps_t));
    }
    st_plain<VEC>(W + row_off, w);
    st_plain<VEC>(m + row_off, mm);
    st_plain<VEC>(v + row_off, vv);
  }
};

template <int VEC, int TPR, typename Op>
__global__ void __launch_bounds__(kGatherThreads)
row_update_kernel(const int64_t* __restrict__ unique_ids, const float* __restrict__ rows,
                  const int32_t* __restrict__ num_unique, int D, int64_t V, int64_t ldw,
                  int64_t ld_rows, Op op) {
  constexpr int GPB = kGatherThreads / TPR;
  const int U = num_unique[0];
  const int r = threadIdx.x % TPR;
  const bool lane_ok = r * VEC < D;
  for (int64_t u = (int64_t)blockIdx.x * GPB + threadIdx.x / TPR; u < U;
       u += (int64_t)gridDim.x * GPB) {
    const int64_t id = unique_ids[u];
    if ((uint64_t)id >= (uint64_t)V || !lane_ok) continue;
    const Vec<VEC> g = ld_row<VEC>(rows + (size_t)u * ld_rows + r * VEC);
    op.template apply<VEC>((size_t)id * ldw + r * VEC, g, r);
  }
}

// AdaGrad with ONE accumulator per row needs the row-mean of g^2 -> its own kernel.
template <int VEC, int TPR>
__global__ void __launch_bounds__(kGatherThreads)
row_adagrad_kernel(float* __restrict__ W, float* __restrict__ g2sum,
                   const int64_t* __restrict__ unique_ids, const float* __restrict__ rows,
                   const int32_t* __restrict__ num_unique, int D, int64_t V, int64_t ldw,
                   int64_t ld_rows, float lr, float g0, float lo, float hi) {
  constexpr int GPB = kGatherThreads / TPR;
  const int U = num_unique[0];
  const int r = threadIdx.x % TPR;
  const bool lane_ok = r * VEC < D;
  // whole warps iterate together so the group shuffles stay converged
  const int64_t groups_total = (int64_t)gridDim.x * GPB;
  const int64_t U_pad = ((int64_t)U + 32 / TPR - 1) / (32 / TPR) * (32 / TPR);
  for (int64_t u = (int64_t)blockIdx.x * GPB + threadIdx.x / TPR; u < U_pad; u += groups_total) {
    const bool live = u < U;
    int64_t id = live ? unique_ids[u] : -1;
    const bool ok = live && (uint64_t)id < (uint64_t)V && lane_ok;
    Vec<VEC> g = vzero<VEC>();
    if (ok) g = ld_row<VEC>(rows + (size_t)u * ld_rows + r * VEC);
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < VEC; ++k) sq = fmaf(g.v[k], g.v[k], sq);
    sq = group_sum<TPR>(sq);
    if (ok) {
      const float acc = g2sum[id];
      const float scale = sqrtf(g0 / (g0 + acc));
      Vec<VEC> w = *reinterpret_cast<const Vec<VEC>*>(W + (size_t)id * ldw + r * VEC);
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        w.v[k] -= lr * g.v[k] * scale;
        w.v[k] = fminf(fmaxf(w.v[k], lo), hi);
      }
      st_plain<VEC>(W + (size_t)id * ldw + r * VEC, w);
    }
    __syncwarp();
    if (ok && r == 0) g2sum[id] += sq / (float)D;
  }
}

// Wide rows (more than 32 vector chunks, e.g. FFM's [R emb | w1] rows of 352-1252 floats): one
// warp per row, each lane stepping through the row 32*VEC floats at a time.
template <int VEC, typename Op>
__global__ void __launch_bounds__(kGatherThreads)
row_update_wide_kernel(const int64_t* __restrict__ unique_ids, const float* __restrict__ rows,
                       const int32_t* __restrict__ num_unique, int D, int64_t V, int64_t ldw,
                       int64_t ld_rows, Op op) {
  constexpr int WPB = kGatherThreads / 32;
  const int U = num_unique[0];
  const int r = threadIdx.x % 32;
  for (int64_t u = (int64_t)blockIdx.x * WPB + threadIdx.x / 32; u < U;
       u += (int64_t)gridDim.x * WPB) {
    const int64_t id = unique_ids[u];
    if ((uint64_t)id >= (uint64_t)V) continue;
    for (int c = r * VEC; c < D; c += 32 * VEC) {
      const Vec<VEC> g = ld_row<VEC>(rows + (size_t)u * ld_rows + c);
      op.template apply<VEC>((size_t)id * ldw + c, g, r);
    }
  }
}

template <int VEC>
__global__ void __launch_bounds__(kGatherThreads)
row_adagrad_wide_kernel(float* __restrict__ W, float* __restrict__ g2sum,
                        const int64_t* __restrict__ unique_ids, const float* __restrict__ rows,
                        const int32_t* __restrict__ num_unique, int D, int64_t V, int64_t ldw,
                        int64_t ld_rows, float lr, float g0, float lo, float hi) {
  constexpr int WPB = kGatherThreads / 32;
  const int U = num_unique[0];
  const int r = threadIdx.x % 32;
  for (int64_t u = (int64_t)blockIdx.x * WPB + threadIdx.x / 32; u < U;
       u += (int64_t)gridDim.x * WPB) {
    const int64_t id = unique_ids[u];   // the whole warp holds the same row
    if ((uint64_t)id >= (uint64_t)V) continue;
    const float* grow = rows + (size_t)u * ld_rows;
    const float acc = g2sum[id];
    float sq = 0.f;
#pragma unroll 1
    for (int c = r * VEC; c < D; c += 32 * VEC) {
      const Vec<VEC> g = ld_row<VEC>(grow + c);
#pragma unroll
      for (int k = 0; k < VEC; ++k) sq = fmaf(g.v[k], g.v[k], sq);
    }
    sq = group_sum<32>(sq);
    const float scale = sqrtf(g0 / (g0 + acc));
#pragma unroll 1
    for (int c = r * VEC; c < D; c += 32 * VEC) {
      const Vec<VEC> g = ld_row<VEC>(grow + c);
      Vec<VEC> w = *reinterpret_cast<const Vec<VEC>*>(W + (size_t)id * ldw + c);
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        w.v[k] -= lr * g.v[k] * scale;
        w.v[k] = fminf(fmaxf(w.v[k], lo), hi);
      }
      st_plain<VEC>(W + (size_t)id * ldw + c, w);
    }
    __syncwarp();
    if (r == 0) g2sum[id] += sq / (float)D;
  }
}

// Row geometry for the row-wise optimizers: start from the widest vector D allows and narrow it
// until the row strides and base addresses fit (column VIEWS of a table — e.g. the embedding part
// of a [show, click, emb] GPUBox row — start at a 4- or 8-byte offset).  Rows of more than 32
// chunks get tpr = 0: the wide kernels above.
static bool pick_row_shape_for(int D, int64_t ldw, int64_t ld_rows, const void* const* ptrs, int np,
                               RowShape* rs) {
  if (D < 1) return false;
  auto fits = [&](int vec) {
    if (D % vec || ldw % vec || ld_rows % vec) return false;
    for (int i = 0; i < np; ++i)
      if (ptrs[i] != nullptr && reinterpret_cast<uintptr_t>(ptrs[i]) % (vec * 4) != 0) return false;
    return true;
  };
  int vec = (D % 4 == 0) ? 4 : (D % 2 == 0 ? 2 : 1);
  while (vec > 1 && !fits(vec)) vec >>= 1;
  const int chunks = D / vec;
  int tpr = 1;
  while (tpr < chunks) tpr <<= 1;
  rs->vec = vec;
  rs->tpr = chunks > 32 ? 0 : tpr;
  return true;
}

#define B200_DISPATCH_VEC(vec, ...)                                   \
  do {                                                                \
    switch (vec) {                                                    \
      case 4: { constexpr int VEC = 4; __VA_ARGS__; } break;          \
      case 2: { constexpr int VEC = 2; __VA_ARGS__; } break;          \
      default: { constexpr int VEC = 1; __VA_ARGS__; } break;         \
    }                                                                 \
  } while (0)

template <typename Op>
static int launch_row_update(const char* what, const int64_t* unique_ids, const float* rows,
                             const int32_t* num_unique, int64_t n, int D, int64_t V, int64_t ldw,
                             int64_t ld_rows, Op op, const void* a0, const void* a1,
                             const void* a2, cudaStream_t st) {
  RowShape rs;
  const void* ptrs[4] = {rows, a0, a1, a2};
  B200_REQUIRE(ldw >= D && ld_rows >= D, "%s: bad row strides", what);
  B200_REQUIRE(pick_row_shape_for(D, ldw, ld_rows, ptrs, 4, &rs), "%s: unsupported D=%d", what, D);
  if (n == 0) return B200REC_OK;
  if (rs.tpr == 0) {
    constexpr int WPB = kGatherThreads / 32;
    const unsigned grid = (unsigned)min((n + WPB - 1) / WPB, (int64_t)sm_count() * 64);
    B200_DISPATCH_VEC(rs.vec, row_update_wide_kernel<VEC, Op><<<grid, kGatherThreads, 0, st>>>(
                                  unique_ids, rows, num_unique, D, V, ldw, ld_rows, op));
    B200_LAUNCH_CHECK();
    return B200REC_OK;
  }
  B200_DISPATCH_ROW_SHAPE(rs, {
    constexpr int GPB = kGatherThreads / TPR;
    const int64_t want = (n + GPB - 1) / GPB;
    const unsigned grid = (unsigned)min(want, (int64_t)sm_count() * 64);
    row_update_kernel<VEC, TPR, Op><<<grid, kGatherThreads, 0, st>>>(unique_ids, rows, num_unique,
                                                                     D, V, ldw, ld_rows, op);
  });
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_adagrad(float* W, float* g2sum, const int64_t* unique_ids, const float* rows,
                          const int32_t* num_unique, int64_t n, int D, int64_t V, int64_t ldw,
                          int64_t ld_rows, float lr, float g0, float lo, float hi,
                          cudaStream_t st) {
  RowShape rs;
  const void* ptrs[2] = {W, rows};
  B200_REQUIRE(ldw >= D && ld_rows >= D, "sparse_adagrad: bad row strides");
  B200_REQUIRE(pick_row_shape_for(D, ldw, ld_rows, ptrs, 2, &rs), "sparse_adagrad: unsupported D=%d",
               D);
  if (n == 0) return B200REC_OK;
  if (rs.tpr == 0) {
    constexpr int WPB = kGatherThreads / 32;
    const unsigned grid = (unsigned)min((n + WPB - 1) / WPB, (int64_t)sm_count() * 64);
    B200_DISPATCH_VEC(rs.vec, row_adagrad_wide_kernel<VEC><<<grid, kGatherThreads, 0, st>>>(
                                  W, g2sum, unique_ids, rows, num_unique, D, V, ldw, ld_rows, lr,
                                  g0, lo, hi));
    B200_LAUNCH_CHECK();
    return B200REC_OK;
  }
  B200_DISPATCH_ROW_SHAPE(rs, {
    constexpr int GPB = kGatherThreads / TPR;
    const int64_t want = (n + GPB - 1) / GPB;
    const unsigned grid = (unsigned)min(want, (int64_t)sm_count() * 64);
    row_adagrad_kernel<VEC, TPR><<<grid, kGatherThreads, 0, st>>>(
        W, g2sum, unique_ids, rows, num_unique, D, V, ldw, ld_rows, lr, g0, lo, hi);
  });
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

}  // namespace b200rec
