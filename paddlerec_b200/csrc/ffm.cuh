// FFM: the field-aware second-order term of models/rank/ffm/net.py:99-133 fused with its gather,
// forward and backward.
//
// NF = F + Dn fields, R = NF*D.  Row n of a sample is e[n,:] = W[ids[n], 0:R] (n < F) or
// dense[n-F] * dense_w[n-F, :] (n >= F); block m of it is e[n, m*D:(m+1)*D].
//   y1 = sum_f W[ids[f], R] + sum_k dense[k]*dense_w1[k] (+ bias)
//   y2 = sum_{n<m} < e[n, block m], e[m, block n] >
// The reference materialises feat [B, NF, R] and evaluates NF(NF-1)/2 slice pairs; here every
// gathered row crosses HBM once, into shared memory, and a sample leaves as two scalars.
// Table rows use the fused slot layout [R emb | w1 | pad] (row stride ldw, ldw % 4 == 0).
#pragma once

#include "common.cuh"
#include "embed_fm.cuh"    // cp_async_16_cg
#include "segreduce.cuh"   // kHotThreshold

namespace b200rec {

constexpr int kFfmThreads = 256;
constexpr int kFfmMaxFields = 64;   // pair table packs (n, m) into 16 bits each; bounds the loops

__host__ __device__ inline int ffm_staged_cols(int R) { return (R + 1 + 3) / 4 * 4; }   // [R | w1 | pad]

// Shared-memory layout of the forward: dense_w resident [Dn*R] | pair table [P] | reduction
// scratch | nbuf sample buffers of F staged rows (Rs floats each).
struct FfmFwdSmem {
  size_t off_pairs, off_red, off_buf, buf_bytes, total;
  FfmFwdSmem(int F, int Dn, int D, int nbuf) {
    const int NF = F + Dn, R = NF * D, P = NF * (NF - 1) / 2;
    off_pairs = align_up((size_t)Dn * R * 4, 16);
    off_red = align_up(off_pairs + (size_t)P * 4, 16);
    off_buf = off_red + 16 * (kFfmThreads / 32 + 4);
    buf_bytes = (size_t)F * ffm_staged_cols(R) * 4;
    total = off_buf + (size_t)nbuf * buf_bytes;
  }
};

// Persistent CTAs, one sample at a time.  With two buffers the next sample's rows stream in with
// cp.async (16-byte pieces, L1 bypassed) while the current one is reduced.  Padding and
// out-of-range ids stage a zero row.  Pairs are summed in a fixed order: thread t takes pairs
// t, t+256, ...; the 256 partials meet in a fixed shuffle + shared-memory tree.
__global__ void __launch_bounds__(kFfmThreads)
ffm_fwd_kernel(const float* __restrict__ W, int64_t ldw, const int64_t* __restrict__ ids,
               const float* __restrict__ dense, const float* __restrict__ dense_w,
               const float* __restrict__ dense_w1, const float* __restrict__ bias,
               float* __restrict__ y1, float* __restrict__ y2, int64_t B, int F, int Dn, int D,
               int64_t V, int64_t pad, int nbuf, size_t off_pairs, size_t off_red,
               size_t off_buf) {
  extern __shared__ __align__(16) unsigned char ffm_smem[];
  const int NF = F + Dn, R = NF * D, P = NF * (NF - 1) / 2;
  const int Rs = ffm_staged_cols(R), C = Rs / 4;
  float* s_dw = reinterpret_cast<float*>(ffm_smem);
  uint32_t* s_pairs = reinterpret_cast<uint32_t*>(ffm_smem + off_pairs);
  float* s_red = reinterpret_cast<float*>(ffm_smem + off_red);
  float* s_buf = reinterpret_cast<float*>(ffm_smem + off_buf);
  const size_t buf_floats = (size_t)F * Rs;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int i = threadIdx.x; i < Dn * R; i += kFfmThreads) s_dw[i] = __ldg(dense_w + i);
  for (int n = threadIdx.x; n < NF; n += kFfmThreads) {
    const int base = n * NF - n * (n + 1) / 2;   // pairs (n, m > n) in row-major order
    for (int m = n + 1; m < NF; ++m) s_pairs[base + m - n - 1] = ((uint32_t)n << 16) | (uint32_t)m;
  }

  auto stage = [&](int64_t b, float* buf) {
    for (int i = threadIdx.x; i < F * C; i += kFfmThreads) {
      const int f = i / C, c = i - f * C;
      const int64_t id = __ldg(ids + b * F + f);
      const bool in_range = (uint64_t)id < (uint64_t)V;
      float* dst = buf + (size_t)f * Rs + c * 4;
      if (in_range && id != pad)
        cp_async_16_cg(dst, W + (size_t)id * ldw + c * 4);
      else
        *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (!in_range && c == 0) atomicAdd(&g_oob_count, 1ull);
    }
  };

  int64_t b = blockIdx.x;
  if (nbuf == 2 && b < B) stage(b, s_buf);
  cp_async_commit();
  for (int it = 0; b < B; b += gridDim.x, ++it) {
    float* rows;
    if (nbuf == 2) {
      const int64_t nb = b + gridDim.x;
      if (nb < B) stage(nb, s_buf + (size_t)((it + 1) & 1) * buf_floats);
      cp_async_commit();
      cp_async_wait<1>();
      rows = s_buf + (size_t)(it & 1) * buf_floats;
    } else {
      stage(b, s_buf);
      cp_async_commit();
      cp_async_wait<0>();
      rows = s_buf;
    }
    __syncthreads();

    const float* x = dense + b * Dn;
    float acc = 0.f;
    for (int p = threadIdx.x; p < P; p += kFfmThreads) {
      const uint32_t nm = s_pairs[p];
      const int n = (int)(nm >> 16), m = (int)(nm & 0xffffu);
      const float* a = n < F ? rows + (size_t)n * Rs + m * D : s_dw + (size_t)(n - F) * R + m * D;
      const float* c = m < F ? rows + (size_t)m * Rs + n * D : s_dw + (size_t)(m - F) * R + n * D;
      const float sa = n < F ? 1.f : __ldg(x + n - F);
      const float sc = m < F ? 1.f : __ldg(x + m - F);
      float t = 0.f;
      for (int d = 0; d < D; ++d) t = fmaf(a[d], c[d], t);
      acc = fmaf(sa * sc, t, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kFfmThreads / 32; ++w) t += s_red[w];
      float s1 = 0.f, s2 = 0.f;
      for (int f = 0; f < F; ++f) s1 += rows[(size_t)f * Rs + R];
      for (int k = 0; k < Dn; ++k) s2 = fmaf(__ldg(x + k), __ldg(dense_w1 + k), s2);
      float first = s1 + s2;
      if (bias != nullptr) first += __ldg(bias);
      y1[b] = first;
      y2[b] = t;
    }
    __syncthreads();   // the buffer and s_red are free for the next sample
  }
  cp_async_wait<0>();
}

static int ffm_max_smem() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess)
      cached = v;
    else
      cached = 227 * 1024;
  }
  return cached;
}

static int ffm_check_shape(const char* what, int F, int Dn, int D, int64_t ldw) {
  B200_REQUIRE(F >= 1 && Dn >= 0 && D >= 1 && F + Dn <= kFfmMaxFields,
               "%s: need 1 <= F, 0 <= Dn, F+Dn <= %d, D >= 1 (F=%d Dn=%d D=%d)", what,
               kFfmMaxFields, F, Dn, D);
  const int R = (F + Dn) * D;
  B200_REQUIRE(ldw >= R + 1 && ldw % 4 == 0,
               "%s: row stride ldw=%lld must hold [R=%d emb | w1] and be a multiple of 4", what,
               (long long)ldw, R);
  return B200REC_OK;
}

static int launch_ffm_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                          const float* dense_w, const float* dense_w1, const float* bias, float* y1,
                          float* y2, int64_t B, int F, int Dn, int D, int64_t V, int64_t pad,
                          cudaStream_t st) {
  int rc = ffm_check_shape("ffm_fwd", F, Dn, D, ldw);
  if (rc != B200REC_OK) return rc;
  B200_REQUIRE(aligned16(W), "ffm_fwd: W must be 16-byte aligned");
  int nbuf = 2;
  FfmFwdSmem L(F, Dn, D, nbuf);
  if (L.total > (size_t)ffm_max_smem()) {
    nbuf = 1;
    L = FfmFwdSmem(F, Dn, D, nbuf);
  }
  B200_REQUIRE(L.total <= (size_t)ffm_max_smem(),
               "ffm_fwd: one sample (F=%d rows of %d floats) and dense_w (%d x %d) need %zu bytes "
               "of shared memory, more than the %d a CTA may use",
               F, ffm_staged_cols((F + Dn) * D), Dn, (F + Dn) * D, L.total, ffm_max_smem());
  if (B == 0) return B200REC_OK;
  B200_CUDA(cudaFuncSetAttribute(ffm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)L.total));
  int per_sm = 1;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ffm_fwd_kernel, kFfmThreads,
                                                          L.total));
  const int64_t grid = min(B, (int64_t)sm_count() * max(per_sm, 1));
  ffm_fwd_kernel<<<(unsigned)grid, kFfmThreads, L.total, st>>>(
      W, ldw, ids, dense, dense_w, dense_w1, bias, y1, y2, B, F, Dn, D, V, pad, nbuf, L.off_pairs,
      L.off_red, L.off_buf);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

// ------------------------------------------------------------------------------------------------
// Backward.  With g2 = dL/dy2 and g1 = dL/dy1 of sample b:
//   table row of the id at position (b,f): block m (m != f) += g2[b] * e[b, m, block f];
//                                          block f += 0;  column R += g1[b]
//   ddense_w[k, block m] = sum_b g2[b] dense[b,k] e[b, m, block F+k]   (m != F+k)
//   ddense_w1[k] = sum_b g1[b] dense[b,k];   dbias = sum_b g1[b]
// The partner blocks e[b, m, block f] are re-gathered (W row of ids[b,m], or dense x dense_w), so
// nothing of size [B, NF, R] exists in either direction.
struct FfmBwd {
  const float* W;
  int64_t ldw;
  const int64_t* ids;
  const float* dense;
  const float* dense_w;
  const float* gy1;
  const float* gy2;
  int F, Dn, D, R, G;   // G = staged columns [R | g1 | pad], the partial-row width
  int64_t V, pad;

  // e[b, m, f*D + j]
  __device__ __forceinline__ float partner(int64_t b, int m, int f, int j) const {
    if (m < F) {
      const int64_t id = __ldg(ids + b * F + m);
      if ((uint64_t)id >= (uint64_t)V || id == pad) return 0.f;
      return __ldg(W + (size_t)id * ldw + f * D + j);
    }
    return __ldg(dense + b * Dn + (m - F)) * __ldg(dense_w + (size_t)(m - F) * R + f * D + j);
  }
  // Per (id, column) state the scheduling kernels compute once per segment before walking its
  // positions; FFM's contribution needs none.
  struct Col {};
  __device__ __forceinline__ Col column(int /*p*/, int /*c*/) const { return {}; }
  // contribution of position p = b*F + f to column c of its gradient row
  __device__ __forceinline__ float contrib(int p, int c, Col) const {
    const int64_t b = p / F;
    const int f = p - (int)b * F;
    if (c < R) {
      const int m = c / D;
      if (m == f) return 0.f;
      return __ldg(gy2 + b) * partner(b, m, f, c - m * D);
    }
    return c == R ? __ldg(gy1 + b) : 0.f;
  }
  // Dense-parameter columns: [ddense_w (Dn*R) | ddense_w1 (Dn) | dbias].  Each adds sample b to acc.
  __device__ __forceinline__ int w1_cols() const { return Dn; }
  __device__ __forceinline__ float dense_w_acc(float acc, int64_t b, int k, int c) const {
    const int m = c / D, j = c - m * D;
    if (m == F + k) return acc;
    const float s = __ldg(gy2 + b) * __ldg(dense + b * Dn + k);
    return fmaf(s, partner(b, m, F + k, j), acc);
  }
  __device__ __forceinline__ float w1_acc(float acc, int64_t b, int k) const {
    return fmaf(__ldg(gy1 + b), __ldg(dense + b * Dn + k), acc);
  }
  __device__ __forceinline__ float bias_acc(float acc, int64_t b) const { return acc + __ldg(gy1 + b); }
};

constexpr int kFfmHotChunk = 1024;   // positions per hot work item (one CTA)

// workspace: counters [4] | items int32[3*max_items] (segment, chunk | chunks<<16, partial slot) |
// hot partial rows [max_slots, G] | dense partials [slices, Dn*R + Dn + 1]
struct FfmBwdWs {
  size_t off_items, off_part, off_dense, total;
  int64_t max_items, max_slots;
  int slices;
  FfmBwdWs(int64_t B, int F, int Dn, int D) {
    const int64_t n = B * F;
    const int R = (F + Dn) * D, G = ffm_staged_cols(R);
    max_items = n / (kHotThreshold + 1) + 1;
    max_slots = 2 * (n / kFfmHotChunk) + 1;   // only ids split into >= 2 chunks get partial rows
    slices = (int)max((int64_t)1, min((int64_t)256, (B + 255) / 256));
    off_items = 16;
    off_part = align_up(off_items + (size_t)max_items * 3 * 4, 256);
    off_dense = align_up(off_part + (size_t)max_slots * G * 4, 256);
    total = off_dense + (size_t)slices * ((size_t)Dn * R + Dn + 1) * 4 + 256;
  }
};

// One warp per distinct id: walks its sorted positions 32 columns at a time (fixed order per
// column).  Ids with more than kHotThreshold positions are deferred to the hot kernel as
// ceil(len / kFfmHotChunk) work items.  A is the per-position functor (FfmBwd, FatBwd).
template <class A>
__global__ void __launch_bounds__(kFfmThreads)
ffm_bwd_light_kernel(A a, const int32_t* __restrict__ seg_offsets,
                     const int32_t* __restrict__ sorted_pos, const int32_t* __restrict__ num_unique,
                     float* __restrict__ rows, int64_t ld_rows, int32_t* __restrict__ counters,
                     int32_t* __restrict__ items) {
  const int U = num_unique[0];
  const int lane = threadIdx.x & 31;
  constexpr int WPB = kFfmThreads / 32;
  for (int64_t u = (int64_t)blockIdx.x * WPB + (threadIdx.x >> 5); u < U;
       u += (int64_t)gridDim.x * WPB) {
    const int beg = seg_offsets[u], end = seg_offsets[u + 1];
    if (end - beg > kHotThreshold) {
      if (lane == 0) {
        const int chunks = (end - beg + kFfmHotChunk - 1) / kFfmHotChunk;
        const int first = atomicAdd(&counters[0], chunks);
        const int slot = chunks > 1 ? atomicAdd(&counters[1], chunks) : -1;
        for (int c = 0; c < chunks; ++c) {
          items[3 * (first + c)] = (int32_t)u;
          items[3 * (first + c) + 1] = c | (c == 0 ? (chunks << 16) : 0);
          items[3 * (first + c) + 2] = slot < 0 ? -1 : slot + c;
        }
      }
      continue;
    }
    float* out = rows + (size_t)u * ld_rows;
    for (int c0 = 0; c0 < ld_rows; c0 += 32) {
      const int c = c0 + lane;
      float acc = 0.f;
      if (c < a.G) {
        const typename A::Col col = a.column(sorted_pos[beg], c);
        for (int i = beg; i < end; ++i) acc += a.contrib(sorted_pos[i], c, col);
      }
      if (c < ld_rows) out[c] = acc;
    }
  }
}

// One CTA per hot work item: warp w takes positions beg+w, beg+w+8, ...; the 8 warp sums of a
// column meet in warp order.  A single-chunk id writes its row; the chunks of a longer id write
// partial rows that the combine kernel adds in chunk order.
template <class A>
__global__ void __launch_bounds__(kFfmThreads)
ffm_bwd_hot_kernel(A a, const int32_t* __restrict__ seg_offsets,
                   const int32_t* __restrict__ sorted_pos, const int32_t* __restrict__ counters,
                   const int32_t* __restrict__ items, float* __restrict__ partials,
                   float* __restrict__ rows, int64_t ld_rows) {
  constexpr int WPB = kFfmThreads / 32;
  __shared__ float s_acc[WPB][33];
  const int n_items = counters[0];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int h = blockIdx.x; h < n_items; h += gridDim.x) {
    const int u = items[3 * h];
    const int chunk = items[3 * h + 1] & 0xffff;
    const int slot = items[3 * h + 2];
    const int beg = seg_offsets[u] + chunk * kFfmHotChunk;
    const int end = min(seg_offsets[u + 1], beg + kFfmHotChunk);
    float* out = slot < 0 ? rows + (size_t)u * ld_rows : partials + (size_t)slot * a.G;
    const int ncols = slot < 0 ? (int)ld_rows : a.G;
    for (int c0 = 0; c0 < ncols; c0 += 32) {
      const int c = c0 + lane;
      float acc = 0.f;
      if (c < a.G) {
        const typename A::Col col = a.column(sorted_pos[beg], c);
        for (int i = beg + warp; i < end; i += WPB) acc += a.contrib(sorted_pos[i], c, col);
      }
      s_acc[warp][lane] = acc;
      __syncthreads();
      if (warp == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < WPB; ++w) t += s_acc[w][lane];
        if (c < ncols) out[c] = t;
      }
      __syncthreads();
    }
  }
}

__global__ void ffm_bwd_combine_kernel(const int32_t* __restrict__ counters,
                                       const int32_t* __restrict__ items,
                                       const float* __restrict__ partials, float* __restrict__ rows,
                                       int64_t ld_rows, int G) {
  const int n_items = counters[0];
  for (int h = blockIdx.x; h < n_items; h += gridDim.x) {
    const int meta = items[3 * h + 1];
    const int slot = items[3 * h + 2];
    if ((meta & 0xffff) != 0 || slot < 0) continue;   // not the head of a multi-chunk id
    const int chunks = meta >> 16;
    float* out = rows + (size_t)items[3 * h] * ld_rows;
    for (int c = threadIdx.x; c < ld_rows; c += blockDim.x) {
      float t = 0.f;
      if (c < G)
        for (int k = 0; k < chunks; ++k) t += partials[(size_t)(slot + k) * G + c];
      out[c] = t;
    }
  }
}

// Dense-parameter gradients: thread = one output column q of [ddense_w (Dn*R) | w1 part
// (a.w1_cols()) | dbias], blockIdx.y = a slice of the batch; each slice writes one partial row.
template <class A>
__global__ void __launch_bounds__(kFfmThreads)
ffm_bwd_dense_kernel(A a, int64_t B, int per_slice, float* __restrict__ partials) {
  const int n1 = a.w1_cols();
  const int len = a.Dn * a.R + n1 + 1;
  const int q = blockIdx.x * kFfmThreads + threadIdx.x;
  if (q >= len) return;
  const int64_t b0 = (int64_t)blockIdx.y * per_slice;
  const int64_t b1 = min(B, b0 + per_slice);
  float acc = 0.f;
  if (q < a.Dn * a.R) {
    const int k = q / a.R, c = q - k * a.R;
#pragma unroll 4
    for (int64_t b = b0; b < b1; ++b) acc = a.dense_w_acc(acc, b, k, c);
  } else if (q < a.Dn * a.R + n1) {
    const int k = q - a.Dn * a.R;
    for (int64_t b = b0; b < b1; ++b) acc = a.w1_acc(acc, b, k);
  } else {
    for (int64_t b = b0; b < b1; ++b) acc = a.bias_acc(acc, b);
  }
  partials[(size_t)blockIdx.y * len + q] = acc;
}

// out[q] = sum over slices of partials[slice][q], slices added in order.  n1 = the w1 part's
// width (Dn for FFM, 0 for a model without dense_w1).
__global__ void ffm_bwd_dense_reduce_kernel(const float* __restrict__ partials, int slices, int Dn,
                                            int R, int n1, float* __restrict__ ddense_w,
                                            float* __restrict__ ddense_w1, float* __restrict__ dbias) {
  const int len = Dn * R + n1 + 1;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= len) return;
  float t = 0.f;
  for (int s = 0; s < slices; ++s) t += partials[(size_t)s * len + q];
  if (q < Dn * R)
    ddense_w[q] = t;
  else if (q < Dn * R + n1)
    ddense_w1[q - Dn * R] = t;
  else if (dbias != nullptr)
    *dbias = t;
}

// The backward's launch sequence over the grouping of the B*F ids: light warps, then (when some id
// may be hot) the hot CTAs and the chunk combine, then the sliced dense-parameter partials and their
// reduce.  The functor a decides what each position contributes; n1 is its w1 part's width.
template <class A>
static int run_ffm_bwd_schedule(const A& a, const FfmBwdWs& L, int64_t B, int n1,
                                const int32_t* seg_offsets, const int32_t* sorted_pos,
                                const int32_t* num_unique, float* dW_rows, int64_t ld_dw,
                                float* ddense_w, float* ddense_w1, float* dbias, void* ws,
                                cudaStream_t st) {
  unsigned char* base = static_cast<unsigned char*>(ws);
  int32_t* counters = reinterpret_cast<int32_t*>(base);
  int32_t* items = reinterpret_cast<int32_t*>(base + L.off_items);
  float* partials = reinterpret_cast<float*>(base + L.off_part);
  float* dense_part = reinterpret_cast<float*>(base + L.off_dense);
  const int Dn = a.Dn, R = a.R;

  B200_CUDA(cudaMemsetAsync(counters, 0, 16, st));
  const int64_t n = B * a.F;
  constexpr int WPB = kFfmThreads / 32;
  const unsigned lgrid = (unsigned)min((n + WPB - 1) / WPB, (int64_t)sm_count() * 16);
  ffm_bwd_light_kernel<A><<<lgrid, kFfmThreads, 0, st>>>(a, seg_offsets, sorted_pos, num_unique,
                                                         dW_rows, ld_dw, counters, items);
  B200_LAUNCH_CHECK();
  if (n > kHotThreshold) {
    const unsigned hgrid = (unsigned)min(L.max_items, (int64_t)sm_count() * 8);
    ffm_bwd_hot_kernel<A><<<hgrid, kFfmThreads, 0, st>>>(a, seg_offsets, sorted_pos, counters,
                                                         items, partials, dW_rows, ld_dw);
    B200_LAUNCH_CHECK();
    ffm_bwd_combine_kernel<<<hgrid, 256, 0, st>>>(counters, items, partials, dW_rows, ld_dw, a.G);
    B200_LAUNCH_CHECK();
  }
  const int len = Dn * R + n1 + 1;
  const int per_slice = (int)((B + L.slices - 1) / L.slices);
  const dim3 dgrid((unsigned)((len + kFfmThreads - 1) / kFfmThreads), (unsigned)L.slices);
  ffm_bwd_dense_kernel<A><<<dgrid, kFfmThreads, 0, st>>>(a, B, per_slice, dense_part);
  B200_LAUNCH_CHECK();
  ffm_bwd_dense_reduce_kernel<<<(unsigned)((len + 255) / 256), 256, 0, st>>>(
      dense_part, L.slices, Dn, R, n1, ddense_w, ddense_w1, dbias);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_ffm_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                          const float* dense_w, const float* gy1, const float* gy2,
                          const int32_t* seg_offsets, const int32_t* sorted_pos,
                          const int32_t* num_unique, float* dW_rows, int64_t ld_dw, float* ddense_w,
                          float* ddense_w1, float* dbias, int64_t B, int F, int Dn, int D, int64_t V,
                          int64_t pad, void* ws, size_t ws_bytes, cudaStream_t st) {
  int rc = ffm_check_shape("ffm_bwd", F, Dn, D, ldw);
  if (rc != B200REC_OK) return rc;
  const int R = (F + Dn) * D, G = ffm_staged_cols(R);
  B200_REQUIRE(ld_dw >= R + 1, "ffm_bwd: ld_dw=%lld must hold R+1=%d columns", (long long)ld_dw,
               R + 1);
  B200_REQUIRE(B * F < (int64_t)INT32_MAX && (int64_t)(F + Dn) * R + F + Dn < (int64_t)INT32_MAX,
               "ffm_bwd: B*F must fit int32");
  B200_REQUIRE(B * F < (int64_t)32767 * kFfmHotChunk, "ffm_bwd: B*F=%lld too large",
               (long long)(B * F));
  const FfmBwdWs L(B, F, Dn, D);
  if (ws_bytes < L.total) {
    set_error("ffm_bwd: workspace %zu < %zu bytes", ws_bytes, L.total);
    return B200REC_ERR_WORKSPACE;
  }
  if (B == 0) {
    if (Dn > 0) {
      B200_CUDA(cudaMemsetAsync(ddense_w, 0, (size_t)Dn * R * sizeof(float), st));
      B200_CUDA(cudaMemsetAsync(ddense_w1, 0, (size_t)Dn * sizeof(float), st));
    }
    if (dbias != nullptr) B200_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float), st));
    return B200REC_OK;
  }
  const FfmBwd a{W, ldw, ids, dense, dense_w, gy1, gy2, F, Dn, D, R, G, V, pad};
  return run_ffm_bwd_schedule(a, L, B, Dn, seg_offsets, sorted_pos, num_unique, dW_rows, ld_dw,
                              ddense_w, ddense_w1, dbias, ws, st);
}

}  // namespace b200rec
