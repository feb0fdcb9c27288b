// FAT-DeepFFM: CENet field attention and the field-aware Hadamard interaction of
// models/rank/fat_deepffm/net.py (CENLayer :105-151, DeepFFM :219-251) fused with their gather,
// forward and backward.
//
// NF = F + Dn fields, R = NF*D, P = NF(NF-1)/2.  Row n of a sample is e[n,:] = W[ids[n], 0:R]
// (n < F) or dense[n-F] * dense_w[n-F, :] (n >= F); block m of it is e[n, m*D:(m+1)*D].
//   pool[n*NF+m] = max_d e[n, m*D+d]                 (first maximum wins the gradient)
//   attn         = the CENet MLP of pool              (tower GEMMs, outside these kernels)
//   s[n,m,:]     = attn[n*NF+m] * e[n, block m]
//   y1           = sum_{n,m,d} s[n,m,d] (+ bias)
//   h[p(n,m)*D+d] = s[n,m,d] * s[m,n,d]               (n < m, row-major pair order)
// The reference materialises feat [B, NF*NF, D] and the attention-weighted copy of it; here every
// gathered row crosses HBM once per kernel and nothing of size [B, NF, R] exists in either
// direction.  Table rows use FFM's fused slot layout [R emb | w1 | pad]; the w1 column is unused.
#pragma once

#include "ffm.cuh"

namespace b200rec {

__host__ __device__ inline int fat_pair_index(int n, int m, int NF) {   // n < m
  return n * NF - n * (n + 1) / 2 + (m - n - 1);
}

// P = NF(NF-1)/2 field pairs; 0 at NF = 1, where h and dh have no elements
inline int64_t fat_pairs(int F, int Dn) {
  const int64_t NF = (int64_t)F + Dn;
  return NF * (NF - 1) / 2;
}

// ---- pool forward ------------------------------------------------------------------------------
// One thread per (sample, block): a streaming gather in which each row is read once.  Padding and
// out-of-range ids read as a zero row and are counted here (once per position), not by the
// kernels that gather the same ids later in the step.
__global__ void __launch_bounds__(256)
fat_ffm_pool_kernel(const float* __restrict__ W, int64_t ldw, const int64_t* __restrict__ ids,
                    const float* __restrict__ dense, const float* __restrict__ dense_w,
                    float* __restrict__ pool, int64_t B, int F, int Dn, int D, int64_t V,
                    int64_t pad) {
  const int NF = F + Dn, R = NF * D, NN = NF * NF;
  const int64_t total = B * NN;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / NN;
    const int q = (int)(i - b * NN);
    const int n = q / NF, m = q - n * NF;
    float best = 0.f;
    if (n < F) {
      const int64_t id = __ldg(ids + b * F + n);
      const bool in_range = (uint64_t)id < (uint64_t)V;
      if (!in_range && m == 0) atomicAdd(&g_oob_count, 1ull);
      if (in_range && id != pad) {
        const float* w = W + (size_t)id * ldw + m * D;
        best = __ldg(w);
        for (int d = 1; d < D; ++d) best = fmaxf(best, __ldg(w + d));
      }
    } else {
      const float x = __ldg(dense + b * Dn + (n - F));
      const float* w = dense_w + (size_t)(n - F) * R + m * D;
      best = x * __ldg(w);
      for (int d = 1; d < D; ++d) best = fmaxf(best, x * __ldg(w + d));
    }
    pool[i] = best;
  }
}

// ---- per-sample kernels: interaction forward and attention backward ----------------------------
// Shared-memory layout: dense_w resident [Dn*R] | pair table [P] | the sample's attention row
// [NF*NF] | reduction scratch | nbuf sample buffers of F staged rows (Rs floats each).
struct FatSmem {
  size_t off_pairs, off_attn, off_red, off_buf, buf_bytes, total;
  FatSmem(int F, int Dn, int D, int nbuf) {
    const int NF = F + Dn, R = NF * D, P = NF * (NF - 1) / 2;
    off_pairs = align_up((size_t)Dn * R * 4, 16);
    off_attn = align_up(off_pairs + (size_t)P * 4, 16);
    off_red = align_up(off_attn + (size_t)NF * NF * 4, 16);
    off_buf = off_red + 16 * (kFfmThreads / 32 + 4);
    buf_bytes = (size_t)F * ffm_staged_cols(R) * 4;
    total = off_buf + (size_t)nbuf * buf_bytes;
  }
};

struct FatSampleArgs {
  const float* W;
  int64_t ldw;
  const int64_t* ids;
  const float* dense;
  const float* dense_w;
  const float* attn;   // [B, NF*NF]
  const float* bias;   // forward: [1] or null
  const float* gy1;    // backward: [B]
  const float* dh;     // backward: [B, P*D]
  float* y1;           // forward: [B]
  float* out;          // forward: h [B, P*D]; backward: dattn [B, NF*NF]
  int64_t B;
  int F, Dn, D;
  int64_t V, pad;
};

// Persistent CTAs, one sample at a time, staged as ffm_fwd_kernel stages them: the sample's F rows
// stream into shared memory with 16-byte cp.async, double-buffered when two samples fit, and
// dense_w stays resident.  kBwd = false: y1 (fixed-order block sum) and h, written coalesced in the
// reference's pair order.  kBwd = true: dattn[n,m] = sum_d e[n,m,d] * ds[n,m,d] with
// ds = gy1 + [n != m] * dh[p(n,m), d] * s[m,n,d]; dh is read from global memory (each element
// twice, by the two blocks of its pair), which keeps the sample buffers small enough to double.
template <bool kBwd>
__global__ void __launch_bounds__(kFfmThreads)
fat_ffm_sample_kernel(FatSampleArgs a, int nbuf, size_t off_pairs, size_t off_attn, size_t off_red,
                      size_t off_buf) {
  extern __shared__ __align__(16) unsigned char fat_smem[];
  const int F = a.F, Dn = a.Dn, D = a.D;
  const int NF = F + Dn, R = NF * D, P = NF * (NF - 1) / 2, NN = NF * NF;
  const int Rs = ffm_staged_cols(R), C = Rs / 4;
  float* s_dw = reinterpret_cast<float*>(fat_smem);
  uint32_t* s_pairs = reinterpret_cast<uint32_t*>(fat_smem + off_pairs);
  float* s_attn = reinterpret_cast<float*>(fat_smem + off_attn);
  float* s_red = reinterpret_cast<float*>(fat_smem + off_red);
  float* s_buf = reinterpret_cast<float*>(fat_smem + off_buf);
  const size_t buf_floats = (size_t)F * Rs;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int i = threadIdx.x; i < Dn * R; i += kFfmThreads) s_dw[i] = __ldg(a.dense_w + i);
  for (int n = threadIdx.x; n < NF; n += kFfmThreads) {
    const int base = fat_pair_index(n, n + 1, NF);
    for (int m = n + 1; m < NF; ++m) s_pairs[base + m - n - 1] = ((uint32_t)n << 16) | (uint32_t)m;
  }

  auto stage = [&](int64_t b, float* buf) {
    for (int i = threadIdx.x; i < F * C; i += kFfmThreads) {
      const int f = i / C, c = i - f * C;
      const int64_t id = __ldg(a.ids + b * F + f);
      float* dst = buf + (size_t)f * Rs + c * 4;
      if ((uint64_t)id < (uint64_t)a.V && id != a.pad)
        cp_async_16_cg(dst, a.W + (size_t)id * a.ldw + c * 4);
      else
        *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };

  int64_t b = blockIdx.x;
  if (nbuf == 2 && b < a.B) stage(b, s_buf);
  cp_async_commit();
  for (int it = 0; b < a.B; b += gridDim.x, ++it) {
    float* rows;
    if (nbuf == 2) {
      const int64_t nb = b + gridDim.x;
      if (nb < a.B) stage(nb, s_buf + (size_t)((it + 1) & 1) * buf_floats);
      cp_async_commit();
      cp_async_wait<1>();
      rows = s_buf + (size_t)(it & 1) * buf_floats;
    } else {
      stage(b, s_buf);
      cp_async_commit();
      cp_async_wait<0>();
      rows = s_buf;
    }
    for (int q = threadIdx.x; q < NN; q += kFfmThreads) s_attn[q] = __ldg(a.attn + b * NN + q);
    __syncthreads();

    const float* x = a.dense + b * Dn;
    // e[n, c] exactly as the reference forms it (a dense row is the fp32 product dense * dense_w)
    auto e = [&](int n, int c) -> float {
      return n < F ? rows[(size_t)n * Rs + c] : __ldg(x + n - F) * s_dw[(size_t)(n - F) * R + c];
    };

    if constexpr (!kBwd) {
      float acc = 0.f;
      for (int q = threadIdx.x; q < NN; q += kFfmThreads) {
        const int n = q / NF, m = q - n * NF;
        float t = 0.f;
        for (int d = 0; d < D; ++d) t += e(n, m * D + d);
        acc = fmaf(s_attn[q], t, acc);
      }
      float* h = a.out + b * (int64_t)P * D;
      for (int i = threadIdx.x; i < P * D; i += kFfmThreads) {
        const int p = i / D, d = i - p * D;
        const uint32_t nm = s_pairs[p];
        const int n = (int)(nm >> 16), m = (int)(nm & 0xffffu);
        h[i] = (s_attn[n * NF + m] * e(n, m * D + d)) * (s_attn[m * NF + n] * e(m, n * D + d));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) s_red[warp] = acc;
      __syncthreads();
      if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < kFfmThreads / 32; ++w) t += s_red[w];
        if (a.bias != nullptr) t += __ldg(a.bias);
        a.y1[b] = t;
      }
    } else {
      const float g = __ldg(a.gy1 + b);
      const float* dh = a.dh + b * (int64_t)P * D;
      for (int q = threadIdx.x; q < NN; q += kFfmThreads) {
        const int n = q / NF, m = q - n * NF;
        float acc = 0.f;
        if (n == m) {
          for (int d = 0; d < D; ++d) acc = fmaf(e(n, m * D + d), g, acc);
        } else {
          const float* dhp = dh + (size_t)fat_pair_index(min(n, m), max(n, m), NF) * D;
          const float a_mn = s_attn[m * NF + n];
          for (int d = 0; d < D; ++d) {
            const float ds = fmaf(__ldg(dhp + d), a_mn * e(m, n * D + d), g);
            acc = fmaf(e(n, m * D + d), ds, acc);
          }
        }
        a.out[b * NN + q] = acc;
      }
    }
    __syncthreads();   // the buffer, s_attn and s_red are free for the next sample
  }
  cp_async_wait<0>();
}

// ---- table and dense-parameter backward ---------------------------------------------------------
// Gradient of e at (b, n, block m, column j):
//   de = attn[n,m] * (gy1 + [m != n] * dh[p(n,m), j] * attn[m,n] * e[m, n*D+j])
//        + [j = first argmax_d e[n, m*D+d]] * dpool[n*NF+m]
// A table row takes de of every position of its id (column R, the unused w1, and the padding
// columns stay 0); ddense_w[k, c] = sum_b dense[b,k] * de(b, F+k, c); dbias = sum_b gy1[b].
// Runs on FFM's scheduling (ffm.cuh) as its per-position functor.
struct FatBwd {
  const float* W;
  int64_t ldw;
  const int64_t* ids;
  const float* dense;
  const float* dense_w;
  const float* gy1;
  const float* dh;
  const float* attn;
  const float* dpool;
  int F, Dn, D, R, G, NF;
  int64_t V, pad;

  // e[b, m, c]
  __device__ __forceinline__ float elem(int64_t b, int m, int c) const {
    if (m < F) {
      const int64_t id = __ldg(ids + b * F + m);
      if ((uint64_t)id >= (uint64_t)V || id == pad) return 0.f;
      return __ldg(W + (size_t)id * ldw + c);
    }
    return __ldg(dense + b * Dn + (m - F)) * __ldg(dense_w + (size_t)(m - F) * R + c);
  }
  // everything of de but the pool route, for row n = field n of sample b
  __device__ __forceinline__ float attn_route(int64_t b, int n, int m, int j) const {
    const float* at = attn + b * NF * NF;
    float ds = __ldg(gy1 + b);
    if (m != n) {
      const int p = fat_pair_index(min(n, m), max(n, m), NF);
      const float s_mn = __ldg(at + m * NF + n) * elem(b, m, n * D + j);
      ds = fmaf(__ldg(dh + (b * (NF * (NF - 1) / 2) + p) * D + j), s_mn, ds);
    }
    return __ldg(at + n * NF + m) * ds;
  }

  // The argmax of a sparse field's block depends only on the table row, so it is found once per
  // (id, column) by the scheduling kernels, not once per position.
  struct Col {
    bool is_max;
  };
  __device__ __forceinline__ Col column(int p, int c) const {
    if (c >= R) return {false};
    const int64_t id = __ldg(ids + p);
    const int m = c / D, j = c - m * D;
    const float* w = W + (size_t)id * ldw + m * D;
    int best = 0;
    float bv = __ldg(w);
    for (int d = 1; d < D; ++d) {
      const float v = __ldg(w + d);
      if (v > bv) { bv = v; best = d; }
    }
    return {best == j};
  }
  // contribution of position p = b*F + f to column c of its gradient row
  __device__ __forceinline__ float contrib(int p, int c, Col col) const {
    if (c >= R) return 0.f;
    const int64_t b = p / F;
    const int f = p - (int)b * F;
    const int m = c / D, j = c - m * D;
    float g = attn_route(b, f, m, j);
    if (col.is_max) g += __ldg(dpool + b * NF * NF + f * NF + m);
    return g;
  }

  __device__ __forceinline__ int w1_cols() const { return 0; }
  __device__ __forceinline__ float dense_w_acc(float acc, int64_t b, int k, int c) const {
    const int n = F + k, m = c / D, j = c - m * D;
    const float x = __ldg(dense + b * Dn + k);
    // first argmax of the block on the fp32 product, exactly as the pool forward forms it
    const float* w = dense_w + (size_t)k * R + m * D;
    int best = 0;
    float bv = x * __ldg(w);
    for (int d = 1; d < D; ++d) {
      const float v = x * __ldg(w + d);
      if (v > bv) { bv = v; best = d; }
    }
    float g = attn_route(b, n, m, j);
    if (best == j) g += __ldg(dpool + b * NF * NF + n * NF + m);
    return fmaf(x, g, acc);
  }
  __device__ __forceinline__ float w1_acc(float acc, int64_t, int) const { return acc; }
  __device__ __forceinline__ float bias_acc(float acc, int64_t b) const { return acc + __ldg(gy1 + b); }
};

// ---- launchers ---------------------------------------------------------------------------------
static int fat_check(const char* what, int64_t B, int F, int Dn, int D, int64_t ldw) {
  int rc = ffm_check_shape(what, F, Dn, D, ldw);
  if (rc != B200REC_OK) return rc;
  const int64_t NF = F + Dn;
  B200_REQUIRE(B >= 0 && NF * NF * D < (int64_t)INT32_MAX, "%s: NF*NF*D=%lld must fit int32", what,
               (long long)(NF * NF * D));
  return B200REC_OK;
}

static int launch_fat_ffm_pool(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                               const float* dense_w, float* pool, int64_t B, int F, int Dn, int D,
                               int64_t V, int64_t pad, cudaStream_t st) {
  int rc = fat_check("fat_ffm_pool_fwd", B, F, Dn, D, ldw);
  if (rc != B200REC_OK) return rc;
  if (B == 0) return B200REC_OK;
  const int64_t total = B * (F + Dn) * (F + Dn);
  const int64_t grid = min((total + 255) / 256, (int64_t)sm_count() * 16);
  fat_ffm_pool_kernel<<<(unsigned)grid, 256, 0, st>>>(W, ldw, ids, dense, dense_w, pool, B, F, Dn, D,
                                                      V, pad);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

template <bool kBwd>
static int launch_fat_sample(const char* what, const FatSampleArgs& a, cudaStream_t st) {
  int rc = fat_check(what, a.B, a.F, a.Dn, a.D, a.ldw);
  if (rc != B200REC_OK) return rc;
  B200_REQUIRE(aligned16(a.W), "%s: W must be 16-byte aligned", what);
  int nbuf = 2;
  FatSmem L(a.F, a.Dn, a.D, nbuf);
  if (L.total > (size_t)ffm_max_smem()) {
    nbuf = 1;
    L = FatSmem(a.F, a.Dn, a.D, nbuf);
  }
  const int NF = a.F + a.Dn;
  B200_REQUIRE(L.total <= (size_t)ffm_max_smem(),
               "%s: one sample (F=%d rows of %d floats, %d attention weights) and dense_w (%d x %d) "
               "need %zu bytes of shared memory, more than the %d a CTA may use",
               what, a.F, ffm_staged_cols(NF * a.D), NF * NF, a.Dn, NF * a.D, L.total,
               ffm_max_smem());
  if (a.B == 0) return B200REC_OK;
  B200_CUDA(cudaFuncSetAttribute(fat_ffm_sample_kernel<kBwd>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total));
  int per_sm = 1;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fat_ffm_sample_kernel<kBwd>,
                                                          kFfmThreads, L.total));
  const int64_t grid = min(a.B, (int64_t)sm_count() * max(per_sm, 1));
  fat_ffm_sample_kernel<kBwd><<<(unsigned)grid, kFfmThreads, L.total, st>>>(
      a, nbuf, L.off_pairs, L.off_attn, L.off_red, L.off_buf);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_fat_ffm_bwd(const FatBwd& a, const int32_t* seg_offsets,
                              const int32_t* sorted_pos, const int32_t* num_unique, float* dW_rows,
                              int64_t ld_dw, float* ddense_w, float* dbias, int64_t B, void* ws,
                              size_t ws_bytes, cudaStream_t st) {
  int rc = fat_check("fat_ffm_bwd", B, a.F, a.Dn, a.D, a.ldw);
  if (rc != B200REC_OK) return rc;
  B200_REQUIRE(ld_dw >= a.R + 1, "fat_ffm_bwd: ld_dw=%lld must hold R+1=%d columns",
               (long long)ld_dw, a.R + 1);
  B200_REQUIRE(B * a.F < (int64_t)INT32_MAX && (int64_t)a.NF * a.R + a.NF < (int64_t)INT32_MAX,
               "fat_ffm_bwd: B*F must fit int32");
  B200_REQUIRE(B * a.F < (int64_t)32767 * kFfmHotChunk, "fat_ffm_bwd: B*F=%lld too large",
               (long long)(B * a.F));
  const FfmBwdWs L(B, a.F, a.Dn, a.D);
  if (ws_bytes < L.total) {
    set_error("fat_ffm_bwd: workspace %zu < %zu bytes", ws_bytes, L.total);
    return B200REC_ERR_WORKSPACE;
  }
  if (B == 0) {
    if (a.Dn > 0) B200_CUDA(cudaMemsetAsync(ddense_w, 0, (size_t)a.Dn * a.R * sizeof(float), st));
    if (dbias != nullptr) B200_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float), st));
    return B200REC_OK;
  }
  return run_ffm_bwd_schedule(a, L, B, 0, seg_offsets, sorted_pos, num_unique, dW_rows, ld_dw,
                              ddense_w, nullptr, dbias, ws, st);
}

}  // namespace b200rec
