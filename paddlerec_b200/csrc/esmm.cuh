// ESMM's two width-2 heads and the CTCVR product (models/multitask/esmm/net.py:85-111) as one
// streaming kernel each way, on the towers' last ReLU'd activations h_t [B,K] (t = ctr, cvr):
//
//   forward   z_t = h_t @ W_t + b_t                      (W_t [K,2], exact fp32 FMAs)
//             p1_t = 1/(1+expf(z0-z1)),  p0_t = 1/(1+expf(z1-z0))     each class on its own, so the
//                                                        small one keeps its relative accuracy
//             ctr_out = p_ctr, ctr_one = p1_ctr, cvr_out = p_cvr, cvr_one = p1_cvr,
//             ctcvr_one = p1_ctr * p1_cvr,  ctcvr_prop = [1 - ctcvr_one, ctcvr_one]
//   backward  G_t = g_t_out + [0, g_t_one]              (every incoming gradient may be NULL)
//             Gc = g_ctcvr_prop[:,1] + g_ctcvr_one - g_ctcvr_prop[:,0]
//             G_ctr1 += Gc * p1_cvr,  G_cvr1 += Gc * p1_ctr
//             s_t = p0_t p1_t (G_t1 - G_t0),  dz_t = [-s_t, s_t]
//             dh_t = dz_t @ W_t^T,  dW_t = h_t^T @ dz_t,  db_t = colsum(dz_t)
//
// LPR lanes own one row; a lane owns the same 4-column chunks of every row it visits, so its dW
// sums stay in registers.  Lanes holding the same chunks are summed with a fixed xor butterfly,
// the warps of a CTA in warp order in shared memory, and the CTAs by reduce_partials_kernel in CTA
// order: no float atomics, and a second run is bit-identical.
#pragma once

#include "common.cuh"

namespace b200rec {

constexpr int kEsmmThreads = 256;
constexpr int kEsmmWarps = kEsmmThreads / 32;
constexpr int kEsmmMaxK = 256;       // keeps the backward's shared memory under 48 KB

struct EsmmGrads {                   // incoming gradients of the six outputs, each may be NULL
  const float* ctr_out;              // [B,2]
  const float* ctr_one;              // [B,1]
  const float* cvr_out;              // [B,2]
  const float* cvr_one;              // [B,1]
  const float* ctcvr_prop;           // [B,2]
  const float* ctcvr_one;            // [B,1]
};

__device__ __forceinline__ float esmm_ld(const float* p, int64_t i) {
  return p != nullptr ? __ldg(p + i) : 0.f;
}

template <int LPR>
__global__ void __launch_bounds__(kEsmmThreads)
esmm_head_fwd_kernel(const float* __restrict__ h_ctr, const float* __restrict__ h_cvr, int K,
                     const float* __restrict__ W_ctr, const float* __restrict__ b_ctr,
                     const float* __restrict__ W_cvr, const float* __restrict__ b_cvr,
                     float* __restrict__ ctr_out, float* __restrict__ ctr_one,
                     float* __restrict__ cvr_out, float* __restrict__ cvr_one,
                     float* __restrict__ ctcvr_prop, float* __restrict__ ctcvr_one, int64_t B) {
  extern __shared__ float s_w[];     // [2K] W_ctr, then [2K] W_cvr (row k: columns 0, 1)
  for (int i = threadIdx.x; i < 2 * K; i += kEsmmThreads) {
    s_w[i] = W_ctr[i];
    s_w[2 * K + i] = W_cvr[i];
  }
  __syncthreads();
  constexpr int RPW = 32 / LPR;      // rows per warp
  const int lane = threadIdx.x & 31, sub = lane % LPR;
  const int64_t row0 = ((int64_t)blockIdx.x * kEsmmWarps + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const int64_t stride = (int64_t)gridDim.x * kEsmmWarps * RPW;
  const int chunks = K / 4;
  const float bc0 = __ldg(b_ctr), bc1 = __ldg(b_ctr + 1);
  const float bv0 = __ldg(b_cvr), bv1 = __ldg(b_cvr + 1);
  // every lane of a warp runs the same trip count, so the shuffles below see all 32 lanes
  const int64_t trips = (B - (row0 - lane / LPR) + stride - 1) / stride;
  int64_t b = row0;
  for (int64_t it = 0; it < trips; ++it, b += stride) {
    const bool live = b < B;
    float zc0 = 0.f, zc1 = 0.f, zv0 = 0.f, zv1 = 0.f;
    if (live) {
      const float4* hc = reinterpret_cast<const float4*>(h_ctr + b * K);
      const float4* hv = reinterpret_cast<const float4*>(h_cvr + b * K);
      for (int c = sub; c < chunks; c += LPR) {
        const float4 x = __ldg(hc + c), y = __ldg(hv + c);
        const float xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = 4 * c + j;
          zc0 = fmaf(xs[j], s_w[2 * k], zc0);
          zc1 = fmaf(xs[j], s_w[2 * k + 1], zc1);
          zv0 = fmaf(ys[j], s_w[2 * K + 2 * k], zv0);
          zv1 = fmaf(ys[j], s_w[2 * K + 2 * k + 1], zv1);
        }
      }
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
      zc0 += __shfl_xor_sync(0xffffffffu, zc0, o);
      zc1 += __shfl_xor_sync(0xffffffffu, zc1, o);
      zv0 += __shfl_xor_sync(0xffffffffu, zv0, o);
      zv1 += __shfl_xor_sync(0xffffffffu, zv1, o);
    }
    if (live && sub == 0) {
      zc0 += bc0; zc1 += bc1; zv0 += bv0; zv1 += bv1;
      const float pc1 = 1.f / (1.f + expf(zc0 - zc1)), pc0 = 1.f / (1.f + expf(zc1 - zc0));
      const float pv1 = 1.f / (1.f + expf(zv0 - zv1)), pv0 = 1.f / (1.f + expf(zv1 - zv0));
      const float one = pc1 * pv1;
      ctr_out[2 * b] = pc0; ctr_out[2 * b + 1] = pc1; ctr_one[b] = pc1;
      cvr_out[2 * b] = pv0; cvr_out[2 * b + 1] = pv1; cvr_one[b] = pv1;
      ctcvr_prop[2 * b] = 1.f - one; ctcvr_prop[2 * b + 1] = one; ctcvr_one[b] = one;
    }
  }
}

template <int LPR, int NITER>
__global__ void __launch_bounds__(kEsmmThreads)
esmm_head_bwd_kernel(EsmmGrads g, const float* __restrict__ p_ctr, const float* __restrict__ p_cvr,
                     const float* __restrict__ h_ctr, const float* __restrict__ h_cvr, int K,
                     const float* __restrict__ W_ctr, const float* __restrict__ W_cvr,
                     float* __restrict__ dh_ctr, float* __restrict__ dh_cvr,
                     float* __restrict__ part_ctr, float* __restrict__ part_cvr, int64_t B) {
  // [4K] weights (as the forward), then [warps][2 towers][2K + 2] per-warp dW | db partials
  extern __shared__ float s_buf[];
  float* s_w = s_buf;
  float* s_part = s_buf + 4 * K;
  const int L = 2 * K + 2;
  for (int i = threadIdx.x; i < 2 * K; i += kEsmmThreads) {
    s_w[i] = W_ctr[i];
    s_w[2 * K + i] = W_cvr[i];
  }
  __syncthreads();
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane % LPR, warp = threadIdx.x >> 5;
  const int64_t b0 = ((int64_t)blockIdx.x * kEsmmWarps + warp) * RPW + lane / LPR;
  const int64_t stride = (int64_t)gridDim.x * kEsmmWarps * RPW;
  const int chunks = K / 4;
  float acc[2][NITER][8];            // [tower][iter][4 columns x 2 classes], dW row-major
#pragma unroll
  for (int t = 0; t < 2; ++t)
#pragma unroll
    for (int i = 0; i < NITER; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[t][i][j] = 0.f;
  float db[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int64_t b = b0; b < B; b += stride) {
    const float pc0 = __ldg(p_ctr + 2 * b), pc1 = __ldg(p_ctr + 2 * b + 1);
    const float pv0 = __ldg(p_cvr + 2 * b), pv1 = __ldg(p_cvr + 2 * b + 1);
    const float Gc = esmm_ld(g.ctcvr_prop, 2 * b + 1) + esmm_ld(g.ctcvr_one, b) -
                     esmm_ld(g.ctcvr_prop, 2 * b);
    const float Gc0 = esmm_ld(g.ctr_out, 2 * b);
    const float Gc1 = esmm_ld(g.ctr_out, 2 * b + 1) + esmm_ld(g.ctr_one, b) + Gc * pv1;
    const float Gv0 = esmm_ld(g.cvr_out, 2 * b);
    const float Gv1 = esmm_ld(g.cvr_out, 2 * b + 1) + esmm_ld(g.cvr_one, b) + Gc * pc1;
    const float s[2] = {pc0 * pc1 * (Gc1 - Gc0), pv0 * pv1 * (Gv1 - Gv0)};
    if (sub == 0) {
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        db[t][0] -= s[t];
        db[t][1] += s[t];
      }
    }
    float4 x[2][NITER];              // every load of the row in flight before the first use
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int i = 0; i < NITER; ++i) {
        const int c = sub + LPR * i;
        x[t][i] = c < chunks
                      ? __ldg(reinterpret_cast<const float4*>((t == 0 ? h_ctr : h_cvr) + b * K) + c)
                      : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const float* w = s_w + 2 * K * t;
#pragma unroll
      for (int i = 0; i < NITER; ++i) {
        const int c = sub + LPR * i;
        if (c < chunks) {
          const float xs[4] = {x[t][i].x, x[t][i].y, x[t][i].z, x[t][i].w};
          float d[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int k = 4 * c + j;
            d[j] = fmaf(s[t], w[2 * k + 1], -s[t] * w[2 * k]);
            acc[t][i][2 * j] = fmaf(xs[j], -s[t], acc[t][i][2 * j]);
            acc[t][i][2 * j + 1] = fmaf(xs[j], s[t], acc[t][i][2 * j + 1]);
          }
          *(reinterpret_cast<float4*>((t == 0 ? dh_ctr : dh_cvr) + b * K) + c) =
              make_float4(d[0], d[1], d[2], d[3]);
        }
      }
    }
  }
  // rows of one warp that own the same chunks: fixed xor butterfly across the RPW row groups
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) {
#pragma unroll
    for (int t = 0; t < 2; ++t) {
#pragma unroll
      for (int i = 0; i < NITER; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[t][i][j] += __shfl_xor_sync(0xffffffffu, acc[t][i][j], o);
      db[t][0] += __shfl_xor_sync(0xffffffffu, db[t][0], o);
      db[t][1] += __shfl_xor_sync(0xffffffffu, db[t][1], o);
    }
  }
  float* mine = s_part + (size_t)warp * 2 * L;
  if (lane < LPR) {
#pragma unroll
    for (int t = 0; t < 2; ++t) {
#pragma unroll
      for (int i = 0; i < NITER; ++i) {
        const int c = lane + LPR * i;
        if (c < chunks)
#pragma unroll
          for (int j = 0; j < 8; ++j) mine[t * L + 8 * c + j] = acc[t][i][j];
      }
      if (lane == 0) {
        mine[t * L + 2 * K] = db[t][0];
        mine[t * L + 2 * K + 1] = db[t][1];
      }
    }
  }
  __syncthreads();
  // CTA sum in warp order, one partial row per CTA and tower: [2K] dW (row-major [K,2]) | [2] db
  for (int k = threadIdx.x; k < 2 * L; k += kEsmmThreads) {
    float sum = 0.f;
#pragma unroll
    for (int wv = 0; wv < kEsmmWarps; ++wv) sum += s_part[(size_t)wv * 2 * L + k];
    if (k < L)
      part_ctr[(size_t)blockIdx.x * L + k] = sum;
    else
      part_cvr[(size_t)blockIdx.x * L + k - L] = sum;
  }
}

static int esmm_lpr(int K) { return K <= 32 ? 8 : (K <= 64 ? 16 : 32); }

static size_t esmm_bwd_smem(int K) {
  return ((size_t)4 * K + (size_t)kEsmmWarps * 2 * (2 * K + 2)) * sizeof(float);
}

template <typename Kern>
static int esmm_grid(Kern kern, size_t smem, int64_t rows_per_cta, int64_t B, int* grid) {
  int per_sm = 0;
  B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kEsmmThreads, smem));
  const int64_t need = (B + rows_per_cta - 1) / rows_per_cta;
  const int64_t cap = (int64_t)sm_count() * (per_sm > 0 ? per_sm : 1);
  *grid = (int)(need < 1 ? 1 : (need < cap ? need : cap));
  return B200REC_OK;
}

// the backward's grid for (B, K): its partials need grid * 2 * (2K + 2) floats of workspace
static int esmm_bwd_grid(int64_t B, int K, int* grid) {
  const int lpr = esmm_lpr(K);
  const int niter = (K / 4 + lpr - 1) / lpr;
  const int64_t rows = (int64_t)kEsmmWarps * (32 / lpr);
  const size_t smem = esmm_bwd_smem(K);
  if (lpr == 8) return esmm_grid(esmm_head_bwd_kernel<8, 1>, smem, rows, B, grid);
  if (lpr == 16) return esmm_grid(esmm_head_bwd_kernel<16, 1>, smem, rows, B, grid);
  if (niter <= 1) return esmm_grid(esmm_head_bwd_kernel<32, 1>, smem, rows, B, grid);
  return esmm_grid(esmm_head_bwd_kernel<32, 2>, smem, rows, B, grid);
}

static bool esmm_k_ok(int K) { return K > 0 && K % 4 == 0 && K <= kEsmmMaxK; }

static int esmm_head_bwd_ws_bytes(int64_t B, int K, size_t* bytes) {
  int grid = 0;
  const int rc = esmm_bwd_grid(B, K, &grid);
  if (rc != B200REC_OK) return rc;
  *bytes = (size_t)grid * 2 * (2 * K + 2) * sizeof(float);
  return B200REC_OK;
}

static int launch_esmm_head_fwd(const float* h_ctr, const float* h_cvr, int K, const float* W_ctr,
                                const float* b_ctr, const float* W_cvr, const float* b_cvr,
                                float* ctr_out, float* ctr_one, float* cvr_out, float* cvr_one,
                                float* ctcvr_prop, float* ctcvr_one, int64_t B, cudaStream_t st) {
  B200_REQUIRE(B >= 0 && esmm_k_ok(K), "esmm_head_fwd: K=%d must be a multiple of 4 in [4, %d]", K,
               kEsmmMaxK);
  B200_REQUIRE(aligned16(h_ctr) && aligned16(h_cvr),
               "esmm_head_fwd: h_ctr and h_cvr must be 16-byte aligned");
  if (B == 0) return B200REC_OK;
  const size_t smem = (size_t)4 * K * sizeof(float);
  const int lpr = esmm_lpr(K);
  const int64_t rows = (int64_t)kEsmmWarps * (32 / lpr);
  int grid = 0;
#define B200_ESMM_FWD(LPR)                                                                         \
  do {                                                                                             \
    auto kern = esmm_head_fwd_kernel<LPR>;                                                         \
    const int rc = esmm_grid(kern, smem, rows, B, &grid);                                          \
    if (rc != B200REC_OK) return rc;                                                               \
    kern<<<grid, kEsmmThreads, smem, st>>>(h_ctr, h_cvr, K, W_ctr, b_ctr, W_cvr, b_cvr, ctr_out,   \
                                           ctr_one, cvr_out, cvr_one, ctcvr_prop, ctcvr_one, B);   \
  } while (0)
  if (lpr == 8) B200_ESMM_FWD(8);
  else if (lpr == 16) B200_ESMM_FWD(16);
  else B200_ESMM_FWD(32);
#undef B200_ESMM_FWD
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_esmm_head_bwd(const EsmmGrads& g, const float* p_ctr, const float* p_cvr,
                                const float* h_ctr, const float* h_cvr, int K, const float* W_ctr,
                                const float* W_cvr, float* dh_ctr, float* dh_cvr, float* dW_ctr,
                                float* db_ctr, float* dW_cvr, float* db_cvr, int64_t B, void* ws,
                                size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(B >= 0 && esmm_k_ok(K), "esmm_head_bwd: K=%d must be a multiple of 4 in [4, %d]", K,
               kEsmmMaxK);
  B200_REQUIRE(aligned16(h_ctr) && aligned16(h_cvr) && aligned16(dh_ctr) && aligned16(dh_cvr),
               "esmm_head_bwd: h and dh must be 16-byte aligned");
  if (B == 0) {
    B200_CUDA(cudaMemsetAsync(dW_ctr, 0, (size_t)2 * K * sizeof(float), st));
    B200_CUDA(cudaMemsetAsync(dW_cvr, 0, (size_t)2 * K * sizeof(float), st));
    B200_CUDA(cudaMemsetAsync(db_ctr, 0, 2 * sizeof(float), st));
    B200_CUDA(cudaMemsetAsync(db_cvr, 0, 2 * sizeof(float), st));
    return B200REC_OK;
  }
  size_t need = 0;
  int rc = esmm_head_bwd_ws_bytes(B, K, &need);
  if (rc != B200REC_OK) return rc;
  if (ws == nullptr || ws_bytes < need) {
    set_error("esmm_head_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return B200REC_ERR_WORKSPACE;
  }
  int grid = 0;
  rc = esmm_bwd_grid(B, K, &grid);
  if (rc != B200REC_OK) return rc;
  const int L = 2 * K + 2;
  float* part_ctr = static_cast<float*>(ws);
  float* part_cvr = part_ctr + (size_t)grid * L;
  const size_t smem = esmm_bwd_smem(K);
  const int lpr = esmm_lpr(K);
  const int niter = (K / 4 + lpr - 1) / lpr;
#define B200_ESMM_BWD(LPR, NI)                                                                     \
  esmm_head_bwd_kernel<LPR, NI><<<grid, kEsmmThreads, smem, st>>>(                                 \
      g, p_ctr, p_cvr, h_ctr, h_cvr, K, W_ctr, W_cvr, dh_ctr, dh_cvr, part_ctr, part_cvr, B)
  if (lpr == 8) B200_ESMM_BWD(8, 1);
  else if (lpr == 16) B200_ESMM_BWD(16, 1);
  else if (niter <= 1) B200_ESMM_BWD(32, 1);
  else B200_ESMM_BWD(32, 2);
#undef B200_ESMM_BWD
  B200_LAUNCH_CHECK();
  reduce_partials_kernel<<<reduce_partials_grid(L), kRedThreads, 0, st>>>(part_ctr, grid, L, dW_ctr,
                                                                          2 * K, db_ctr);
  B200_LAUNCH_CHECK();
  reduce_partials_kernel<<<reduce_partials_grid(L), kRedThreads, 0, st>>>(part_cvr, grid, L, dW_cvr,
                                                                          2 * K, db_cvr);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

}  // namespace b200rec
