// Tower epilogues: the elementwise halves of the dense MLP tower when its GEMMs run on the bf16
// tensor cores with a hi/lo split of the fp32 operands ("bf16x3": a*b ~ a_hi*b_hi + a_lo*b_hi +
// a_hi*b_lo, exact products accumulated in fp32, ~2^-16 relative error — meets the 1e-4 bar that
// plain TF32 misses).
//
// Reference: DNN.forward models/rank/deepfm/net.py:169-174 (Linear -> ReLU chain) and its autograd.
// The GEMMs themselves are library calls (cuBLASLt through torch.mm(out_dtype=fp32)); what the
// reference spreads over bias-add / ReLU / cast kernels is one streaming pass per layer here:
//   forward : y(fp32) --(+bias, ReLU, split)--> [hi | lo] bf16, directly the next GEMM's A operand
//   backward: dy(fp32) --(ReLU mask from the saved hi half, split, bias column-sum)--> [hi | lo]
//   weights : W(fp32) --> the three bf16 operand layouts the forward/backward GEMMs consume
// All HBM-bound: 8 B/element forward, 10 B/element backward.
#pragma once

#include <cuda_bf16.h>

#include "common.cuh"

namespace b200rec {

constexpr int kTowerThreads = 256;

__device__ __forceinline__ void split1(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

struct alignas(8) Bf16x4 {
  __nv_bfloat16 v[4];
};

// out[m, k] = hi(f(x[m,k])), out[m, K+k] = lo(...), f = optional (+bias[k]) then optional ReLU.
template <int VEC>
__global__ void __launch_bounds__(kTowerThreads)
tower_split_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ bias,
                   int relu, __nv_bfloat16* __restrict__ out, int64_t ldp, int64_t M, int K,
                   int ones_col) {
  const int chunks = K / VEC;
  const int64_t total = M * chunks;
  for (int64_t i = (int64_t)blockIdx.x * kTowerThreads + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * kTowerThreads) {
    const int64_t m = i / chunks;
    const int k = (int)(i - m * chunks) * VEC;
    Vec<VEC> a = ld_row<VEC>(x + (size_t)m * ldx + k);
    if (bias != nullptr) {
      const Vec<VEC> b = ld_cached<VEC>(bias + k);
#pragma unroll
      for (int j = 0; j < VEC; ++j) a.v[j] += b.v[j];
    }
    if (relu) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) a.v[j] = fmaxf(a.v[j], 0.f);
    }
    __nv_bfloat16* row = out + (size_t)m * 2 * ldp;
    if (ones_col && k == 0) {   // column K of the hi plane = 1: the dW GEMM then yields colsum(g)
      row[K] = __float2bfloat16_rn(1.f);
      row[ldp + K] = __float2bfloat16_rn(0.f);
    }
    if (VEC == 4) {
      Bf16x4 hi, lo;
#pragma unroll
      for (int j = 0; j < 4; ++j) split1(a.v[j], hi.v[j], lo.v[j]);
      *reinterpret_cast<Bf16x4*>(row + k) = hi;
      *reinterpret_cast<Bf16x4*>(row + ldp + k) = lo;
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) split1(a.v[j], row[k + j], row[ldp + k + j]);
    }
  }
}

// dz = dy * (act_hi > 0) (mask skipped if act == nullptr); dz_out = [hi | lo]; partial column sums
// of dz per row-slice (thread owns its columns => register accumulation, fixed order).
template <int VEC>
__device__ __forceinline__ void relu_bwd_split_row(Vec<VEC>& g, const __nv_bfloat16* a,
                                                   __nv_bfloat16* row, int64_t N, int c) {
  if (a != nullptr) {
    if (VEC == 4) {
      const Bf16x4 h = *reinterpret_cast<const Bf16x4*>(a);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (!(__bfloat162float(h.v[j]) > 0.f)) g.v[j] = 0.f;
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        if (!(__bfloat162float(a[j]) > 0.f)) g.v[j] = 0.f;
    }
  }
  if (VEC == 4) {
    Bf16x4 hi, lo;
#pragma unroll
    for (int j = 0; j < 4; ++j) split1(g.v[j], hi.v[j], lo.v[j]);
    *reinterpret_cast<Bf16x4*>(row + c) = hi;
    *reinterpret_cast<Bf16x4*>(row + N + c) = lo;
  } else {
#pragma unroll
    for (int j = 0; j < VEC; ++j) split1(g.v[j], row[c + j], row[N + c + j]);
  }
}

// blockDim = (TX column chunks, TY rows); a thread owns its columns and walks rows
// blockIdx.y*TY + ty, stepping gridDim.y*TY, four rows in flight.
constexpr int kBwdUnroll = 4;

template <int VEC>
__global__ void __launch_bounds__(kTowerThreads)
tower_relu_bwd_split_kernel(const float* __restrict__ dy, const __nv_bfloat16* __restrict__ act,
                            int64_t ld_act, __nv_bfloat16* __restrict__ dz, int64_t ldp,
                            float* __restrict__ partials, int64_t M, int N) {
  const int chunks = N / VEC;
  const int chunk = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = chunk * VEC;
  const bool col_ok = chunk < chunks;
  const int64_t row_step = (int64_t)gridDim.y * blockDim.y;
  Vec<VEC> acc = vzero<VEC>();
  if (col_ok) {
    int64_t m = (int64_t)blockIdx.y * blockDim.y + threadIdx.y;
    for (; m + (kBwdUnroll - 1) * row_step < M; m += kBwdUnroll * row_step) {
      Vec<VEC> g[kBwdUnroll];
#pragma unroll
      for (int u = 0; u < kBwdUnroll; ++u)
        g[u] = ld_row<VEC>(dy + (size_t)(m + u * row_step) * N + c);
#pragma unroll
      for (int u = 0; u < kBwdUnroll; ++u) {
        const int64_t mm = m + u * row_step;
        relu_bwd_split_row<VEC>(g[u], act ? act + (size_t)mm * 2 * ld_act + c : nullptr,
                                dz + (size_t)mm * 2 * ldp, ldp, c);
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc.v[j] += g[u].v[j];
      }
    }
    for (; m < M; m += row_step) {
      Vec<VEC> g = ld_row<VEC>(dy + (size_t)m * N + c);
      relu_bwd_split_row<VEC>(g, act ? act + (size_t)m * 2 * ld_act + c : nullptr,
                              dz + (size_t)m * 2 * ldp, ldp, c);
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc.v[j] += g.v[j];
    }
  }
  // reduce the TY row-threads of the block in shared memory (fixed order), one partial per block
  __shared__ float s_part[kTowerThreads * 4];
#pragma unroll
  for (int j = 0; j < VEC; ++j)
    s_part[(threadIdx.y * blockDim.x + threadIdx.x) * VEC + j] = acc.v[j];
  __syncthreads();
  if (threadIdx.y == 0 && col_ok) {
    Vec<VEC> t = vzero<VEC>();
    for (int y = 0; y < (int)blockDim.y; ++y)
#pragma unroll
      for (int j = 0; j < VEC; ++j) t.v[j] += s_part[(y * blockDim.x + threadIdx.x) * VEC + j];
    st_plain<VEC>(partials + (size_t)blockIdx.y * N + c, t);
  }
}

// Backward of the GateNet hidden gate z = y * tanh(a), a = y @ G (gatenet/net.py:116-118), given dz:
//   planes(g) with g = dz * y * (1 - tanh(a)^2)   (the operand of dG = y^T g and of g @ G^T)
//   r = dz * tanh(a)                               (fp32, the addend of that dX GEMM)
// y = hi + lo of its planes, exactly the value the forward epilogue multiplied.  One streaming pass.
template <int VEC>
__global__ void __launch_bounds__(kTowerThreads)
tower_gate_bwd_kernel(const float* __restrict__ dz, const __nv_bfloat16* __restrict__ y, int64_t ldy,
                      const float* __restrict__ a, __nv_bfloat16* __restrict__ g, int64_t ldp,
                      float* __restrict__ r, int64_t M, int N) {
  const int chunks = N / VEC;
  const int64_t total = M * chunks;
  for (int64_t i = (int64_t)blockIdx.x * kTowerThreads + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * kTowerThreads) {
    const int64_t m = i / chunks;
    const int c = (int)(i - m * chunks) * VEC;
    const Vec<VEC> d = ld_row<VEC>(dz + (size_t)m * N + c);
    const Vec<VEC> t = ld_row<VEC>(a + (size_t)m * N + c);
    const __nv_bfloat16* yr = y + (size_t)m * 2 * ldy + c;
    Vec<VEC> gv, rv;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float yv = __bfloat162float(yr[j]) + __bfloat162float(yr[ldy + j]);
      const float th = tanhf(t.v[j]);
      gv.v[j] = d.v[j] * yv * (1.f - th * th);
      rv.v[j] = d.v[j] * th;
    }
    st_plain<VEC>(r + (size_t)m * N + c, rv);
    __nv_bfloat16* row = g + (size_t)m * 2 * ldp;
    if (VEC == 4) {
      Bf16x4 hi, lo;
#pragma unroll
      for (int j = 0; j < 4; ++j) split1(gv.v[j], hi.v[j], lo.v[j]);
      *reinterpret_cast<Bf16x4*>(row + c) = hi;
      *reinterpret_cast<Bf16x4*>(row + ldp + c) = lo;
    } else {
#pragma unroll
      for (int j = 0; j < VEC; ++j) split1(gv.v[j], row[c + j], row[ldp + c + j]);
    }
  }
}

// W fp32 [K,N] -> W2r bf16 [2K,N] = [hi; hi],  W2c bf16 [K,2N] = [hi | hi],  Wlo bf16 [K,N]
__global__ void tower_prep_weight_kernel(const float* __restrict__ W,
                                         __nv_bfloat16* __restrict__ W2r,
                                         __nv_bfloat16* __restrict__ W2c,
                                         __nv_bfloat16* __restrict__ Wlo, int K, int N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * N) return;
  const int k = (int)(i / N);
  const int n = (int)(i - (int64_t)k * N);
  __nv_bfloat16 hi, lo;
  split1(W[i], hi, lo);
  W2r[i] = hi;
  W2r[(int64_t)K * N + i] = hi;
  W2c[(int64_t)k * 2 * N + n] = hi;
  W2c[(int64_t)k * 2 * N + N + n] = hi;
  Wlo[i] = lo;
}

// dW[k,n] = Mx[k,n] + Mx[k,N+n] + Mx[K+k,n]   with Mx = [a_hi|a_lo]^T @ [dz_hi|dz_lo]  ([2K,2N])
__global__ void tower_fold_dw_kernel(const float* __restrict__ Mx, float* __restrict__ dW, int K,
                                     int N) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)K * N) return;
  const int k = (int)(i / N);
  const int n = (int)(i - (int64_t)k * N);
  const size_t r0 = (size_t)k * 2 * N, r1 = (size_t)(K + k) * 2 * N;
  dW[i] = (Mx[r0 + n] + Mx[r0 + N + n]) + Mx[r1 + n];
}

// ------------------------------------------------------------------------------------------------
// The width-1 head of a CTR tower (deepfm/net.py:169-174 last Linear: 400 -> 1) as two streaming
// kernels instead of three 128 x 16-column GEMM tiles that would each re-stream the activations:
//   head_fwd : y[m] = sum_k (a_hi + a_lo)[m,k] * w[k] + b                      reads 4K B/sample
//   head_bwd : g[m,k] = dy[m] * w[k] * (a_hi[m,k] > 0)  -> planes (the next dX/dW operand),
//              dW[k] = sum_m (a_hi + a_lo)[m,k] * dy[m],  db = sum_m dy[m]      reads 4K, writes 4K
// One warp per row; a lane owns the same 8-column chunks for every row it visits, so the dW sums
// stay in registers; warps -> CTA in shared memory, CTAs -> result in fixed order (deterministic).
constexpr int kHeadThreads = 256;
constexpr int kHeadMaxIter = 8;      // K <= 8 * 256

__device__ __forceinline__ void bf16x8_to_float(const uint4& q, float (&f)[8]) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    f[2 * j] = __uint_as_float(w[j] << 16);
    f[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
  }
}

__global__ void __launch_bounds__(kHeadThreads)
tower_head_fwd_kernel(const __nv_bfloat16* __restrict__ a, int64_t lda, int K,
                      const float* __restrict__ w, const float* __restrict__ bias,
                      float* __restrict__ y, int64_t M) {
  extern __shared__ float s_w[];
  for (int k = threadIdx.x; k < K; k += kHeadThreads) s_w[k] = w[k];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (int64_t)blockIdx.x * (kHeadThreads / 32) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (kHeadThreads / 32);
  const float b = bias != nullptr ? __ldg(bias) : 0.f;
  const int chunks = K / 8;
  constexpr int R = 4;      // rows in flight per warp: one row alone leaves the LSU idle
  for (int64_t m0 = warp0 * R; m0 < M; m0 += nwarps * R) {
    float acc[R];
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;
    for (int c = lane; c < chunks; c += 32) {
      uint4 qh[R], ql[R];
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const int64_t m = m0 + i < M ? m0 + i : M - 1;
        const __nv_bfloat16* row = a + m * 2 * lda;
        qh[i] = __ldg(reinterpret_cast<const uint4*>(row) + c);
        ql[i] = __ldg(reinterpret_cast<const uint4*>(row + lda) + c);
      }
#pragma unroll
      for (int i = 0; i < R; ++i) {
        float h[8], l[8];
        bf16x8_to_float(qh[i], h);
        bf16x8_to_float(ql[i], l);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i] = fmaf(h[j] + l[j], s_w[c * 8 + j], acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int64_t m = m0 + i;
      if (m < M) {
        const __nv_bfloat16* row = a + m * 2 * lda;
        for (int k = chunks * 8 + lane; k < K; k += 32)
          acc[i] = fmaf(__bfloat162float(row[k]) + __bfloat162float(row[lda + k]), s_w[k], acc[i]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
      if (lane == 0 && m < M) y[m] = acc[i] + b;
    }
  }
}

template <int NITER>
__global__ void __launch_bounds__(kHeadThreads)
tower_head_bwd_kernel(const __nv_bfloat16* __restrict__ a, int64_t lda, int K,
                      const float* __restrict__ w, const float* __restrict__ dy,
                      __nv_bfloat16* __restrict__ g, int64_t ldg, float* __restrict__ partials,
                      int64_t M) {
  extern __shared__ float s_buf[];      // [K] w, then [warps][K + 1] per-warp dW partials
  float* s_w = s_buf;
  float* s_part = s_buf + K;
  for (int k = threadIdx.x; k < K; k += kHeadThreads) s_w[k] = w[k];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t warp0 = (int64_t)blockIdx.x * (kHeadThreads / 32) + warp;
  const int64_t nwarps = (int64_t)gridDim.x * (kHeadThreads / 32);
  const int chunks = K / 8;             // K % 8 == 0 (checked on the host)
  float acc[NITER][8];
#pragma unroll
  for (int i = 0; i < NITER; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float dsum = 0.f;
  for (int64_t m = warp0; m < M; m += nwarps) {
    const __nv_bfloat16* row = a + m * 2 * lda;
    __nv_bfloat16* grow = g + m * 2 * ldg;
    const float d = __ldg(dy + m);
    dsum += d;
    uint4 qhs[NITER], qls[NITER];        // every load of the row in flight before the first use
#pragma unroll
    for (int i = 0; i < NITER; ++i) {
      const int c = lane + 32 * i;
      if (c < chunks) {
        qhs[i] = __ldg(reinterpret_cast<const uint4*>(row) + c);
        qls[i] = __ldg(reinterpret_cast<const uint4*>(row + lda) + c);
      }
    }
#pragma unroll
    for (int i = 0; i < NITER; ++i) {
      const int c = lane + 32 * i;
      if (c < chunks) {
        const uint4 qh = qhs[i];
        const uint4 ql = qls[i];
        float h[8], l[8];
        bf16x8_to_float(qh, h);
        bf16x8_to_float(ql, l);
        uint32_t oh[4], ol[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float v0 = h[2 * j] > 0.f ? d * s_w[c * 8 + 2 * j] : 0.f;
          float v1 = h[2 * j + 1] > 0.f ? d * s_w[c * 8 + 2 * j + 1] : 0.f;
          const __nv_bfloat162 h2 = __floats2bfloat162_rn(v0, v1);
          oh[j] = *reinterpret_cast<const uint32_t*>(&h2);
          v0 -= __uint_as_float(oh[j] << 16);
          v1 -= __uint_as_float(oh[j] & 0xFFFF0000u);
          const __nv_bfloat162 l2 = __floats2bfloat162_rn(v0, v1);
          ol[j] = *reinterpret_cast<const uint32_t*>(&l2);
        }
        *(reinterpret_cast<uint4*>(grow) + c) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
        *(reinterpret_cast<uint4*>(grow + ldg) + c) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(h[j] + l[j], d, acc[i][j]);
      }
    }
  }
  // warp partials -> shared memory, CTA sum in fixed warp order, one partial row per CTA:
  // partials[cta][0..K) = dW, partials[cta][K] = db
  float* mine = s_part + (size_t)warp * (K + 1);
#pragma unroll
  for (int i = 0; i < NITER; ++i) {
    const int c = lane + 32 * i;
    if (c < chunks)
#pragma unroll
      for (int j = 0; j < 8; ++j) mine[c * 8 + j] = acc[i][j];
  }
  if (lane == 0) mine[K] = dsum;
  __syncthreads();
  for (int k = threadIdx.x; k <= K; k += kHeadThreads) {
    float t = 0.f;
#pragma unroll
    for (int wv = 0; wv < kHeadThreads / 32; ++wv) t += s_part[(size_t)wv * (K + 1) + k];
    partials[(size_t)blockIdx.x * (K + 1) + k] = t;
  }
}

constexpr int kTowerRowSlices = 132 * 4;
static int tower_row_slices(int64_t M) {
  return (int)min((int64_t)kTowerRowSlices, M > 0 ? M : (int64_t)1);
}

static int launch_tower_split(const float* x, int64_t ldx, const float* bias, int relu, void* out,
                              int64_t ldp, int64_t M, int K, int ones_col, cudaStream_t st) {
  B200_REQUIRE(K > 0 && M >= 0 && ldx >= K && ldp >= K + (ones_col ? 1 : 0),
               "tower_split: bad sizes");
  if (M == 0) return B200REC_OK;
  const bool v4 = (K % 4 == 0) && (ldx % 4 == 0) && (ldp % 4 == 0) && aligned16(x) &&
                  aligned8(out) && (!bias || aligned16(bias));
  const int64_t total = M * (v4 ? K / 4 : K);
  const unsigned grid =
      (unsigned)min((total + kTowerThreads - 1) / kTowerThreads, (int64_t)sm_count() * 16);
  __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out);
  if (v4)
    tower_split_kernel<4><<<grid, kTowerThreads, 0, st>>>(x, ldx, bias, relu, o, ldp, M, K,
                                                          ones_col);
  else
    tower_split_kernel<1><<<grid, kTowerThreads, 0, st>>>(x, ldx, bias, relu, o, ldp, M, K,
                                                          ones_col);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_tower_relu_bwd_split(const float* dy, const void* act, int64_t ld_act, void* dz,
                                       int64_t ldp, float* dbias, int64_t M, int N, void* ws,
                                       size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(N > 0 && M >= 0 && ldp >= N && (!act || ld_act >= N),
               "tower_relu_bwd_split: bad sizes");
  const int slices = tower_row_slices(M);
  const size_t need = (size_t)slices * N * sizeof(float);
  if (ws_bytes < need) {
    set_error("tower_relu_bwd_split: workspace %zu < %zu bytes", ws_bytes, need);
    return B200REC_ERR_WORKSPACE;
  }
  if (M == 0) {
    B200_CUDA(cudaMemsetAsync(dbias, 0, (size_t)N * sizeof(float), st));
    return B200REC_OK;
  }
  const bool v4 = (N % 4 == 0) && (ldp % 4 == 0) && (!act || ld_act % 4 == 0) && aligned16(dy) &&
                  aligned8(dz) && (!act || aligned8(act)) && aligned16(ws);
  const int chunks = v4 ? N / 4 : N;
  // TX = column chunks per block (power of two <= 256), TY = rows per block
  int tx = 32;
  while (tx < chunks && tx < kTowerThreads) tx <<= 1;
  const int ty = kTowerThreads / tx;
  dim3 block(tx, ty);
  dim3 grid((chunks + tx - 1) / tx, slices);
  float* partials = static_cast<float*>(ws);
  const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(act);
  __nv_bfloat16* z = static_cast<__nv_bfloat16*>(dz);
  if (v4)
    tower_relu_bwd_split_kernel<4><<<grid, block, 0, st>>>(dy, a, ld_act, z, ldp, partials, M, N);
  else
    tower_relu_bwd_split_kernel<1><<<grid, block, 0, st>>>(dy, a, ld_act, z, ldp, partials, M, N);
  B200_LAUNCH_CHECK();
  reduce_partials_kernel<<<reduce_partials_grid(N), kRedThreads, 0, st>>>(partials, slices, N, dbias, N,
                                                                          nullptr);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_tower_gate_bwd(const float* dz, const void* y, int64_t ldy, const float* a,
                                 void* g, int64_t ldp, float* r, int64_t M, int N, cudaStream_t st) {
  B200_REQUIRE(N > 0 && M >= 0 && ldy >= N && ldp >= N, "tc_gate_bwd: bad sizes");
  if (M == 0) return B200REC_OK;
  const bool v4 = (N % 4 == 0) && (ldy % 4 == 0) && (ldp % 4 == 0) && aligned16(dz) &&
                  aligned16(a) && aligned16(r) && aligned8(y) && aligned8(g);
  const int64_t total = M * (v4 ? N / 4 : N);
  const unsigned grid =
      (unsigned)min((total + kTowerThreads - 1) / kTowerThreads, (int64_t)sm_count() * 16);
  const __nv_bfloat16* yp = static_cast<const __nv_bfloat16*>(y);
  __nv_bfloat16* gp = static_cast<__nv_bfloat16*>(g);
  if (v4)
    tower_gate_bwd_kernel<4><<<grid, kTowerThreads, 0, st>>>(dz, yp, ldy, a, gp, ldp, r, M, N);
  else
    tower_gate_bwd_kernel<1><<<grid, kTowerThreads, 0, st>>>(dz, yp, ldy, a, gp, ldp, r, M, N);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int head_grid() { return sm_count() * 2; }

static int launch_tower_head_fwd(const void* a, int64_t lda, int K, const float* w,
                                 const float* bias, float* y, int64_t M, cudaStream_t st) {
  B200_REQUIRE(K > 0 && M >= 0 && lda >= K && lda % 8 == 0 && aligned16(a),
               "tower_head_fwd: bad sizes / alignment");
  if (M == 0) return B200REC_OK;
  const size_t smem = (size_t)K * sizeof(float);
  B200_REQUIRE(smem <= 48 * 1024, "tower_head_fwd: K=%d too large", K);
  const int64_t rows_per_cta = kHeadThreads / 32;
  const int grid = (int)min((int64_t)head_grid(), (M + rows_per_cta - 1) / rows_per_cta);
  tower_head_fwd_kernel<<<grid, kHeadThreads, smem, st>>>(static_cast<const __nv_bfloat16*>(a), lda, K,
                                                         w, bias, y, M);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static size_t tower_head_bwd_ws_bytes(int K) { return (size_t)head_grid() * (K + 1) * sizeof(float); }

static int launch_tower_head_bwd(const void* a, int64_t lda, int K, const float* w, const float* dy,
                                 void* g, int64_t ldg, float* dW, float* db, int64_t M, void* ws,
                                 size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(K > 0 && K % 8 == 0 && K <= kHeadMaxIter * 256 && lda >= K && ldg >= K &&
                   lda % 8 == 0 && ldg % 8 == 0 && aligned16(a) && aligned16(g),
               "tower_head_bwd: K must be a multiple of 8 and <= %d, planes 16-byte aligned",
               kHeadMaxIter * 256);
  if (ws_bytes < tower_head_bwd_ws_bytes(K)) {
    set_error("tower_head_bwd: workspace %zu < %zu bytes", ws_bytes, tower_head_bwd_ws_bytes(K));
    return B200REC_ERR_WORKSPACE;
  }
  if (M == 0) {
    B200_CUDA(cudaMemsetAsync(dW, 0, (size_t)K * sizeof(float), st));
    B200_CUDA(cudaMemsetAsync(db, 0, sizeof(float), st));
    return B200REC_OK;
  }
  const size_t smem = ((size_t)K + (size_t)(kHeadThreads / 32) * (K + 1)) * sizeof(float);
  const int64_t rows_per_cta = kHeadThreads / 32;
  const int grid = (int)min((int64_t)head_grid(), (M + rows_per_cta - 1) / rows_per_cta);
  const int niter = (K / 8 + 31) / 32;
  const __nv_bfloat16* ap = static_cast<const __nv_bfloat16*>(a);
  __nv_bfloat16* gp = static_cast<__nv_bfloat16*>(g);
  float* partials = static_cast<float*>(ws);
#define B200_HEAD_BWD(NI)                                                                          \
  do {                                                                                             \
    auto kern = tower_head_bwd_kernel<NI>;                                                         \
    if (smem > 48 * 1024)                                                                          \
      B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, kHeadThreads, smem, st>>>(ap, lda, K, w, dy, gp, ldg, partials, M);               \
  } while (0)
  if (niter <= 1) B200_HEAD_BWD(1);
  else if (niter <= 2) B200_HEAD_BWD(2);
  else if (niter <= 4) B200_HEAD_BWD(4);
  else B200_HEAD_BWD(8);
#undef B200_HEAD_BWD
  B200_LAUNCH_CHECK();
  reduce_partials_kernel<<<reduce_partials_grid(K + 1), kRedThreads, 0, st>>>(partials, grid, K + 1, dW,
                                                                              K, db);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

}  // namespace b200rec
