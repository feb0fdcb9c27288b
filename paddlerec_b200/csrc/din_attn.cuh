// K4: DIN attention pooling — attention-unit MLP over [h, t, h-t, h*t], additive mask, E^-0.5
// scale, softmax over the history and weighted-sum pooling, fused (forward).
//
// Reference: DINLayer.forward, models/rank/din/net.py:155-173 (≈12 Paddle ops that materialise the
// [B,L,4E] concat = 205 KB/sample at L=100, E=128).  Here the concat never exists:
//     [h, t, h-t, h*t] W1 = h (Wa+Wc) + (h*t) Wd + t (Wb-Wc)
// so per history position only two E x 80 products remain (half the FLOPs of the reference's
// formulation) and the t-term  tb = t (Wb-Wc) + b1  is one [B,E]x[E,80] GEMM done once per sample
// by the caller.  FLOP-bound (2*L*(2E*80 + 80*40 + 40) flop per sample, 4.8 MFLOP at L=100) on the
// fp32 SIMT pipe: this round's kernel is a register-tiled shared-memory GEMM, not tensor-core code
// (the 1e-4 parity bar rules out single-pass TF32/BF16; a split-precision wgmma version is listed
// in DESIGN.md as next).
//
//   kernel A (din_scores_kernel): persistent CTAs over tiles of 64 flattened (b,l) positions;
//     both E x 80 weight blocks live transposed+padded in shared memory for the whole kernel;
//     thread (og,pg) owns a 4-position x 5-output register tile; layer 2 (80->40) and layer 3
//     (40->1) run from shared memory / warp shuffles; writes the masked, scaled score per position.
//   kernel B (din_softmax_pool_kernel): one CTA per sample: softmax over L, then
//     out[b,:] = sum_l w_l h[b,l,:]  (h is re-read; it was just touched and mostly sits in L2).
#pragma once

#include "common.cuh"

namespace b200rec {

constexpr int kDinH1 = 80;
constexpr int kDinH2 = 40;
constexpr int kDinTile = 64;      // positions per tile
constexpr int kDinThreads = 256;  // 16 output groups x 16 position groups
constexpr int kDinMaxE = 128;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

struct DinSmem {
  // all sizes in floats; EP = E + 4 (row padding keeps the 128-bit LDS conflict-free)
  static __host__ __device__ size_t floats(int E) {
    const size_t EP = E + 4;
    return 2 * (size_t)kDinH1 * EP            // WacT, WdT  [80][EP]
           + (size_t)kDinH1 * kDinH2          // W2s [80][40]
           + (size_t)kDinTile * EP            // hs [64][EP]
           + hts_floats(E)                    // hts [64][EP], reused for z1s [64][81]
           + 2 * kDinH2 + 8;                  // b2, W3
  }
  static __host__ __device__ size_t hts_floats(int E) {
    const size_t EP = E + 4;
    return (size_t)kDinTile * (EP > (size_t)(kDinH1 + 1) ? EP : (size_t)(kDinH1 + 1));
  }
};

__global__ void __launch_bounds__(kDinThreads, 1)
din_scores_kernel(const float* __restrict__ hist, const float* __restrict__ tseq,
                  const float* __restrict__ tb, const float* __restrict__ Wac,
                  const float* __restrict__ Wd, const float* __restrict__ W2,
                  const float* __restrict__ b2, const float* __restrict__ W3,
                  const float* __restrict__ b3, const int64_t* __restrict__ mask,
                  float* __restrict__ scores, int64_t P, int L, int E, float scale) {
  extern __shared__ __align__(16) float sm[];
  const int EP = E + 4;
  float* WacT = sm;                               // [80][EP]
  float* WdT = WacT + (size_t)kDinH1 * EP;        // [80][EP]
  float* W2s = WdT + (size_t)kDinH1 * EP;         // [80][40]
  float* hs = W2s + kDinH1 * kDinH2;              // [64][EP]
  float* hts = hs + (size_t)kDinTile * EP;        // [64][EP]
  float* z1s = hts;                               // [64][81]  (after GEMM1)
  float* b2s = hts + DinSmem::hts_floats(E);      // [40]
  float* W3s = b2s + kDinH2;                      // [40]

  const int tid = threadIdx.x;
  // one-time: weights -> shared (transposed [o][k])
  for (int i = tid; i < E * kDinH1; i += kDinThreads) {
    const int k = i / kDinH1, o = i - k * kDinH1;
    WacT[(size_t)o * EP + k] = Wac[i];
    WdT[(size_t)o * EP + k] = Wd[i];
  }
  for (int i = tid; i < kDinH1 * kDinH2; i += kDinThreads) W2s[i] = W2[i];
  if (tid < kDinH2) {
    b2s[tid] = b2[tid];
    W3s[tid] = W3[tid];
  }
  const float b3v = b3[0];
  __syncthreads();

  const int og = tid & 15;        // outputs og + 16*j, j<5
  const int pg = tid >> 4;        // positions pg*4 + i, i<4
  const int p2 = tid >> 2;        // layer 2: position
  const int qg = tid & 3;         // layer 2: outputs qg*10 + j, j<10
  const int chunks = E / 4;
  const int64_t ntiles = (P + kDinTile - 1) / kDinTile;

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t p0 = tile * kDinTile;
    // ---- load h and h*t rows of the tile ------------------------------------------------------
    for (int i = tid; i < kDinTile * chunks; i += kDinThreads) {
      const int row = i / chunks, c = i - row * chunks;
      const int64_t p = p0 + row;
      float4 h = make_float4(0.f, 0.f, 0.f, 0.f), tt = h;
      if (p < P) {
        const int64_t b = p / L;
        h = __ldg(reinterpret_cast<const float4*>(hist + (size_t)p * E) + c);
        tt = __ldg(reinterpret_cast<const float4*>(tseq + (size_t)b * E) + c);
      }
      *reinterpret_cast<float4*>(hs + (size_t)row * EP + c * 4) = h;
      *reinterpret_cast<float4*>(hts + (size_t)row * EP + c * 4) =
          make_float4(h.x * tt.x, h.y * tt.y, h.z * tt.z, h.w * tt.w);
    }
    __syncthreads();

    // ---- GEMM1: [64 x 2E] @ [2E x 80], 4x5 register tile --------------------------------------
    float acc[4][5];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j) acc[i][j] = 0.f;
    for (int c = 0; c < chunks; ++c) {
      float4 hv[4], htv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        hv[i] = *reinterpret_cast<const float4*>(hs + (size_t)(pg * 4 + i) * EP + c * 4);
        htv[i] = *reinterpret_cast<const float4*>(hts + (size_t)(pg * 4 + i) * EP + c * 4);
      }
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float4 wa = *reinterpret_cast<const float4*>(WacT + (size_t)(og + 16 * j) * EP + c * 4);
        const float4 wd = *reinterpret_cast<const float4*>(WdT + (size_t)(og + 16 * j) * EP + c * 4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float a = acc[i][j];
          a = fmaf(hv[i].x, wa.x, a); a = fmaf(hv[i].y, wa.y, a);
          a = fmaf(hv[i].z, wa.z, a); a = fmaf(hv[i].w, wa.w, a);
          a = fmaf(htv[i].x, wd.x, a); a = fmaf(htv[i].y, wd.y, a);
          a = fmaf(htv[i].z, wd.z, a); a = fmaf(htv[i].w, wd.w, a);
          acc[i][j] = a;
        }
      }
    }
    __syncthreads();  // everyone is done reading hts before it becomes z1s
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = pg * 4 + i;
      const int64_t p = p0 + row;
      const int64_t b = (p < P) ? p / L : 0;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const int o = og + 16 * j;
        z1s[row * (kDinH1 + 1) + o] = sigmoidf_(acc[i][j] + __ldg(tb + (size_t)b * kDinH1 + o));
      }
    }
    __syncthreads();

    // ---- layer 2 (80 -> 40, sigmoid) and layer 3 (40 -> 1) -------------------------------------
    float a2[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) a2[j] = 0.f;
    for (int o = 0; o < kDinH1; ++o) {
      const float z = z1s[p2 * (kDinH1 + 1) + o];
      const float* w = W2s + o * kDinH2 + qg * 10;
#pragma unroll
      for (int j = 0; j < 10; ++j) a2[j] = fmaf(z, w[j], a2[j]);
    }
    float part = 0.f;
#pragma unroll
    for (int j = 0; j < 10; ++j)
      part = fmaf(sigmoidf_(a2[j] + b2s[qg * 10 + j]), W3s[qg * 10 + j], part);
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 2);
    const int64_t p = p0 + p2;
    if (qg == 0 && p < P) {
      const float m = (mask != nullptr) ? (float)mask[p] : 0.f;
      scores[p] = ((part + b3v) + m) * scale;   // mask is added BEFORE the scale (net.py:166-168)
    }
    __syncthreads();  // smem tile is reused by the next iteration
  }
}

// One CTA per sample: w = softmax(scores[b,:]); out[b,:] = sum_l w_l * hist[b,l,:].
__global__ void __launch_bounds__(128)
din_softmax_pool_kernel(const float* __restrict__ hist, const float* __restrict__ scores,
                        float* __restrict__ weights, float* __restrict__ out, int L, int E) {
  extern __shared__ float sw[];  // [L]
  __shared__ float red[4];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* sc = scores + (size_t)b * L;
  float mx = -INFINITY;
  for (int l = tid; l < L; l += 128) {
    const float v = sc[l];
    sw[l] = v;
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int l = tid; l < L; l += 128) {
    const float e = __expf(sw[l] - mx);
    sw[l] = e;
    sum += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  const float inv = 1.f / (((red[0] + red[1]) + red[2]) + red[3]);
  for (int l = tid; l < L; l += 128) {
    const float w = sw[l] * inv;
    sw[l] = w;
    weights[(size_t)b * L + l] = w;
  }
  __syncthreads();
  const float* hb = hist + (size_t)b * L * E;
  for (int e = tid; e < E; e += 128) {
    float acc = 0.f;
    for (int l = 0; l < L; ++l) acc = fmaf(sw[l], hb[(size_t)l * E + e], acc);
    out[(size_t)b * E + e] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// Backward.
//   kernel B' (din_softmax_bwd_kernel), one CTA per sample:
//       dw_l = <dout[b], h_l>,  da_l = scale * w_l * (dw_l - sum_j w_j dw_j)
//   kernel A' (din_scores_bwd_kernel), persistent CTAs over the same 64-position tiles as forward:
//       recomputes z1, z2 (nothing but the softmax weights was saved), back-propagates
//       da -> layer 3 -> layer 2 -> g = d(pre-activation of layer 1)  [64 x 80], then
//         dhist[p]  = w_p*dout[b] + g Wac^T + (g Wd^T) * t          (second register-tiled GEMM)
//         dtseq[b] += (g Wd^T) * h_p ;  dtb[b] += g_p               (atomics, <= a few per sample)
//         dWac += h^T g,  dWd += (h*t)^T g,  dW2, db2, dW3          (per-thread register
//             accumulators over ALL tiles of the CTA, one partial per CTA, fixed-order reduce)
//   The caller finishes the t-path with two small GEMMs (see ops.raw_din_attn_bwd).
// out[k] = sum_g partials[g][k] in ascending g, split over five consecutive output arrays
__global__ void din_reduce_partials_kernel(const float* __restrict__ partials, int G, int len,
                                           float* __restrict__ o0, int n0, float* __restrict__ o1,
                                           int n1, float* __restrict__ o2, int n2,
                                           float* __restrict__ o3, int n3, float* __restrict__ o4) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= len) return;
  float t = 0.f;
#pragma unroll 8
  for (int g = 0; g < G; ++g) t += partials[(size_t)g * len + k];   // loads hoisted, adds in order
  if (k < n0) { o0[k] = t; return; }
  k -= n0;
  if (k < n1) { o1[k] = t; return; }
  k -= n1;
  if (k < n2) { o2[k] = t; return; }
  k -= n2;
  if (k < n3) { o3[k] = t; return; }
  o4[k - n3] = t;
}

struct DinBwdSmem {
  static __host__ __device__ size_t floats(int E) {
    const size_t EP = E + 4;
    return 2 * (size_t)kDinH1 * EP + (size_t)kDinH1 * kDinH2 + 2 * (size_t)kDinTile * EP +
           (size_t)kDinTile * (kDinH1 + 1) + (size_t)kDinTile * (kDinH2 + 1) + 2 * kDinH2 + 8;
  }
};
// per-CTA partial layout (floats): dWac[E*80] | dWd[E*80] | dW2[80*40] | db2[40] | dW3[40]
static __host__ __device__ inline size_t din_partial_floats(int E) {
  return 2 * (size_t)E * kDinH1 + (size_t)kDinH1 * kDinH2 + 2 * kDinH2;
}

__global__ void __launch_bounds__(128)
din_softmax_bwd_kernel(const float* __restrict__ hist, const float* __restrict__ weights,
                       const float* __restrict__ dout, float* __restrict__ da, int L, int E,
                       float scale) {
  extern __shared__ float sdw[];  // [L]
  __shared__ float red[4];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* hb = hist + (size_t)b * L * E;
  const float* w = weights + (size_t)b * L;
  const float* g = dout + (size_t)b * E;
  for (int l = warp; l < L; l += 4) {
    float acc = 0.f;
    for (int e = lane; e < E; e += 32) acc = fmaf(g[e], hb[(size_t)l * E + e], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) sdw[l] = acc;
  }
  __syncthreads();
  float dot = 0.f;
  for (int l = tid; l < L; l += 128) dot = fmaf(w[l], sdw[l], dot);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  if (lane == 0) red[warp] = dot;
  __syncthreads();
  dot = ((red[0] + red[1]) + red[2]) + red[3];
  for (int l = tid; l < L; l += 128) da[(size_t)b * L + l] = scale * w[l] * (sdw[l] - dot);
}

__global__ void __launch_bounds__(kDinThreads, 1)
din_scores_bwd_kernel(const float* __restrict__ hist, const float* __restrict__ tseq,
                      const float* __restrict__ tb, const float* __restrict__ Wac,
                      const float* __restrict__ Wd, const float* __restrict__ W2,
                      const float* __restrict__ b2, const float* __restrict__ W3,
                      const float* __restrict__ weights, const float* __restrict__ dout,
                      const float* __restrict__ da, float* __restrict__ dhist,
                      float* __restrict__ dtseq, float* __restrict__ dtb,
                      float* __restrict__ partials, int64_t P, int L, int E) {
  extern __shared__ __align__(16) float sm[];
  const int EP = E + 4;
  float* WacT = sm;                                   // [80][EP]
  float* WdT = WacT + (size_t)kDinH1 * EP;            // [80][EP]
  float* W2s = WdT + (size_t)kDinH1 * EP;             // [80][40]
  float* hs = W2s + kDinH1 * kDinH2;                  // [64][EP]
  float* hts = hs + (size_t)kDinTile * EP;            // [64][EP]
  float* z1s = hts + (size_t)kDinTile * EP;           // [64][81]   z1, later g
  float* dz2s = z1s + kDinTile * (kDinH1 + 1);        // [64][41]
  float* b2s = dz2s + kDinTile * (kDinH2 + 1);        // [40]
  float* W3s = b2s + kDinH2;                          // [40]

  const int tid = threadIdx.x;
  for (int i = tid; i < E * kDinH1; i += kDinThreads) {
    const int k = i / kDinH1, o = i - k * kDinH1;
    WacT[(size_t)o * EP + k] = Wac[i];
    WdT[(size_t)o * EP + k] = Wd[i];
  }
  for (int i = tid; i < kDinH1 * kDinH2; i += kDinThreads) W2s[i] = W2[i];
  if (tid < kDinH2) {
    b2s[tid] = b2[tid];
    W3s[tid] = W3[tid];
  }
  __syncthreads();

  const int og = tid & 15, pg = tid >> 4;     // GEMM1 / dz1 tile: outputs og+16j, positions pg*4+i
  const int p2 = tid >> 2, qg = tid & 3;      // layer 2: position p2, outputs qg*10+j
  const int chunks = E / 4;
  const int64_t ntiles = (P + kDinTile - 1) / kDinTile;

  // persistent weight-gradient accumulators
  //   dWac/dWd: thread (og, kg=pg) owns k = kg + 16*i (i < E/16 <= 8) x o = og + 16*j (j<5)
  float aWac[8][5], aWd[8][5];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 5; ++j) aWac[i][j] = aWd[i][j] = 0.f;
  //   dW2: thread t < 240 owns q = t % 40, o = t/40 + 6*i (i < 14)
  const int q2 = tid % kDinH2, o2 = tid / kDinH2;
  float aW2[14];
#pragma unroll
  for (int i = 0; i < 14; ++i) aW2[i] = 0.f;
  float ab2 = 0.f, aW3 = 0.f;  // thread t < 40 owns db2[t], dW3[t]
  const int kreps = (E + 15) / 16;

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t p0 = tile * kDinTile;
    for (int i = tid; i < kDinTile * chunks; i += kDinThreads) {
      const int row = i / chunks, c = i - row * chunks;
      const int64_t p = p0 + row;
      float4 h = make_float4(0.f, 0.f, 0.f, 0.f), tt = h;
      if (p < P) {
        const int64_t b = p / L;
        h = __ldg(reinterpret_cast<const float4*>(hist + (size_t)p * E) + c);
        tt = __ldg(reinterpret_cast<const float4*>(tseq + (size_t)b * E) + c);
      }
      *reinterpret_cast<float4*>(hs + (size_t)row * EP + c * 4) = h;
      *reinterpret_cast<float4*>(hts + (size_t)row * EP + c * 4) =
          make_float4(h.x * tt.x, h.y * tt.y, h.z * tt.z, h.w * tt.w);
    }
    __syncthreads();

    // ---- recompute GEMM1 -> z1 -----------------------------------------------------------------
    {
      float acc[4][5];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 5; ++j) acc[i][j] = 0.f;
      for (int c = 0; c < chunks; ++c) {
        float4 hv[4], htv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          hv[i] = *reinterpret_cast<const float4*>(hs + (size_t)(pg * 4 + i) * EP + c * 4);
          htv[i] = *reinterpret_cast<const float4*>(hts + (size_t)(pg * 4 + i) * EP + c * 4);
        }
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const float4 wa = *reinterpret_cast<const float4*>(WacT + (size_t)(og + 16 * j) * EP + c * 4);
          const float4 wd = *reinterpret_cast<const float4*>(WdT + (size_t)(og + 16 * j) * EP + c * 4);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float a = acc[i][j];
            a = fmaf(hv[i].x, wa.x, a); a = fmaf(hv[i].y, wa.y, a);
            a = fmaf(hv[i].z, wa.z, a); a = fmaf(hv[i].w, wa.w, a);
            a = fmaf(htv[i].x, wd.x, a); a = fmaf(htv[i].y, wd.y, a);
            a = fmaf(htv[i].z, wd.z, a); a = fmaf(htv[i].w, wd.w, a);
            acc[i][j] = a;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = pg * 4 + i;
        const int64_t p = p0 + row;
        const int64_t b = (p < P) ? p / L : 0;
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          const int o = og + 16 * j;
          z1s[row * (kDinH1 + 1) + o] = sigmoidf_(acc[i][j] + __ldg(tb + (size_t)b * kDinH1 + o));
        }
      }
    }
    __syncthreads();

    // ---- layer 2 forward, then back through layers 3 and 2: dz2pre -> dz2s ---------------------
    {
      float a2[10];
#pragma unroll
      for (int j = 0; j < 10; ++j) a2[j] = 0.f;
      for (int o = 0; o < kDinH1; ++o) {
        const float z = z1s[p2 * (kDinH1 + 1) + o];
        const float* w = W2s + o * kDinH2 + qg * 10;
#pragma unroll
        for (int j = 0; j < 10; ++j) a2[j] = fmaf(z, w[j], a2[j]);
      }
      const int64_t p = p0 + p2;
      const float dav = (p < P) ? __ldg(da + p) : 0.f;
#pragma unroll
      for (int j = 0; j < 10; ++j) {
        const float z2 = sigmoidf_(a2[j] + b2s[qg * 10 + j]);
        // da * W3[q] * z2(1-z2); keep da*z2 for dW3 in the unused (negative-index-free) slot below
        dz2s[p2 * (kDinH2 + 1) + qg * 10 + j] = dav * W3s[qg * 10 + j] * z2 * (1.f - z2);
        a2[j] = dav * z2;  // contribution to dW3[q]
      }
      // dW3[q] += sum_p da_p z2[p][q]: stage through hts? no - use shuffles over the 8 positions of
      // the warp (lanes with equal qg), then one shared-memory atomic-free slot per warp via dz2s
      // column kDinH2 is not wide enough -> accumulate with a tiny smem array instead (below).
#pragma unroll
      for (int j = 0; j < 10; ++j) {
        float v = a2[j];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        a2[j] = v;  // lanes 0..3 (qg) of each warp hold the warp's partial for q = qg*10+j
      }
      // stash warp partials in hs' padding-free scratch: reuse the first 8*40 floats of dz2s'
      // neighbour? -> use a dedicated static array
      __shared__ float s_w3[8][kDinH2];
      if ((tid & 31) < 4) {
#pragma unroll
        for (int j = 0; j < 10; ++j) s_w3[tid >> 5][qg * 10 + j] = a2[j];
      }
      __syncthreads();
      if (tid < kDinH2) {
        float t3 = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t3 += s_w3[w][tid];
        aW3 += t3;
        float tb2 = 0.f;
        for (int pp = 0; pp < kDinTile; ++pp) tb2 += dz2s[pp * (kDinH2 + 1) + tid];
        ab2 += tb2;
      }
    }
    // dW2[o][q] += sum_p z1[p][o] dz2pre[p][q]
    if (tid < 6 * kDinH2) {
      for (int pp = 0; pp < kDinTile; ++pp) {
        const float d = dz2s[pp * (kDinH2 + 1) + q2];
#pragma unroll
        for (int i = 0; i < 14; ++i) {
          const int o = o2 + 6 * i;
          if (o < kDinH1) aW2[i] = fmaf(z1s[pp * (kDinH1 + 1) + o], d, aW2[i]);
        }
      }
    }
    // dz1 = dz2pre W2^T ; g = dz1 * z1 (1 - z1)    (4x5 tile as GEMM1)
    float gv[4][5];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j) gv[i][j] = 0.f;
    for (int q = 0; q < kDinH2; ++q) {
      float d[4], w[5];
#pragma unroll
      for (int i = 0; i < 4; ++i) d[i] = dz2s[(pg * 4 + i) * (kDinH2 + 1) + q];
#pragma unroll
      for (int j = 0; j < 5; ++j) w[j] = W2s[(og + 16 * j) * kDinH2 + q];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 5; ++j) gv[i][j] = fmaf(d[i], w[j], gv[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const float z = z1s[(pg * 4 + i) * (kDinH1 + 1) + og + 16 * j];
        gv[i][j] *= z * (1.f - z);
      }
    __syncthreads();  // all reads of z1s (dW2, g) are done
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 5; ++j) z1s[(pg * 4 + i) * (kDinH1 + 1) + og + 16 * j] = gv[i][j];
    __syncthreads();
    float* gs = z1s;  // [64][81] now holds g

    // ---- dtb[b][o] += sum over the tile's positions of sample b ---------------------------------
    if (tid < kDinH1) {
      float run = 0.f;
      int64_t cur = -1;
      for (int pp = 0; pp < kDinTile; ++pp) {
        const int64_t p = p0 + pp;
        if (p >= P) break;
        const int64_t b = p / L;
        if (b != cur) {
          if (cur >= 0) atomicAdd(dtb + (size_t)cur * kDinH1 + tid, run);
          cur = b;
          run = 0.f;
        }
        run += gs[pp * (kDinH1 + 1) + tid];
      }
      if (cur >= 0) atomicAdd(dtb + (size_t)cur * kDinH1 + tid, run);
    }

    // ---- dWac += h^T g, dWd += (h*t)^T g  (thread owns k = pg + 16 i, o = og + 16 j) ------------
    for (int pp = 0; pp < kDinTile; ++pp) {
      float gg[5];
#pragma unroll
      for (int j = 0; j < 5; ++j) gg[j] = gs[pp * (kDinH1 + 1) + og + 16 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (i < kreps) {
          const int k = pg + 16 * i;
          if (k < E) {
            const float hv = hs[(size_t)pp * EP + k];
            const float htv = hts[(size_t)pp * EP + k];
#pragma unroll
            for (int j = 0; j < 5; ++j) {
              aWac[i][j] = fmaf(hv, gg[j], aWac[i][j]);
              aWd[i][j] = fmaf(htv, gg[j], aWd[i][j]);
            }
          }
        }
      }
    }

    // ---- dh GEMM: [64 x 80] @ [80 x E] (Wac^T and Wd^T); thread: k-chunk kc, 8 positions --------
    for (int kc = tid & 31; kc < chunks; kc += 32) {
      const int pg8 = tid >> 5;  // positions pg8*8 + i
      float4 dA[8], dD[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) dA[i] = dD[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int o = 0; o < kDinH1; ++o) {
        const float4 wa = *reinterpret_cast<const float4*>(WacT + (size_t)o * EP + kc * 4);
        const float4 wd = *reinterpret_cast<const float4*>(WdT + (size_t)o * EP + kc * 4);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float g1 = gs[(pg8 * 8 + i) * (kDinH1 + 1) + o];
          dA[i].x = fmaf(g1, wa.x, dA[i].x); dA[i].y = fmaf(g1, wa.y, dA[i].y);
          dA[i].z = fmaf(g1, wa.z, dA[i].z); dA[i].w = fmaf(g1, wa.w, dA[i].w);
          dD[i].x = fmaf(g1, wd.x, dD[i].x); dD[i].y = fmaf(g1, wd.y, dD[i].y);
          dD[i].z = fmaf(g1, wd.z, dD[i].z); dD[i].w = fmaf(g1, wd.w, dD[i].w);
        }
      }
      float4 run = make_float4(0.f, 0.f, 0.f, 0.f);
      int64_t cur = -1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = pg8 * 8 + i;
        const int64_t p = p0 + row;
        if (p < P) {
          const int64_t b = p / L;
          const float4 tt = __ldg(reinterpret_cast<const float4*>(tseq + (size_t)b * E) + kc);
          const float4 go = __ldg(reinterpret_cast<const float4*>(dout + (size_t)b * E) + kc);
          const float wp = __ldg(weights + p);
          const float4 h = *reinterpret_cast<const float4*>(hs + (size_t)row * EP + kc * 4);
          float4 r;
          r.x = fmaf(wp, go.x, fmaf(dD[i].x, tt.x, dA[i].x));
          r.y = fmaf(wp, go.y, fmaf(dD[i].y, tt.y, dA[i].y));
          r.z = fmaf(wp, go.z, fmaf(dD[i].z, tt.z, dA[i].z));
          r.w = fmaf(wp, go.w, fmaf(dD[i].w, tt.w, dA[i].w));
          *reinterpret_cast<float4*>(dhist + (size_t)p * E + kc * 4) = r;
          if (b != cur) {
            if (cur >= 0) {
              float* dst = dtseq + (size_t)cur * E + kc * 4;
              atomicAdd(dst + 0, run.x); atomicAdd(dst + 1, run.y);
              atomicAdd(dst + 2, run.z); atomicAdd(dst + 3, run.w);
            }
            cur = b;
            run = make_float4(0.f, 0.f, 0.f, 0.f);
          }
          run.x = fmaf(dD[i].x, h.x, run.x); run.y = fmaf(dD[i].y, h.y, run.y);
          run.z = fmaf(dD[i].z, h.z, run.z); run.w = fmaf(dD[i].w, h.w, run.w);
        }
      }
      if (cur >= 0) {
        float* dst = dtseq + (size_t)cur * E + kc * 4;
        atomicAdd(dst + 0, run.x); atomicAdd(dst + 1, run.y);
        atomicAdd(dst + 2, run.z); atomicAdd(dst + 3, run.w);
      }
    }
    __syncthreads();  // tile buffers are reused by the next iteration
  }

  // ---- one partial per CTA ----------------------------------------------------------------------
  float* part = partials + (size_t)blockIdx.x * din_partial_floats(E);
  float* pWac = part;
  float* pWd = pWac + (size_t)E * kDinH1;
  float* pW2 = pWd + (size_t)E * kDinH1;
  float* pb2 = pW2 + kDinH1 * kDinH2;
  float* pW3 = pb2 + kDinH2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = pg + 16 * i;
    if (i < kreps && k < E) {
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        pWac[(size_t)k * kDinH1 + og + 16 * j] = aWac[i][j];
        pWd[(size_t)k * kDinH1 + og + 16 * j] = aWd[i][j];
      }
    }
  }
  if (tid < 6 * kDinH2) {
#pragma unroll
    for (int i = 0; i < 14; ++i) {
      const int o = o2 + 6 * i;
      if (o < kDinH1) pW2[o * kDinH2 + q2] = aW2[i];
    }
  }
  if (tid < kDinH2) {
    pb2[tid] = ab2;
    pW3[tid] = aW3;
  }
}

static int din_bwd_grid(int64_t P) {
  const int64_t ntiles = (P + kDinTile - 1) / kDinTile;
  return (int)min(ntiles, (int64_t)sm_count());
}

static int launch_din_attn_bwd(const float* hist, const float* tseq, const float* tb,
                               const float* Wac, const float* Wd, const float* W2, const float* b2,
                               const float* W3, const float* weights, const float* dout, float* da,
                               float* dhist, float* dtseq, float* dtb, float* dWac, float* dWd,
                               float* dW2, float* db2, float* dW3, int64_t B, int L, int E,
                               float scale, void* ws, size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(E > 0 && E % 4 == 0 && E <= kDinMaxE, "din_attn_bwd: E=%d must be a multiple of 4, <=%d",
               E, kDinMaxE);
  B200_REQUIRE(L > 0 && L <= 8192, "din_attn_bwd: L=%d out of range", L);
  const size_t plen = din_partial_floats(E);
  if (B == 0) {
    B200_CUDA(cudaMemsetAsync(dWac, 0, (size_t)E * kDinH1 * 4, st));
    B200_CUDA(cudaMemsetAsync(dWd, 0, (size_t)E * kDinH1 * 4, st));
    B200_CUDA(cudaMemsetAsync(dW2, 0, (size_t)kDinH1 * kDinH2 * 4, st));
    B200_CUDA(cudaMemsetAsync(db2, 0, kDinH2 * 4, st));
    B200_CUDA(cudaMemsetAsync(dW3, 0, kDinH2 * 4, st));
    return B200REC_OK;
  }
  const int64_t P = B * L;
  const int grid = din_bwd_grid(P);
  const size_t need = (size_t)grid * plen * sizeof(float);
  if (ws_bytes < need) {
    set_error("din_attn_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return B200REC_ERR_WORKSPACE;
  }
  B200_CUDA(cudaMemsetAsync(dtseq, 0, (size_t)B * E * sizeof(float), st));
  B200_CUDA(cudaMemsetAsync(dtb, 0, (size_t)B * kDinH1 * sizeof(float), st));
  din_softmax_bwd_kernel<<<(unsigned)B, 128, (size_t)L * sizeof(float), st>>>(hist, weights, dout, da,
                                                                              L, E, scale);
  B200_LAUNCH_CHECK();
  const size_t smem = DinBwdSmem::floats(E) * sizeof(float);
  B200_CUDA(cudaFuncSetAttribute(din_scores_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
  float* partials = static_cast<float*>(ws);
  din_scores_bwd_kernel<<<grid, kDinThreads, smem, st>>>(hist, tseq, tb, Wac, Wd, W2, b2, W3, weights,
                                                         dout, da, dhist, dtseq, dtb, partials, P, L,
                                                         E);
  B200_LAUNCH_CHECK();
  // fixed-order reduction of the per-CTA partials into the five outputs
  const int len = (int)plen;
  const int nW = E * kDinH1;
  din_reduce_partials_kernel<<<(len + 127) / 128, 128, 0, st>>>(
      partials, grid, len, dWac, nW, dWd, nW, dW2, kDinH1 * kDinH2, db2, kDinH2, dW3);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_din_attn_fwd(const float* hist, const float* tseq, const float* tb,
                               const float* Wac, const float* Wd, const float* W2, const float* b2,
                               const float* W3, const float* b3, const int64_t* mask, float* scores,
                               float* weights, float* out, int64_t B, int L, int E, float scale,
                               cudaStream_t st) {
  B200_REQUIRE(E > 0 && E % 4 == 0 && E <= kDinMaxE, "din_attn_fwd: E=%d must be a multiple of 4, <=%d",
               E, kDinMaxE);
  B200_REQUIRE(L > 0 && L <= 8192, "din_attn_fwd: L=%d out of range", L);
  B200_REQUIRE(aligned16(hist) && aligned16(tseq), "din_attn_fwd: hist/tseq must be 16-byte aligned");
  if (B == 0) return B200REC_OK;
  const int64_t P = B * L;
  const size_t smem = DinSmem::floats(E) * sizeof(float);
  B200_CUDA(cudaFuncSetAttribute(din_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
  const int64_t ntiles = (P + kDinTile - 1) / kDinTile;
  const unsigned grid = (unsigned)min(ntiles, (int64_t)sm_count());
  din_scores_kernel<<<grid, kDinThreads, smem, st>>>(hist, tseq, tb, Wac, Wd, W2, b2, W3, b3, mask,
                                                     scores, P, L, E, scale);
  B200_LAUNCH_CHECK();
  din_softmax_pool_kernel<<<(unsigned)B, 128, (size_t)L * sizeof(float), st>>>(hist, scores, weights,
                                                                               out, L, E);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

}  // namespace b200rec
