// K6 — DLRM dot interaction (models/rank/dlrm/net.py:97-115), forward and backward.
//
//   T [B, N, d]   N = num_field + 1 feature vectors per sample: the 26 embedding rows, then the
//                 bottom-MLP output x as the LAST row (net.py:97-100)
//   R [B, d + P]  R[:, :d] = x  (the concat of net.py:115 fused in),
//                 R[:, d + p] = <T_i, T_j> for the pairs (i, j) of the upper triangle in row-major
//                 order; P = N(N-1)/2 (i < j), or N(N+1)/2 with self_interaction, where — exactly
//                 as the reference's triu(Z,1) + tril(MIN_FLOAT,-1) + masked_select evaluates —
//                 the diagonal entries are selected but carry 0, not <T_i, T_i> (net.py:105-113).
//
// One warp per sample, persistent grid.  The sample's N*d floats are staged in shared memory with a
// row pitch of d+1 (consecutive pairs differ in j, so lanes hit consecutive rows: pitch d+1 is
// conflict-free, the shared i row is a broadcast); lanes then own pairs p = lane, lane+32, ... and
// write R coalesced.  Backward stages T the same way, mirrors dZ into a full N x N matrix
// with a zero diagonal, and lane (i, c) accumulates dT[i][c] = sum_j dZ[i][j] * T[j][c]
// (+ dR[:, c] for the x row) — no atomics, deterministic.  HBM-bound: algorithmic bytes per sample 4*(N*d + d + P) forward (3 196 B at
// N=27, d=16) and 4*(2*N*d + d + P) backward.
#pragma once

#include "common.cuh"

namespace b200rec {

constexpr int kDotWarps = 4;  // samples in flight per CTA (fewer when N*N floats would not fit)

struct DotShape {
  int N, d, self, P, pitch;
  __host__ __device__ DotShape(int N_, int d_, int self_)
      : N(N_), d(d_), self(self_), P(self_ ? N_ * (N_ + 1) / 2 : N_ * (N_ - 1) / 2), pitch(d_ + 1) {}
  // first output index of row i of the (strict / with-diagonal) upper triangle
  __host__ __device__ int row_start(int i) const {
    return self ? i * N - i * (i - 1) / 2 : i * (N - 1) - i * (i - 1) / 2;
  }
  __host__ __device__ int row_len(int i) const { return self ? N - i : N - 1 - i; }
  // output index of the pair (i, j), i < j (or i <= j with self)
  __host__ __device__ int pair(int i, int j) const { return row_start(i) + (self ? j - i : j - i - 1); }
  __host__ __device__ size_t smem_floats_fwd() const { return (size_t)N * pitch; }
  __host__ __device__ size_t smem_floats_bwd() const { return (size_t)N * pitch + (size_t)N * N; }
};

__device__ __forceinline__ void dot_stage_rows(const float* __restrict__ src, float* __restrict__ dst,
                                               const DotShape& s, int lane) {
  const int total = s.N * s.d;
  for (int e = lane; e < total; e += 32) {
    const int r = e / s.d, c = e - r * s.d;
    dst[r * s.pitch + c] = __ldg(src + e);
  }
}

__global__ void __launch_bounds__(kDotWarps * 32)
dot_interact_fwd_kernel(const float* __restrict__ T, float* __restrict__ R, int64_t B, DotShape s) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* tile = smem + (size_t)warp * s.smem_floats_fwd();
  const int out_w = s.d + s.P;
  const int warps = blockDim.x >> 5;
  for (int64_t b = (int64_t)blockIdx.x * warps + warp; b < B; b += (int64_t)gridDim.x * warps) {
    dot_stage_rows(T + b * s.N * s.d, tile, s, lane);
    __syncwarp();
    float* out = R + b * out_w;
    for (int c = lane; c < s.d; c += 32) __stcs(out + c, tile[(s.N - 1) * s.pitch + c]);
    // walk the triangle: (i, j) of this lane's first pair, then advance by 32 pairs each round
    int i = 0, off = lane;  // off = position inside row i
    for (int p = lane; p < s.P; p += 32) {
      while (off >= s.row_len(i)) { off -= s.row_len(i); ++i; }
      const int j = s.self ? i + off : i + 1 + off;
      float acc = 0.f;
      if (j != i) {
        const float* a = tile + i * s.pitch;
        const float* bb = tile + j * s.pitch;
#pragma unroll 4
        for (int c = 0; c < s.d; ++c) acc = fmaf(a[c], bb[c], acc);
      }
      __stcs(out + s.d + p, acc);
      off += 32;
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kDotWarps * 32)
dot_interact_bwd_kernel(const float* __restrict__ T, const float* __restrict__ dR,
                        float* __restrict__ dT, int64_t B, DotShape s) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* tile = smem + (size_t)warp * s.smem_floats_bwd();
  float* dzf = tile + (size_t)s.N * s.pitch;  // dZ mirrored into a full N x N matrix, zero diagonal
  const int out_w = s.d + s.P;
  const int warps = blockDim.x >> 5;
  for (int64_t b = (int64_t)blockIdx.x * warps + warp; b < B; b += (int64_t)gridDim.x * warps) {
    dot_stage_rows(T + b * s.N * s.d, tile, s, lane);
    const float* g = dR + b * out_w;
    for (int i = lane; i < s.N; i += 32) dzf[i * s.N + i] = 0.f;
    {
      int i = 0, off = lane;
      for (int p = lane; p < s.P; p += 32) {
        while (off >= s.row_len(i)) { off -= s.row_len(i); ++i; }
        const int j = s.self ? i + off : i + 1 + off;
        if (j != i) {
          const float v = __ldg(g + s.d + p);
          dzf[i * s.N + j] = v;
          dzf[j * s.N + i] = v;
        }
        off += 32;
      }
    }
    __syncwarp();
    float* out = dT + b * s.N * s.d;
    const int total = s.N * s.d;
    for (int e = lane; e < total; e += 32) {
      const int i = e / s.d, c = e - i * s.d;
      float acc = (i == s.N - 1) ? __ldg(g + c) : 0.f;   // x is both the last row of T and R[:, :d]
      const float* zr = dzf + i * s.N;
#pragma unroll 3
      for (int j = 0; j < s.N; ++j) acc = fmaf(zr[j], tile[j * s.pitch + c], acc);
      __stcs(out + e, acc);                                // the diagonal carries no gradient
    }
    __syncwarp();
  }
}

// ================================================================================================
// v2 — EXPERIMENTAL, opt-in with B200REC_K6_V2=1 (d % 4 == 0).  Written after the round's GPU budget
// was spent: it compiles for sm_90a but has NOT run on hardware yet; the default path above is the
// validated one.  Parity test: tests/test_gpu_kernels.py::test_dot_interact_v2_matches_v1 (enabled
// with B200REC_TEST_EXPERIMENTAL=1); timing: tools/dot_bench.py --v2.
//
// What the v1 measurement said (0.20 of HBM peak forward, on the GPU the project first targeted):
// ~530 warp instructions per sample, two scalar shared-memory loads per FMA, and no overlap between
// a warp's global loads and its math.  v2 changes exactly those two things:
//   * rows live at a pitch of d+4 floats, so every row is 16-byte aligned and the inner product
//     reads float4 (LDS.128): 4x fewer shared-memory instructions; 8 consecutive rows at a pitch of
//     d+4 words start in 8 different 4-bank groups (d = 16: 0,20,8,28,16,4,24,12), so a quarter-warp
//     phase of LDS.128 is conflict-free;
//   * the NEXT sample of the warp is staged with cp.async (16-byte copies) into a second buffer
//     while the current one is being multiplied.
extern __shared__ __align__(16) float dot_smem_v2[];

__device__ __forceinline__ void cp_async_16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                   static_cast<unsigned>(__cvta_generic_to_shared(smem))),
               "l"(gmem)
               : "memory");
}

__device__ __forceinline__ void dot_stage_rows_async(const float* __restrict__ src, float* dst, int N,
                                                     int d4, int pitch, int lane) {
  const int chunks = N * d4;
  for (int e = lane; e < chunks; e += 32) {
    const int r = e / d4, c = e - r * d4;
    cp_async_16(dst + r * pitch + 4 * c, src + 4 * e);
  }
  cp_async_commit();
}

__host__ __device__ inline size_t dot_v2_smem_floats(const DotShape& s, bool bwd) {
  const size_t tile = (size_t)s.N * (s.d + 4);
  return bwd ? tile + (((size_t)s.N * s.N + 3) & ~size_t(3)) : 2 * tile;
}

__global__ void __launch_bounds__(kDotWarps * 32)
dot_interact_fwd_v2_kernel(const float* __restrict__ T, float* __restrict__ R, int64_t B, DotShape s) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  const int pitch = s.d + 4, d4 = s.d >> 2;
  float* buf0 = dot_smem_v2 + (size_t)warp * dot_v2_smem_floats(s, false);
  float* buf1 = buf0 + (size_t)s.N * pitch;
  const int out_w = s.d + s.P;
  const int64_t stride = (int64_t)gridDim.x * warps;
  int64_t b = (int64_t)blockIdx.x * warps + warp;
  if (b < B) dot_stage_rows_async(T + b * s.N * s.d, buf0, s.N, d4, pitch, lane);
  for (int cur = 0; b < B; b += stride, cur ^= 1) {
    const float* tile = cur ? buf1 : buf0;
    if (b + stride < B) {
      dot_stage_rows_async(T + (b + stride) * s.N * s.d, cur ? buf0 : buf1, s.N, d4, pitch, lane);
      cp_async_wait<1>();   // this sample's copies have landed; the next sample's may be in flight
    } else {
      cp_async_wait<0>();
    }
    __syncwarp();
    float* out = R + b * out_w;
    for (int c = lane; c < s.d; c += 32) __stcs(out + c, tile[(s.N - 1) * pitch + c]);
    int i = 0, off = lane;
    for (int p = lane; p < s.P; p += 32) {
      while (off >= s.row_len(i)) { off -= s.row_len(i); ++i; }
      const int j = s.self ? i + off : i + 1 + off;
      float acc = 0.f;
      if (j != i) {
        const float4* a4 = reinterpret_cast<const float4*>(tile + i * pitch);
        const float4* b4 = reinterpret_cast<const float4*>(tile + j * pitch);
#pragma unroll 4
        for (int c = 0; c < d4; ++c) {
          const float4 x = a4[c], y = b4[c];
          acc = fmaf(x.x, y.x, acc);
          acc = fmaf(x.y, y.y, acc);
          acc = fmaf(x.z, y.z, acc);
          acc = fmaf(x.w, y.w, acc);
        }
      }
      __stcs(out + s.d + p, acc);
      off += 32;
    }
    __syncwarp();   // every lane is done with `tile` before the copy two iterations on reuses it
  }
}

__global__ void __launch_bounds__(kDotWarps * 32)
dot_interact_bwd_v2_kernel(const float* __restrict__ T, const float* __restrict__ dR,
                           float* __restrict__ dT, int64_t B, DotShape s) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  const int pitch = s.d + 4, d4 = s.d >> 2;
  float* tile = dot_smem_v2 + (size_t)warp * dot_v2_smem_floats(s, true);
  float* dzf = tile + (size_t)s.N * pitch;
  const int out_w = s.d + s.P;
  for (int64_t b = (int64_t)blockIdx.x * warps + warp; b < B; b += (int64_t)gridDim.x * warps) {
    dot_stage_rows_async(T + b * s.N * s.d, tile, s.N, d4, pitch, lane);
    const float* g = dR + b * out_w;
    for (int i = lane; i < s.N; i += 32) dzf[i * s.N + i] = 0.f;
    {
      int i = 0, off = lane;
      for (int p = lane; p < s.P; p += 32) {
        while (off >= s.row_len(i)) { off -= s.row_len(i); ++i; }
        const int j = s.self ? i + off : i + 1 + off;
        if (j != i) {
          const float v = __ldg(g + s.d + p);
          dzf[i * s.N + j] = v;
          dzf[j * s.N + i] = v;
        }
        off += 32;
      }
    }
    cp_async_wait<0>();
    __syncwarp();
    float* out = dT + b * s.N * s.d;
    const int items = s.N * d4;
    for (int e = lane; e < items; e += 32) {
      const int i = e / d4, c = e - i * d4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i == s.N - 1) {   // dR rows are d+P floats apart: not 16-byte aligned, so four scalar loads
        acc = make_float4(__ldg(g + 4 * c), __ldg(g + 4 * c + 1), __ldg(g + 4 * c + 2), __ldg(g + 4 * c + 3));
      }
      const float* zr = dzf + i * s.N;
#pragma unroll 3
      for (int j = 0; j < s.N; ++j) {
        const float z = zr[j];
        const float4 t = *reinterpret_cast<const float4*>(tile + j * pitch + 4 * c);
        acc.x = fmaf(z, t.x, acc.x);
        acc.y = fmaf(z, t.y, acc.y);
        acc.z = fmaf(z, t.z, acc.z);
        acc.w = fmaf(z, t.w, acc.w);
      }
      __stcs(reinterpret_cast<float4*>(out + 4 * e), acc);
    }
    __syncwarp();
  }
}

}  // namespace b200rec
