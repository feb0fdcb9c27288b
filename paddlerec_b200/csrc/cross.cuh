// K3: CrossNet fused epilogues (DCN-V2).
//
// Reference: CrossNetV2.forward, models/rank/dcn_v2/net.py:222-226
//     X_{i+1} = X_i + X_0 * (X_i W_i + b_i)
// The contraction X_i W_i is a dense GEMM (tensor-core library call on the host side); what the
// reference then runs as 3 separate elementwise kernels (bias add, Hadamard, residual) is one
// streaming pass here, and the backward (dxw, dx0 accumulation, bias column-sum) is one pass too.
// Both are HBM-bound: forward moves 4*4C bytes per sample (x0, xl, xw in; out), backward 5*4C.
#pragma once

#include "common.cuh"

namespace b200rec {

constexpr int kCrossThreads = 256;

template <int VEC>
__global__ void __launch_bounds__(kCrossThreads)
cross_v2_fwd_kernel(const float* __restrict__ x0, const float* __restrict__ xl,
                    const float* __restrict__ xw, const float* __restrict__ bias,
                    float* __restrict__ out, int64_t B, int C) {
  const int chunks = C / VEC;
  const int64_t total = B * chunks;
  for (int64_t i = (int64_t)blockIdx.x * kCrossThreads + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * kCrossThreads) {
    const int c = (int)(i % chunks) * VEC;
    const size_t off = (size_t)(i / chunks) * C + c;
    const Vec<VEC> a0 = ld_row<VEC>(x0 + off);
    const Vec<VEC> al = ld_row<VEC>(xl + off);
    const Vec<VEC> aw = ld_row<VEC>(xw + off);
    const Vec<VEC> bb = ld_cached<VEC>(bias + c);
    Vec<VEC> o;
#pragma unroll
    for (int k = 0; k < VEC; ++k) o.v[k] = fmaf(a0.v[k], aw.v[k] + bb.v[k], al.v[k]);
    st_plain<VEC>(out + off, o);
  }
}

// Each thread owns one column chunk and walks a strided slice of rows, so the bias column-sum is
// a register accumulation; partial sums per row-slice go to the workspace and are added in a
// fixed order by reduce_partials_kernel (deterministic).
constexpr int kCrossRowSlices = 132 * 2;

template <int VEC>
__global__ void __launch_bounds__(kCrossThreads)
cross_v2_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ x0,
                    const float* __restrict__ xw, const float* __restrict__ bias,
                    float* __restrict__ dxw, float* __restrict__ dx0,
                    float* __restrict__ partials /*[gridDim.y, C]*/, int64_t B, int C) {
  const int chunks = C / VEC;
  const int chunk = blockIdx.x * kCrossThreads + threadIdx.x;
  if (chunk >= chunks) return;
  const int c = chunk * VEC;
  const Vec<VEC> bb = ld_cached<VEC>(bias + c);
  Vec<VEC> acc = vzero<VEC>();
  for (int64_t b = blockIdx.y; b < B; b += gridDim.y) {
    const size_t off = (size_t)b * C + c;
    const Vec<VEC> g = ld_row<VEC>(dout + off);
    const Vec<VEC> a0 = ld_row<VEC>(x0 + off);
    const Vec<VEC> aw = ld_row<VEC>(xw + off);
    Vec<VEC> d0;
    Vec<VEC> dw;
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      dw.v[k] = g.v[k] * a0.v[k];
      d0.v[k] = g.v[k] * (aw.v[k] + bb.v[k]);
      acc.v[k] += dw.v[k];
    }
    st_plain<VEC>(dxw + off, dw);
    st_plain<VEC>(dx0 + off, d0);
  }
  st_plain<VEC>(partials + (size_t)blockIdx.y * C + c, acc);
}

static int cross_row_slices(int64_t B) {
  return (int)min((int64_t)kCrossRowSlices, B > 0 ? B : (int64_t)1);
}

static int launch_cross_v2_fwd(const float* x0, const float* xl, const float* xw,
                               const float* bias, float* out, int64_t B, int C, cudaStream_t st) {
  B200_REQUIRE(C > 0, "cross_v2_fwd: C must be positive");
  if (B == 0) return B200REC_OK;
  const bool v4 = (C % 4 == 0) && aligned16(x0) && aligned16(xl) && aligned16(xw) &&
                  aligned16(bias) && aligned16(out);
  const int64_t total = B * (v4 ? C / 4 : C);
  const unsigned grid =
      (unsigned)min((total + kCrossThreads - 1) / kCrossThreads, (int64_t)sm_count() * 16);
  if (v4)
    cross_v2_fwd_kernel<4><<<grid, kCrossThreads, 0, st>>>(x0, xl, xw, bias, out, B, C);
  else
    cross_v2_fwd_kernel<1><<<grid, kCrossThreads, 0, st>>>(x0, xl, xw, bias, out, B, C);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_cross_v2_bwd(const float* dout, const float* x0, const float* xw,
                               const float* bias, float* dxw, float* dx0, float* dbias,
                               int64_t B, int C, void* ws, size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(C > 0, "cross_v2_bwd: C must be positive");
  const int slices = cross_row_slices(B);
  const size_t need = (size_t)slices * C * sizeof(float);
  if (ws_bytes < need) {
    set_error("cross_v2_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return B200REC_ERR_WORKSPACE;
  }
  if (B == 0) {
    B200_CUDA(cudaMemsetAsync(dbias, 0, (size_t)C * sizeof(float), st));
    return B200REC_OK;
  }
  const bool v4 = (C % 4 == 0) && aligned16(dout) && aligned16(x0) && aligned16(xw) &&
                  aligned16(bias) && aligned16(dxw) && aligned16(dx0) && aligned16(ws);
  const int chunks = v4 ? C / 4 : C;
  dim3 grid((chunks + kCrossThreads - 1) / kCrossThreads, slices);
  float* partials = static_cast<float*>(ws);
  if (v4)
    cross_v2_bwd_kernel<4><<<grid, kCrossThreads, 0, st>>>(dout, x0, xw, bias, dxw, dx0,
                                                           partials, B, C);
  else
    cross_v2_bwd_kernel<1><<<grid, kCrossThreads, 0, st>>>(dout, x0, xw, bias, dxw, dx0,
                                                           partials, B, C);
  B200_LAUNCH_CHECK();
  reduce_partials_kernel<<<reduce_partials_grid(C), kRedThreads, 0, st>>>(partials, slices, C, dbias, C,
                                                                          nullptr);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

}  // namespace b200rec
