// The scalar tail of a CTR step as three kernels instead of ~25 elementwise launches:
//   sum_sigmoid : pred = sigmoid(a + b + c)            (deepfm/net.py:47, wide_deep/net.py:99-101)
//   log_loss_mean fwd/bwd : mean_i( -y log(p+eps) - (1-y) log(1-p+eps) ), Paddle's log_loss with
//       eps = 1e-4 followed by paddle.mean (deepfm/dygraph_model.py:53-58)
// At 65536 samples these are launch-latency bound: each torch op costs a launch the host has to
// issue (the step is host-bound whenever the loss is read back every step).  Deterministic: block
// partial sums are combined in block order by the last block to finish.
#pragma once

#include "common.cuh"

namespace b200rec {

constexpr int kHeadOpThreads = 256;

// pred[i] = sigmoid(a[i] + b[i] + c[i]); b / c may be null
__global__ void sum_sigmoid_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                       const float* __restrict__ c, float* __restrict__ pred,
                                       int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x = a[i];
  if (b != nullptr) x += b[i];
  if (c != nullptr) x += c[i];
  // full-precision expf: the logit bar is 1e-4 relative
  pred[i] = 1.f / (1.f + expf(-x));
}

// dlogit[i] = dpred[i] * p (1 - p)
__global__ void sum_sigmoid_bwd_kernel(const float* __restrict__ pred,
                                       const float* __restrict__ dpred,
                                       float* __restrict__ dlogit, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float p = pred[i];
  dlogit[i] = dpred[i] * p * (1.f - p);
}

template <typename LabelT>
__global__ void __launch_bounds__(kHeadOpThreads)
log_loss_mean_fwd_kernel(const float* __restrict__ pred, const LabelT* __restrict__ label,
                         float eps, float* __restrict__ partials, unsigned int* __restrict__ ticket,
                         float* __restrict__ loss, int64_t n) {
  __shared__ float s_red[kHeadOpThreads / 32];
  __shared__ bool s_last;
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * kHeadOpThreads + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * kHeadOpThreads) {
    const float p = pred[i];
    const float y = (float)label[i];
    acc += -y * logf(p + eps) - (1.f - y) * logf(1.f - p + eps);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kHeadOpThreads / 32; ++w) t += s_red[w];
    partials[blockIdx.x] = t;
    __threadfence();
    s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {       // fixed block order: deterministic
    __threadfence();
    double t = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) t += (double)__ldcg(partials + b);
    loss[0] = (float)(t / (double)n);
    *ticket = 0u;                         // ready for the next launch
  }
}

// dpred[i] = dloss * ( -y/(p+eps) + (1-y)/(1-p+eps) ) / n
template <typename LabelT>
__global__ void log_loss_mean_bwd_kernel(const float* __restrict__ pred,
                                         const LabelT* __restrict__ label, float eps,
                                         const float* __restrict__ dloss, float* __restrict__ dpred,
                                         int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float p = pred[i];
  const float y = (float)label[i];
  const float g = __ldg(dloss) / (float)n;
  dpred[i] = g * (-y / (p + eps) + (1.f - y) / (1.f - p + eps));
}

// paddle.metric.Auc.update (deepfm/dygraph_model.py:75-87): bucket = clamp(int(p * T), 0, T);
// stat_pos / stat_neg [T+1] += 1.  Integer atomics: the result does not depend on their order.
template <typename LabelT>
__global__ void auc_update_kernel(const float* __restrict__ pred, const LabelT* __restrict__ label,
                                  long long* __restrict__ pos, long long* __restrict__ neg,
                                  int num_thresholds, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long b = (long long)(pred[i] * (float)num_thresholds);
  b = b < 0 ? 0 : (b > num_thresholds ? num_thresholds : b);
  const bool is_pos = label[i] != (LabelT)0;
  atomicAdd(reinterpret_cast<unsigned long long*>(is_pos ? pos : neg) + b, 1ull);
}

constexpr int kLossBlocks = 132;
static size_t log_loss_ws_bytes() { return (size_t)kLossBlocks * sizeof(float) + 16; }

}  // namespace b200rec
