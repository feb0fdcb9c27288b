// GateNet's embedding gate (models/rank/gatenet/net.py:88-103) fused with the gather and the concat
// of the tower input (:110):
//
//   forward   per (sample b, field f): e = W[id], s = sum_d e_d * w_f, g = sigmoid(s);
//             out[b, f*D + d] = e_d * g, then out[b, F*D + j] = dense[b, j]
//   backward  per (b, f), the row re-gathered (nothing is saved):
//             q = sum_d dout_d * e_d, c = q * g * (1 - g)
//             drow[b*F + f, d] = dout_d * g + c * w_f      (then group_ids + segment_reduce)
//             dgate_w[f] = sum_b c * sum_d e_d              (per-CTA partials, fixed-order reduce)
//
// Out-of-range ids give a zero row and no gradient (counted in the forward); there is no padding id
// (the reference's Embedding has none).  g uses full-precision expf: at s -> -inf expf(-s) = inf and
// g = 0; at s -> +inf g = 1, so the output stays finite.
//
// One thread per (b, f): a CTA iteration covers spb = kGateEmbedThreads / F whole samples, thread
// t < spb * F owns field t % F for the whole run (the grid stride is a multiple of F positions), so
// its gate-weight contribution is one register summed in sample order.  Grid-stride over samples.
#pragma once

#include "common.cuh"

namespace b200rec {

constexpr int kGateEmbedThreads = 256;
constexpr int kGateEmbedMaxFields = kGateEmbedThreads;

static int gate_embed_grid(int64_t B, int F) {
  const int spb = kGateEmbedThreads / F;
  const int64_t need = (B + spb - 1) / spb;
  const int64_t cap = (int64_t)sm_count() * 8;
  return (int)(need < 1 ? 1 : (need < cap ? need : cap));
}

__device__ __forceinline__ float gate_embed_sigmoid(const float* e, bool ok, float wf, int D) {
  float s = 0.f;
  if (ok)
    for (int d = 0; d < D; ++d) s += __ldg(e + d) * wf;     // multiply, then sum in column order
  return 1.f / (1.f + expf(-s));
}

__global__ void __launch_bounds__(kGateEmbedThreads)
gate_embed_fwd_kernel(const float* __restrict__ W, int64_t ldw, const int64_t* __restrict__ ids,
                      const float* __restrict__ gate_w, const float* __restrict__ dense,
                      float* __restrict__ out, int64_t ld_out, int64_t B, int F, int D, int Dn,
                      int64_t V) {
  const int spb = kGateEmbedThreads / F;
  const int t = threadIdx.x;
  if (t >= spb * F) return;
  const int f = t % F;
  const float wf = __ldg(gate_w + f);
  for (int64_t b = (int64_t)blockIdx.x * spb + t / F; b < B; b += (int64_t)gridDim.x * spb) {
    const int64_t id = __ldg(ids + b * F + f);
    const bool ok = (uint64_t)id < (uint64_t)V;
    if (!ok) atomicAdd(&g_oob_count, 1ull);
    const float* e = W + (ok ? id : 0) * ldw;
    const float g = gate_embed_sigmoid(e, ok, wf, D);
    float* o = out + b * ld_out + (int64_t)f * D;
    for (int d = 0; d < D; ++d) o[d] = ok ? __ldg(e + d) * g : 0.f;
    for (int j = f; j < Dn; j += F) out[b * ld_out + (int64_t)F * D + j] = __ldg(dense + b * Dn + j);
  }
}

__global__ void __launch_bounds__(kGateEmbedThreads)
gate_embed_bwd_kernel(const float* __restrict__ W, int64_t ldw, const int64_t* __restrict__ ids,
                      const float* __restrict__ gate_w, const float* __restrict__ dout,
                      int64_t ld_out, float* __restrict__ drow, float* __restrict__ partials,
                      int64_t B, int F, int D, int64_t V) {
  __shared__ float s_acc[kGateEmbedThreads];
  const int spb = kGateEmbedThreads / F;
  const int t = threadIdx.x;
  float acc = 0.f;
  if (t < spb * F) {
    const int f = t % F;
    const float wf = __ldg(gate_w + f);
    for (int64_t b = (int64_t)blockIdx.x * spb + t / F; b < B; b += (int64_t)gridDim.x * spb) {
      const int64_t id = __ldg(ids + b * F + f);
      const bool ok = (uint64_t)id < (uint64_t)V;
      const float* e = W + (ok ? id : 0) * ldw;
      const float* go = dout + b * ld_out + (int64_t)f * D;
      float* dr = drow + (b * F + f) * D;
      if (!ok) {
        for (int d = 0; d < D; ++d) dr[d] = 0.f;
        continue;
      }
      const float g = gate_embed_sigmoid(e, true, wf, D);
      float q = 0.f, se = 0.f;
      for (int d = 0; d < D; ++d) {
        const float ed = __ldg(e + d);
        q += __ldg(go + d) * ed;
        se += ed;
      }
      const float c = q * g * (1.f - g);
      for (int d = 0; d < D; ++d) dr[d] = __ldg(go + d) * g + c * wf;
      acc += c * se;
    }
  }
  s_acc[t] = acc;
  __syncthreads();
  if (t < F) {                                   // the CTA's samples of field t, in sample order
    float sum = 0.f;
    for (int s = 0; s < spb; ++s) sum += s_acc[s * F + t];
    partials[(int64_t)blockIdx.x * F + t] = sum;
  }
}

// dgate_w[f] = sum over CTAs of partials[cta, f], in CTA order
__global__ void gate_embed_reduce_kernel(const float* __restrict__ partials, int n_cta, int F,
                                         float* __restrict__ dgate_w) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  float sum = 0.f;
  for (int c = 0; c < n_cta; ++c) sum += partials[(int64_t)c * F + f];
  dgate_w[f] = sum;
}

static size_t gate_embed_bwd_ws_bytes(int64_t B, int F) {
  return (size_t)gate_embed_grid(B, F) * F * sizeof(float);
}

static int launch_gate_embed_fwd(const float* W, int64_t ldw, const int64_t* ids,
                                 const float* gate_w, const float* dense, float* out,
                                 int64_t ld_out, int64_t B, int F, int D, int Dn, int64_t V,
                                 cudaStream_t st) {
  B200_REQUIRE(B >= 0 && F > 0 && F <= kGateEmbedMaxFields && D > 0 && Dn >= 0 && V > 0 &&
                   ldw >= D && ld_out >= (int64_t)F * D + Dn,
               "gate_embed_fwd: bad sizes");
  if (B == 0) return B200REC_OK;
  gate_embed_fwd_kernel<<<gate_embed_grid(B, F), kGateEmbedThreads, 0, st>>>(
      W, ldw, ids, gate_w, dense, out, ld_out, B, F, D, Dn, V);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_gate_embed_bwd(const float* W, int64_t ldw, const int64_t* ids,
                                 const float* gate_w, const float* dout, int64_t ld_out,
                                 float* drow, float* dgate_w, int64_t B, int F, int D, int64_t V,
                                 void* ws, size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(B >= 0 && F > 0 && F <= kGateEmbedMaxFields && D > 0 && V > 0 && ldw >= D &&
                   ld_out >= (int64_t)F * D,
               "gate_embed_bwd: bad sizes");
  if (B == 0) {
    B200_CUDA(cudaMemsetAsync(dgate_w, 0, (size_t)F * sizeof(float), st));
    return B200REC_OK;
  }
  const size_t need = gate_embed_bwd_ws_bytes(B, F);
  if (ws == nullptr || ws_bytes < need) {
    set_error("gate_embed_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return B200REC_ERR_WORKSPACE;
  }
  const int grid = gate_embed_grid(B, F);
  float* partials = static_cast<float*>(ws);
  gate_embed_bwd_kernel<<<grid, kGateEmbedThreads, 0, st>>>(W, ldw, ids, gate_w, dout, ld_out, drow,
                                                            partials, B, F, D, V);
  B200_LAUNCH_CHECK();
  gate_embed_reduce_kernel<<<(F + 255) / 256, 256, 0, st>>>(partials, grid, F, dgate_w);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

}  // namespace b200rec
