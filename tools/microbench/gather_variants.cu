// Micro-benchmark: how should 64-byte random rows be fetched on the H100?
// Variants of the load instruction x cudaLimitMaxL2FetchGranularity, timed with CUDA events.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gather_variants gather_variants.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1);} } while (0)

template <int MODE> __device__ __forceinline__ float4 ld(const float* p) {
  float4 r;
  if (MODE == 0) asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 1) asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 2) asm volatile("ld.global.ca.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 3) asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 4) asm volatile("ld.global.cs.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 5) asm volatile("ld.global.L2::64B.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 6) asm volatile("ld.global.lu.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  if (MODE == 7) asm volatile("ld.global.nc.L1::no_allocate.L2::64B.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x),"=f"(r.y),"=f"(r.z),"=f"(r.w) : "l"(p));
  return r;
}

// TPR lanes per row (D = 4*TPR floats), ROWS rows in flight per lane group; sum-reduce the rows of
// a group of RPG consecutive ids and write one row (so output traffic is small: isolates reads).
template <int MODE, int TPR, int ROWS>
__global__ void gather_sum(const float* __restrict__ W, const int64_t* __restrict__ ids, float* __restrict__ out, int64_t n, int D) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) / TPR, r = threadIdx.x % TPR;
  const int64_t base = (int64_t)g * ROWS;
  if (base >= n) return;
  float4 acc = make_float4(0, 0, 0, 0);
  float4 e[ROWS];
#pragma unroll
  for (int j = 0; j < ROWS; ++j) { int64_t id = ids[base + j]; e[j] = ld<MODE>(W + id * D + r * 4); }
#pragma unroll
  for (int j = 0; j < ROWS; ++j) { acc.x += e[j].x; acc.y += e[j].y; acc.z += e[j].z; acc.w += e[j].w; }
  *reinterpret_cast<float4*>(out + (int64_t)g * D + r * 4) = acc;
}

// scalar 4-byte gather (the first-order table W1[V])
template <int MODE>
__global__ void gather_scalar(const float* __restrict__ W1, const int64_t* __restrict__ ids, float* __restrict__ out, int64_t n) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= n) return;
  float a = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float v; const float* p = W1 + ids[i + j];
    if (MODE == 0) asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    if (MODE == 2) asm volatile("ld.global.ca.f32 %0, [%1];" : "=f"(v) : "l"(p));
    if (MODE == 3) asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(p));
    a += v;
  }
  out[i / 4] = a;
}

template <int MODE, int TPR>
float run(const float* W, const int64_t* ids, float* out, int64_t n, int D) {
  constexpr int ROWS = 8;
  int64_t groups = n / ROWS; int threads = 256; int64_t blocks = (groups * TPR + threads - 1) / threads;
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < 3; ++i) gather_sum<MODE, TPR, ROWS><<<blocks, threads>>>(W, ids, out, n, D);
  cudaEventRecord(a);
  for (int i = 0; i < 10; ++i) gather_sum<MODE, TPR, ROWS><<<blocks, threads>>>(W, ids + (i % 4) * n, out, n, D);
  cudaEventRecord(b); CK(cudaEventSynchronize(b));
  float ms; cudaEventElapsedTime(&ms, a, b); return ms / 10;
}

int main() {
  const int64_t V = 100000000; const int64_t n = 65536 * 26;
  size_t lim = 0; cudaDeviceGetLimit(&lim, cudaLimitMaxL2FetchGranularity);
  printf("default cudaLimitMaxL2FetchGranularity = %zu\n", lim);
  float* W; CK(cudaMalloc(&W, V * 16 * sizeof(float))); CK(cudaMemset(W, 0, V * 16 * sizeof(float)));
  std::vector<int64_t> h(n * 4); uint64_t s = 88172645463325252ull;
  for (auto& x : h) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; x = (int64_t)(s % (uint64_t)V); }
  int64_t* ids; CK(cudaMalloc(&ids, n * 4 * 8)); CK(cudaMemcpy(ids, h.data(), n * 4 * 8, cudaMemcpyHostToDevice));
  float* out; CK(cudaMalloc(&out, n * 16 * sizeof(float)));
  for (int gran : {0, 32, 64, 128}) {
    if (gran) { cudaError_t e = cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran); printf("set granularity %d: %s\n", gran, cudaGetErrorString(e)); }
    const char* names[] = {"nc.noalloc", "nc", "ca", "cg", "cs", "L2::64B", "lu", "nc.noalloc.L2::64B"};
    float t[8];
    t[0] = run<0, 4>(W, ids, out, n, 16); t[1] = run<1, 4>(W, ids, out, n, 16); t[2] = run<2, 4>(W, ids, out, n, 16);
    t[3] = run<3, 4>(W, ids, out, n, 16); t[4] = run<4, 4>(W, ids, out, n, 16); t[5] = run<5, 4>(W, ids, out, n, 16);
    t[6] = run<6, 4>(W, ids, out, n, 16); t[7] = run<7, 4>(W, ids, out, n, 16);
    for (int m = 0; m < 8; ++m)
      printf("D=16 (64B rows) %-20s %.4f ms  rows: %.0f GB/s useful\n", names[m], t[m], n * 64.0 / t[m] / 1e6);
    // 128B rows (D=32) and 256B rows (D=64) from the same buffer for comparison (V/2, V/4 rows)
    {
      std::vector<int64_t> h2(n * 4); for (size_t i = 0; i < h2.size(); ++i) h2[i] = h[i] / 2;
      int64_t* ids2; CK(cudaMalloc(&ids2, n * 4 * 8)); CK(cudaMemcpy(ids2, h2.data(), n * 4 * 8, cudaMemcpyHostToDevice));
      float a = run<0, 8>(W, ids2, out, n, 32); printf("D=32 (128B rows) nc.noalloc %.4f ms  %.0f GB/s useful\n", a, n * 128.0 / a / 1e6);
      for (size_t i = 0; i < h2.size(); ++i) h2[i] = h[i] / 4;
      CK(cudaMemcpy(ids2, h2.data(), n * 4 * 8, cudaMemcpyHostToDevice));
      a = run<0, 16>(W, ids2, out, n, 64); printf("D=64 (256B rows) nc.noalloc %.4f ms  %.0f GB/s useful\n", a, n * 256.0 / a / 1e6);
      cudaFree(ids2);
    }
    // scalar gathers
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); float ms;
#define SC(MODE, NAME) { for (int i = 0; i < 2; ++i) gather_scalar<MODE><<<(n / 4 + 255) / 256, 256>>>(W, ids, out, n); cudaEventRecord(a); \
      for (int i = 0; i < 10; ++i) gather_scalar<MODE><<<(n / 4 + 255) / 256, 256>>>(W, ids + (i % 4) * n, out, n); cudaEventRecord(b); cudaEventSynchronize(b); \
      cudaEventElapsedTime(&ms, a, b); printf("scalar 4B gather %-12s %.4f ms (%.0f M lookups/s)\n", NAME, ms / 10, n / (ms / 10) / 1e3); }
    SC(0, "nc.noalloc") SC(2, "ca") SC(3, "cg")
  }
  return 0;
}
