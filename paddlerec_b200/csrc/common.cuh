// Shared helpers for the b200rec kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "b200rec.h"

namespace b200rec {

// ---- error reporting across the C ABI (never throw) --------------------------------------
void set_error(const char* fmt, ...);

#define B200_CUDA(expr)                                                                  \
  do {                                                                                   \
    cudaError_t e__ = (expr);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      ::b200rec::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,            \
                           cudaGetErrorString(e__));                                     \
      return B200REC_ERR_CUDA;                                                           \
    }                                                                                    \
  } while (0)

#define B200_LAUNCH_CHECK() B200_CUDA(cudaPeekAtLastError())

#define B200_REQUIRE(cond, ...)                                                          \
  do {                                                                                   \
    if (!(cond)) {                                                                       \
      ::b200rec::set_error(__VA_ARGS__);                                                 \
      return B200REC_ERR_INVALID;                                                        \
    }                                                                                    \
  } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// H100 SXM: 132 SMs.  Queried once; used to size persistent grids.
int sm_count();

// out-of-range id counter.  The library is ONE translation unit (b200rec.cu includes every
// *.cuh), so this is the single definition.
__device__ unsigned long long g_oob_count = 0ull;

// ---- vector access ---------------------------------------------------------------------
// Vec<VEC> is VEC consecutive floats moved by one LSU instruction (128/64/32 bit).
template <int VEC>
struct Vec;
template <>
struct alignas(16) Vec<4> {
  float v[4];
};
template <>
struct alignas(8) Vec<2> {
  float v[2];
};
template <>
struct Vec<1> {
  float v[1];
};

// read-only, no L1 allocation: the random table rows are touched once per kernel.
template <int VEC>
__device__ __forceinline__ Vec<VEC> ld_row(const float* p);
template <>
__device__ __forceinline__ Vec<4> ld_row<4>(const float* p) {
  Vec<4> r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3])
               : "l"(p));
  return r;
}
template <>
__device__ __forceinline__ Vec<2> ld_row<2>(const float* p) {
  Vec<2> r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];"
               : "=f"(r.v[0]), "=f"(r.v[1])
               : "l"(p));
  return r;
}
template <>
__device__ __forceinline__ Vec<1> ld_row<1>(const float* p) {
  Vec<1> r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r.v[0]) : "l"(p));
  return r;
}

// Predicated variants: branch-free "load if pred else zeros" (the predicate is a PTX guard, so the
// compiler cannot turn it into a divergent branch around the volatile asm).  ALLOC selects whether
// the line may allocate in L1 (rows whose line is re-read by a neighbouring scalar lookup).
template <int VEC, bool ALLOC>
__device__ __forceinline__ Vec<VEC> ld_row_pred(const float* p, bool pred);
#define B200_LD_PRED(VECN, ALLOCB, PTXOP, OUTS, REGS)                                           \
  template <>                                                                                    \
  __device__ __forceinline__ Vec<VECN> ld_row_pred<VECN, ALLOCB>(const float* p, bool pred) {    \
    Vec<VECN> r = vzero_init<VECN>();                                                            \
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %" #REGS ", 0;\n\t@q " PTXOP          \
                 ";\n\t}"                                                                       \
                 : OUTS                                                                          \
                 : "l"(p), "r"((int)pred));                                                      \
    return r;                                                                                    \
  }
template <int VEC>
__device__ __forceinline__ Vec<VEC> vzero_init() {
  Vec<VEC> r;
#pragma unroll
  for (int i = 0; i < VEC; ++i) r.v[i] = 0.f;
  return r;
}
#define B200_OUT4 "+f"(r.v[0]), "+f"(r.v[1]), "+f"(r.v[2]), "+f"(r.v[3])
#define B200_OUT2 "+f"(r.v[0]), "+f"(r.v[1])
#define B200_OUT1 "+f"(r.v[0])
B200_LD_PRED(4, false, "ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4]", B200_OUT4, 5)
B200_LD_PRED(4, true, "ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4]", B200_OUT4, 5)
B200_LD_PRED(2, false, "ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2]", B200_OUT2, 3)
B200_LD_PRED(2, true, "ld.global.nc.v2.f32 {%0,%1}, [%2]", B200_OUT2, 3)
B200_LD_PRED(1, false, "ld.global.nc.L1::no_allocate.f32 %0, [%1]", B200_OUT1, 2)
B200_LD_PRED(1, true, "ld.global.nc.f32 %0, [%1]", B200_OUT1, 2)
#undef B200_LD_PRED

// cp.async (LDGSTS) helpers: global -> shared without register staging
__device__ __forceinline__ void cp_async_8(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(
                   (unsigned)__cvta_generic_to_shared(smem)),
               "l"(gmem)
               : "memory");
}
__device__ __forceinline__ void cp_async_4(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(
                   (unsigned)__cvta_generic_to_shared(smem)),
               "l"(gmem)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// cached read (small broadcast operands: dense_w, S rows, bias)
template <int VEC>
__device__ __forceinline__ Vec<VEC> ld_cached(const float* p);
template <>
__device__ __forceinline__ Vec<4> ld_cached<4>(const float* p) {
  float4 t = __ldg(reinterpret_cast<const float4*>(p));
  Vec<4> r;
  r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  return r;
}
template <>
__device__ __forceinline__ Vec<2> ld_cached<2>(const float* p) {
  float2 t = __ldg(reinterpret_cast<const float2*>(p));
  Vec<2> r;
  r.v[0] = t.x; r.v[1] = t.y;
  return r;
}
template <>
__device__ __forceinline__ Vec<1> ld_cached<1>(const float* p) {
  Vec<1> r;
  r.v[0] = __ldg(p);
  return r;
}

// streaming store (write-once outputs larger than L2: evict-first)
template <int VEC>
__device__ __forceinline__ void st_stream(float* p, const Vec<VEC>& x);
template <>
__device__ __forceinline__ void st_stream<4>(float* p, const Vec<4>& x) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(x.v[0]), "f"(x.v[1]),
               "f"(x.v[2]), "f"(x.v[3])
               : "memory");
}
template <>
__device__ __forceinline__ void st_stream<2>(float* p, const Vec<2>& x) {
  asm volatile("st.global.cs.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(x.v[0]), "f"(x.v[1])
               : "memory");
}
template <>
__device__ __forceinline__ void st_stream<1>(float* p, const Vec<1>& x) {
  asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(x.v[0]) : "memory");
}

// plain store (outputs that the next kernel re-reads from L2)
template <int VEC>
__device__ __forceinline__ void st_plain(float* p, const Vec<VEC>& x);
template <>
__device__ __forceinline__ void st_plain<4>(float* p, const Vec<4>& x) {
  *reinterpret_cast<float4*>(p) = make_float4(x.v[0], x.v[1], x.v[2], x.v[3]);
}
template <>
__device__ __forceinline__ void st_plain<2>(float* p, const Vec<2>& x) {
  *reinterpret_cast<float2*>(p) = make_float2(x.v[0], x.v[1]);
}
template <>
__device__ __forceinline__ void st_plain<1>(float* p, const Vec<1>& x) {
  *p = x.v[0];
}

template <int VEC>
__device__ __forceinline__ Vec<VEC> vzero() {
  Vec<VEC> r;
#pragma unroll
  for (int i = 0; i < VEC; ++i) r.v[i] = 0.f;
  return r;
}

// xor-shuffle sum over the TPR lanes that share one row (TPR is a power of two <= 32).
template <int TPR>
__device__ __forceinline__ float group_sum(float x) {
#pragma unroll
  for (int o = TPR / 2; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// Row geometry chosen on the host: VEC floats per lane, TPR lanes per row, D = row length.
// A lane with chunk index r is active iff r*VEC < D.
struct RowShape {
  int vec;  // 4, 2 or 1
  int tpr;  // lanes per row (power of two)
};
static inline bool pick_row_shape(int D, RowShape* rs) {
  int vec = (D % 4 == 0) ? 4 : (D % 2 == 0 ? 2 : 1);
  int chunks = D / vec;
  if (chunks > 32) return false;
  int tpr = 1;
  while (tpr < chunks) tpr <<= 1;
  rs->vec = vec;
  rs->tpr = tpr;
  return true;
}

// Dispatch a functor templated on <VEC,TPR>.
#define B200_DISPATCH_ROW_SHAPE(rs, ...)                    \
  do {                                                        \
    switch ((rs).vec * 100 + (rs).tpr) {                      \
      case 401: { constexpr int VEC = 4, TPR = 1; __VA_ARGS__; } break;  \
      case 402: { constexpr int VEC = 4, TPR = 2; __VA_ARGS__; } break;  \
      case 404: { constexpr int VEC = 4, TPR = 4; __VA_ARGS__; } break;  \
      case 408: { constexpr int VEC = 4, TPR = 8; __VA_ARGS__; } break;  \
      case 416: { constexpr int VEC = 4, TPR = 16; __VA_ARGS__; } break;  \
      case 432: { constexpr int VEC = 4, TPR = 32; __VA_ARGS__; } break;  \
      case 201: { constexpr int VEC = 2, TPR = 1; __VA_ARGS__; } break;  \
      case 202: { constexpr int VEC = 2, TPR = 2; __VA_ARGS__; } break;  \
      case 204: { constexpr int VEC = 2, TPR = 4; __VA_ARGS__; } break;  \
      case 208: { constexpr int VEC = 2, TPR = 8; __VA_ARGS__; } break;  \
      case 216: { constexpr int VEC = 2, TPR = 16; __VA_ARGS__; } break;  \
      case 232: { constexpr int VEC = 2, TPR = 32; __VA_ARGS__; } break;  \
      case 101: { constexpr int VEC = 1, TPR = 1; __VA_ARGS__; } break;  \
      case 102: { constexpr int VEC = 1, TPR = 2; __VA_ARGS__; } break;  \
      case 104: { constexpr int VEC = 1, TPR = 4; __VA_ARGS__; } break;  \
      case 108: { constexpr int VEC = 1, TPR = 8; __VA_ARGS__; } break;  \
      case 116: { constexpr int VEC = 1, TPR = 16; __VA_ARGS__; } break;  \
      case 132: { constexpr int VEC = 1, TPR = 32; __VA_ARGS__; } break;  \
      default:                                                \
        ::b200rec::set_error("unsupported row shape");        \
        return B200REC_ERR_INVALID;                           \
    }                                                         \
  } while (0)

}  // namespace b200rec
