// Hand-written wgmma / TMA GEMMs for the dense tower in split precision ("bf16x3").
//
// Reference path: DNN.forward models/rank/deepfm/net.py:169-174 (Linear -> ReLU chain), its autograd
// (tools/trainer.py:151 loss.backward()), and the same chain in dcn_v2/net.py:178-184,
// wide_deep/net.py:95-97, din/net.py:175-184.  An fp32 product a@w is evaluated on the Hopper
// tensor cores as a_hi@w_hi + a_lo@w_hi + a_hi@w_lo (bf16 operands, exact products, fp32
// accumulation in registers; ~2^-16 relative), which meets the 1e-4 logit bar that plain TF32 misses.
//
// Operand format ("planes"): a matrix X[R, C] lives in HBM as bf16 [R, 2*ld] with the rounded value
// hi(X) in columns [0, C) and the residual lo(X) = bf16(X - hi) in columns [ld, ld + C); ld is C
// rounded up to 8 so that both planes are 16-byte aligned TMA tensors.  Same bytes as fp32.
//
// Two kernels, both warp-specialised over three warpgroups (warpgroup 0 = TMA producer, warpgroups
// 1 and 2 = wgmma.mma_async consumers owning 64 output rows each, fp32 accumulators in registers)
// with an mbarrier pipeline full/empty over the shared-memory stages:
//
//   tc_gemm_kmajor_kernel   D[M,N] = A[M,K] . B[N,K]^T     both operands K-major (reduction dim
//       contiguous): forward (A = activations, B = W^T planes) and dX (A = dZ planes, B = W
//       planes).  Persistent over 128 x BN output tiles; the producer streams the next tile's
//       k-blocks while the consumers run the epilogue of the current one.  Fused epilogues, staged
//       through shared memory per warp and stored row-contiguously: +bias, ReLU, hi/lo split (emits
//       the NEXT GEMM's operand directly), ReLU mask + bias column-sum in backward, CrossNet, or
//       plain fp32.
//   tc_gemm_dw_kernel       dW[K,N] = sum_m A[m,K] . G[m,N]   both operands MN-major (the batch dim
//       is the reduction; wgmma reads both transposed), split over the batch across CTAs, fp32
//       partial tiles + fixed-order reduce (deterministic, no atomics).
//
// Shared-memory tiles are swizzled exactly as TMA writes them (CU_TENSOR_MAP_SWIZZLE_128B, or 64B
// for 32-wide k-blocks) and described to wgmma by 64-bit shared-memory matrix descriptors.
#pragma once

#include <cuda.h>  // CUtensorMap and enums only; cuTensorMapEncodeTiled is resolved at run time
#include <cuda_bf16.h>

#include <type_traits>

#include "common.cuh"

namespace b200rec {
namespace tc {

constexpr int kBM = 128;          // output rows per tile: two consumer warpgroups x wgmma M = 64
constexpr int kUK = 16;           // wgmma K for 16-bit operands
constexpr int kThreads = 384;     // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma + epilogue
constexpr int kConsumerWarps = 8;
constexpr int kMaxBN = 256;       // wgmma N limit; the accumulator is BN / 2 registers per thread
constexpr int kDwBR = 32;         // batch rows per k-block of the dW kernel
constexpr uint32_t kSmemBudget = 227u * 1024u - 2048u;

// device-side error word: a pipeline wait that exceeds its budget records where and traps, so a
// protocol bug surfaces as a CUDA error instead of a hung GPU.
__device__ unsigned int g_tc_timeout = 0u;

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, unsigned where) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) {  // ~2 s at 2 GHz
      atomicExch(&g_tc_timeout, where | 0x80000000u);
      __trap();
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
// 2-D tiled TMA load: box lands in shared memory swizzled, completion on an mbarrier.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar,
                                            int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(m), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
// move registers from the producer warpgroup to the consumers (all 128 threads of a warpgroup)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
// at most N committed wgmma groups of this warpgroup still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// the accumulator registers are written asynchronously: keep the compiler from moving their reads
// (the epilogue) above the wgmma_wait that completes them
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ------------------------------------------------------------------------------------------------
// descriptors
// ------------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (bits: [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4,
// [62,64) swizzle: 1 = 128B, 2 = 64B).  K-major: SBO = stride between 8-row groups, LBO unused
// (one swizzle row spans the whole k-block).  MN-major: LBO = stride between 64-element column
// chunks, SBO = stride between 8-row (k) groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes,
                                              uint32_t sbo_bytes, uint32_t layout) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}

// wgmma.mma_async m64nNk16, bf16 x bf16 -> fp32: d (N / 2 registers per thread) += A . B with both
// operands read from shared memory through descriptors; TA / TB = 1: the operand is stored
// MN-major.  acc = 0 overwrites d instead of accumulating.
template <int N, int TA, int TB>
struct Wgmma;

template <int TA, int TB>
struct Wgmma<16, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7"
        "}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

template <int TA, int TB>
struct Wgmma<64, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
        "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),
          "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

template <int TA, int TB>
struct Wgmma<128, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
        "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, "
        "%34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
        "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),
          "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]),
          "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]),
          "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
          "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]),
          "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

template <int TA, int TB>
struct Wgmma<208, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[104], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %106, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n208k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
        "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, "
        "%34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
        "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, "
        "%66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, "
        "%82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, "
        "%98, %99, %100, %101, %102, %103"
        "}, %104, %105, p, 1, 1, %107, %108;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),
          "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]),
          "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]),
          "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
          "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]),
          "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]),
          "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]),
          "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]),
          "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]),
          "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]),
          "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

template <int TA, int TB>
struct Wgmma<256, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, "
        "%18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, "
        "%34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, "
        "%50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, "
        "%66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, "
        "%82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, "
        "%98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, "
        "%111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, "
        "%124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, %131, %132;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]),
          "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]),
          "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]),
          "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]),
          "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]),
          "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]),
          "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]),
          "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]),
          "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]),
          "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]),
          "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]),
          "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]),
          "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]),
          "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]),
          "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]),
          "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

// ------------------------------------------------------------------------------------------------
// epilogue description (plain pointers: this struct crosses into the kernel by value)
// ------------------------------------------------------------------------------------------------
struct Epilogue {
  const float* bias;                // [N] added before ReLU, or null
  int relu;                         // max(., 0)
  float* out_f32;                   // [M, ld_f32] or null
  int64_t ld_f32;
  __nv_bfloat16* out_planes;        // [M, 2*ldp] hi | lo, or null
  int64_t ldp;
  const __nv_bfloat16* mask_src;    // keep v where mask_src[m, n] > 0 (hi plane of the saved
  int64_t ld_mask;                  //   activation; row pitch in elements), or null
  float* colsum;                    // [tiles_m, N] per-tile column sums of the emitted v, or null
  // CrossNetV2 (dcn_v2/net.py:222-226): v = x0[m,n] * (acc + bias[n]) + xl[m,n]
  const float* cross_x0;
  const float* cross_xl;
  int64_t ld_cross;
  // also write out_planes[m, N] = 1.0 (hi) / 0 (lo): the column of ones that makes the dW GEMM of
  // the next layer produce its bias gradient as row N (needs ldp > N)
  int ones_col;
  const float* addend;              // [M, ld_add] added to acc (+bias) before everything else, or null
  int64_t ld_add;
  float* aux_f32;                   // [M, ld_aux] receives acc + bias + addend, i.e. the value BEFORE
  int64_t ld_aux;                   //   the CrossNet / ReLU / mask transforms, or null
  // GateNet hidden gate (gatenet/net.py:116-118): v = y[m,n] * tanhf(acc), y = hi + lo of the planes
  // [M, 2*ld_gate] at gate_y (the GEMM's own A operand).  Read only by the kernels compiled with
  // kGate, so the other instantiations keep their code.
  const __nv_bfloat16* gate_y;
  int64_t ld_gate;
  // filled in by launch_gemm_kmajor, not by the callers:
  int vec;                          // kVec* bits: the operand allows one 16-byte (fp32) or 8-byte
                                    //   (bf16) access per 4 columns at every row
  int extra;                        // addend, aux_f32 or CrossNet in use (the second epilogue body)
};

enum : int {
  kVecBias = 1, kVecF32 = 2, kVecPlanes = 4, kVecMask = 8, kVecAdd = 16, kVecAux = 32,
  kVecCross = 64, kVecGate = 128,
};

__device__ __forceinline__ void split_bf16(float x, float& hi_f, __nv_bfloat16& hi,
                                           __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  hi_f = __bfloat162float(hi);
  lo = __float2bfloat16_rn(x - hi_f);
}

// hi/lo split of two values, packed for a 32-bit store (element a at the lower address)
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  hi = *reinterpret_cast<const uint32_t*>(&h2);
  const float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xFFFF0000u);
  const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - ha, b - hb);
  lo = *reinterpret_cast<const uint32_t*>(&l2);
}

__device__ __forceinline__ bool al8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

__device__ __forceinline__ void st_pair(float* p, bool two, float x, float y) {
  if (two && al8(p)) {
    *reinterpret_cast<float2*>(p) = make_float2(x, y);
  } else {
    p[0] = x;
    if (two) p[1] = y;
  }
}

// p[0 .. n), n in 1..4, as one access where `vec` allows it; missing elements read as 0
__device__ __forceinline__ float4 ld4(const float* p, int n, bool vec) {
  if (vec && n == 4) return __ldg(reinterpret_cast<const float4*>(p));
  float4 v = make_float4(__ldg(p), 0.f, 0.f, 0.f);
  if (n > 1) v.y = __ldg(p + 1);
  if (n > 2) v.z = __ldg(p + 2);
  if (n > 3) v.w = __ldg(p + 3);
  return v;
}
__device__ __forceinline__ void st4(float* p, int n, bool vec, float4 v) {
  if (vec && n == 4) {
    *reinterpret_cast<float4*>(p) = v;
    return;
  }
  p[0] = v.x;
  if (n > 1) p[1] = v.y;
  if (n > 2) p[2] = v.z;
  if (n > 3) p[3] = v.w;
}
// four bf16 packed in two 32-bit words (element 0 in the low half of w.x)
__device__ __forceinline__ uint2 ld4_bf16(const __nv_bfloat16* p, int n, bool vec) {
  if (vec && n == 4) return __ldg(reinterpret_cast<const uint2*>(p));
  const unsigned short* q = reinterpret_cast<const unsigned short*>(p);
  uint2 w = make_uint2(__ldg(q), 0u);
  if (n > 1) w.x |= (uint32_t)__ldg(q + 1) << 16;
  if (n > 2) w.y = __ldg(q + 2);
  if (n > 3) w.y |= (uint32_t)__ldg(q + 3) << 16;
  return w;
}
__device__ __forceinline__ void st4_bf16(__nv_bfloat16* p, int n, bool vec, uint2 w) {
  if (vec && n == 4) {
    *reinterpret_cast<uint2*>(p) = w;
    return;
  }
  unsigned short* q = reinterpret_cast<unsigned short*>(p);
  q[0] = (unsigned short)(w.x & 0xFFFFu);
  if (n > 1) q[1] = (unsigned short)(w.x >> 16);
  if (n > 2) q[2] = (unsigned short)(w.y & 0xFFFFu);
  if (n > 3) q[3] = (unsigned short)(w.y >> 16);
}

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
// the 128-byte lines of `bytes` bytes at p, spread over the two lanes (lane & 1) of a row
__device__ __forceinline__ void prefetch_row_l2(const void* p, int bytes, int lane) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(p) & ~(uintptr_t)127;
  const uintptr_t a1 = reinterpret_cast<uintptr_t>(p) + (uintptr_t)bytes - 1;
  for (uintptr_t a = a0 + 128u * (uintptr_t)(lane & 1); a <= a1; a += 256u)
    prefetch_l2(reinterpret_cast<const void*>(a));
}

// Epilogue staging: each consumer warp passes its 16 x BN accumulator rows through shared memory
// in chunks of 16 rows x 32 columns (fp32, rows padded to 40 floats: the fragment's float2 writes
// and the row-contiguous float4 reads are both free of bank conflicts).  Read back row-contiguously,
// every global access of a quarter-warp covers one row segment of 4 x 8 columns: 128-byte fp32
// stores, 64-byte stores into each bf16 plane.
constexpr int kEpCols = 32;
constexpr int kEpPitch = 40;
constexpr uint32_t kEpWarpFloats = 16u * kEpPitch;
constexpr uint32_t kEpSmemBytes = kConsumerWarps * kEpWarpFloats * 4u;

// Accumulator fragment columns [32 c, 32 c + 32) -> the warp's staging chunk (wgmma layout: the
// thread holds rows lane / 4 and + 8, columns 8 j + 2 (lane % 4) + {0, 1}).  The chunk index is a
// run-time value; the accumulator registers are selected by a chain of compile-time cases.
template <int BN, int C = 0>
__device__ __forceinline__ void stage_chunk(const float (&acc)[BN / 2], float* stg, int c, int lane) {
  if (c == C) {
    constexpr int CW = BN - kEpCols * C < kEpCols ? BN - kEpCols * C : kEpCols;
    constexpr int j0 = kEpCols / 8 * C;
    const int lc = 2 * (lane & 3), rr = lane >> 2;
#pragma unroll
    for (int jj = 0; jj < CW / 8; ++jj) {
      *reinterpret_cast<float2*>(stg + rr * kEpPitch + 8 * jj + lc) =
          make_float2(acc[4 * (j0 + jj)], acc[4 * (j0 + jj) + 1]);
      *reinterpret_cast<float2*>(stg + (rr + 8) * kEpPitch + 8 * jj + lc) =
          make_float2(acc[4 * (j0 + jj) + 2], acc[4 * (j0 + jj) + 3]);
    }
    return;
  }
  if constexpr (kEpCols * (C + 1) < BN) stage_chunk<BN, C + 1>(acc, stg, c, lane);
}

// One chunk of a consumer warp's epilogue: matrix columns [c0, c0 + cw) of the warp's 16 rows (first
// row r0).  Lane l handles columns c0 + 4 (l % 8) .. + 3 in rows l / 8 + 4 p, p = 0..3.  The side
// inputs of the chunk are loaded first, then stage() puts the raw accumulators into `stg`.  The
// transforms apply in this order: + bias, + addend, aux store, CrossNet fma, ReLU, mask, then the
// fp32 and hi/lo stores, the same per-element arithmetic as an unstaged epilogue.  kExtra: the
// addend / aux / CrossNet body; without it those fields are ignored.  kGate (with kExtra): the hidden
// gate v = y * tanhf(v) right after the aux store.  With s_cs (the warp's column sums of this chunk)
// the emitted values are summed over the warp's rows in a fixed order.
template <bool kExtra, typename Stage, bool kGate = false>
__device__ __forceinline__ void epilogue_rows(const Epilogue& ep, const float* stg, int M, int N,
                                              int64_t r0, int c0, int cw, int lane, float* s_cs,
                                              Stage stage) {
  const int g = lane & 7, lr = lane >> 3;
  const int col = c0 + 4 * g;
  int n = 4 * g < cw ? N - col : 0;           // valid columns of this lane (<= 0: none)
  n = n > 4 ? 4 : n;
  const int vec = ep.vec;

  float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ep.bias != nullptr && n > 0) bias = ld4(ep.bias + col, n, vec & kVecBias);
  uint2 mw[4];
  if (ep.mask_src != nullptr) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int64_t row = r0 + lr + 4 * p;
      mw[p] = n > 0 && row < M ? ld4_bf16(ep.mask_src + row * ep.ld_mask + col, n, vec & kVecMask)
                               : make_uint2(0u, 0u);
    }
  }
  __syncwarp();                                // the previous chunk's reads are done
  stage();
  __syncwarp();

  float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int64_t row = r0 + lr + 4 * p;
    if (n <= 0 || row >= M) continue;
    float4 v = *reinterpret_cast<const float4*>(stg + (lr + 4 * p) * kEpPitch + 4 * g);
    if (ep.bias != nullptr) {
      v.x += bias.x; v.y += bias.y; v.z += bias.z; v.w += bias.w;
    }
    if (kExtra) {
      if (ep.addend != nullptr) {
        const float4 a = ld4(ep.addend + row * ep.ld_add + col, n, vec & kVecAdd);
        v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
      }
      if (ep.aux_f32 != nullptr) st4(ep.aux_f32 + row * ep.ld_aux + col, n, vec & kVecAux, v);
      if (ep.cross_x0 != nullptr) {
        const float4 x0 = ld4(ep.cross_x0 + row * ep.ld_cross + col, n, vec & kVecCross);
        const float4 xl = ld4(ep.cross_xl + row * ep.ld_cross + col, n, vec & kVecCross);
        v.x = fmaf(x0.x, v.x, xl.x); v.y = fmaf(x0.y, v.y, xl.y);
        v.z = fmaf(x0.z, v.z, xl.z); v.w = fmaf(x0.w, v.w, xl.w);
      }
      if (kGate) {
        // accurate tanhf (tanh.approx's ~2^-11 relative error would show in the logit)
        const __nv_bfloat16* yp = ep.gate_y + row * 2 * ep.ld_gate + col;
        const uint2 h = ld4_bf16(yp, n, vec & kVecGate), l = ld4_bf16(yp + ep.ld_gate, n, vec & kVecGate);
        v.x = (__uint_as_float(h.x << 16) + __uint_as_float(l.x << 16)) * tanhf(v.x);
        v.y = (__uint_as_float(h.x & 0xFFFF0000u) + __uint_as_float(l.x & 0xFFFF0000u)) * tanhf(v.y);
        v.z = (__uint_as_float(h.y << 16) + __uint_as_float(l.y << 16)) * tanhf(v.z);
        v.w = (__uint_as_float(h.y & 0xFFFF0000u) + __uint_as_float(l.y & 0xFFFF0000u)) * tanhf(v.w);
      }
    }
    if (ep.relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    if (ep.mask_src != nullptr) {
      // bf16 > 0  <=>  its bit pattern, as a signed integer in the high half, is > 0
      if (!((int)(mw[p].x << 16) > 0)) v.x = 0.f;
      if (!((int)(mw[p].x & 0xFFFF0000u) > 0)) v.y = 0.f;
      if (!((int)(mw[p].y << 16) > 0)) v.z = 0.f;
      if (!((int)(mw[p].y & 0xFFFF0000u) > 0)) v.w = 0.f;
    }
    if (n < 4) {                               // columns past N: nothing stored, 0 in the sums
      if (n < 2) v.y = 0.f;
      if (n < 3) v.z = 0.f;
      v.w = 0.f;
    }
    if (ep.out_f32 != nullptr) st4(ep.out_f32 + row * ep.ld_f32 + col, n, vec & kVecF32, v);
    if (ep.out_planes != nullptr) {
      __nv_bfloat16* oh = ep.out_planes + row * 2 * ep.ldp + col;
      uint2 h, l;
      split_pack2(v.x, v.y, h.x, l.x);
      split_pack2(v.z, v.w, h.y, l.y);
      st4_bf16(oh, n, vec & kVecPlanes, h);
      st4_bf16(oh + ep.ldp, n, vec & kVecPlanes, l);
    }
    cs.x += v.x; cs.y += v.y; cs.z += v.z; cs.w += v.w;
  }
  if (s_cs != nullptr) {                       // fixed-order tree over the 4 lanes of a column group
#pragma unroll
    for (int h = 8; h <= 16; h <<= 1) {
      cs.x += __shfl_xor_sync(0xffffffffu, cs.x, h);
      cs.y += __shfl_xor_sync(0xffffffffu, cs.y, h);
      cs.z += __shfl_xor_sync(0xffffffffu, cs.z, h);
      cs.w += __shfl_xor_sync(0xffffffffu, cs.w, h);
    }
    if (lane < 8 && 4 * lane < cw) *reinterpret_cast<float4*>(s_cs + 4 * lane) = cs;
  }
}

// One consumer warp's 16 x BN share of a 128 x BN accumulator tile -> outputs, in chunks of 32
// columns.  r0: the warp's first matrix row.  With s_cs ([kMaxBN]) the warp's column sums of the
// emitted values land there.  The chunk loop is not unrolled: one copy of each epilogue body.
template <int BN, bool kGate = false>
__device__ __forceinline__ void epilogue_tile(const Epilogue& ep, const float (&acc)[BN / 2],
                                              float* stg, int M, int N, int64_t r0, int n0, int lane,
                                              float* s_colsum) {
  constexpr int kChunks = (BN + kEpCols - 1) / kEpCols;
#pragma unroll 1
  for (int c = 0; c < kChunks; ++c) {
    const int cw = BN - kEpCols * c < kEpCols ? BN - kEpCols * c : kEpCols;
    float* s_cs = s_colsum != nullptr ? s_colsum + kEpCols * c : nullptr;
    auto stage = [&] { stage_chunk<BN>(acc, stg, c, lane); };
    if constexpr (kGate)
      epilogue_rows<true, decltype(stage), true>(ep, stg, M, N, r0, n0 + kEpCols * c, cw, lane, s_cs,
                                                 stage);
    else if (ep.extra)
      epilogue_rows<true>(ep, stg, M, N, r0, n0 + kEpCols * c, cw, lane, s_cs, stage);
    else
      epilogue_rows<false>(ep, stg, M, N, r0, n0 + kEpCols * c, cw, lane, s_cs, stage);
  }
  if (ep.ones_col && ep.out_planes != nullptr && n0 + BN >= N && lane < 16 && r0 + lane < M) {
    __nv_bfloat16* oh = ep.out_planes + (r0 + lane) * 2 * ep.ldp + N;
    oh[0] = __float2bfloat16_rn(1.f);
    oh[ep.ldp] = __float2bfloat16_rn(0.f);
  }
}

// The side inputs a warp's epilogue will read for its 16 rows of a tile, fetched into L2 while the
// tile's products run (the saved activations they come from are far larger than L2).
__device__ __forceinline__ void epilogue_prefetch(const Epilogue& ep, int M, int N, int BN,
                                                 int64_t r0, int n0, int lane) {
  const int64_t row = r0 + (lane >> 1);
  if (row >= M) return;
  const int w = N - n0 < BN ? N - n0 : BN;
  if (ep.mask_src != nullptr) prefetch_row_l2(ep.mask_src + row * ep.ld_mask + n0, 2 * w, lane);
  if (ep.extra) {
    if (ep.addend != nullptr) prefetch_row_l2(ep.addend + row * ep.ld_add + n0, 4 * w, lane);
    if (ep.cross_x0 != nullptr) {
      prefetch_row_l2(ep.cross_x0 + row * ep.ld_cross + n0, 4 * w, lane);
      prefetch_row_l2(ep.cross_xl + row * ep.ld_cross + n0, 4 * w, lane);
    }
  }
}

// The gate's y planes (hi and lo) of a warp's 16 rows, fetched like the side inputs above.
__device__ __forceinline__ void epilogue_prefetch_gate(const Epilogue& ep, int M, int N, int BN,
                                                      int64_t r0, int n0, int lane) {
  const int64_t row = r0 + (lane >> 1);
  if (row >= M) return;
  const int w = N - n0 < BN ? N - n0 : BN;
  const __nv_bfloat16* y = ep.gate_y + row * 2 * ep.ld_gate + n0;
  prefetch_row_l2(y, 2 * w, lane);
  prefetch_row_l2(y + ep.ld_gate, 2 * w, lane);
}

// ------------------------------------------------------------------------------------------------
// K-major GEMM: D[M,N] = A[M,K] . B[N,K]^T  (three wgmma per 16-wide k step)
//   BK = 64: 128-byte swizzle rows (2 pipeline stages at BN = 208)
//   BK = 32: 64-byte swizzle rows, half-size stages -> 4 stages at BN = 208: about the same bytes in
//            shared memory, but a freed slot is refilled twice as early, which hides the TMA latency
// The producer warpgroup hands registers to the consumers (setmaxnreg): a consumer thread holds
// BN / 2 accumulators through the whole epilogue.  kGate: the GateNet hidden-gate epilogue
// (Epilogue::gate_y), a separate instantiation so the plain and CrossNet kernels stay as they are.
// ------------------------------------------------------------------------------------------------
template <int BN, int BK, bool kGate = false>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_kmajor_kernel(const __grid_constant__ CUtensorMap tmA_hi,
                      const __grid_constant__ CUtensorMap tmA_lo,
                      const __grid_constant__ CUtensorMap tmB_hi,
                      const __grid_constant__ CUtensorMap tmB_lo, int M, int N, int K, int stages,
                      const __grid_constant__ Epilogue ep) {
  constexpr uint32_t kRow = BK * 2;                       // bytes per operand row in a stage
  constexpr uint32_t kLayout = BK == 64 ? 1u : 2u;        // SWIZZLE_128B / SWIZZLE_64B
  constexpr uint32_t kSbo = 8u * kRow;                    // 8-row swizzle atom
  constexpr uint32_t a_bytes = kBM * kRow;
  constexpr uint32_t b_bytes = BN * kRow;
  constexpr uint32_t stage_bytes = 2u * a_bytes + 2u * b_bytes;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;          // swizzled tiles: atom-aligned
  uint8_t* sm = smem_raw + (base - raw);
  // [stages][full barriers][empty barriers][colsum scratch: 8 warps x kMaxBN][epilogue staging]
  const uint32_t bar_full = base + (uint32_t)stages * stage_bytes;
  const uint32_t bar_empty = bar_full + 8u * stages;
  float* s_colsum = reinterpret_cast<float*>(sm + (size_t)stages * stage_bytes + 16 * stages);
  float* s_stage = s_colsum + kConsumerWarps * kMaxBN;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + kBM - 1) / kBM, tiles_n = (N + BN - 1) / BN;
  const int n_tiles = tiles_m * tiles_n;
  const int nkb = (K + BK - 1) / BK;
  // the consumers split the k-blocks into nfull blocks of BK / 16 real k-steps and, if tail > 0, a
  // last block of tail < BK / 16 steps
  const int last_steps = (K - (nkb - 1) * BK + kUK - 1) / kUK;
  const int tail = last_steps == BK / kUK ? 0 : last_steps;
  const int nfull = tail ? nkb - 1 : nkb;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA_hi); prefetch_tmap(&tmA_lo); prefetch_tmap(&tmB_hi); prefetch_tmap(&tmB_lo);
    for (int s = 0; s < stages; ++s) {
      mbar_init(bar_full + 8u * s, 1);
      mbar_init(bar_empty + 8u * s, kConsumerWarps);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * kBM, n0 = (tile % tiles_n) * BN;
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(bar_empty + 8u * stage, phase ^ 1u, 0x100u + stage);
          const uint32_t full = bar_full + 8u * stage;
          const uint32_t sA = base + (uint32_t)stage * stage_bytes;
          mbar_expect_tx(full, stage_bytes);
          tma_load_2d(sA, &tmA_hi, full, kb * BK, m0);
          tma_load_2d(sA + a_bytes, &tmA_lo, full, kb * BK, m0);
          tma_load_2d(sA + 2u * a_bytes, &tmB_hi, full, kb * BK, n0);
          tma_load_2d(sA + 2u * a_bytes + b_bytes, &tmB_lo, full, kb * BK, n0);
          if (++stage == stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();            // 128 x 40 + 256 x 232 registers <= 64 K
    const int cw = warp - 4;          // consumer warp 0..7; warpgroup = cw / 4 owns rows 64 (cw / 4)..
    const int wg = cw >> 2;
    const bool want_colsum = ep.colsum != nullptr;
    float* const stg = s_stage + cw * kEpWarpFloats;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int m_blk = tile / tiles_n;
      const int m0 = m_blk * kBM, n0 = (tile % tiles_n) * BN;
      const int64_t r0 = (int64_t)m0 + 64 * wg + 16 * (cw & 3);   // this warp's first row
      epilogue_prefetch(ep, M, N, BN, r0, n0, lane);
      if constexpr (kGate) epilogue_prefetch_gate(ep, M, N, BN, r0, n0, lane);
      int prev = 0;
      // one k-block of NS 16-wide k-steps: three wgmma per step, one commit group per block
      auto kblock = [&](auto ns, int kb) {
        mbar_wait(bar_full + 8u * stage, phase, 0x300u + stage);
        const uint32_t sA = base + (uint32_t)stage * stage_bytes + (uint32_t)wg * (64u * kRow);
        const uint32_t sB = base + (uint32_t)stage * stage_bytes + 2u * a_bytes;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < decltype(ns)::value; ++j) {
          const uint32_t ko = (uint32_t)j * (kUK * 2);   // 32 bytes further inside the swizzle row
          const uint64_t a_hi = gmma_desc(sA + ko, 16, kSbo, kLayout);
          const uint64_t a_lo = gmma_desc(sA + a_bytes + ko, 16, kSbo, kLayout);
          const uint64_t b_hi = gmma_desc(sB + ko, 16, kSbo, kLayout);
          const uint64_t b_lo = gmma_desc(sB + b_bytes + ko, 16, kSbo, kLayout);
          Wgmma<BN, 0, 0>::mma(acc, a_hi, b_hi, (kb | j) != 0 ? 1u : 0u);
          Wgmma<BN, 0, 0>::mma(acc, a_lo, b_hi, 1u);
          Wgmma<BN, 0, 0>::mma(acc, a_hi, b_lo, 1u);
        }
        wgmma_commit();
        if (kb > 0) {           // the previous k-block's products are done: its slot is free
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(bar_empty + 8u * prev);
        }
        prev = stage;
        if (++stage == stages) { stage = 0; phase ^= 1u; }
      };
      constexpr int kSteps = BK / kUK;
      for (int kb = 0; kb < nfull; ++kb) kblock(std::integral_constant<int, kSteps>(), kb);
      // A last block with fewer real k-steps skips the steps that would multiply TMA's zero fill.
      // Each tail length runs as a loop of 0 or 1 trips, not as a branch: wgmma issued inside a
      // conditional path is serialized by ptxas.
      for (int t = 0; t < (tail == 1); ++t) kblock(std::integral_constant<int, 1>(), nfull);
      if constexpr (kSteps > 2)
        for (int t = 0; t < (tail == 2); ++t) kblock(std::integral_constant<int, 2>(), nfull);
      if constexpr (kSteps > 3)
        for (int t = 0; t < (tail == 3); ++t) kblock(std::integral_constant<int, 3>(), nfull);
      wgmma_wait<0>();
      fence_acc(acc);
      if (lane == 0) mbar_arrive(bar_empty + 8u * prev);
      epilogue_tile<BN, kGate>(ep, acc, stg, M, N, r0, n0, lane,
                        want_colsum ? s_colsum + cw * kMaxBN : nullptr);
      if (want_colsum) {
        named_bar_sync(1, 32 * kConsumerWarps);
        const int n_tile = (N - n0) < BN ? (N - n0) : BN;
        for (int c = threadIdx.x - 128; c < n_tile; c += 32 * kConsumerWarps) {
          float s = 0.f;
#pragma unroll
          for (int w = 0; w < kConsumerWarps; ++w) s += s_colsum[w * kMaxBN + c];
          ep.colsum[(int64_t)m_blk * N + n0 + c] = s;
        }
        named_bar_sync(1, 32 * kConsumerWarps);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// dW GEMM: P[split][K,N] = sum_{m in split} A[m,K]^T G[m,N]   (both operands MN-major)
// ------------------------------------------------------------------------------------------------
struct DwDebug {
  uint32_t lbo_a, lbo_b, sbo;   // 0 = default
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
tc_gemm_dw_kernel(const __grid_constant__ CUtensorMap tmA_hi,
                  const __grid_constant__ CUtensorMap tmA_lo,
                  const __grid_constant__ CUtensorMap tmG_hi,
                  const __grid_constant__ CUtensorMap tmG_lo, int M, int Kin, int N, int stages,
                  int rows_per_split, float* __restrict__ partials, DwDebug dbg) {
  constexpr int nb = BN / 64;                             // 64-column chunks of the G tile
  constexpr uint32_t chunk = kDwBR * 128u;                // one TMA box: BR rows x 128 B
  constexpr uint32_t a_bytes = 2u * chunk, b_bytes = (uint32_t)nb * chunk;
  constexpr uint32_t stage_bytes = 2u * a_bytes + 2u * b_bytes;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bar_full = base + (uint32_t)stages * stage_bytes, bar_empty = bar_full + 8u * stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_n = (N + BN - 1) / BN;
  const int k0 = (blockIdx.x / tiles_n) * kBM, n0 = (blockIdx.x % tiles_n) * BN;
  const int split = blockIdx.y;
  const int r0 = split * rows_per_split;
  int r1 = r0 + rows_per_split;
  r1 = r1 > M ? M : r1;
  const int nkb = r1 > r0 ? (r1 - r0 + kDwBR - 1) / kDwBR : 0;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA_hi); prefetch_tmap(&tmA_lo); prefetch_tmap(&tmG_hi); prefetch_tmap(&tmG_lo);
    for (int s = 0; s < stages; ++s) {
      mbar_init(bar_full + 8u * s, 1);
      mbar_init(bar_empty + 8u * s, kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(bar_empty + 8u * stage, phase ^ 1u, 0x500u + stage);
        const uint32_t full = bar_full + 8u * stage;
        const uint32_t sA = base + (uint32_t)stage * stage_bytes;
        const uint32_t sB = sA + 2u * a_bytes;
        const int r = r0 + kb * kDwBR;
        mbar_expect_tx(full, stage_bytes);
        for (int c = 0; c < 2; ++c) {
          tma_load_2d(sA + c * chunk, &tmA_hi, full, k0 + c * 64, r);
          tma_load_2d(sA + a_bytes + c * chunk, &tmA_lo, full, k0 + c * 64, r);
        }
        for (int c = 0; c < nb; ++c) {
          tma_load_2d(sB + c * chunk, &tmG_hi, full, n0 + c * 64, r);
          tma_load_2d(sB + b_bytes + c * chunk, &tmG_lo, full, n0 + c * 64, r);
        }
        if (++stage == stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    const int cw = warp - 4, wg = cw >> 2;
    const uint32_t lbo_a = dbg.lbo_a ? dbg.lbo_a : chunk;
    const uint32_t lbo_b = dbg.lbo_b ? dbg.lbo_b : chunk;
    const uint32_t sbo = dbg.sbo ? dbg.sbo : 1024u;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      mbar_wait(bar_full + 8u * stage, phase, 0x600u + stage);
      // this warpgroup's 64 output rows (features k0 + 64 wg ..) are the wg-th column chunk of A
      const uint32_t sA = base + (uint32_t)stage * stage_bytes + (uint32_t)wg * chunk;
      const uint32_t sB = base + (uint32_t)stage * stage_bytes + 2u * a_bytes;
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < kDwBR / kUK; ++j) {
        const uint32_t ko = (uint32_t)j * (kUK * 128u);  // 16 batch rows further down the box
        const uint64_t a_hi = gmma_desc(sA + ko, lbo_a, sbo, 1u);
        const uint64_t a_lo = gmma_desc(sA + a_bytes + ko, lbo_a, sbo, 1u);
        const uint64_t g_hi = gmma_desc(sB + ko, lbo_b, sbo, 1u);
        const uint64_t g_lo = gmma_desc(sB + b_bytes + ko, lbo_b, sbo, 1u);
        Wgmma<BN, 1, 1>::mma(acc, a_hi, g_hi, 1u);
        Wgmma<BN, 1, 1>::mma(acc, a_lo, g_hi, 1u);
        Wgmma<BN, 1, 1>::mma(acc, a_hi, g_lo, 1u);
      }
      wgmma_commit();
      if (kb > 0) {
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(bar_empty + 8u * prev);
      }
      prev = stage;
      if (++stage == stages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    fence_acc(acc);
    const int kr0 = k0 + 64 * wg + 16 * (cw & 3) + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = n0 + 8 * j + 2 * (lane & 3);
      if (col >= N) continue;
      const bool two = col + 1 < N;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int krow = kr0 + 8 * h;
        if (krow < Kin)
          st_pair(partials + ((size_t)split * Kin + (size_t)krow) * N + col, two, acc[4 * j + 2 * h],
                  acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

// dW[k,n] = sum_s P[s][k,n] in fixed order
__global__ void tc_dw_reduce_kernel(const float* __restrict__ P, int splits, int64_t KN,
                                    float* __restrict__ dW) {
  const int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 >= KN) return;
  if (i4 + 4 <= KN && (KN & 3) == 0) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < splits; ++s) {
      const float4 p = __ldg(reinterpret_cast<const float4*>(P + (size_t)s * KN + i4));
      acc.x += p.x; acc.y += p.y; acc.z += p.z; acc.w += p.w;
    }
    *reinterpret_cast<float4*>(dW + i4) = acc;
  } else {
    for (int64_t i = i4; i < KN && i < i4 + 4; ++i) {
      float acc = 0.f;
      for (int s = 0; s < splits; ++s) acc += P[(size_t)s * KN + i];
      dW[i] = acc;
    }
  }
}

// out[n] = sum_t P[t][n] (per-tile column sums -> bias gradient), fixed order, coalesced over n
__global__ void tc_colsum_reduce_kernel(const float* __restrict__ P, int tiles, int N,
                                        float* __restrict__ out) {
  // blockDim = (32 columns, 8 row-slices): slice y sums tiles y, y+8, ...; then a fixed-order
  // combine over the 8 slices in shared memory.
  __shared__ float s[8][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  float acc = 0.f;
  if (n < N)
    for (int t = threadIdx.y; t < tiles; t += 8) acc += P[(size_t)t * N + n];
  s[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += s[y][threadIdx.x];
    out[n] = t;
  }
}

// W fp32 [K,N] -> Wp planes [K, 2*ldn] (straight) and WTp planes [N, 2*ldk] (transposed)
__global__ void tc_prep_weight_kernel(const float* __restrict__ W, int K, int N,
                                      __nv_bfloat16* __restrict__ Wp, int64_t ldn,
                                      __nv_bfloat16* __restrict__ WTp, int64_t ldk) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int y = threadIdx.y; y < 32; y += blockDim.y) {
    const int k = k0 + y, n = n0 + threadIdx.x;
    float w = 0.f;
    if (k < K && n < N) {
      w = W[(size_t)k * N + n];
      float hf;
      __nv_bfloat16 h, l;
      split_bf16(w, hf, h, l);
      if (Wp != nullptr) {
        Wp[(size_t)k * 2 * ldn + n] = h;
        Wp[(size_t)k * 2 * ldn + ldn + n] = l;
      }
    }
    tile[y][threadIdx.x] = w;
  }
  __syncthreads();
  if (WTp == nullptr) return;
  for (int y = threadIdx.y; y < 32; y += blockDim.y) {
    const int n = n0 + y, k = k0 + threadIdx.x;
    if (k < K && n < N) {
      float hf;
      __nv_bfloat16 h, l;
      split_bf16(tile[threadIdx.x][y], hf, h, l);
      WTp[(size_t)n * 2 * ldk + k] = h;
      WTp[(size_t)n * 2 * ldk + ldk + k] = l;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// bf16 matrix [rows, width] with row pitch `pitch_elems`; box = box_w x box_rows, 128B swizzle
// (64B for 32-wide boxes), out-of-bounds elements read as zero.
static int make_map(CUtensorMap* m, const void* base, int64_t width, int64_t rows,
                    int64_t pitch_elems, int box_w, int box_rows) {
  const CUtensorMapSwizzle swz = box_w == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  EncodeTiledFn enc = encode_tiled_fn();
  if (enc == nullptr) {
    set_error("tc_gemm: cuTensorMapEncodeTiled is not available from this driver");
    return B200REC_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15u) != 0 || (pitch_elems * 2) % 16 != 0) {
    set_error("tc_gemm: operand planes must be 16-byte aligned with a pitch multiple of 8 "
              "(base %p, pitch %lld)", base, (long long)pitch_elems);
    return B200REC_ERR_INVALID;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)pitch_elems * 2};
  const cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("tc_gemm: cuTensorMapEncodeTiled failed (%d) width %lld rows %lld pitch %lld box %dx%d",
              (int)r, (long long)width, (long long)rows, (long long)pitch_elems, box_w, box_rows);
    return B200REC_ERR_CUDA;
  }
  return B200REC_OK;
}

static DwDebug g_dw_debug = {0u, 0u, 0u};
static int g_bn_override = 0;
// k-block of the K-major kernel: 32 (SWIZZLE_64B, 4 stages at BN = 208) or 64 (SWIZZLE_128B, 2
// stages).  At every forward and dX shape of the DeepFM tower 32 is faster or within 2 % of 64
// (tools/tc_probe.py perf), so it is not chosen per shape.
static int g_bk = 32;

// Tile widths the K-major kernel is compiled for.  The choice minimises the padded output width
// plus a per-tile charge of 64 columns for re-reading the A tile (N = 400 -> 2 x 208, 624 -> 3 x 208,
// 1560 -> 8 x 208, 512 -> 2 x 256, 1 -> 16).  A forced width (tc_debug key 0) rounds up to the next
// compiled one.
static const int kTileBN[] = {16, 64, 128, 208, 256};

static int pick_bn(int N) {
  if (g_bn_override > 0) {
    for (int bn : kTileBN)
      if (bn >= g_bn_override) return bn;
    return kMaxBN;
  }
  int best = kMaxBN;
  int64_t best_cost = -1;
  for (int bn : kTileBN) {
    const int64_t cost = (int64_t)((N + bn - 1) / bn) * (bn + 64);
    if (best_cost < 0 || cost <= best_cost) {
      best = bn;
      best_cost = cost;
    }
  }
  return best;
}

template <int BN, int BK, bool kGate>
static int launch_kmajor_tiles(const CUtensorMap (&mp)[4], int64_t M, int N, int K,
                               const Epilogue& ep, cudaStream_t st) {
  constexpr uint32_t stage_bytes = (2u * kBM + 2u * BN) * (uint32_t)BK * 2u;
  constexpr uint32_t scratch = kConsumerWarps * kMaxBN * 4u + kEpSmemBytes;
  constexpr uint32_t fixed = scratch + 16u * 8u + 1024u;
  int stages = (int)((kSmemBudget - fixed) / stage_bytes);
  stages = stages > 8 ? 8 : stages;
  B200_REQUIRE(stages >= 2, "tc_gemm: tile does not fit shared memory");
  const size_t smem = (size_t)stages * stage_bytes + 16 * stages + scratch + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    B200_CUDA(cudaFuncSetAttribute(tc_gemm_kmajor_kernel<BN, BK, kGate>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  const int tiles = (int)((M + kBM - 1) / kBM) * ((N + BN - 1) / BN);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  tc_gemm_kmajor_kernel<BN, BK, kGate><<<grid, kThreads, smem, st>>>(mp[0], mp[1], mp[2], mp[3],
                                                                     (int)M, N, K, stages, ep);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

template <int BK, bool kGate>
static int launch_kmajor_bk(int BN, const CUtensorMap (&mp)[4], int64_t M, int N, int K,
                            const Epilogue& ep, cudaStream_t st) {
  switch (BN) {
    case 16: return launch_kmajor_tiles<16, BK, kGate>(mp, M, N, K, ep, st);
    case 64: return launch_kmajor_tiles<64, BK, kGate>(mp, M, N, K, ep, st);
    case 128: return launch_kmajor_tiles<128, BK, kGate>(mp, M, N, K, ep, st);
    case 208: return launch_kmajor_tiles<208, BK, kGate>(mp, M, N, K, ep, st);
    default: return launch_kmajor_tiles<256, BK, kGate>(mp, M, N, K, ep, st);
  }
}

// D = A . B^T with A planes [M, 2*lda] (logical [M,K]) and B planes [N, 2*ldb] (logical [N,K]).
// p is set, and 4 elements at any row and any column multiple of 4 are one `bytes`-aligned access
static bool aligned_rows(const void* p, int64_t ld, unsigned bytes) {
  return p != nullptr && reinterpret_cast<uintptr_t>(p) % bytes == 0 && ld % 4 == 0;
}

static int launch_gemm_kmajor(const void* A, int64_t lda, const void* B, int64_t ldb, int64_t M,
                              int N, int K, const Epilogue& ep_in, cudaStream_t st) {
  B200_REQUIRE(M >= 0 && N > 0 && K > 0, "tc_gemm: bad sizes M=%lld N=%d K=%d", (long long)M, N, K);
  B200_REQUIRE(M < (1ll << 31), "tc_gemm: M too large");
  if (M == 0) return B200REC_OK;
  Epilogue ep = ep_in;
  ep.vec = (aligned_rows(ep.bias, 0, 16) ? kVecBias : 0) |
           (aligned_rows(ep.out_f32, ep.ld_f32, 16) ? kVecF32 : 0) |
           (aligned_rows(ep.out_planes, ep.ldp, 8) ? kVecPlanes : 0) |
           (aligned_rows(ep.mask_src, ep.ld_mask, 8) ? kVecMask : 0) |
           (aligned_rows(ep.addend, ep.ld_add, 16) ? kVecAdd : 0) |
           (aligned_rows(ep.aux_f32, ep.ld_aux, 16) ? kVecAux : 0) |
           (aligned_rows(ep.cross_x0, ep.ld_cross, 16) && aligned_rows(ep.cross_xl, ep.ld_cross, 16)
                ? kVecCross : 0) |
           (aligned_rows(ep.gate_y, ep.ld_gate, 8) ? kVecGate : 0);
  ep.extra = ep.addend != nullptr || ep.aux_f32 != nullptr || ep.cross_x0 != nullptr ||
             ep.gate_y != nullptr;
  const bool gate = ep.gate_y != nullptr;
  const int BN = pick_bn(N);
  const int BK = g_bk;
  const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(A);
  const __nv_bfloat16* b = static_cast<const __nv_bfloat16*>(B);
  CUtensorMap mp[4];
  int rc;
  if ((rc = make_map(&mp[0], a, K, M, 2 * lda, BK, kBM)) != B200REC_OK) return rc;
  if ((rc = make_map(&mp[1], a + lda, K, M, 2 * lda, BK, kBM)) != B200REC_OK) return rc;
  if ((rc = make_map(&mp[2], b, K, N, 2 * ldb, BK, BN)) != B200REC_OK) return rc;
  if ((rc = make_map(&mp[3], b + ldb, K, N, 2 * ldb, BK, BN)) != B200REC_OK) return rc;
  if (gate)
    return BK == 64 ? launch_kmajor_bk<64, true>(BN, mp, M, N, K, ep, st)
                    : launch_kmajor_bk<32, true>(BN, mp, M, N, K, ep, st);
  return BK == 64 ? launch_kmajor_bk<64, false>(BN, mp, M, N, K, ep, st)
                  : launch_kmajor_bk<32, false>(BN, mp, M, N, K, ep, st);
}

struct DwPlan {
  int BN, tiles, splits, rows_per_split, stages;
  size_t smem, ws_bytes;
};

static DwPlan plan_dw(int64_t M, int K, int N) {
  DwPlan p;
  // the G tile is loaded in 64-column chunks: widths 64, 128 or 256
  p.BN = N <= 64 ? 64 : (N <= 128 ? 128 : 256);
  if (g_bn_override > 0) p.BN = g_bn_override <= 64 ? 64 : (g_bn_override <= 128 ? 128 : 256);
  p.tiles = ((K + kBM - 1) / kBM) * ((N + p.BN - 1) / p.BN);
  int splits = sm_count() / p.tiles;
  splits = splits < 1 ? 1 : splits;
  int64_t rps = (M + splits - 1) / splits;
  rps = (rps + kDwBR - 1) / kDwBR * kDwBR;
  rps = rps < kDwBR ? kDwBR : rps;
  p.rows_per_split = (int)rps;
  p.splits = (int)((M + rps - 1) / rps);
  p.splits = p.splits < 1 ? 1 : p.splits;
  const int nb = p.BN / 64;
  const uint32_t stage_bytes = (4u + 2u * nb) * kDwBR * 128u;
  p.stages = (int)((kSmemBudget - 4096u) / stage_bytes);
  p.stages = p.stages > 8 ? 8 : p.stages;
  p.smem = (size_t)p.stages * stage_bytes + 16 * p.stages + 1024;
  p.ws_bytes = (size_t)p.splits * K * N * sizeof(float);
  return p;
}

template <int BN>
static int launch_dw_tiles(const DwPlan& p, const CUtensorMap (&mp)[4], int M, int K, int N,
                           float* P, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    B200_CUDA(cudaFuncSetAttribute(tc_gemm_dw_kernel<BN>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  dim3 grid(p.tiles, p.splits);
  tc_gemm_dw_kernel<BN><<<grid, kThreads, p.smem, st>>>(mp[0], mp[1], mp[2], mp[3], M, K, N,
                                                        p.stages, p.rows_per_split, P, g_dw_debug);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

// dW[K,N] = A^T G with A planes [M, 2*lda] (logical [M,K]) and G planes [M, 2*ldg] (logical [M,N])
static int launch_gemm_dw(const void* A, int64_t lda, const void* G, int64_t ldg, int64_t M, int K,
                          int N, float* dW, void* ws, size_t ws_bytes, cudaStream_t st) {
  B200_REQUIRE(M >= 0 && N > 0 && K > 0, "tc_gemm_dw: bad sizes");
  B200_REQUIRE(M < (1ll << 31), "tc_gemm_dw: M too large");
  const int64_t KN = (int64_t)K * N;
  if (M == 0) {
    B200_CUDA(cudaMemsetAsync(dW, 0, (size_t)KN * sizeof(float), st));
    return B200REC_OK;
  }
  const DwPlan p = plan_dw(M, K, N);
  if (ws_bytes < p.ws_bytes) {
    set_error("tc_gemm_dw: workspace %zu < %zu bytes", ws_bytes, p.ws_bytes);
    return B200REC_ERR_WORKSPACE;
  }
  const __nv_bfloat16* a = static_cast<const __nv_bfloat16*>(A);
  const __nv_bfloat16* g = static_cast<const __nv_bfloat16*>(G);
  CUtensorMap mp[4];
  int rc;
  if ((rc = make_map(&mp[0], a, K, M, 2 * lda, 64, kDwBR)) != B200REC_OK) return rc;
  if ((rc = make_map(&mp[1], a + lda, K, M, 2 * lda, 64, kDwBR)) != B200REC_OK) return rc;
  if ((rc = make_map(&mp[2], g, N, M, 2 * ldg, 64, kDwBR)) != B200REC_OK) return rc;
  if ((rc = make_map(&mp[3], g + ldg, N, M, 2 * ldg, 64, kDwBR)) != B200REC_OK) return rc;
  float* P = p.splits == 1 ? dW : static_cast<float*>(ws);
  switch (p.BN) {
    case 64: rc = launch_dw_tiles<64>(p, mp, (int)M, K, N, P, st); break;
    case 128: rc = launch_dw_tiles<128>(p, mp, (int)M, K, N, P, st); break;
    default: rc = launch_dw_tiles<256>(p, mp, (int)M, K, N, P, st); break;
  }
  if (rc != B200REC_OK) return rc;
  if (p.splits > 1) {
    const int64_t n4 = (KN + 3) / 4;
    tc_dw_reduce_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(P, p.splits, KN, dW);
    B200_LAUNCH_CHECK();
  }
  return B200REC_OK;
}

}  // namespace tc
}  // namespace b200rec
