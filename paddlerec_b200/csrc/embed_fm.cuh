// K1 / K2: DeepFM's fused multi-slot gather + FM interaction, forward and backward.
//
// Replaces FM.forward of the reference (models/rank/deepfm/net.py:105-139) and its autograd
// (SURVEY.md §8a rows A1-A3, A7).  HBM-bound: per sample the forward moves
//   F*8 (ids) + Dn*4 (dense) + F*4D (rows) + F*4 (first-order) + (F+Dn)*4D (feat) + 8 (y1,y2)
// algorithmic bytes (4532 B at F=26, Dn=13, D=16) and ~3 flops per byte, so the design goal is
// to keep as many independent 128-bit row loads in flight as the LSU allows and to touch
// every byte once:
//   * ids/dense of a tile of samples are staged to shared memory with coalesced loads;
//   * TPR lanes share one sample, each lane owns VEC consecutive floats of every row, so one
//     warp instruction fetches 32/TPR random rows with full 32 B-sector use (D=16: 8 rows);
//   * the running sum S and sum of squares Q stay in registers over all F+Dn fields; the
//     first-order lookups are spread over the TPR lanes; a xor-shuffle finishes y1/y2;
//   * feat is written once with evict-first stores (it is larger than L2 at B=65536).
#pragma once

#include <stdlib.h>

#include "common.cuh"
#include "segreduce.cuh"

namespace b200rec {

// Tunables (env B200REC_K1_UNROLL = 8|13|26, B200REC_K1_CACHE = 0|1, B200REC_K1_CTAS = persistent
// CTAs per SM), read once per process:
// U = independent row loads in flight per lane; CACHE = let row loads allocate in L1 (useful for
// the fused slot layout, where the first-order weight sits in the same 128-byte line as the row).
struct K1Config {
  int unroll;
  int cache_rows;
  int ctas_per_sm;
  int debug;
  int tma;  // 1: shared-memory-staged variant with a bulk (TMA) store of the feat tile
  int minb;  // __launch_bounds__ min blocks/SM (register cap) variants: 4 (default), 5, 6, 8
  int warp_sched;  // 1: per-warp pipeline with a dynamic group scheduler (no CTA barriers)
};
static K1Config k1_config() {
  static K1Config cfg = [] {
    K1Config c{13, 0, 8, 0, 0, 4, 0};
    if (const char* s = getenv("B200REC_K1_WARP")) c.warp_sched = atoi(s);
    if (const char* s = getenv("B200REC_K1_UNROLL")) c.unroll = atoi(s);
    if (const char* s = getenv("B200REC_K1_CACHE")) c.cache_rows = atoi(s);
    if (const char* s = getenv("B200REC_K1_CTAS")) c.ctas_per_sm = atoi(s);
    if (const char* s = getenv("B200REC_K1_DEBUG")) c.debug = atoi(s);
    if (const char* s = getenv("B200REC_K1_TMA")) c.tma = atoi(s);
    if (const char* s = getenv("B200REC_K1_MINB")) c.minb = atoi(s);
    if (c.ctas_per_sm < 1 || c.ctas_per_sm > 16) c.ctas_per_sm = 8;
    if (c.unroll != 8 && c.unroll != 13 && c.unroll != 26) c.unroll = 13;
    return c;
  }();
  return cfg;
}

template <int TPR>
struct FwdGeom {
  static constexpr int kThreads = 128;
  static constexpr int kSamples = kThreads / TPR;  // samples per tile (32 at D=16)
};

// Persistent CTAs: each loops over tiles of kSamples samples (static stride).  While tile t is
// processed, the ids/dense of tile t+gridDim.x stream into the other shared-memory buffer with
// cp.async, so the id round trip is off the critical path.  Per tile and lane: all row loads and
// first-order lookups of a batch of kFieldUnroll fields are issued (predicated PTX, no branches)
// before the first one is consumed.
template <int VEC, int TPR, int kFieldUnroll, bool CACHE, int MINB = 4>
__global__ void __launch_bounds__(FwdGeom<TPR>::kThreads, MINB)
embed_fm_fwd_kernel(const float* __restrict__ W, const float* __restrict__ W1,
                    const int64_t* __restrict__ ids, const float* __restrict__ dense,
                    const float* __restrict__ dense_w, const float* __restrict__ dense_w1,
                    float* __restrict__ feat, float* __restrict__ y1, float* __restrict__ y2,
                    float* __restrict__ S, int64_t B, int F, int Dn, int D, int64_t V,
                    int64_t pad, int64_t ldw, int64_t ldw1, int dbg) {
  // dbg (env B200REC_K1_DEBUG, measurement only): bit 0 = skip the feat stores, bit 1 = skip the
  // table loads.  0 in production.
  constexpr int kThreads = FwdGeom<TPR>::kThreads;
  constexpr int SPB = FwdGeom<TPR>::kSamples;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const size_t ids_elems = (size_t)SPB * F;
  const size_t dense_elems = (size_t)SPB * Dn;
  const size_t buf_bytes = (ids_elems * 8 + dense_elems * 4 + 15) / 16 * 16;

  const int64_t ntiles = (B + SPB - 1) / SPB;
  const int s = threadIdx.x / TPR;
  const int r = threadIdx.x % TPR;
  const bool lane_ok = r * VEC < D;
  const int N = F + Dn;

  auto stage = [&](int64_t tile, int buf) {
    int64_t* s_ids = reinterpret_cast<int64_t*>(smem_raw + (size_t)buf * buf_bytes);
    float* s_dense = reinterpret_cast<float*>(s_ids + ids_elems);
    const int64_t b0 = tile * SPB;
    const int nb = (int)min((int64_t)SPB, B - b0);
    for (int i = threadIdx.x; i < nb * F; i += kThreads) cp_async_8(s_ids + i, ids + b0 * F + i);
    for (int i = threadIdx.x; i < nb * Dn; i += kThreads)
      cp_async_4(s_dense + i, dense + b0 * Dn + i);
  };

  int64_t tile = blockIdx.x;
  if (tile < ntiles) stage(tile, 0);
  cp_async_commit();
  for (int it = 0; tile < ntiles; tile += gridDim.x, ++it) {
    const int64_t next = tile + gridDim.x;
    if (next < ntiles) stage(next, (it + 1) & 1);
    cp_async_commit();
    cp_async_wait<1>();  // everything but the newest group (the next tile) has landed
    __syncthreads();

    const int64_t* s_ids = reinterpret_cast<const int64_t*>(smem_raw + (size_t)(it & 1) * buf_bytes);
    const float* s_dense = reinterpret_cast<const float*>(s_ids + ids_elems);
    const int64_t b0 = tile * SPB;
    const int nb = (int)min((int64_t)SPB, B - b0);
    const bool sample_ok = s < nb;
    const int64_t b = b0 + s;

    Vec<VEC> Ssum = vzero<VEC>();
    Vec<VEC> Q = vzero<VEC>();
    float first = 0.f;

    if (sample_ok) {
      const int64_t* my_ids = s_ids + (size_t)s * F;
      float* feat_row = feat + (size_t)b * N * D + r * VEC;
      for (int f0 = 0; f0 < F; f0 += kFieldUnroll) {
        Vec<VEC> e[kFieldUnroll];
        float w1v[kFieldUnroll];
        // phase 1: issue every load of the batch before anything consumes one
#pragma unroll
        for (int j = 0; j < kFieldUnroll; ++j) {
          const int f = f0 + j;
          const int64_t id = (f < F) ? my_ids[f] : pad;
          const bool in_range = (uint64_t)id < (uint64_t)V;
          const bool live = (f < F) && in_range && id != pad && !(dbg & 2);
          const size_t row = live ? (size_t)id : 0;
          e[j] = ld_row_pred<VEC, CACHE>(W + row * ldw + r * VEC, live && lane_ok);
          w1v[j] = ld_row_pred<1, true>(W1 + row * ldw1, live && ((f & (TPR - 1)) == r)).v[0];
          if ((f < F) && !in_range && r == 0) atomicAdd(&g_oob_count, 1ull);
        }
        // phase 2: consume
#pragma unroll
        for (int j = 0; j < kFieldUnroll; ++j) {
          const int f = f0 + j;
          if (f < F) {
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
              Ssum.v[k] += e[j].v[k];
              Q.v[k] = fmaf(e[j].v[k], e[j].v[k], Q.v[k]);
            }
            if (lane_ok && !(dbg & 1)) st_stream<VEC>(feat_row + (size_t)f * D, e[j]);
          }
        }
#pragma unroll
        for (int j = 0; j < kFieldUnroll; ++j) first += w1v[j];
      }
      const float* my_dense = s_dense + (size_t)s * Dn;
      for (int j = 0; j < Dn; ++j) {
        const float x = my_dense[j];
        Vec<VEC> e = vzero<VEC>();
        if (lane_ok) {
          const Vec<VEC> w = ld_cached<VEC>(dense_w + (size_t)j * D + r * VEC);
#pragma unroll
          for (int k = 0; k < VEC; ++k) e.v[k] = x * w.v[k];
          if (!(dbg & 1)) st_stream<VEC>(feat_row + (size_t)(F + j) * D, e);
        }
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
          Ssum.v[k] += e.v[k];
          Q.v[k] = fmaf(e.v[k], e.v[k], Q.v[k]);
        }
        if ((j & (TPR - 1)) == r) first = fmaf(x, __ldg(dense_w1 + j), first);
      }
    }

    float t = 0.f;
#pragma unroll
    for (int k = 0; k < VEC; ++k) t += Ssum.v[k] * Ssum.v[k] - Q.v[k];
    t = group_sum<TPR>(t);
    first = group_sum<TPR>(first);
    if (sample_ok) {
      if (r == 0) {
        y1[b] = first;
        y2[b] = 0.5f * t;
      }
      if (S != nullptr && lane_ok) st_plain<VEC>(S + (size_t)b * D + r * VEC, Ssum);
    }
    __syncthreads();  // buffer (it&1) is free for the prefetch issued two iterations later
  }
  cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// K1, warp-scheduled variant: the same per-sample arithmetic, but every WARP runs its own
// double-buffered pipeline over groups of 32/TPR samples and takes its next group from a global
// atomic counter.  Compared with the CTA-tiled kernel above there is no __syncthreads (the four
// warps of a CTA no longer wait for the slowest one twice per tile), no static tile-to-CTA map
// (2048 tiles over 1184 CTAs leaves a 1-vs-2 tile imbalance), and the id round trip of a warp's
// FIRST group is the only one that is exposed.  sched[0] = next group, sched[1] = warps that have
// finished; the last warp to finish resets both, so the buffer needs no memset between launches
// (one launch at a time per scheduler buffer).
__device__ unsigned int g_k1_sched[2] = {0u, 0u};

template <int VEC, int TPR, int kFieldUnroll, bool CACHE>
__global__ void __launch_bounds__(128, 4)
embed_fm_fwd_warp_kernel(const float* __restrict__ W, const float* __restrict__ W1,
                         const int64_t* __restrict__ ids, const float* __restrict__ dense,
                         const float* __restrict__ dense_w, const float* __restrict__ dense_w1,
                         float* __restrict__ feat, float* __restrict__ y1, float* __restrict__ y2,
                         float* __restrict__ S, int64_t B, int F, int Dn, int D, int64_t V,
                         int64_t pad, int64_t ldw, int64_t ldw1, int dbg) {
  constexpr int SPW = 32 / TPR;                      // samples per warp-group (8 at D=16)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const size_t ids_elems = (size_t)SPW * F;
  const size_t dense_elems = (size_t)SPW * Dn;
  const size_t buf_bytes = (ids_elems * 8 + dense_elems * 4 + 15) / 16 * 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* my_smem = smem_raw + (size_t)warp * 2 * buf_bytes;
  const unsigned ngroups = (unsigned)((B + SPW - 1) / SPW);
  const int s = lane / TPR;
  const int r = lane % TPR;
  const bool lane_ok = r * VEC < D;
  const int N = F + Dn;

  auto grab = [&]() -> unsigned {
    unsigned g = 0;
    if (lane == 0) g = atomicAdd(&g_k1_sched[0], 1u);
    return __shfl_sync(0xffffffffu, g, 0);
  };
  auto stage = [&](unsigned g, int buf) {
    int64_t* s_ids = reinterpret_cast<int64_t*>(my_smem + (size_t)buf * buf_bytes);
    float* s_dense = reinterpret_cast<float*>(s_ids + ids_elems);
    const int64_t b0 = (int64_t)g * SPW;
    const int nb = (int)min((int64_t)SPW, B - b0);
    for (int i = lane; i < nb * F; i += 32) cp_async_8(s_ids + i, ids + b0 * F + i);
    for (int i = lane; i < nb * Dn; i += 32) cp_async_4(s_dense + i, dense + b0 * Dn + i);
  };

  unsigned g = grab();
  if (g < ngroups) stage(g, 0);
  cp_async_commit();
  unsigned gn = grab();
  for (int it = 0; g < ngroups; ++it) {
    if (gn < ngroups) stage(gn, (it + 1) & 1);
    cp_async_commit();
    const unsigned gnn = grab();   // consumed one iteration later: its latency hides behind this group
    cp_async_wait<1>();
    __syncwarp();

    const int64_t* s_ids = reinterpret_cast<const int64_t*>(my_smem + (size_t)(it & 1) * buf_bytes);
    const float* s_dense = reinterpret_cast<const float*>(s_ids + ids_elems);
    const int64_t b0 = (int64_t)g * SPW;
    const int nb = (int)min((int64_t)SPW, B - b0);
    const bool sample_ok = s < nb;
    const int64_t b = b0 + s;

    Vec<VEC> Ssum = vzero<VEC>();
    Vec<VEC> Q = vzero<VEC>();
    float first = 0.f;
    if (sample_ok) {
      const int64_t* my_ids = s_ids + (size_t)s * F;
      float* feat_row = feat + (size_t)b * N * D + r * VEC;
      for (int f0 = 0; f0 < F; f0 += kFieldUnroll) {
        Vec<VEC> e[kFieldUnroll];
        float w1v[kFieldUnroll];
#pragma unroll
        for (int j = 0; j < kFieldUnroll; ++j) {
          const int f = f0 + j;
          const int64_t id = (f < F) ? my_ids[f] : pad;
          const bool in_range = (uint64_t)id < (uint64_t)V;
          const bool live = (f < F) && in_range && id != pad && !(dbg & 2);
          const size_t row = live ? (size_t)id : 0;
          e[j] = ld_row_pred<VEC, CACHE>(W + row * ldw + r * VEC, live && lane_ok);
          w1v[j] = ld_row_pred<1, true>(W1 + row * ldw1, live && ((f & (TPR - 1)) == r)).v[0];
          if ((f < F) && !in_range && r == 0) atomicAdd(&g_oob_count, 1ull);
        }
#pragma unroll
        for (int j = 0; j < kFieldUnroll; ++j) {
          const int f = f0 + j;
          if (f < F) {
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
              Ssum.v[k] += e[j].v[k];
              Q.v[k] = fmaf(e[j].v[k], e[j].v[k], Q.v[k]);
            }
            if (lane_ok && !(dbg & 1)) st_stream<VEC>(feat_row + (size_t)f * D, e[j]);
          }
        }
#pragma unroll
        for (int j = 0; j < kFieldUnroll; ++j) first += w1v[j];
      }
      const float* my_dense = s_dense + (size_t)s * Dn;
      for (int j = 0; j < Dn; ++j) {
        const float x = my_dense[j];
        Vec<VEC> e = vzero<VEC>();
        if (lane_ok) {
          const Vec<VEC> w = ld_cached<VEC>(dense_w + (size_t)j * D + r * VEC);
#pragma unroll
          for (int k = 0; k < VEC; ++k) e.v[k] = x * w.v[k];
          if (!(dbg & 1)) st_stream<VEC>(feat_row + (size_t)(F + j) * D, e);
        }
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
          Ssum.v[k] += e.v[k];
          Q.v[k] = fmaf(e.v[k], e.v[k], Q.v[k]);
        }
        if ((j & (TPR - 1)) == r) first = fmaf(x, __ldg(dense_w1 + j), first);
      }
    }
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < VEC; ++k) t += Ssum.v[k] * Ssum.v[k] - Q.v[k];
    t = group_sum<TPR>(t);
    first = group_sum<TPR>(first);
    if (sample_ok) {
      if (r == 0) {
        y1[b] = first;
        y2[b] = 0.5f * t;
      }
      if (S != nullptr && lane_ok) st_plain<VEC>(S + (size_t)b * D + r * VEC, Ssum);
    }
    __syncwarp();   // every lane is done with buffer (it&1) before the next iteration refills it
    g = gn;
    gn = gnn;
  }
  cp_async_wait<0>();
  if (lane == 0) {
    const unsigned total_warps = gridDim.x * (blockDim.x >> 5);
    const unsigned done = atomicAdd(&g_k1_sched[1], 1u);
    if (done == total_warps - 1) {   // nobody else will touch the scheduler in this launch
      g_k1_sched[0] = 0u;
      g_k1_sched[1] = 0u;
      __threadfence();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K1, shared-memory-staged variant (D % 4 == 0): the tile of `feat` is ASSEMBLED IN SHARED MEMORY in
// exactly its global layout ([sample][field][D], contiguous over the tile) and leaves the SM as ONE
// bulk asynchronous copy (cp.async.bulk / TMA, SASS UBLKCP) — no per-thread global stores at all.
//   * the random table rows are fetched with cp.async 16 B (LDGSTS) straight into their place in
//     the tile: all F rows of a lane are in flight at once at zero register cost (the register
//     variant above can afford 13);
//   * first-order scalars land in a [sample][field] side tile the same way; padding / out-of-range
//     ids store zeros;
//   * the dense-feature rows are computed into the tile while the gathers fly;
//   * after cp.async.wait_group + barrier each lane re-reads its 39 chunks (LDS.128, conflict-free)
//     for S, Q, y1, y2; fence.proxy.async; one thread issues the bulk store and the CTA only
//     waits for it (wait_group.read) right before it overwrites the tile for its next iteration —
//     the second CTA of the SM gathers meanwhile.
// ids/dense of the next tile are prefetched with cp.async into a second small buffer.
// STATUS: correct (same tests as the register variant) but it was slower where it was measured
// (on the GPU the project first targeted; not re-measured on the H100): one 32-sample tile is
// 80 KB, so only 2 CTAs = 8 warps fit per SM and the per-field issue chain (LDS id -> compare ->
// address -> LDGSTS) is not hidden.  Opt-in with B200REC_K1_TMA=1; the register variant is default.
constexpr int kTmaThreads = 128;

__device__ __forceinline__ void cp_async_16_cg(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(
                   (unsigned)__cvta_generic_to_shared(smem)),
               "l"(gmem)
               : "memory");
}
__device__ __forceinline__ void bulk_store_smem_to_global(void* gdst, const void* ssrc,
                                                          unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"((unsigned)__cvta_generic_to_shared(ssrc)), "r"(bytes)
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

struct K1TmaSmem {
  size_t feat_bytes, w1_bytes, ids_bytes, dense_bytes, total;
  __host__ __device__ K1TmaSmem(int spb, int F, int Dn, int D) {
    feat_bytes = ((size_t)spb * (F + Dn) * D * 4 + 127) / 128 * 128;
    w1_bytes = ((size_t)spb * F * 4 + 15) / 16 * 16;
    ids_bytes = ((size_t)spb * F * 8 + 15) / 16 * 16;
    dense_bytes = ((size_t)spb * Dn * 4 + 15) / 16 * 16;
    total = feat_bytes + w1_bytes + 2 * (ids_bytes + dense_bytes);
  }
};

template <int TPR>
__global__ void __launch_bounds__(kTmaThreads)
embed_fm_fwd_tma_kernel(const float* __restrict__ W, const float* __restrict__ W1,
                        const int64_t* __restrict__ ids, const float* __restrict__ dense,
                        const float* __restrict__ dense_w, const float* __restrict__ dense_w1,
                        float* __restrict__ feat, float* __restrict__ y1, float* __restrict__ y2,
                        float* __restrict__ S, int64_t B, int F, int Dn, int D, int64_t V,
                        int64_t pad, int64_t ldw, int64_t ldw1) {
  constexpr int VEC = 4;
  constexpr int SPB = kTmaThreads / TPR;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const K1TmaSmem L(SPB, F, Dn, D);
  float* feat_tile = reinterpret_cast<float*>(smem_raw);
  float* w1_tile = reinterpret_cast<float*>(smem_raw + L.feat_bytes);
  unsigned char* stage0 = smem_raw + L.feat_bytes + L.w1_bytes;
  const size_t stage_bytes = L.ids_bytes + L.dense_bytes;

  const int N = F + Dn;
  const int row_floats = N * D;  // one sample of feat
  const int64_t ntiles = (B + SPB - 1) / SPB;
  const int s = threadIdx.x / TPR;
  const int r = threadIdx.x % TPR;
  const bool lane_ok = r * VEC < D;

  auto stage = [&](int64_t tile, int buf) {
    int64_t* s_ids = reinterpret_cast<int64_t*>(stage0 + (size_t)buf * stage_bytes);
    float* s_dense = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(s_ids) + L.ids_bytes);
    const int64_t b0 = tile * SPB;
    const int nb = (int)min((int64_t)SPB, B - b0);
    for (int i = threadIdx.x; i < nb * F; i += kTmaThreads) cp_async_8(s_ids + i, ids + b0 * F + i);
    for (int i = threadIdx.x; i < nb * Dn; i += kTmaThreads)
      cp_async_4(s_dense + i, dense + b0 * Dn + i);
  };

  int64_t tile = blockIdx.x;
  if (tile < ntiles) stage(tile, 0);
  cp_async_commit();
  for (int it = 0; tile < ntiles; tile += gridDim.x, ++it) {
    const int64_t next = tile + gridDim.x;
    if (next < ntiles) stage(next, (it + 1) & 1);
    cp_async_commit();
    cp_async_wait<1>();
    // the previous iteration's bulk store must have finished READING the tile before we refill it
    if (threadIdx.x == 0) bulk_store_wait_read();
    __syncthreads();

    const int64_t* s_ids = reinterpret_cast<const int64_t*>(stage0 + (size_t)(it & 1) * stage_bytes);
    const float* s_dense = reinterpret_cast<const float*>(
        reinterpret_cast<const unsigned char*>(s_ids) + L.ids_bytes);
    const int64_t b0 = tile * SPB;
    const int nb = (int)min((int64_t)SPB, B - b0);
    const bool sample_ok = s < nb;
    const int64_t b = b0 + s;
    float* my_feat = feat_tile + (size_t)s * row_floats + r * VEC;
    float* my_w1 = w1_tile + (size_t)s * F;

    // ---- issue: every row of this lane, straight into its place in the tile -------------------
    if (sample_ok) {
      const int64_t* my_ids = s_ids + (size_t)s * F;
      for (int f = 0; f < F; ++f) {
        const int64_t id = my_ids[f];
        const bool in_range = (uint64_t)id < (uint64_t)V;
        const bool live = in_range && id != pad;
        if (lane_ok) {
          if (live)
            cp_async_16_cg(my_feat + (size_t)f * D, W + (size_t)id * ldw + r * VEC);
          else
            *reinterpret_cast<float4*>(my_feat + (size_t)f * D) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if ((f & (TPR - 1)) == r) {
          if (live)
            cp_async_4(my_w1 + f, W1 + (size_t)id * ldw1);
          else
            my_w1[f] = 0.f;
        }
        if (!in_range && r == 0) atomicAdd(&g_oob_count, 1ull);
      }
    }
    cp_async_commit();
    // ---- dense-feature rows while the gathers are in flight -----------------------------------
    float first = 0.f;
    if (sample_ok) {
      const float* my_dense = s_dense + (size_t)s * Dn;
      for (int j = 0; j < Dn; ++j) {
        const float x = my_dense[j];
        if (lane_ok) {
          const float4 w = __ldg(reinterpret_cast<const float4*>(dense_w + (size_t)j * D) + r);
          *reinterpret_cast<float4*>(my_feat + (size_t)(F + j) * D) =
              make_float4(x * w.x, x * w.y, x * w.z, x * w.w);
        }
        if ((j & (TPR - 1)) == r) first = fmaf(x, __ldg(dense_w1 + j), first);
      }
    }
    cp_async_wait<0>();
    __syncthreads();

    // ---- consume from the tile ----------------------------------------------------------------
    float4 Ssum = make_float4(0.f, 0.f, 0.f, 0.f), Q = Ssum;
    if (sample_ok) {
      if (lane_ok) {
#pragma unroll 13
        for (int n = 0; n < N; ++n) {
          const float4 e = *reinterpret_cast<const float4*>(my_feat + (size_t)n * D);
          Ssum.x += e.x; Ssum.y += e.y; Ssum.z += e.z; Ssum.w += e.w;
          Q.x = fmaf(e.x, e.x, Q.x); Q.y = fmaf(e.y, e.y, Q.y);
          Q.z = fmaf(e.z, e.z, Q.z); Q.w = fmaf(e.w, e.w, Q.w);
        }
      }
      for (int f = r; f < F; f += TPR) first += my_w1[f];
    }
    float t = (Ssum.x * Ssum.x - Q.x) + (Ssum.y * Ssum.y - Q.y) + (Ssum.z * Ssum.z - Q.z) +
              (Ssum.w * Ssum.w - Q.w);
    t = group_sum<TPR>(t);
    first = group_sum<TPR>(first);
    if (sample_ok) {
      if (r == 0) {
        y1[b] = first;
        y2[b] = 0.5f * t;
      }
      if (S != nullptr && lane_ok)
        *reinterpret_cast<float4*>(S + (size_t)b * D + r * VEC) = Ssum;
    }
    // ---- the whole tile leaves as one bulk copy -----------------------------------------------
    fence_proxy_async_smem();  // generic-proxy writes (st.shared, cp.async) -> visible to the TMA
    __syncthreads();
    if (threadIdx.x == 0)
      bulk_store_smem_to_global(feat + (size_t)b0 * row_floats, feat_tile,
                                (unsigned)((size_t)nb * row_floats * sizeof(float)));
  }
  if (threadIdx.x == 0) bulk_store_wait_read();
  cp_async_wait<0>();
}

struct K1Args {
  const float* W; const float* W1; const int64_t* ids; const float* dense; const float* dense_w;
  const float* dense_w1; float* feat; float* y1; float* y2; float* S;
  int64_t B; int F, Dn, D; int64_t V, pad, ldw, ldw1;
};

template <int TPR>
static int k1_tma_launch(const K1Args& a, cudaStream_t st) {
  constexpr int SPB = kTmaThreads / TPR;
  const K1TmaSmem L(SPB, a.F, a.Dn, a.D);
  auto kern = embed_fm_fwd_tma_kernel<TPR>;
  B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.total));
  const int64_t ntiles = (a.B + SPB - 1) / SPB;
  const int per_sm = (int)max((size_t)1, min((size_t)8, (size_t)(220 * 1024) / L.total));
  const int64_t grid = min(ntiles, (int64_t)sm_count() * per_sm);
  kern<<<(unsigned)grid, kTmaThreads, L.total, st>>>(a.W, a.W1, a.ids, a.dense, a.dense_w, a.dense_w1,
                                                    a.feat, a.y1, a.y2, a.S, a.B, a.F, a.Dn, a.D, a.V,
                                                    a.pad, a.ldw, a.ldw1);
  return B200REC_OK;
}

template <int VEC, int TPR, int U>
static int k1_warp_launch(const K1Args& a, int ctas_per_sm, cudaStream_t st) {
  constexpr int SPW = 32 / TPR;
  const size_t buf = ((size_t)SPW * a.F * sizeof(int64_t) + (size_t)SPW * a.Dn * sizeof(float) + 15) /
                     16 * 16;
  const size_t smem = 4 * 2 * buf;     // 4 warps x 2 buffers
  auto kern = embed_fm_fwd_warp_kernel<VEC, TPR, U, false>;
  if (smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t ngroups = (a.B + SPW - 1) / SPW;
  const int64_t grid = min((ngroups + 3) / 4, (int64_t)sm_count() * ctas_per_sm);
  kern<<<(unsigned)grid, 128, smem, st>>>(a.W, a.W1, a.ids, a.dense, a.dense_w, a.dense_w1, a.feat,
                                          a.y1, a.y2, a.S, a.B, a.F, a.Dn, a.D, a.V, a.pad, a.ldw,
                                          a.ldw1, k1_config().debug);
  return B200REC_OK;
}

template <int VEC, int TPR, int U, bool C, int MINB = 4>
static int k1_launch(const K1Args& a, int64_t grid, size_t smem, cudaStream_t st) {
  auto kern = embed_fm_fwd_kernel<VEC, TPR, U, C, MINB>;
  if (smem > 48 * 1024)
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)grid, FwdGeom<TPR>::kThreads, smem, st>>>(
      a.W, a.W1, a.ids, a.dense, a.dense_w, a.dense_w1, a.feat, a.y1, a.y2, a.S, a.B, a.F, a.Dn, a.D,
      a.V, a.pad, a.ldw, a.ldw1, k1_config().debug);
  return B200REC_OK;
}

static int launch_embed_fm_fwd(const float* W, const float* W1, const int64_t* ids,
                               const float* dense, const float* dense_w, const float* dense_w1,
                               float* feat, float* y1, float* y2, float* S, int64_t B, int F,
                               int Dn, int D, int64_t V, int64_t pad, int64_t ldw, int64_t ldw1,
                               cudaStream_t st) {
  RowShape rs;
  B200_REQUIRE(pick_row_shape(D, &rs), "embed_fm_fwd: unsupported D=%d", D);
  B200_REQUIRE(ldw >= D && ldw1 >= 1 && ldw % rs.vec == 0,
               "embed_fm_fwd: bad row strides ldw=%lld ldw1=%lld", (long long)ldw, (long long)ldw1);
  if (rs.vec == 4)
    B200_REQUIRE(aligned16(W) && aligned16(feat) && aligned16(dense_w) && (!S || aligned16(S)),
                 "embed_fm_fwd: W/feat/dense_w/S must be 16-byte aligned for D%%4==0");
  if (rs.vec == 2)
    B200_REQUIRE(aligned8(W) && aligned8(feat) && aligned8(dense_w) && (!S || aligned8(S)),
                 "embed_fm_fwd: W/feat/dense_w/S must be 8-byte aligned for D%%2==0");
  if (B == 0) return B200REC_OK;
  B200_DISPATCH_ROW_SHAPE(rs, {
    constexpr int SPB = FwdGeom<TPR>::kSamples;
    const size_t buf = ((size_t)SPB * F * sizeof(int64_t) + (size_t)SPB * Dn * sizeof(float) + 15) /
                       16 * 16;
    const size_t smem = 2 * buf;
    B200_REQUIRE(smem <= 200 * 1024, "embed_fm_fwd: F=%d Dn=%d tile does not fit shared memory", F,
                 Dn);
    const K1Config cfg = k1_config();
    // same 128-byte line as the row (fused slot layout)?  then let the row load allocate in L1
    const bool same_line = (W1 >= W && W1 < W + ldw && ldw1 == ldw);
    const bool cache = cfg.cache_rows < 0 ? same_line : cfg.cache_rows != 0;
    const int64_t ntiles = (B + SPB - 1) / SPB;
    const int64_t grid = min(ntiles, (int64_t)sm_count() * cfg.ctas_per_sm);
    K1Args a{W, W1, ids, dense, dense_w, dense_w1, feat, y1, y2, S, B, F, Dn, D, V, pad, ldw, ldw1};
    int rc;
    if (VEC == 4 && cfg.tma && cfg.debug == 0 && aligned16(dense_w) && (ldw % 4 == 0) &&
        K1TmaSmem(kTmaThreads / TPR, F, Dn, D).total <= 110 * 1024)
      rc = k1_tma_launch<TPR>(a, st);
    else if (cfg.warp_sched && cfg.unroll == 8)
      rc = k1_warp_launch<VEC, TPR, 8>(a, cfg.ctas_per_sm, st);
    else if (cfg.warp_sched)
      rc = k1_warp_launch<VEC, TPR, 13>(a, cfg.ctas_per_sm, st);
    else if (cfg.minb == 5 && cfg.unroll == 13)
      rc = k1_launch<VEC, TPR, 13, false, 5>(a, grid, smem, st);
    else if (cfg.minb == 6 && cfg.unroll == 13)
      rc = k1_launch<VEC, TPR, 13, false, 6>(a, grid, smem, st);
    else if (cfg.minb == 6 && cfg.unroll == 8)
      rc = k1_launch<VEC, TPR, 8, false, 6>(a, grid, smem, st);
    else if (cfg.minb == 8 && cfg.unroll == 8)
      rc = k1_launch<VEC, TPR, 8, false, 8>(a, grid, smem, st);
    else if (cfg.unroll == 8)
      rc = cache ? k1_launch<VEC, TPR, 8, true>(a, grid, smem, st)
                 : k1_launch<VEC, TPR, 8, false>(a, grid, smem, st);
    else if (cfg.unroll == 26)
      rc = cache ? k1_launch<VEC, TPR, 26, true>(a, grid, smem, st)
                 : k1_launch<VEC, TPR, 26, false>(a, grid, smem, st);
    else
      rc = cache ? k1_launch<VEC, TPR, 13, true>(a, grid, smem, st)
                 : k1_launch<VEC, TPR, 13, false>(a, grid, smem, st);
    if (rc != B200REC_OK) return rc;
  });
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

// ------------------------------------------------------------------------------------------
// K2a: sparse part of the backward.  One group of TPR lanes per DISTINCT id (segment of the
// sorted positions).  dfeat is never materialised for the sparse fields:
//   dfeat[p] = gy2[b]*(S[b]-feat[p]) + dfeat_dnn[p]      (net.py:123-137 differentiated)
// and summed in the fixed (stable-sort) order of the segment => deterministic.
constexpr int kBwdThreads = 256;

struct FmRowContrib {
  const float* feat;
  const float* S;
  const float* dfeat_dnn;  // may be null
  const float* gy1;
  const float* gy2;
  int F, N, D;
  template <int VEC>
  __device__ __forceinline__ void add(int p, int r, bool lane_ok, Vec<VEC>& acc,
                                      float& acc1) const {
    const int b = p / F;
    const int f = p - b * F;
    const float g2 = __ldg(gy2 + b);
    acc1 += __ldg(gy1 + b);
    if (lane_ok) {
      const size_t off = ((size_t)b * N + f) * D + r * VEC;
      const Vec<VEC> fe = ld_row<VEC>(feat + off);
      const Vec<VEC> sv = ld_cached<VEC>(S + (size_t)b * D + r * VEC);
      Vec<VEC> dd = vzero<VEC>();
      if (dfeat_dnn != nullptr) dd = ld_row<VEC>(dfeat_dnn + off);
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc.v[k] += fmaf(g2, sv.v[k] - fe.v[k], dd.v[k]);
    }
  }
};

// K2b: dense-feature part: ddense_w[j,:] = sum_b dense[b,j]*dfeat[b,F+j,:],
// ddense_w1[j] = sum_b gy1[b]*dense[b,j].  Persistent CTAs accumulate in registers over a
// strided set of samples, reduce once, and write one partial per CTA; a second tiny kernel adds
// the partials in a fixed order (deterministic, no float atomics).
constexpr int kDenseChunk = 8;  // dense features held in registers at once (Dn=13 -> 2 passes)

template <int VEC, int TPR>
__global__ void __launch_bounds__(kBwdThreads, 2)
embed_fm_bwd_dense_kernel(const float* __restrict__ feat, const float* __restrict__ S,
                          const float* __restrict__ dfeat_dnn, const float* __restrict__ gy1,
                          const float* __restrict__ gy2, const float* __restrict__ dense,
                          float* __restrict__ partials /*[grid, Dn*D + Dn]*/, int64_t B, int F,
                          int Dn, int D) {
  constexpr int SPB = kBwdThreads / TPR;
  constexpr int kWarps = kBwdThreads / 32;
  __shared__ float s_red[kWarps][32 * VEC];
  __shared__ float s_red1[kWarps];
  const int s = threadIdx.x / TPR;
  const int r = threadIdx.x % TPR;
  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const bool lane_ok = r * VEC < D;
  const int N = F + Dn;
  float* my_partial = partials + (size_t)blockIdx.x * ((size_t)Dn * D + Dn);

  for (int j0 = 0; j0 < Dn; j0 += kDenseChunk) {
    Vec<VEC> acc[kDenseChunk];
    float acc1[kDenseChunk];
#pragma unroll
    for (int j = 0; j < kDenseChunk; ++j) {
      acc[j] = vzero<VEC>();
      acc1[j] = 0.f;
    }
    for (int64_t b = (int64_t)blockIdx.x * SPB + s; b < B; b += (int64_t)gridDim.x * SPB) {
      const float g2 = __ldg(gy2 + b);
      const float g1 = __ldg(gy1 + b);
      Vec<VEC> sv = vzero<VEC>();
      if (lane_ok) sv = ld_cached<VEC>(S + (size_t)b * D + r * VEC);
#pragma unroll
      for (int j = 0; j < kDenseChunk; ++j) {
        if (j0 + j < Dn) {
          const float x = __ldg(dense + (size_t)b * Dn + j0 + j);
          if (lane_ok) {
            const size_t off = ((size_t)b * N + F + j0 + j) * D + r * VEC;
            const Vec<VEC> fe = ld_row<VEC>(feat + off);
            Vec<VEC> dd = vzero<VEC>();
            if (dfeat_dnn != nullptr) dd = ld_row<VEC>(dfeat_dnn + off);
#pragma unroll
            for (int k = 0; k < VEC; ++k)
              acc[j].v[k] = fmaf(x, fmaf(g2, sv.v[k] - fe.v[k], dd.v[k]), acc[j].v[k]);
          }
          if (r == 0) acc1[j] = fmaf(g1, x, acc1[j]);
        }
      }
    }
    // reduce over the samples of the CTA, one dense feature at a time
#pragma unroll
    for (int j = 0; j < kDenseChunk; ++j) {
      if (j0 + j < Dn) {  // uniform across the CTA
        Vec<VEC> a = acc[j];
        float a1 = acc1[j];
#pragma unroll
        for (int o = TPR; o < 32; o <<= 1) {
#pragma unroll
          for (int k = 0; k < VEC; ++k) a.v[k] += __shfl_xor_sync(0xffffffffu, a.v[k], o);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        if (lane < TPR) {
#pragma unroll
          for (int k = 0; k < VEC; ++k) s_red[warp][lane * VEC + k] = a.v[k];
        }
        if (lane == 0) s_red1[warp] = a1;
        __syncthreads();
        if (threadIdx.x < D) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < kWarps; ++w) t += s_red[w][threadIdx.x];
          my_partial[(size_t)(j0 + j) * D + threadIdx.x] = t;
        }
        if (threadIdx.x == 0) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < kWarps; ++w) t += s_red1[w];
          my_partial[(size_t)Dn * D + j0 + j] = t;
        }
        __syncthreads();
      }
    }
  }
}

// out[k] = sum_g partials[g][k] (deterministic: fixed strided order + fixed shared-memory tree).
// `len` is small (<= a few thousand) but G can be hundreds: 32 columns x 8 g-lanes per block so
// the G-long sums are not one serial dependent chain per column.
constexpr int kRedCols = 32;
constexpr int kRedLanes = 32;   // r1 had 8: 74 dependent L2 round trips per thread = 30 us/launch
__global__ void __launch_bounds__(kRedCols * kRedLanes)
reduce_partials_kernel(const float* __restrict__ partials, int G, int len,
                       float* __restrict__ out0, int len0, float* __restrict__ out1) {
  __shared__ float s[kRedLanes][kRedCols + 1];
  const int cx = threadIdx.x % kRedCols, gy = threadIdx.x / kRedCols;
  const int k = blockIdx.x * kRedCols + cx;
  float t = 0.f;
  if (k < len) {
    int g = gy;
    for (; g + 3 * kRedLanes < G; g += 4 * kRedLanes) {   // four loads in flight, fixed add order
      const float a0 = partials[(size_t)g * len + k];
      const float a1 = partials[(size_t)(g + kRedLanes) * len + k];
      const float a2 = partials[(size_t)(g + 2 * kRedLanes) * len + k];
      const float a3 = partials[(size_t)(g + 3 * kRedLanes) * len + k];
      t += a0; t += a1; t += a2; t += a3;
    }
    for (; g < G; g += kRedLanes) t += partials[(size_t)g * len + k];
  }
  s[gy][cx] = t;
  __syncthreads();
  if (gy == 0 && k < len) {
    float r = 0.f;
#pragma unroll
    for (int y = 0; y < kRedLanes; ++y) r += s[y][cx];
    if (k < len0)
      out0[k] = r;
    else
      out1[k - len0] = r;
  }
}
static inline unsigned reduce_partials_grid(int len) { return (unsigned)((len + kRedCols - 1) / kRedCols); }
constexpr int kRedThreads = kRedCols * kRedLanes;

static int bwd_dense_grid() { return sm_count() * 2; }

static int launch_embed_fm_bwd(const float* feat, const float* S, const float* dfeat_dnn,
                               const float* gy1, const float* gy2, const float* dense,
                               const int32_t* seg_offsets, const int32_t* sorted_pos,
                               const int32_t* num_unique, float* dW_rows, float* dW1_rows,
                               SegOut so, float* ddense_w, float* ddense_w1, int64_t B, int F,
                               int Dn, int D, void* ws, size_t ws_bytes, cudaStream_t st) {
  RowShape rs;
  B200_REQUIRE(pick_row_shape(D, &rs), "embed_fm_bwd: unsupported D=%d", D);
  const int align = rs.vec * 4;
  auto ok = [&](const void* p) { return (reinterpret_cast<uintptr_t>(p) % align) == 0; };
  B200_REQUIRE(ok(feat) && ok(S) && ok(dfeat_dnn) && ok(dW_rows),
               "embed_fm_bwd: feat/S/dfeat_dnn/dW_rows must be %d-byte aligned", align);
  B200_REQUIRE(so.ld_rows >= D && so.ld_rows % rs.vec == 0 && so.ld_rows1 >= 1 && so.zero_pad >= 0,
               "embed_fm_bwd: bad output strides");
  B200_REQUIRE(B * F < (int64_t)INT32_MAX, "embed_fm_bwd: B*F must fit int32");
  const int G = bwd_dense_grid();
  const size_t dense_bytes = align_up((size_t)G * ((size_t)Dn * D + Dn) * sizeof(float), 256);
  const size_t need = dense_bytes + seg_workspace_bytes(B * F, D);
  if (ws_bytes < need) {
    set_error("embed_fm_bwd: workspace %zu < %zu bytes", ws_bytes, need);
    return B200REC_ERR_WORKSPACE;
  }
  if (B == 0) {
    if (Dn > 0) {
      B200_CUDA(cudaMemsetAsync(ddense_w, 0, (size_t)Dn * D * sizeof(float), st));
      B200_CUDA(cudaMemsetAsync(ddense_w1, 0, (size_t)Dn * sizeof(float), st));
    }
    return B200REC_OK;
  }
  const int N = F + Dn;
  int rc = B200REC_OK;
  B200_DISPATCH_ROW_SHAPE(rs, {
    const int64_t n = B * F;
    if (n > 0) {
      FmRowContrib contrib{feat, S, dfeat_dnn, gy1, gy2, F, N, D};
      rc = launch_seg_reduce<VEC, TPR, FmRowContrib>(seg_offsets, sorted_pos, num_unique, contrib,
                                                     dW_rows, dW1_rows, so, n, D,
                                                     static_cast<unsigned char*>(ws) + dense_bytes,
                                                     st);
    }
    if (rc == B200REC_OK && Dn > 0) {
      embed_fm_bwd_dense_kernel<VEC, TPR><<<G, kBwdThreads, 0, st>>>(
          feat, S, dfeat_dnn, gy1, gy2, dense, static_cast<float*>(ws), B, F, Dn, D);
    }
  });
  if (rc != B200REC_OK) return rc;
  B200_LAUNCH_CHECK();
  if (Dn > 0) {
    const int len = Dn * D + Dn;
    reduce_partials_kernel<<<reduce_partials_grid(len), kRedThreads, 0, st>>>(
        static_cast<const float*>(ws), G, len, ddense_w, Dn * D, ddense_w1);
    B200_LAUNCH_CHECK();
  }
  return B200REC_OK;
}

}  // namespace b200rec
