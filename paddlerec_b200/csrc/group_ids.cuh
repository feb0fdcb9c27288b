// Grouping of lookup positions by id: the "merge" half of Paddle's SelectedRows gradient
// (lookup_table_v2_grad + merge_add), done once per step and shared by every consumer
// (segmented reduce, fused FM backward, row-wise optimizers).
//
//   keys  = id (or a sentinel V for padding / out-of-range ids, which sorts last)
//   stable LSD radix sort of (key, position) over only the ceil(log2(V+1)) significant bits
//   head flags -> inclusive scan -> segment table
//
// The radix sort and the scan are CUB device primitives (shipped with the CUDA toolkit and
// compiled here for sm_90a); the key building and segment-table kernels are ours.
#pragma once

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace b200rec {

template <typename KeyT>
__global__ void build_keys_kernel(const int64_t* __restrict__ ids, int64_t n, int64_t V,
                                  int64_t pad, KeyT* __restrict__ keys,
                                  int32_t* __restrict__ pos) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t id = ids[i];
  const bool in_range = (uint64_t)id < (uint64_t)V;
  if (!in_range) atomicAdd(&g_oob_count, 1ull);
  keys[i] = (in_range && id != pad) ? (KeyT)id : (KeyT)V;
  pos[i] = (int32_t)i;
}

template <typename KeyT>
__global__ void head_flags_kernel(const KeyT* __restrict__ keys, int64_t n,
                                  int32_t* __restrict__ flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

template <typename KeyT>
__global__ void segment_table_kernel(const KeyT* __restrict__ keys,
                                     const int32_t* __restrict__ segidx /*inclusive scan*/,
                                     int64_t n, int64_t V, int64_t* __restrict__ unique_ids,
                                     int32_t* __restrict__ seg_offsets,
                                     int32_t* __restrict__ num_unique) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const KeyT k = keys[i];
  const bool head = (i == 0) || (k != keys[i - 1]);
  const bool sentinel = (k == (KeyT)V);
  const int32_t u = segidx[i] - 1;
  if (head) {
    seg_offsets[u] = (int32_t)i;  // for the sentinel run this is seg_offsets[U] = #kept
    if (!sentinel) unique_ids[u] = (int64_t)k;
    if (sentinel) {
      num_unique[0] = u;
      num_unique[1] = (int32_t)i;
    }
  }
  if (i == n - 1 && !sentinel) {
    seg_offsets[u + 1] = (int32_t)n;
    num_unique[0] = u + 1;
    num_unique[1] = (int32_t)n;
  }
}

static inline int key_bits(int64_t V) {
  int bits = 1;
  while (bits < 64 && ((uint64_t)V >> bits) != 0) ++bits;
  return bits;  // V itself (the sentinel) is representable
}

struct GroupPlan {
  bool wide;  // 64-bit keys
  size_t key_bytes, off_keys_in, off_keys_out, off_pos_in, off_flags, off_cub, cub_bytes, total;
};

template <typename KeyT>
static cudaError_t cub_sort_bytes(int64_t n, int bits, size_t* bytes) {
  return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const KeyT*)nullptr, (KeyT*)nullptr,
                                         (const int32_t*)nullptr, (int32_t*)nullptr, (int)n, 0,
                                         bits);
}

static int make_group_plan(int64_t n, int64_t V, GroupPlan* p) {
  B200_REQUIRE(n >= 0 && n < (int64_t)INT32_MAX, "group_ids: n=%lld must fit int32", (long long)n);
  B200_REQUIRE(V > 0, "group_ids: V must be positive");
  p->wide = V >= (int64_t)0xffffffffll;
  p->key_bytes = p->wide ? 8 : 4;
  const int bits = key_bits(V);
  size_t sort_bytes = 0, scan_bytes = 0;
  if (p->wide)
    B200_CUDA(cub_sort_bytes<uint64_t>(n, bits, &sort_bytes));
  else
    B200_CUDA(cub_sort_bytes<uint32_t>(n, bits, &sort_bytes));
  B200_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int32_t*)nullptr,
                                          (int32_t*)nullptr, (int)n));
  p->cub_bytes = sort_bytes > scan_bytes ? sort_bytes : scan_bytes;
  size_t off = 0;
  p->off_keys_in = off;  off += align_up((size_t)n * p->key_bytes, 256);
  p->off_keys_out = off; off += align_up((size_t)n * p->key_bytes, 256);
  p->off_pos_in = off;   off += align_up((size_t)n * 4, 256);
  p->off_flags = off;    off += align_up((size_t)n * 4, 256);
  p->off_cub = off;      off += align_up(p->cub_bytes, 256);
  p->total = off + 256;
  return B200REC_OK;
}

template <typename KeyT>
static int run_group_ids(const GroupPlan& p, const int64_t* ids, int64_t n, int64_t V, int64_t pad,
                         int64_t* unique_ids, int32_t* seg_offsets, int32_t* sorted_pos,
                         int32_t* num_unique, unsigned char* ws, cudaStream_t st) {
  KeyT* keys_in = reinterpret_cast<KeyT*>(ws + p.off_keys_in);
  KeyT* keys_out = reinterpret_cast<KeyT*>(ws + p.off_keys_out);
  int32_t* pos_in = reinterpret_cast<int32_t*>(ws + p.off_pos_in);
  int32_t* flags = reinterpret_cast<int32_t*>(ws + p.off_flags);
  void* cub_ws = ws + p.off_cub;
  size_t cub_bytes = p.cub_bytes;
  const unsigned grid = (unsigned)((n + 255) / 256);
  build_keys_kernel<KeyT><<<grid, 256, 0, st>>>(ids, n, V, pad, keys_in, pos_in);
  B200_LAUNCH_CHECK();
  B200_CUDA(cub::DeviceRadixSort::SortPairs(cub_ws, cub_bytes, keys_in, keys_out, pos_in,
                                            sorted_pos, (int)n, 0, key_bits(V), st));
  head_flags_kernel<KeyT><<<grid, 256, 0, st>>>(keys_out, n, flags);
  B200_LAUNCH_CHECK();
  cub_bytes = p.cub_bytes;
  B200_CUDA(cub::DeviceScan::InclusiveSum(cub_ws, cub_bytes, flags, flags, (int)n, st));
  segment_table_kernel<KeyT><<<grid, 256, 0, st>>>(keys_out, flags, n, V, unique_ids, seg_offsets,
                                                   num_unique);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int launch_group_ids(const int64_t* ids, int64_t n, int64_t V, int64_t pad,
                            int64_t* unique_ids, int32_t* seg_offsets, int32_t* sorted_pos,
                            int32_t* num_unique, void* ws, size_t ws_bytes, cudaStream_t st) {
  GroupPlan p;
  int rc = make_group_plan(n, V, &p);
  if (rc != B200REC_OK) return rc;
  if (n == 0) {
    B200_CUDA(cudaMemsetAsync(num_unique, 0, 2 * sizeof(int32_t), st));
    B200_CUDA(cudaMemsetAsync(seg_offsets, 0, sizeof(int32_t), st));
    return B200REC_OK;
  }
  if (ws_bytes < p.total) {
    set_error("group_ids: workspace %zu < %zu bytes", ws_bytes, p.total);
    return B200REC_ERR_WORKSPACE;
  }
  // 256-byte align the workspace base
  unsigned char* base = static_cast<unsigned char*>(ws);
  unsigned char* aligned = reinterpret_cast<unsigned char*>(align_up((size_t)(uintptr_t)base, 256));
  if (p.wide)
    return run_group_ids<uint64_t>(p, ids, n, V, pad, unique_ids, seg_offsets, sorted_pos,
                                   num_unique, aligned, st);
  return run_group_ids<uint32_t>(p, ids, n, V, pad, unique_ids, seg_offsets, sorted_pos, num_unique,
                                 aligned, st);
}

}  // namespace b200rec
