// libb200rec.so — the single translation unit behind include/b200rec.h.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -shared -Xcompiler -fPIC
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
// kernels (order matters: embed_fm.cuh defines reduce_partials_kernel used by cross.cuh)
#include "embed_fm.cuh"
#include "group_ids.cuh"
#include "gather_scatter.cuh"
#include "cross.cuh"
#include "shard.cuh"
#include "tower.cuh"
#include "tc_gemm.cuh"
#include "ctr_head.cuh"
#include "cvm.cuh"
#include "hash_keys.cuh"
#include "dot_interact.cuh"
#include "din_attn.cuh"
#include "ffm.cuh"
#include "fat_ffm.cuh"
#include "gate_embed.cuh"
#include "esmm.cuh"

namespace b200rec {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 132;
  }
  return cached;
}

}  // namespace b200rec

using namespace b200rec;

#define ST(s) static_cast<cudaStream_t>(s)
#define NOT_NULL(p) B200_REQUIRE((p) != nullptr, "%s: argument `%s` is NULL", __func__, #p)

extern "C" {

int b200rec_abi_version(void) { return B200REC_ABI_VERSION; }

const char* b200rec_last_error(void) { return g_err; }

int b200rec_oob_count(uint64_t* count_host, int reset, void* stream) {
  NOT_NULL(count_host);
  unsigned long long v = 0;
  B200_CUDA(cudaStreamSynchronize(ST(stream)));
  B200_CUDA(cudaMemcpyFromSymbol(&v, g_oob_count, sizeof(v)));
  *count_host = (uint64_t)v;
  if (reset) {
    v = 0;
    B200_CUDA(cudaMemcpyToSymbol(g_oob_count, &v, sizeof(v)));
  }
  return B200REC_OK;
}

int b200rec_embed_fm_fwd(const float* W, int64_t ldw, const float* W1, int64_t ldw1,
                         const int64_t* ids, const float* dense, const float* dense_w,
                         const float* dense_w1, float* feat, float* y1, float* y2, float* S,
                         int64_t B, int F, int Dn, int D, int64_t V, int64_t padding_idx,
                         void* stream) {
  B200_REQUIRE(B >= 0 && F >= 0 && Dn >= 0 && D > 0 && V > 0, "embed_fm_fwd: bad sizes");
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(W1); NOT_NULL(feat); NOT_NULL(y1); NOT_NULL(y2);
    if (F > 0) NOT_NULL(ids);
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); NOT_NULL(dense_w1); }
  }
  return launch_embed_fm_fwd(W, W1, ids, dense, dense_w, dense_w1, feat, y1, y2, S, B, F, Dn, D, V,
                             padding_idx, ldw, ldw1, ST(stream));
}

int b200rec_group_ids_workspace_bytes(int64_t n, int64_t V, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  GroupPlan p;
  int rc = make_group_plan(n, V, &p);
  if (rc != B200REC_OK) return rc;
  *bytes_host = p.total;
  return B200REC_OK;
}

int b200rec_group_ids(const int64_t* ids, int64_t n, int64_t V, int64_t padding_idx,
                      int64_t* unique_ids, int32_t* seg_offsets, int32_t* sorted_pos,
                      int32_t* num_unique, void* workspace, size_t workspace_bytes, void* stream) {
  NOT_NULL(seg_offsets); NOT_NULL(num_unique);
  if (n > 0) { NOT_NULL(ids); NOT_NULL(unique_ids); NOT_NULL(sorted_pos); NOT_NULL(workspace); }
  return launch_group_ids(ids, n, V, padding_idx, unique_ids, seg_offsets, sorted_pos, num_unique,
                          workspace, workspace_bytes, ST(stream));
}

int b200rec_embed_fm_bwd_workspace_bytes(int64_t B, int F, int Dn, int D, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  *bytes_host = align_up((size_t)bwd_dense_grid() * ((size_t)Dn * D + Dn) * sizeof(float), 256) +
                seg_workspace_bytes(B * F, D);
  return B200REC_OK;
}

int b200rec_embed_fm_bwd(const float* feat, const float* S, const float* dfeat_dnn,
                         const float* gy1, const float* gy2, const float* dense,
                         const int32_t* seg_offsets, const int32_t* sorted_pos,
                         const int32_t* num_unique, float* dW_rows, int64_t ld_dw,
                         float* dW1_rows, int64_t ld_dw1, int dw1_zero_pad, float* ddense_w,
                         float* ddense_w1, int64_t B, int F, int Dn, int D, void* workspace,
                         size_t workspace_bytes, void* stream) {
  B200_REQUIRE(B >= 0 && F >= 0 && Dn >= 0 && D > 0, "embed_fm_bwd: bad sizes");
  if (B > 0) {
    NOT_NULL(feat); NOT_NULL(S); NOT_NULL(gy1); NOT_NULL(gy2);
    if (F > 0) {
      NOT_NULL(seg_offsets); NOT_NULL(sorted_pos); NOT_NULL(num_unique);
      NOT_NULL(dW_rows); NOT_NULL(dW1_rows);
    }
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(ddense_w); NOT_NULL(ddense_w1); }
    NOT_NULL(workspace);
  }
  return launch_embed_fm_bwd(feat, S, dfeat_dnn, gy1, gy2, dense, seg_offsets, sorted_pos,
                             num_unique, dW_rows, dW1_rows, SegOut{ld_dw, ld_dw1, dw1_zero_pad},
                             ddense_w, ddense_w1, B, F, Dn, D, workspace, workspace_bytes,
                             ST(stream));
}

int b200rec_ffm_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                    const float* dense_w, const float* dense_w1, const float* bias, float* y1,
                    float* y2, int64_t B, int F, int Dn, int D, int64_t V, int64_t padding_idx,
                    void* stream) {
  B200_REQUIRE(B >= 0 && V > 0, "ffm_fwd: bad sizes");
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(y1); NOT_NULL(y2);
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); NOT_NULL(dense_w1); }
  }
  return launch_ffm_fwd(W, ldw, ids, dense, dense_w, dense_w1, bias, y1, y2, B, F, Dn, D, V,
                        padding_idx, ST(stream));
}

int b200rec_ffm_bwd_workspace_bytes(int64_t B, int F, int Dn, int D, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  B200_REQUIRE(B >= 0 && F >= 1 && Dn >= 0 && D >= 1 && F + Dn <= kFfmMaxFields,
               "ffm_bwd_workspace_bytes: bad sizes");
  *bytes_host = FfmBwdWs(B, F, Dn, D).total;
  return B200REC_OK;
}

int b200rec_ffm_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                    const float* dense_w, const float* gy1, const float* gy2,
                    const int32_t* seg_offsets, const int32_t* sorted_pos,
                    const int32_t* num_unique, float* dW_rows, int64_t ld_dw, float* ddense_w,
                    float* ddense_w1, float* dbias, int64_t B, int F, int Dn, int D, int64_t V,
                    int64_t padding_idx, void* workspace, size_t workspace_bytes, void* stream) {
  B200_REQUIRE(B >= 0 && V > 0, "ffm_bwd: bad sizes");
  if (Dn > 0) { NOT_NULL(ddense_w); NOT_NULL(ddense_w1); }
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(gy1); NOT_NULL(gy2); NOT_NULL(seg_offsets);
    NOT_NULL(sorted_pos); NOT_NULL(num_unique); NOT_NULL(dW_rows); NOT_NULL(workspace);
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); }
  }
  return launch_ffm_bwd(W, ldw, ids, dense, dense_w, gy1, gy2, seg_offsets, sorted_pos,
                        num_unique, dW_rows, ld_dw, ddense_w, ddense_w1, dbias, B, F, Dn, D, V,
                        padding_idx, workspace, workspace_bytes, ST(stream));
}

int b200rec_fat_ffm_pool_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                             const float* dense_w, float* pool, int64_t B, int F, int Dn, int D,
                             int64_t V, int64_t padding_idx, void* stream) {
  B200_REQUIRE(B >= 0 && V > 0, "fat_ffm_pool_fwd: bad sizes");
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(pool);
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); }
  }
  return launch_fat_ffm_pool(W, ldw, ids, dense, dense_w, pool, B, F, Dn, D, V, padding_idx,
                             ST(stream));
}

int b200rec_fat_ffm_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                        const float* dense_w, const float* attn, const float* bias, float* y1,
                        float* h, int64_t B, int F, int Dn, int D, int64_t V, int64_t padding_idx,
                        void* stream) {
  B200_REQUIRE(B >= 0 && V > 0, "fat_ffm_fwd: bad sizes");
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(attn); NOT_NULL(y1);
    if (fat_pairs(F, Dn) * D > 0) NOT_NULL(h);     // one field: no pairs, h has no elements
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); }
  }
  const FatSampleArgs a{W, ldw, ids, dense, dense_w, attn, bias, nullptr, nullptr, y1, h,
                        B, F, Dn, D, V, padding_idx};
  return launch_fat_sample<false>("fat_ffm_fwd", a, ST(stream));
}

int b200rec_fat_ffm_bwd_attn(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                             const float* dense_w, const float* attn, const float* gy1,
                             const float* dh, float* dattn, int64_t B, int F, int Dn, int D,
                             int64_t V, int64_t padding_idx, void* stream) {
  B200_REQUIRE(B >= 0 && V > 0, "fat_ffm_bwd_attn: bad sizes");
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(attn); NOT_NULL(gy1); NOT_NULL(dattn);
    if (fat_pairs(F, Dn) * D > 0) NOT_NULL(dh);
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); }
  }
  const FatSampleArgs a{W, ldw, ids, dense, dense_w, attn, nullptr, gy1, dh, nullptr, dattn,
                        B, F, Dn, D, V, padding_idx};
  return launch_fat_sample<true>("fat_ffm_bwd_attn", a, ST(stream));
}

int b200rec_fat_ffm_bwd_workspace_bytes(int64_t B, int F, int Dn, int D, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  B200_REQUIRE(B >= 0 && F >= 1 && Dn >= 0 && D >= 1 && F + Dn <= kFfmMaxFields,
               "fat_ffm_bwd_workspace_bytes: bad sizes");
  *bytes_host = FfmBwdWs(B, F, Dn, D).total;
  return B200REC_OK;
}

int b200rec_fat_ffm_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                        const float* dense_w, const float* attn, const float* gy1, const float* dh,
                        const float* dpool, const int32_t* seg_offsets, const int32_t* sorted_pos,
                        const int32_t* num_unique, float* dW_rows, int64_t ld_dw, float* ddense_w,
                        float* dbias, int64_t B, int F, int Dn, int D, int64_t V,
                        int64_t padding_idx, void* workspace, size_t workspace_bytes,
                        void* stream) {
  B200_REQUIRE(B >= 0 && V > 0, "fat_ffm_bwd: bad sizes");
  if (Dn > 0) NOT_NULL(ddense_w);
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(attn); NOT_NULL(gy1); NOT_NULL(dpool);
    NOT_NULL(seg_offsets); NOT_NULL(sorted_pos); NOT_NULL(num_unique); NOT_NULL(dW_rows);
    NOT_NULL(workspace);
    if (fat_pairs(F, Dn) * D > 0) NOT_NULL(dh);
    if (Dn > 0) { NOT_NULL(dense); NOT_NULL(dense_w); }
  }
  const int NF = F + Dn, R = NF * D;
  const FatBwd a{W, ldw, ids, dense, dense_w, gy1, dh, attn, dpool, F, Dn, D, R,
                 ffm_staged_cols(R), NF, V, padding_idx};
  return launch_fat_ffm_bwd(a, seg_offsets, sorted_pos, num_unique, dW_rows, ld_dw, ddense_w,
                            dbias, B, workspace, workspace_bytes, ST(stream));
}

int b200rec_gather(const float* W, int64_t ldw, const int64_t* ids, float* out, int64_t n, int D,
                   int64_t V, int64_t padding_idx, void* stream) {
  B200_REQUIRE(n >= 0 && D > 0 && V > 0, "gather: bad sizes");
  if (n > 0) { NOT_NULL(W); NOT_NULL(ids); NOT_NULL(out); }
  return launch_gather(W, ids, out, n, D, V, padding_idx, ldw, ST(stream));
}

int b200rec_gate_embed_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* gate_w,
                           const float* dense, float* out, int64_t ld_out, int64_t B, int F, int D,
                           int Dn, int64_t V, void* stream) {
  if (B > 0) {
    NOT_NULL(W); NOT_NULL(ids); NOT_NULL(gate_w); NOT_NULL(out);
    if (Dn > 0) NOT_NULL(dense);
  }
  return launch_gate_embed_fwd(W, ldw, ids, gate_w, dense, out, ld_out, B, F, D, Dn, V, ST(stream));
}

int b200rec_gate_embed_bwd_workspace_bytes(int64_t B, int F, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  B200_REQUIRE(B >= 0 && F > 0 && F <= kGateEmbedMaxFields, "gate_embed_bwd_workspace_bytes: bad sizes");
  *bytes_host = gate_embed_bwd_ws_bytes(B, F) + 16;
  return B200REC_OK;
}

int b200rec_gate_embed_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* gate_w,
                           const float* dout, int64_t ld_out, float* drow, float* dgate_w,
                           int64_t B, int F, int D, int64_t V, void* workspace,
                           size_t workspace_bytes, void* stream) {
  NOT_NULL(dgate_w);
  if (B > 0) { NOT_NULL(W); NOT_NULL(ids); NOT_NULL(gate_w); NOT_NULL(dout); NOT_NULL(drow); }
  return launch_gate_embed_bwd(W, ldw, ids, gate_w, dout, ld_out, drow, dgate_w, B, F, D, V,
                               workspace, workspace_bytes, ST(stream));
}

int b200rec_segment_reduce_workspace_bytes(int64_t n, int D, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  B200_REQUIRE(n >= 0, "segment_reduce: bad sizes");
  *bytes_host = seg_workspace_bytes(n, D);
  return B200REC_OK;
}

int b200rec_gather_pool_sum(const float* W, int64_t ldw, const int64_t* keys,
                            const int64_t* offsets, float* out, int32_t* bag_of_pos, int64_t n_bags,
                            int D, int64_t V, int64_t padding_idx, void* stream) {
  B200_REQUIRE(n_bags >= 0 && D > 0 && V > 0, "gather_pool_sum: bad sizes");
  if (n_bags > 0) { NOT_NULL(W); NOT_NULL(offsets); NOT_NULL(out); }
  return launch_gather_pool(W, keys, offsets, out, bag_of_pos, n_bags, D, V, padding_idx, ldw,
                            ST(stream));
}

int b200rec_segment_reduce(const float* dOut, const int32_t* row_of_pos,
                           const int32_t* seg_offsets, const int32_t* sorted_pos,
                           const int32_t* num_unique, float* rows, int64_t n, int D,
                           void* workspace, size_t workspace_bytes, void* stream) {
  B200_REQUIRE(n >= 0 && D > 0, "segment_reduce: bad sizes");
  if (n > 0) { NOT_NULL(dOut); NOT_NULL(seg_offsets); NOT_NULL(sorted_pos); NOT_NULL(num_unique); NOT_NULL(rows); NOT_NULL(workspace); }
  return launch_segment_reduce(dOut, row_of_pos, seg_offsets, sorted_pos, num_unique, rows, n, D,
                               workspace,
                               workspace_bytes, ST(stream));
}

int b200rec_rows_to_dense(const int64_t* unique_ids, const float* rows, int64_t ld_rows,
                          const int32_t* num_unique, float* dW, int64_t ld_dw, int64_t n, int D,
                          int64_t V, void* stream) {
  B200_REQUIRE(n >= 0 && D > 0 && V > 0, "rows_to_dense: bad sizes");
  if (n > 0) { NOT_NULL(unique_ids); NOT_NULL(rows); NOT_NULL(num_unique); NOT_NULL(dW); }
  RowsToDenseOp op{dW};
  return launch_row_update("rows_to_dense", unique_ids, rows, num_unique, n, D, V, ld_dw, ld_rows,
                           op, dW, nullptr, nullptr, ST(stream));
}

int b200rec_sparse_sgd(float* W, int64_t ldw, const int64_t* unique_ids, const float* rows,
                       int64_t ld_rows, const int32_t* num_unique, int64_t n, int D, int64_t V,
                       double lr, void* stream) {
  B200_REQUIRE(n >= 0 && D > 0 && V > 0, "sparse_sgd: bad sizes");
  if (n > 0) { NOT_NULL(W); NOT_NULL(unique_ids); NOT_NULL(rows); NOT_NULL(num_unique); }
  SgdOp op{W, (float)lr};
  return launch_row_update("sparse_sgd", unique_ids, rows, num_unique, n, D, V, ldw, ld_rows, op,
                           W, nullptr, nullptr, ST(stream));
}

int b200rec_sparse_adam(float* W, float* m, float* v, int64_t ldw, const int64_t* unique_ids,
                        const float* rows, int64_t ld_rows, const int32_t* num_unique, int64_t n,
                        int D, int64_t V,
                        double lr, double beta1, double beta2, double eps, double beta1_pow_t,
                        double beta2_pow_t, void* stream) {
  B200_REQUIRE(n >= 0 && D > 0 && V > 0, "sparse_adam: bad sizes");
  if (n > 0) { NOT_NULL(W); NOT_NULL(m); NOT_NULL(v); NOT_NULL(unique_ids); NOT_NULL(rows); NOT_NULL(num_unique); }
  const double c2 = sqrt(1.0 - beta2_pow_t);
  AdamOp op{W, m, v, (float)beta1, (float)beta2, (float)(1.0 - beta1), (float)(1.0 - beta2),
            (float)(lr * c2 / (1.0 - beta1_pow_t)), (float)(eps * c2)};
  return launch_row_update("sparse_adam", unique_ids, rows, num_unique, n, D, V, ldw, ld_rows, op,
                           W, m, v, ST(stream));
}

int b200rec_sparse_adagrad(float* W, float* g2sum, int64_t ldw, const int64_t* unique_ids,
                           const float* rows, int64_t ld_rows, const int32_t* num_unique, int64_t n,
                           int D, int64_t V, double lr,
                           double initial_g2sum, double lo, double hi, void* stream) {
  B200_REQUIRE(n >= 0 && D > 0 && V > 0, "sparse_adagrad: bad sizes");
  if (n > 0) { NOT_NULL(W); NOT_NULL(g2sum); NOT_NULL(unique_ids); NOT_NULL(rows); NOT_NULL(num_unique); }
  return launch_adagrad(W, g2sum, unique_ids, rows, num_unique, n, D, V, ldw, ld_rows, (float)lr,
                        (float)initial_g2sum, (float)lo, (float)hi,
                        ST(stream));
}

int b200rec_cross_v2_fwd(const float* x0, const float* xl, const float* xw, const float* bias,
                         float* out, int64_t B, int C, void* stream) {
  if (B > 0) { NOT_NULL(x0); NOT_NULL(xl); NOT_NULL(xw); NOT_NULL(bias); NOT_NULL(out); }
  return launch_cross_v2_fwd(x0, xl, xw, bias, out, B, C, ST(stream));
}

int b200rec_cross_bwd_workspace_bytes(int64_t B, int C, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  *bytes_host = (size_t)cross_row_slices(B) * (size_t)C * sizeof(float) + 16;
  return B200REC_OK;
}

int b200rec_cross_v2_bwd(const float* dout, const float* x0, const float* xw, const float* bias,
                         float* dxw, float* dx0, float* dbias, int64_t B, int C,
                         void* workspace, size_t workspace_bytes, void* stream) {
  NOT_NULL(dbias);
  if (B > 0) { NOT_NULL(dout); NOT_NULL(x0); NOT_NULL(xw); NOT_NULL(bias); NOT_NULL(dxw); NOT_NULL(dx0); NOT_NULL(workspace); }
  return launch_cross_v2_bwd(dout, x0, xw, bias, dxw, dx0, dbias, B, C, workspace,
                             workspace_bytes, ST(stream));
}

int b200rec_shard_bucketize_workspace_bytes(int64_t n, int world, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  ShardPlan p;
  int rc = make_shard_plan(n, world, &p);
  if (rc != B200REC_OK) return rc;
  *bytes_host = p.total;
  return B200REC_OK;
}

int b200rec_shard_bucketize(const int64_t* ids, int64_t n, int world, int64_t V, int64_t* send_ids,
                            int64_t* perm, int32_t* inv_perm, int64_t* counts, void* workspace,
                            size_t workspace_bytes, void* stream) {
  NOT_NULL(counts);
  if (n > 0) { NOT_NULL(ids); NOT_NULL(send_ids); NOT_NULL(perm); NOT_NULL(inv_perm); NOT_NULL(workspace); }
  return launch_shard_bucketize(ids, n, world, V, send_ids, perm, inv_perm, counts, workspace,
                                workspace_bytes, ST(stream));
}

int b200rec_shard_gather_push(const float* shard, int64_t ldw, int D, int64_t V_loc,
                              int64_t local_pad, const int64_t* recv_ids, const int64_t* seg_dev,
                              const int64_t* dst_dev, const uint64_t* peer_ptrs_host, int64_t ld_dst,
                              int world, int64_t n, void* stream) {
  NOT_NULL(peer_ptrs_host);
  if (n > 0) { NOT_NULL(shard); NOT_NULL(recv_ids); NOT_NULL(seg_dev); NOT_NULL(dst_dev); }
  return launch_shard_gather_push(shard, ldw, D, V_loc, local_pad, recv_ids, seg_dev, dst_dev,
                                  peer_ptrs_host, ld_dst, world, n, ST(stream));
}

int b200rec_shard_fm_grads_push(const float* feat, const float* S, const float* dfeat_dnn,
                                const float* gy1, const float* gy2, const int32_t* inv_perm,
                                const int64_t* seg_dev, const int64_t* dst_dev,
                                const uint64_t* peer_ptrs_host, int64_t ld_dst, int world, int64_t B,
                                int F, int Dn, int D, int G, void* stream) {
  NOT_NULL(peer_ptrs_host);
  if (B > 0 && F > 0) {
    NOT_NULL(feat); NOT_NULL(S); NOT_NULL(gy1); NOT_NULL(gy2); NOT_NULL(inv_perm); NOT_NULL(seg_dev);
    NOT_NULL(dst_dev);
  }
  return launch_shard_fm_grads_push(feat, S, dfeat_dnn, gy1, gy2, inv_perm, seg_dev, dst_dev,
                                    peer_ptrs_host, ld_dst, world, B, F, Dn, D, G, ST(stream));
}

int b200rec_shard_push_rows(const float* rows, int64_t ld, int D, const int64_t* seg_dev,
                            const int64_t* dst_dev, const uint64_t* peer_ptrs_host, int64_t ld_dst,
                            int world, int64_t n, void* stream) {
  NOT_NULL(peer_ptrs_host);
  if (n > 0) { NOT_NULL(rows); NOT_NULL(seg_dev); NOT_NULL(dst_dev); }
  return launch_shard_push_rows(rows, ld, D, seg_dev, dst_dev, peer_ptrs_host, ld_dst, world, n,
                                ST(stream));
}

int b200rec_tower_split(const float* x, const float* bias, int relu, void* out_bf16, int64_t M,
                        int K, void* stream) {
  if (M > 0) { NOT_NULL(x); NOT_NULL(out_bf16); }
  return launch_tower_split(x, K, bias, relu, out_bf16, K, M, K, 0, ST(stream));
}

int b200rec_tower_bwd_workspace_bytes(int64_t M, int N, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  *bytes_host = (size_t)tower_row_slices(M) * (size_t)N * sizeof(float) + 16;
  return B200REC_OK;
}

int b200rec_tower_relu_bwd_split(const float* dy, const void* act_bf16, void* dz_bf16,
                                 float* dbias, int64_t M, int N, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  NOT_NULL(dbias);
  if (M > 0) { NOT_NULL(dy); NOT_NULL(dz_bf16); NOT_NULL(workspace); }
  return launch_tower_relu_bwd_split(dy, act_bf16, N, dz_bf16, N, dbias, M, N, workspace,
                                     workspace_bytes, ST(stream));
}

/* ---- wgmma tower GEMMs (csrc/tc_gemm.cuh) ------------------------------------------------ */
int b200rec_tc_split(const float* x, int64_t ldx, const float* bias, int relu, void* planes,
                     int64_t ldp, int64_t M, int K, int ones_col, void* stream) {
  if (M > 0) { NOT_NULL(x); NOT_NULL(planes); }
  return launch_tower_split(x, ldx, bias, relu, planes, ldp, M, K, ones_col, ST(stream));
}

int b200rec_tc_split_bwd(const float* dy, const void* mask_planes, int64_t ld_mask, void* g_planes,
                         int64_t ldp, float* dbias, int64_t M, int N, void* workspace,
                         size_t workspace_bytes, void* stream) {
  NOT_NULL(dbias);
  if (M > 0) { NOT_NULL(dy); NOT_NULL(g_planes); NOT_NULL(workspace); }
  return launch_tower_relu_bwd_split(dy, mask_planes, ld_mask, g_planes, ldp, dbias, M, N,
                                     workspace, workspace_bytes, ST(stream));
}

int b200rec_tc_prep_weight(const float* W, int K, int N, void* w_planes, int64_t ldn,
                           void* wt_planes, int64_t ldk, void* stream) {
  B200_REQUIRE(K > 0 && N > 0, "tc_prep_weight: bad sizes");
  NOT_NULL(W);
  B200_REQUIRE(w_planes == nullptr || ldn >= N, "tc_prep_weight: ldn < N");
  B200_REQUIRE(wt_planes == nullptr || ldk >= K, "tc_prep_weight: ldk < K");
  dim3 grid((N + 31) / 32, (K + 31) / 32), block(32, 8);
  tc::tc_prep_weight_kernel<<<grid, block, 0, ST(stream)>>>(
      W, K, N, static_cast<__nv_bfloat16*>(w_planes), ldn, static_cast<__nv_bfloat16*>(wt_planes),
      ldk);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_tc_linear_fwd(const void* a_planes, int64_t lda, const void* wt_planes, int64_t ldk,
                          const float* bias, int relu, float* out_f32, int64_t ld_f32,
                          void* out_planes, int64_t ldp, int ones_col, int64_t M, int N, int K,
                          void* stream) {
  if (M > 0) { NOT_NULL(a_planes); NOT_NULL(wt_planes); }
  B200_REQUIRE(out_f32 != nullptr || out_planes != nullptr, "tc_linear_fwd: no output");
  B200_REQUIRE(out_f32 == nullptr || ld_f32 >= N, "tc_linear_fwd: ld_f32 < N");
  B200_REQUIRE(out_planes == nullptr || ldp >= N + (ones_col ? 1 : 0), "tc_linear_fwd: ldp < N");
  tc::Epilogue ep = {};
  ep.bias = bias; ep.relu = relu; ep.ones_col = ones_col;
  ep.out_f32 = out_f32; ep.ld_f32 = ld_f32;
  ep.out_planes = static_cast<__nv_bfloat16*>(out_planes); ep.ldp = ldp;
  return tc::launch_gemm_kmajor(a_planes, lda, wt_planes, ldk, M, N, K, ep, ST(stream));
}

int b200rec_tc_cross_fwd(const void* xl_planes, int64_t lda, const void* wt_planes, int64_t ldk,
                         const float* bias, const float* x0, const float* xl, int64_t ld_x,
                         float* u_f32, float* out_f32, int64_t ld_f32, void* out_planes,
                         int64_t ldp, int ones_col, int64_t M, int C, void* stream) {
  if (M > 0) { NOT_NULL(xl_planes); NOT_NULL(wt_planes); NOT_NULL(x0); NOT_NULL(xl); }
  B200_REQUIRE(out_f32 != nullptr || out_planes != nullptr, "tc_cross_fwd: no output");
  B200_REQUIRE(out_planes == nullptr || ldp >= C + (ones_col ? 1 : 0), "tc_cross_fwd: ldp < C");
  tc::Epilogue ep = {};
  ep.bias = bias;
  ep.ones_col = ones_col;
  ep.aux_f32 = u_f32; ep.ld_aux = ld_f32;
  ep.cross_x0 = x0; ep.cross_xl = xl; ep.ld_cross = ld_x;
  ep.out_f32 = out_f32; ep.ld_f32 = ld_f32;
  ep.out_planes = static_cast<__nv_bfloat16*>(out_planes); ep.ldp = ldp;
  return tc::launch_gemm_kmajor(xl_planes, lda, wt_planes, ldk, M, C, C, ep, ST(stream));
}

int b200rec_tc_gate_fwd(const void* y_planes, int64_t ldy, const void* gt_planes, int64_t ldk,
                        float* a_f32, float* out_f32, int64_t ld_f32, void* out_planes, int64_t ldp,
                        int ones_col, int64_t M, int N, void* stream) {
  if (M > 0) { NOT_NULL(y_planes); NOT_NULL(gt_planes); }
  B200_REQUIRE(out_f32 != nullptr || out_planes != nullptr, "tc_gate_fwd: no output");
  B200_REQUIRE(ldy >= N && ld_f32 >= N, "tc_gate_fwd: ldy or ld_f32 < N");
  B200_REQUIRE(out_planes == nullptr || ldp >= N + (ones_col ? 1 : 0), "tc_gate_fwd: ldp < N");
  tc::Epilogue ep = {};
  ep.ones_col = ones_col;
  ep.aux_f32 = a_f32; ep.ld_aux = ld_f32;
  ep.gate_y = static_cast<const __nv_bfloat16*>(y_planes); ep.ld_gate = ldy;
  ep.out_f32 = out_f32; ep.ld_f32 = ld_f32;
  ep.out_planes = static_cast<__nv_bfloat16*>(out_planes); ep.ldp = ldp;
  return tc::launch_gemm_kmajor(y_planes, ldy, gt_planes, ldk, M, N, N, ep, ST(stream));
}

int b200rec_tc_gate_bwd(const float* dz, const void* y_planes, int64_t ldy, const float* a,
                        void* g_planes, int64_t ldp, float* r, int64_t M, int N, void* stream) {
  if (M > 0) { NOT_NULL(dz); NOT_NULL(y_planes); NOT_NULL(a); NOT_NULL(g_planes); NOT_NULL(r); }
  return launch_tower_gate_bwd(dz, y_planes, ldy, a, g_planes, ldp, r, M, N, ST(stream));
}

int b200rec_tc_linear_bwd_workspace_bytes(int64_t M, int K, int N, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  B200_REQUIRE(M >= 0 && K > 0 && N > 0, "tc_linear_bwd_workspace_bytes: bad sizes");
  const size_t colsum = (size_t)((M + tc::kBM - 1) / tc::kBM) * (size_t)K * sizeof(float);
  const size_t dw = tc::plan_dw(M, K, N).ws_bytes;
  *bytes_host = (colsum > dw ? colsum : dw) + 256;
  return B200REC_OK;
}

int b200rec_tc_linear_bwd_dx(const void* g_planes, int64_t ldg, const void* w_planes, int64_t ldn,
                             const void* mask_planes, int64_t ld_mask, const float* addend,
                             float* dx_f32, int64_t ld_f32, void* dx_planes, int64_t ldp,
                             float* dbias_prev, int64_t M, int K, int N, void* workspace,
                             size_t workspace_bytes, void* stream) {
  if (M > 0) { NOT_NULL(g_planes); NOT_NULL(w_planes); }
  B200_REQUIRE(dx_f32 != nullptr || dx_planes != nullptr, "tc_linear_bwd_dx: no output");
  B200_REQUIRE(dx_f32 == nullptr || ld_f32 >= K, "tc_linear_bwd_dx: ld_f32 < K");
  B200_REQUIRE(dx_planes == nullptr || ldp >= K, "tc_linear_bwd_dx: ldp < K");
  tc::Epilogue ep = {};
  ep.out_f32 = dx_f32; ep.ld_f32 = ld_f32;
  ep.out_planes = static_cast<__nv_bfloat16*>(dx_planes); ep.ldp = ldp;
  ep.mask_src = static_cast<const __nv_bfloat16*>(mask_planes); ep.ld_mask = 2 * ld_mask;
  ep.addend = addend; ep.ld_add = K;
  const int tiles_m = (int)((M + tc::kBM - 1) / tc::kBM);
  if (dbias_prev != nullptr) {
    const size_t need = (size_t)tiles_m * K * sizeof(float);
    if (workspace_bytes < need || (M > 0 && workspace == nullptr)) {
      set_error("tc_linear_bwd_dx: workspace %zu < %zu bytes", workspace_bytes, need);
      return B200REC_ERR_WORKSPACE;
    }
    if (M == 0) {
      B200_CUDA(cudaMemsetAsync(dbias_prev, 0, (size_t)K * sizeof(float), ST(stream)));
      return B200REC_OK;
    }
    ep.colsum = static_cast<float*>(workspace);
  }
  // D[M,K] = G[M,N] . W[K,N]^T : the reduction runs over N, the output width is K
  const int rc = tc::launch_gemm_kmajor(g_planes, ldg, w_planes, ldn, M, K, N, ep, ST(stream));
  if (rc != B200REC_OK) return rc;
  if (dbias_prev != nullptr && M > 0) {
    dim3 block(32, 8);
    tc::tc_colsum_reduce_kernel<<<(K + 31) / 32, block, 0, ST(stream)>>>(ep.colsum, tiles_m, K,
                                                                         dbias_prev);
    B200_LAUNCH_CHECK();
  }
  return B200REC_OK;
}

int b200rec_tc_linear_bwd_dw(const void* a_planes, int64_t lda, const void* g_planes, int64_t ldg,
                             float* dW, int64_t M, int K, int N, void* workspace,
                             size_t workspace_bytes, void* stream) {
  NOT_NULL(dW);
  if (M > 0) { NOT_NULL(a_planes); NOT_NULL(g_planes); }
  return tc::launch_gemm_dw(a_planes, lda, g_planes, ldg, M, K, N, dW, workspace, workspace_bytes,
                            ST(stream));
}

int b200rec_tc_head_fwd(const void* a_planes, int64_t lda, int K, const float* w, const float* bias,
                        float* y, int64_t M, void* stream) {
  if (M > 0) { NOT_NULL(a_planes); NOT_NULL(w); NOT_NULL(y); }
  return launch_tower_head_fwd(a_planes, lda, K, w, bias, y, M, ST(stream));
}

int b200rec_tc_head_bwd_workspace_bytes(int K, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  *bytes_host = tower_head_bwd_ws_bytes(K) + 16;
  return B200REC_OK;
}

int b200rec_tc_head_bwd(const void* a_planes, int64_t lda, int K, const float* w, const float* dy,
                        void* g_planes, int64_t ldg, float* dW, float* db, int64_t M,
                        void* workspace, size_t workspace_bytes, void* stream) {
  NOT_NULL(dW); NOT_NULL(db);
  if (M > 0) { NOT_NULL(a_planes); NOT_NULL(w); NOT_NULL(dy); NOT_NULL(g_planes); NOT_NULL(workspace); }
  return launch_tower_head_bwd(a_planes, lda, K, w, dy, g_planes, ldg, dW, db, M, workspace,
                               workspace_bytes, ST(stream));
}

int b200rec_esmm_head_fwd(const float* h_ctr, const float* h_cvr, int K, const float* W_ctr,
                          const float* b_ctr, const float* W_cvr, const float* b_cvr, float* ctr_out,
                          float* ctr_one, float* cvr_out, float* cvr_one, float* ctcvr_prop,
                          float* ctcvr_one, int64_t B, void* stream) {
  if (B > 0) {
    NOT_NULL(h_ctr); NOT_NULL(h_cvr); NOT_NULL(W_ctr); NOT_NULL(b_ctr); NOT_NULL(W_cvr);
    NOT_NULL(b_cvr); NOT_NULL(ctr_out); NOT_NULL(ctr_one); NOT_NULL(cvr_out); NOT_NULL(cvr_one);
    NOT_NULL(ctcvr_prop); NOT_NULL(ctcvr_one);
  }
  return launch_esmm_head_fwd(h_ctr, h_cvr, K, W_ctr, b_ctr, W_cvr, b_cvr, ctr_out, ctr_one,
                              cvr_out, cvr_one, ctcvr_prop, ctcvr_one, B, ST(stream));
}

int b200rec_esmm_head_bwd_workspace_bytes(int64_t B, int K, size_t* bytes_host) {
  NOT_NULL(bytes_host);
  B200_REQUIRE(B >= 0 && esmm_k_ok(K), "esmm_head_bwd_workspace_bytes: K=%d must be a multiple of 4 "
               "in [4, %d]", K, kEsmmMaxK);
  size_t bytes = 0;
  const int rc = esmm_head_bwd_ws_bytes(B, K, &bytes);
  if (rc != B200REC_OK) return rc;
  *bytes_host = bytes + 16;
  return B200REC_OK;
}

int b200rec_esmm_head_bwd(const float* g_ctr_out, const float* g_ctr_one, const float* g_cvr_out,
                          const float* g_cvr_one, const float* g_ctcvr_prop,
                          const float* g_ctcvr_one, const float* p_ctr, const float* p_cvr,
                          const float* h_ctr, const float* h_cvr, int K, const float* W_ctr,
                          const float* W_cvr, float* dh_ctr, float* dh_cvr, float* dW_ctr,
                          float* db_ctr, float* dW_cvr, float* db_cvr, int64_t B, void* workspace,
                          size_t workspace_bytes, void* stream) {
  NOT_NULL(dW_ctr); NOT_NULL(db_ctr); NOT_NULL(dW_cvr); NOT_NULL(db_cvr);
  if (B > 0) {
    NOT_NULL(p_ctr); NOT_NULL(p_cvr); NOT_NULL(h_ctr); NOT_NULL(h_cvr); NOT_NULL(W_ctr);
    NOT_NULL(W_cvr); NOT_NULL(dh_ctr); NOT_NULL(dh_cvr);
  }
  const EsmmGrads g = {g_ctr_out, g_ctr_one, g_cvr_out, g_cvr_one, g_ctcvr_prop, g_ctcvr_one};
  return launch_esmm_head_bwd(g, p_ctr, p_cvr, h_ctr, h_cvr, K, W_ctr, W_cvr, dh_ctr, dh_cvr,
                              dW_ctr, db_ctr, dW_cvr, db_cvr, B, workspace, workspace_bytes,
                              ST(stream));
}

/* ---- CTR head: sigmoid of the summed logits, mean log-loss (csrc/ctr_head.cuh) --------------- */
int b200rec_sum_sigmoid_fwd(const float* a, const float* b, const float* c, float* pred, int64_t n,
                            void* stream) {
  B200_REQUIRE(n >= 0, "sum_sigmoid_fwd: bad n");
  if (n == 0) return B200REC_OK;
  NOT_NULL(a); NOT_NULL(pred);
  sum_sigmoid_fwd_kernel<<<(unsigned)((n + kHeadOpThreads - 1) / kHeadOpThreads), kHeadOpThreads, 0,
                           ST(stream)>>>(a, b, c, pred, n);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_sum_sigmoid_bwd(const float* pred, const float* dpred, float* dlogit, int64_t n,
                            void* stream) {
  B200_REQUIRE(n >= 0, "sum_sigmoid_bwd: bad n");
  if (n == 0) return B200REC_OK;
  NOT_NULL(pred); NOT_NULL(dpred); NOT_NULL(dlogit);
  sum_sigmoid_bwd_kernel<<<(unsigned)((n + kHeadOpThreads - 1) / kHeadOpThreads), kHeadOpThreads, 0,
                           ST(stream)>>>(pred, dpred, dlogit, n);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_log_loss_workspace_bytes(size_t* bytes_host) {
  NOT_NULL(bytes_host);
  *bytes_host = log_loss_ws_bytes();
  return B200REC_OK;
}

/* label_is_i64: labels are int64 (as the readers deliver them) or float32.  `workspace` must be
 * ZERO before its first use (the kernel leaves its ticket word zero again). */
int b200rec_log_loss_mean_fwd(const float* pred, const void* label, int label_is_i64, double eps,
                              float* loss, int64_t n, void* workspace, size_t workspace_bytes,
                              void* stream) {
  B200_REQUIRE(n > 0, "log_loss_mean_fwd: n must be positive");
  NOT_NULL(pred); NOT_NULL(label); NOT_NULL(loss); NOT_NULL(workspace);
  if (workspace_bytes < log_loss_ws_bytes()) {
    set_error("log_loss_mean_fwd: workspace %zu < %zu bytes", workspace_bytes, log_loss_ws_bytes());
    return B200REC_ERR_WORKSPACE;
  }
  unsigned int* ticket = static_cast<unsigned int*>(workspace);
  float* partials = reinterpret_cast<float*>(static_cast<unsigned char*>(workspace) + 16);
  const int64_t want = (n + kHeadOpThreads - 1) / kHeadOpThreads;
  const unsigned grid = (unsigned)(want < kLossBlocks ? want : kLossBlocks);
  if (label_is_i64)
    log_loss_mean_fwd_kernel<int64_t><<<grid, kHeadOpThreads, 0, ST(stream)>>>(
        pred, static_cast<const int64_t*>(label), (float)eps, partials, ticket, loss, n);
  else
    log_loss_mean_fwd_kernel<float><<<grid, kHeadOpThreads, 0, ST(stream)>>>(
        pred, static_cast<const float*>(label), (float)eps, partials, ticket, loss, n);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_log_loss_mean_bwd(const float* pred, const void* label, int label_is_i64, double eps,
                              const float* dloss, float* dpred, int64_t n, void* stream) {
  B200_REQUIRE(n > 0, "log_loss_mean_bwd: n must be positive");
  NOT_NULL(pred); NOT_NULL(label); NOT_NULL(dloss); NOT_NULL(dpred);
  const unsigned grid = (unsigned)((n + kHeadOpThreads - 1) / kHeadOpThreads);
  if (label_is_i64)
    log_loss_mean_bwd_kernel<int64_t><<<grid, kHeadOpThreads, 0, ST(stream)>>>(
        pred, static_cast<const int64_t*>(label), (float)eps, dloss, dpred, n);
  else
    log_loss_mean_bwd_kernel<float><<<grid, kHeadOpThreads, 0, ST(stream)>>>(
        pred, static_cast<const float*>(label), (float)eps, dloss, dpred, n);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_auc_update(const float* pred, const void* label, int label_is_i64, int64_t* stat_pos,
                       int64_t* stat_neg, int num_thresholds, int64_t n, void* stream) {
  B200_REQUIRE(n >= 0 && num_thresholds > 0, "auc_update: bad sizes");
  if (n == 0) return B200REC_OK;
  NOT_NULL(pred); NOT_NULL(label); NOT_NULL(stat_pos); NOT_NULL(stat_neg);
  const unsigned grid = (unsigned)((n + kHeadOpThreads - 1) / kHeadOpThreads);
  long long* p = reinterpret_cast<long long*>(stat_pos);
  long long* q = reinterpret_cast<long long*>(stat_neg);
  if (label_is_i64)
    auc_update_kernel<int64_t><<<grid, kHeadOpThreads, 0, ST(stream)>>>(
        pred, static_cast<const int64_t*>(label), p, q, num_thresholds, n);
  else
    auc_update_kernel<float><<<grid, kHeadOpThreads, 0, ST(stream)>>>(
        pred, static_cast<const float*>(label), p, q, num_thresholds, n);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_tc_debug(int key, int value) {
  switch (key) {
    case 0: tc::g_bn_override = value; break;
    case 1: tc::g_dw_debug.lbo_a = (uint32_t)value; break;
    case 2: tc::g_dw_debug.lbo_b = (uint32_t)value; break;
    case 3: tc::g_dw_debug.sbo = (uint32_t)value; break;
    case 4: tc::g_bk = value == 64 ? 64 : 32; break;
    default: set_error("tc_debug: unknown key %d", key); return B200REC_ERR_INVALID;
  }
  return B200REC_OK;
}

int b200rec_tc_timeout_word(unsigned int* word_host) {
  NOT_NULL(word_host);
  B200_CUDA(cudaMemcpyFromSymbol(word_host, tc::g_tc_timeout, sizeof(unsigned int)));
  return B200REC_OK;
}

int b200rec_tower_prep_weight(const float* W, void* W2r_bf16, void* W2c_bf16, void* Wlo_bf16,
                              int K, int N, void* stream) {
  B200_REQUIRE(K > 0 && N > 0, "tower_prep_weight: bad sizes");
  NOT_NULL(W); NOT_NULL(W2r_bf16); NOT_NULL(W2c_bf16); NOT_NULL(Wlo_bf16);
  const int64_t total = (int64_t)K * N;
  tower_prep_weight_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ST(stream)>>>(
      W, static_cast<__nv_bfloat16*>(W2r_bf16), static_cast<__nv_bfloat16*>(W2c_bf16),
      static_cast<__nv_bfloat16*>(Wlo_bf16), K, N);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_tower_fold_dw(const float* Mx, float* dW, int K, int N, void* stream) {
  B200_REQUIRE(K > 0 && N > 0, "tower_fold_dw: bad sizes");
  NOT_NULL(Mx); NOT_NULL(dW);
  const int64_t total = (int64_t)K * N;
  tower_fold_dw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ST(stream)>>>(Mx, dW, K, N);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_cvm_fwd(const float* x, float* y, int64_t N, int D, int use_cvm, void* stream) {
  B200_REQUIRE(N >= 0 && D > 0, "cvm_fwd: bad sizes");
  if (N == 0) return B200REC_OK;
  NOT_NULL(x); NOT_NULL(y);
  const int64_t total = N * (use_cvm ? D + 2 : D);
  const unsigned grid = (unsigned)min((total + 255) / 256, (int64_t)sm_count() * 16);
  cvm_fwd_kernel<<<grid, 256, 0, ST(stream)>>>(x, y, N, D, use_cvm);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_cvm_bwd(const float* dy, const float* show_click, float* dx, int64_t N, int D,
                    int use_cvm, void* stream) {
  B200_REQUIRE(N >= 0 && D > 0, "cvm_bwd: bad sizes");
  if (N == 0) return B200REC_OK;
  NOT_NULL(dy); NOT_NULL(show_click); NOT_NULL(dx);
  const int64_t total = N * (D + 2);
  const unsigned grid = (unsigned)min((total + 255) / 256, (int64_t)sm_count() * 16);
  cvm_bwd_kernel<<<grid, 256, 0, ST(stream)>>>(dy, show_click, dx, N, D, use_cvm);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

static int dot_interact_launch(bool bwd, const float* T, const float* dR, float* out, int64_t B, int N,
                               int d, int self_interaction, void* stream) {
  B200_REQUIRE(B >= 0 && N >= 2 && N <= 128 && d >= 1 && d <= 256, "dot_interact: bad sizes");
  if (B == 0) return B200REC_OK;
  NOT_NULL(T); NOT_NULL(out);
  const DotShape s(N, d, self_interaction ? 1 : 0);
  // B200REC_K6_V2=1 selects the experimental float4 / cp.async variant (dot_interact.cuh); read per
  // call so that a test can compare both paths in one process
  const char* v2_env = getenv("B200REC_K6_V2");
  const bool v2 = v2_env && atoi(v2_env) != 0 && d % 4 == 0;
  const size_t per_warp = sizeof(float) * (v2 ? dot_v2_smem_floats(s, bwd)
                                              : (bwd ? s.smem_floats_bwd() : s.smem_floats_fwd()));
  int warps = kDotWarps;  // samples in flight per CTA; shrink until the tiles fit
  while (warps > 1 && warps * per_warp > 96 * 1024) warps >>= 1;
  const size_t smem = warps * per_warp;
  B200_REQUIRE(smem <= 200 * 1024, "dot_interact: N*d too large for shared memory");
  const int64_t ctas = (B + warps - 1) / warps;
  const unsigned grid = (unsigned)min(ctas, (int64_t)sm_count() * 8);
  if (bwd) NOT_NULL(dR);
  auto fwd_k = v2 ? dot_interact_fwd_v2_kernel : dot_interact_fwd_kernel;
  auto bwd_k = v2 ? dot_interact_bwd_v2_kernel : dot_interact_bwd_kernel;
  if (smem > 48 * 1024) {
    if (bwd) B200_CUDA(cudaFuncSetAttribute(bwd_k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    else B200_CUDA(cudaFuncSetAttribute(fwd_k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  if (bwd) bwd_k<<<grid, warps * 32, smem, ST(stream)>>>(T, dR, out, B, s);
  else fwd_k<<<grid, warps * 32, smem, ST(stream)>>>(T, out, B, s);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

int b200rec_dot_interact_fwd(const float* T, float* R, int64_t B, int N, int d, int self_interaction,
                             void* stream) {
  return dot_interact_launch(false, T, nullptr, R, B, N, d, self_interaction, stream);
}

int b200rec_dot_interact_bwd(const float* T, const float* dR, float* dT, int64_t B, int N, int d,
                             int self_interaction, void* stream) {
  return dot_interact_launch(true, T, dR, dT, B, N, d, self_interaction, stream);
}

int b200rec_hash_keys(const uint64_t* keys, const int32_t* slot_of_key, int64_t n, int64_t V,
                      int reserve_zero, int64_t* rows, void* stream) {
  B200_REQUIRE(n >= 0, "hash_keys: n < 0");
  B200_REQUIRE(V >= (reserve_zero ? 2 : 1), "hash_keys: table too small for the requested fold");
  if (n == 0) return B200REC_OK;
  NOT_NULL(keys); NOT_NULL(rows);
  const unsigned grid = (unsigned)min((n + 255) / 256, (int64_t)sm_count() * 16);
  hash_keys_kernel<<<grid, 256, 0, ST(stream)>>>(keys, slot_of_key, n, (uint64_t)V, reserve_zero, rows);
  B200_LAUNCH_CHECK();
  return B200REC_OK;
}

#include "din_attn_api.inc"

}  // extern "C"
