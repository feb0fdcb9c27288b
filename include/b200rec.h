/*
 * b200rec.h — C ABI of the H100-native sparse-embedding + feature-interaction engine.
 *
 * This is the drop-in boundary for the one hot path of PaddleRec's rank models
 * (reference checkout /root/reference, commit 656326ad):
 *
 *   paddle.nn.Embedding fwd/bwd   models/rank/deepfm/net.py:66-86,108,117
 *                                 models/rank/dcn_v2/net.py:45-54,95
 *                                 models/rank/din/net.py:33-82,141-147
 *                                 models/rank/wide_deep/net.py:47-53,90
 *   FM first/second order         models/rank/deepfm/net.py:105-139
 *   CrossNetV2 / CrossNetMix      models/rank/dcn_v2/net.py:222-226,278-320
 *   DIN attention pooling         models/rank/din/net.py:155-173
 *   sparse (row-wise) optimizers  models/rank/deepfm/static_model.py:101-103 (lazy Adam),
 *                                 models/rank/din/dygraph_model.py:64-73 (SGD),
 *                                 models/rank/slot_dnn/config_online.yaml:57-79 (AdaGrad rule)
 *   sharded table key exchange    tools/static_gpubox_trainer.py:152-159,244-259 (PSGPU pull/push)
 *
 * PaddleRec has no FFI of its own (SURVEY.md §8b): the arithmetic above lives in Paddle
 * core operators that net.py calls.  A Paddle custom-op (`PD_BUILD_OP`) or any other host
 * binds these entry points; INTEGRATION.md shows the stub.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - the caller owns every buffer (outputs and workspace; query sizes first) — the
 *     library never allocates on the hot path;
 *   - all tensors are dense row-major fp32, all ids int64;
 *   - functions enqueue on `stream` (a cudaStream_t passed as void*) and return
 *     without synchronising; they are re-entrant;
 *   - return 0 on success, a negative B200REC_ERR_* otherwise; the message is
 *     available from b200rec_last_error() (thread-local); nothing throws;
 *   - ids outside [0,V) are treated like the padding row (zero output, no
 *     gradient) and counted in a device-side counter readable with
 *     b200rec_oob_count() (Paddle raises on such ids; we stay UB-free and report).
 */
#ifndef B200REC_H_
#define B200REC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200REC_ABI_VERSION 7

#define B200REC_OK 0
#define B200REC_ERR_INVALID (-1)   /* bad argument (shape, alignment, NULL) */
#define B200REC_ERR_CUDA (-2)      /* a CUDA runtime call or launch failed   */
#define B200REC_ERR_WORKSPACE (-3) /* workspace too small                    */

/* ---- library ------------------------------------------------------------ */
int b200rec_abi_version(void);
const char* b200rec_last_error(void);
/* number of out-of-range ids seen since the last reset (synchronises `stream`). */
int b200rec_oob_count(uint64_t* count_host, int reset, void* stream);

/* ---- K1: fused multi-slot gather + FM (DeepFM forward) ------------------- */
/* Replaces FM.forward, models/rank/deepfm/net.py:105-139.
 *   feat[b,f,:]   = W[ids[b,f],:]                (zeros if ids==padding_idx)     f <  F
 *   feat[b,F+j,:] = dense[b,j] * dense_w[j,:]                                    j <  Dn
 *   y1[b] = sum_f W1[ids[b,f]] + sum_j dense[b,j]*dense_w1[j]
 *   S[b,:] = sum_n feat[b,n,:] ;  y2[b] = 0.5 * sum_d ( S[b,d]^2 - sum_n feat[b,n,d]^2 )
 * feat:[B,F+Dn,D]  y1,y2:[B]  S:[B,D] (saved for backward; may be NULL).
 * padding_idx < 0 means "no padding row".  D must be <=128 (D%4==0), <=64 (D%2==0) or <=32.
 * Row strides (in floats): row i of the second-order table starts at W + i*ldw, its first-order
 * weight is W1[i*ldw1].  Two separate tables: ldw=D, ldw1=1.  The FUSED layout keeps
 * both in one 128-byte slot [D emb | w1 | pad] (ldw = ldw1 = 32, W1 = W + D): a random 64-byte
 * row and a random 4-byte scalar each cost a full 128-byte DRAM access
 * (tools/microbench/gather_variants.cu measures it), so the slot halves the random traffic. */
int b200rec_embed_fm_fwd(const float* W, int64_t ldw, const float* W1, int64_t ldw1,
                         const int64_t* ids, const float* dense, const float* dense_w,
                         const float* dense_w1, float* feat, float* y1, float* y2, float* S,
                         int64_t B, int F, int Dn, int D, int64_t V, int64_t padding_idx,
                         void* stream);

/* ---- grouping of ids (sort + run-length) shared by every backward -------- */
/* Stable-sorts the n ids, dropping padding / out-of-range ones, and produces
 *   unique_ids[u]            the u-th distinct id (ascending)             u < *num_unique
 *   seg_offsets[u..u+1]      range in sorted_pos of the positions holding that id
 *   sorted_pos[i]            original position (0..n-1), ascending inside a segment
 * num_unique is a device int32[2]: {#distinct ids, #positions kept}.
 * Output arrays must hold n (seg_offsets: n+1) elements. */
int b200rec_group_ids_workspace_bytes(int64_t n, int64_t V, size_t* bytes_host);
int b200rec_group_ids(const int64_t* ids, int64_t n, int64_t V, int64_t padding_idx,
                      int64_t* unique_ids, int32_t* seg_offsets, int32_t* sorted_pos,
                      int32_t* num_unique, void* workspace, size_t workspace_bytes, void* stream);

/* ---- K2: DeepFM backward (analytic FM grad fused into the segmented reduce) */
/* Backward of b200rec_embed_fm_fwd (autograd of net.py:105-139, SURVEY.md §8a A7).
 *   dfeat[b,n,:] = gy2[b]*(S[b,:] - feat[b,n,:]) + dfeat_dnn[b,n,:]   (dfeat_dnn may be NULL)
 *   dW_rows[u,:] = sum_{p in segment u} dfeat[p]        dW1_rows[u] = sum_{p in seg u} gy1[b(p)]
 *   ddense_w[j,:] = sum_b dense[b,j]*dfeat[b,F+j,:]     ddense_w1[j] = sum_b gy1[b]*dense[b,j]
 * dW_rows:[n,D], dW1_rows:[n] with n=B*F; only the first num_unique[0] rows are written
 * (a SelectedRows{rows=unique_ids, value=dW_rows} in Paddle terms).  Deterministic.
 * Output strides: dW_rows[u*ld_dw + d], dW1_rows[u*ld_dw1]; separate buffers: ld_dw=D, ld_dw1=1,
 * dw1_zero_pad=0.  Fused gradient rows [D | g1 | 0-pad]: dW1_rows = dW_rows + D, ld_dw = ld_dw1 =
 * D+1+pad, dw1_zero_pad = pad (those floats are written as zeros). */
int b200rec_embed_fm_bwd_workspace_bytes(int64_t B, int F, int Dn, int D, size_t* bytes_host);
int b200rec_embed_fm_bwd(const float* feat, const float* S, const float* dfeat_dnn,
                         const float* gy1, const float* gy2, const float* dense,
                         const int32_t* seg_offsets, const int32_t* sorted_pos,
                         const int32_t* num_unique, float* dW_rows, int64_t ld_dw,
                         float* dW1_rows, int64_t ld_dw1, int dw1_zero_pad, float* ddense_w,
                         float* ddense_w1, int64_t B, int F, int Dn, int D, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---- FFM: field-aware second-order term fused with its gather -------------- */
/* Replaces FFM.forward, models/rank/ffm/net.py:99-133.  NF = F + Dn fields, R = NF*D.
 * W [V, ldw] holds fused rows [R emb | w1 | pad] (ldw >= R+1, ldw % 4 == 0, base 16-byte aligned).
 *   e[b,n,:] = W[ids[b,n], 0:R] (n < F; zeros for padding / out-of-range ids)
 *            = dense[b,n-F] * dense_w[n-F, :]      (n >= F; dense_w [Dn, R])
 *   y1[b] = sum_f W[ids[b,f], R] + sum_k dense[b,k]*dense_w1[k] (+ bias[0] if bias != NULL)
 *   y2[b] = sum_{n<m} < e[b,n, m*D:(m+1)*D], e[b,m, n*D:(n+1)*D] >
 * Nothing of size [B,NF,R] is written.  1 <= F, F+Dn <= 64; one sample's F staged rows plus dense_w
 * must fit a CTA's shared memory (F=26, Dn=13 fits up to D=32), else B200REC_ERR_INVALID. */
int b200rec_ffm_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                    const float* dense_w, const float* dense_w1, const float* bias, float* y1,
                    float* y2, int64_t B, int F, int Dn, int D, int64_t V, int64_t padding_idx,
                    void* stream);
/* Backward of b200rec_ffm_fwd with gy1 = dL/dy1, gy2 = dL/dy2 [B] and the grouping of the B*F ids
 * from b200rec_group_ids:
 *   dW_rows[u, m*D:(m+1)*D] = sum_{(b,f) in segment u, m != f} gy2[b] * e[b,m, f*D:(f+1)*D]
 *   dW_rows[u, R] = sum gy1[b];  columns R+1 .. ld_dw-1 are written as zeros
 *   ddense_w[k, m*D:(m+1)*D] = sum_b gy2[b]*dense[b,k]*e[b,m, (F+k)*D:(F+k+1)*D]   (m != F+k)
 *   ddense_w1[k] = sum_b gy1[b]*dense[b,k];   dbias[0] = sum_b gy1[b] (dbias may be NULL)
 * Only the first num_unique[0] rows of dW_rows are written, so it needs min(B*F, V) rows.
 * Ids with more than 64 positions are split over CTAs; every sum has a fixed order, no float
 * atomics: a second run is bit-identical. */
int b200rec_ffm_bwd_workspace_bytes(int64_t B, int F, int Dn, int D, size_t* bytes_host);
int b200rec_ffm_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                    const float* dense_w, const float* gy1, const float* gy2,
                    const int32_t* seg_offsets, const int32_t* sorted_pos,
                    const int32_t* num_unique, float* dW_rows, int64_t ld_dw, float* ddense_w,
                    float* ddense_w1, float* dbias, int64_t B, int F, int Dn, int D, int64_t V,
                    int64_t padding_idx, void* workspace, size_t workspace_bytes, void* stream);

/* ---- FAT-DeepFFM: CENet field attention + field-aware Hadamard interaction -- */
/* Replaces CENLayer.forward and DeepFFM.forward, models/rank/fat_deepffm/net.py:105-151, 219-251,
 * around the attention MLP (which stays a pair of GEMMs).  NF = F + Dn, R = NF*D, P = NF(NF-1)/2.
 * W [V, ldw] holds FFM's fused rows (ldw >= R+1, ldw % 4 == 0, base 16-byte aligned); its w1
 * column is not read.  e[b,n,:] = W[ids[b,n], 0:R] (n < F; zeros for padding / out-of-range ids),
 * dense[b,n-F] * dense_w[n-F, :] (n >= F).  Same shape limits as b200rec_ffm_fwd, and the sample
 * buffers also hold one [NF*NF] attention row.
 *   pool[b, n*NF+m] = max_d e[b,n, m*D+d]
 * Padding and out-of-range ids are counted (b200rec_oob_count) by this call only. */
int b200rec_fat_ffm_pool_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                             const float* dense_w, float* pool, int64_t B, int F, int Dn, int D,
                             int64_t V, int64_t padding_idx, void* stream);
/* With attn [B, NF*NF] and s[b,n,m,:] = attn[b, n*NF+m] * e[b,n, m*D:(m+1)*D]:
 *   y1[b] = sum_{n,m,d} s[b,n,m,d] (+ bias[0] if bias != NULL), summed in a fixed order
 *   h[b, p(n,m)*D + d] = s[b,n,m,d] * s[b,m,n,d]   for n < m in row-major pair order
 * Nothing of size [B,NF,R] is written.  h may be NULL when P*D = 0 (one field: no pairs). */
int b200rec_fat_ffm_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                        const float* dense_w, const float* attn, const float* bias, float* y1,
                        float* h, int64_t B, int F, int Dn, int D, int64_t V, int64_t padding_idx,
                        void* stream);
/* dattn[b, n*NF+m] = sum_d e[b,n,m*D+d] * (gy1[b] + [n != m] * dh[b, p(n,m)*D+d] * s[b,m,n,d])
 * dh may be NULL when P*D = 0. */
int b200rec_fat_ffm_bwd_attn(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                             const float* dense_w, const float* attn, const float* gy1,
                             const float* dh, float* dattn, int64_t B, int F, int Dn, int D,
                             int64_t V, int64_t padding_idx, void* stream);
/* Table and dense-parameter gradients through both routes (the attention product and the max
 * pool), with the grouping of the B*F ids from b200rec_group_ids.  For row n, block m, column j:
 *   de = attn[n,m] * (gy1 + [m != n] * dh[p(n,m), j] * attn[m,n] * e[m, n*D+j])
 *        + [j = FIRST argmax_d e[n, m*D+d]] * dpool[n*NF+m]
 *   dW_rows[u, 0:R] = sum over the positions of segment u of de;  columns R .. ld_dw-1 are 0
 *   ddense_w[k, c] = sum_b dense[b,k] * de(b, F+k, c);   dbias[0] = sum_b gy1[b] (may be NULL)
 * The argmax of a dense block is taken on the fp32 product dense * dense_w.  Only the first
 * num_unique[0] rows of dW_rows are written, so it needs min(B*F, V) rows.  Every sum has a fixed
 * order, no float atomics: a second run is bit-identical.  dh may be NULL when P*D = 0. */
int b200rec_fat_ffm_bwd_workspace_bytes(int64_t B, int F, int Dn, int D, size_t* bytes_host);
int b200rec_fat_ffm_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* dense,
                        const float* dense_w, const float* attn, const float* gy1, const float* dh,
                        const float* dpool, const int32_t* seg_offsets, const int32_t* sorted_pos,
                        const int32_t* num_unique, float* dW_rows, int64_t ld_dw, float* ddense_w,
                        float* dbias, int64_t B, int F, int Dn, int D, int64_t V,
                        int64_t padding_idx, void* workspace, size_t workspace_bytes,
                        void* stream);

/* ---- plain gather / segmented scatter-add (W&D, DCN-V2, DIN lookups) ------ */
/* out[i,:] = W[ids[i],:]  (zeros if ids[i]==padding_idx).  Replaces paddle.nn.Embedding
 * forward (lookup_table_v2), e.g. models/rank/wide_deep/net.py:90, dcn_v2/net.py:95. */
int b200rec_gather(const float* W, int64_t ldw, const int64_t* ids, float* out, int64_t n, int D,
                   int64_t V, int64_t padding_idx, void* stream);
/* GateNet embedding gate fused with the gather and the tower-input concat
 * (models/rank/gatenet/net.py:88-103,110).  W [V,ldw], ids int64 [B,F] (F <= 256), gate_w [F].
 *   gate_embed_fwd  out [B, ld_out] (ld_out >= F*D + Dn): out[b, f*D + d] = e_d * g with
 *                   e = W[ids[b,f], :D], g = 1/(1 + expf(-sum_d e_d * gate_w[f])); the dense
 *                   features dense [B,Dn] follow at column F*D.  Out-of-range ids: zero row, counted.
 *   gate_embed_bwd  re-gathers the rows; dout is the gradient of out (pitch ld_out).  Writes the
 *                   per-position table-gradient rows drow [B*F, D] (to be merged with group_ids +
 *                   segment_reduce; zero for out-of-range ids) and dgate_w [F], summed in a fixed
 *                   order (no float atomics: bit-identical across runs). */
int b200rec_gate_embed_fwd(const float* W, int64_t ldw, const int64_t* ids, const float* gate_w,
                           const float* dense, float* out, int64_t ld_out, int64_t B, int F, int D,
                           int Dn, int64_t V, void* stream);
int b200rec_gate_embed_bwd_workspace_bytes(int64_t B, int F, size_t* bytes_host);
int b200rec_gate_embed_bwd(const float* W, int64_t ldw, const int64_t* ids, const float* gate_w,
                           const float* dout, int64_t ld_out, float* drow, float* dgate_w,
                           int64_t B, int F, int D, int64_t V, void* workspace,
                           size_t workspace_bytes, void* stream);
/* rows[u,:] = sum_{p in segment u} dOut[p,:]  — the SelectedRows merge of
 * lookup_table_v2_grad.  Deterministic (fixed order inside a segment); ids occurring more than
 * 64 times are reduced by whole CTAs (skew-proof).  row_of_pos (may be NULL) redirects position p to
 * row row_of_pos[p] of dOut (pooled lookups: many positions share one output row). */
int b200rec_segment_reduce_workspace_bytes(int64_t n, int D, size_t* bytes_host);
int b200rec_segment_reduce(const float* dOut, const int32_t* row_of_pos,
                           const int32_t* seg_offsets, const int32_t* sorted_pos,
                           const int32_t* num_unique, float* rows, int64_t n, int D,
                           void* workspace, size_t workspace_bytes, void* stream);
/* Multi-hot slots (LoD): out[bag,:] = sum_{i in [offsets[bag], offsets[bag+1])} W[keys[i],:D]
 * (sequence_pool(sum) after sparse_embedding, models/rank/slot_dnn/net.py:63-75; the pooling half
 * of fused_seqpool_cvm, tools/utils/static_ps/model_util.py:411-415).  Empty bags give zeros.
 * bag_of_pos (int32 [nnz], may be NULL) receives the owning bag of every key position: pass it as
 * `row_of_pos` to b200rec_segment_reduce (with dOut = d/d(out)) for the backward. */
int b200rec_gather_pool_sum(const float* W, int64_t ldw, const int64_t* keys,
                            const int64_t* offsets, float* out, int32_t* bag_of_pos, int64_t n_bags,
                            int D, int64_t V, int64_t padding_idx, void* stream);
/* dW[unique_ids[u],:] += rows[u,:] into a dense [V,D] gradient (small tables / tests). */
int b200rec_rows_to_dense(const int64_t* unique_ids, const float* rows, int64_t ld_rows,
                          const int32_t* num_unique, float* dW, int64_t ld_dw, int64_t n, int D,
                          int64_t V, void* stream);

/* ---- row-wise ("lazy") optimizers applied to the touched rows only -------- */
/* W (and m, v) rows start at i*ldw, gradient rows at u*ld_rows; D columns are updated.  Rows wider
 * than 128 floats (FFM's [R | w1] rows) are updated by one warp per row in 32-lane chunks. */
/* W[id] -= lr * g */
int b200rec_sparse_sgd(float* W, int64_t ldw, const int64_t* unique_ids, const float* rows,
                       int64_t ld_rows, const int32_t* num_unique, int64_t n, int D, int64_t V,
                       double lr, void* stream);
/* Adam(lazy_mode=True): m=b1*m+(1-b1)g; v=b2*v+(1-b2)g^2;
 * W -= lr*sqrt(1-b2^t)/(1-b1^t) * m/(sqrt(v)+eps*sqrt(1-b2^t)); bias terms from the host.
 * Hyper-parameters are doubles: derived constants (1-b1, 1-b2, lr_t) are formed in double on the
 * host and only then rounded to fp32 (1-0.999f would be off by 5e-5 relative). */
int b200rec_sparse_adam(float* W, float* m, float* v, int64_t ldw, const int64_t* unique_ids,
                        const float* rows, int64_t ld_rows, const int32_t* num_unique, int64_t n,
                        int D, int64_t V,
                        double lr, double beta1, double beta2, double eps, double beta1_pow_t,
                        double beta2_pow_t, void* stream);
/* SparseAdaGradSGDRule: one g2sum scalar per row.
 *   W -= lr * g * sqrt(g0/(g0+g2sum)); clamp to [lo,hi]; g2sum += mean_d(g^2). */
int b200rec_sparse_adagrad(float* W, float* g2sum, int64_t ldw, const int64_t* unique_ids,
                           const float* rows, int64_t ld_rows, const int32_t* num_unique, int64_t n,
                           int D, int64_t V, double lr,
                           double initial_g2sum, double lo, double hi, void* stream);

/* ---- K3: CrossNet fused epilogues (GEMM itself is a library GEMM) --------- */
/* CrossNetV2 step, models/rank/dcn_v2/net.py:222-226, after xw = x_l @ W_l:
 *   out = xl + x0 * (xw + bias)           all [B,C], bias [C] */
int b200rec_cross_v2_fwd(const float* x0, const float* xl, const float* xw, const float* bias,
                         float* out, int64_t B, int C, void* stream);
/* Given dout: dxw = dout*x0 ; dx0 = dout*(xw+bias) ; dbias[c] = sum_b dxw[b,c]
 * (the caller finishes dxl = dout + dxw@W^T and dW = xl^T@dxw with library GEMMs).  dbias needs a workspace of b200rec_cross_bwd_workspace_bytes. */
int b200rec_cross_bwd_workspace_bytes(int64_t B, int C, size_t* bytes_host);
int b200rec_cross_v2_bwd(const float* dout, const float* x0, const float* xw, const float* bias,
                         float* dxw, float* dx0, float* dbias, int64_t B, int C,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ---- K4: DIN attention pooling (forward) ---------------------------------- */
/* Replaces the attention unit + masked softmax + pooling of DINLayer.forward,
 * models/rank/din/net.py:155-173, for the reader's tiled target (dinReader.py:85-90):
 *   a[b,l]  = MLP([h, t, h-t, h*t]),  MLP = Linear(4E,80)-sigmoid-Linear(80,40)-sigmoid-Linear(40,1)
 *   w[b,:]  = softmax_l((a[b,:] + mask[b,:]) * scale)            (mask added BEFORE the scale)
 *   out[b,:] = sum_l w[b,l] * hist[b,l,:]
 * with the first layer re-associated:  [h,t,h-t,h*t] W1 = h Wac + (h*t) Wd + tb,
 *   Wac = W1[0:E] + W1[2E:3E],  Wd = W1[3E:4E],  tb = t (W1[E:2E] - W1[2E:3E]) + b1   ([B,80], by
 * the caller: one small library GEMM per step).  hist [B,L,E], tseq [B,E], mask int64 [B,L]
 * (0 / -1e9, may be NULL), scores/weights [B,L] (scratch / saved softmax), out [B,E].
 * E % 4 == 0, E <= 128; hidden sizes are the reference's fixed 80 and 40. */
int b200rec_din_attn_fwd(const float* hist, const float* tseq, const float* tb, const float* Wac,
                         const float* Wd, const float* W2, const float* b2, const float* W3,
                         const float* b3, const int64_t* mask, float* scores, float* weights,
                         float* out, int64_t B, int L, int E, float scale, void* stream);

/* ---- sharded table: the exchange over NVLink peer memory -------------------- */
/* PSGPU pull_sparse / push_sparse (tools/static_gpubox_trainer.py:152-159,244-259) without a
 * collective-library call on the data path: every GPU maps its peers' receive buffers (symmetric
 * memory; `peer_ptrs_host[r]` = base of rank r's buffer in THIS process's address space) and the
 * kernels store straight into them over NVLink.  seg_dev [world+1] / dst_dev [world] are DEVICE
 * int64 tables (outputs of the count exchange): rows [seg[r], seg[r+1]) of the local list go to
 * peer r, starting at row dst[r] of its buffer (row pitch ld_dst floats).  The first `world`
 * peer pointers must be non-null and aligned to the row store width (4*VEC bytes, VEC as for D;
 * 16 bytes for shard_fm_grads_push), else B200REC_ERR_INVALID, checked also when n == 0.
 *   shard_gather_push  owner side of the pull: gather of the requested rows of `shard` (ids are
 *                      LOCAL rows; local_pad / out-of-range -> zeros) fused with their transfer
 *   shard_push_rows    requester side of the push: per-slot gradient rows (bucket order) -> owners
 * The caller publishes the stores with a barrier over the same symmetric memory. */
int b200rec_shard_gather_push(const float* shard, int64_t ldw, int D, int64_t V_loc,
                              int64_t local_pad, const int64_t* recv_ids, const int64_t* seg_dev,
                              const int64_t* dst_dev, const uint64_t* peer_ptrs_host, int64_t ld_dst,
                              int world, int64_t n, void* stream);
/* DeepFM: the sparse half of the FM backward fused with the push — slot k (position b*F+f = inv_perm[k]) receives
 * [ gy2[b]*(S[b]-feat[b,f]) + dfeat_dnn[b,f] | gy1[b] | 0.. ] (G floats) straight in its owner's
 * buffer; no [B*F, G] staging buffer exists.  D % 4 == 0, G % 4 == 0, G >= D+1. */
int b200rec_shard_fm_grads_push(const float* feat, const float* S, const float* dfeat_dnn,
                                const float* gy1, const float* gy2, const int32_t* inv_perm,
                                const int64_t* seg_dev, const int64_t* dst_dev,
                                const uint64_t* peer_ptrs_host, int64_t ld_dst, int world, int64_t B,
                                int F, int Dn, int D, int G, void* stream);
int b200rec_shard_push_rows(const float* rows, int64_t ld, int D, const int64_t* seg_dev,
                            const int64_t* dst_dev, const uint64_t* peer_ptrs_host, int64_t ld_dst,
                            int world, int64_t n, void* stream);

/* ---- tower epilogues (bf16 hi/lo split operands for the tensor-core GEMMs) -- */
/* The MLP tower (DNN.forward, models/rank/deepfm/net.py:169-174) runs its GEMMs on the bf16 tensor
 * cores as a*b ~ a_hi*b_hi + a_lo*b_hi + a_hi*b_lo (fp32 accumulate).  These fuse everything
 * between two GEMMs into one pass.  bf16 buffers are passed as void*.
 *   split:          out[m,0:K] = hi(f(x[m,:])), out[m,K:2K] = lo(...),  f = (+bias) then (ReLU)
 *   relu_bwd_split: dz = dy * (act_hi > 0) (act may be NULL: no mask); dz_out = [hi|lo];
 *                   dbias[n] = sum_m dz[m,n]   (deterministic)
 *   prep_weight:    W[K,N] -> W2r[2K,N]=[hi;hi], W2c[K,2N]=[hi|hi], Wlo[K,N]
 *   fold_dw:        dW = Mx[0:K,0:N] + Mx[0:K,N:2N] + Mx[K:2K,0:N],  Mx = [a_hi|a_lo]^T [dz_hi|dz_lo] */
int b200rec_tower_split(const float* x, const float* bias, int relu, void* out_bf16, int64_t M,
                        int K, void* stream);
int b200rec_tower_bwd_workspace_bytes(int64_t M, int N, size_t* bytes_host);
int b200rec_tower_relu_bwd_split(const float* dy, const void* act_bf16, void* dz_bf16,
                                 float* dbias, int64_t M, int N, void* workspace,
                                 size_t workspace_bytes, void* stream);
int b200rec_tower_prep_weight(const float* W, void* W2r_bf16, void* W2c_bf16, void* Wlo_bf16,
                              int K, int N, void* stream);
int b200rec_tower_fold_dw(const float* Mx, float* dW, int K, int N, void* stream);

/* ---- tower GEMMs on the Hopper tensor cores (csrc/tc_gemm.cuh) ------------ */
/* Hand-written wgmma / TMA kernels that replace the library GEMMs of the dense tower
 * (DNN.forward, models/rank/deepfm/net.py:169-174; dcn_v2/net.py:178-184; CrossNetV2
 * dcn_v2/net.py:222-226) and of its backward (tools/trainer.py:151).  fp32 products are evaluated
 * as a_hi*b_hi + a_lo*b_hi + a_hi*b_lo on bf16 operands with fp32 accumulation ("bf16x3").
 *
 * "planes": a matrix X[R,C] is passed as bf16 [R, 2*ld] (void*), hi(X) in columns [0,C) and
 * lo(X) = bf16(X - hi) in columns [ld, ld+C); ld >= C, ld % 8 == 0, base 16-byte aligned.
 *
 *   tc_split        planes(relu?(x + bias?)) of an fp32 matrix x[M,K] with row pitch ldx
 *   tc_split_bwd    g = dy * (mask_hi > 0) (mask may be NULL) -> planes(g), dbias = colsum(g)
 *   tc_prep_weight  W[K,N] -> planes(W) [K,2*ldn] and planes(W^T) [N,2*ldk] (either may be NULL)
 *   tc_linear_fwd   y = a @ W + bias, optional ReLU; a = planes [M,2*lda], W^T planes; writes y as
 *                   fp32 [M,ld_f32] and/or as planes [M,2*ldp] (the next layer's operand)
 *   tc_cross_fwd    CrossNetV2 layer: out = x0 * u + xl with u = xl @ W + b (x0, xl fp32 [M,C] pitch
 *                   ld_x); u_f32 (may be NULL) receives u [M,C] for the backward (pitch ld_f32)
 *   tc_linear_bwd_dx  dx = g @ W^T (g planes [M,2*ldg], W planes [K,2*ldn]); optional ReLU mask
 *                   from the hi plane of the layer input (mask_planes [M,2*ld_mask]); `addend`
 *                   (fp32 [M,K] contiguous, may be NULL) is added first (residual paths); dx as fp32
 *                   and/or planes; dbias_prev[K] = colsum(masked dx) if not NULL (deterministic)
 *   tc_linear_bwd_dw  dW[K,N] = a^T @ g, batch reduction split across CTAs, fixed-order reduce
 * ones_col (tc_split, tc_linear_fwd): additionally store 1.0 in column C of the emitted planes
 * (needs ld > C).  Passing K+1 as the width of such an operand to tc_linear_bwd_dw makes row K of
 * its output the column sum of g, i.e. the layer's bias gradient, at no extra cost.
 * One workspace size covers bwd_dx and bwd_dw of a layer. */
int b200rec_tc_split(const float* x, int64_t ldx, const float* bias, int relu, void* planes,
                     int64_t ldp, int64_t M, int K, int ones_col, void* stream);
int b200rec_tc_split_bwd(const float* dy, const void* mask_planes, int64_t ld_mask, void* g_planes,
                         int64_t ldp, float* dbias, int64_t M, int N, void* workspace,
                         size_t workspace_bytes, void* stream);
int b200rec_tc_prep_weight(const float* W, int K, int N, void* w_planes, int64_t ldn,
                           void* wt_planes, int64_t ldk, void* stream);
int b200rec_tc_linear_fwd(const void* a_planes, int64_t lda, const void* wt_planes, int64_t ldk,
                          const float* bias, int relu, float* out_f32, int64_t ld_f32,
                          void* out_planes, int64_t ldp, int ones_col, int64_t M, int N, int K,
                          void* stream);
int b200rec_tc_cross_fwd(const void* xl_planes, int64_t lda, const void* wt_planes, int64_t ldk,
                         const float* bias, const float* x0, const float* xl, int64_t ld_x,
                         float* u_f32, float* out_f32, int64_t ld_f32, void* out_planes,
                         int64_t ldp, int ones_col, int64_t M, int C, void* stream);
/* GateNet hidden gate (models/rank/gatenet/net.py:116-118), z = y * tanh(a) with a = y @ G, G [N,N]:
 *   tc_gate_fwd   a = y @ G on the K-major wgmma GEMM (y planes [M,2*ldy] are both the A operand and
 *                 the gate's multiplicand; G^T planes [N,2*ldk]); the epilogue writes a_f32 (may be
 *                 NULL) and z as fp32 (may be NULL) with pitch ld_f32, and/or planes(z) [M,2*ldp]
 *                 with the optional column of ones.  tanhf is the accurate one.
 *   tc_gate_bwd   given dz fp32 [M,N] and a fp32 [M,N] (both contiguous): planes(g) [M,2*ldp] with
 *                 g = dz * y * (1 - tanh(a)^2) and r = dz * tanh(a) fp32 [M,N].  Then
 *                 dG = tc_linear_bwd_dw(y, g) and dy = tc_linear_bwd_dx(g, G, mask = y, addend = r). */
int b200rec_tc_gate_fwd(const void* y_planes, int64_t ldy, const void* gt_planes, int64_t ldk,
                        float* a_f32, float* out_f32, int64_t ld_f32, void* out_planes, int64_t ldp,
                        int ones_col, int64_t M, int N, void* stream);
int b200rec_tc_gate_bwd(const float* dz, const void* y_planes, int64_t ldy, const float* a,
                        void* g_planes, int64_t ldp, float* r, int64_t M, int N, void* stream);
int b200rec_tc_linear_bwd_workspace_bytes(int64_t M, int K, int N, size_t* bytes_host);
int b200rec_tc_linear_bwd_dx(const void* g_planes, int64_t ldg, const void* w_planes, int64_t ldn,
                             const void* mask_planes, int64_t ld_mask, const float* addend,
                             float* dx_f32, int64_t ld_f32, void* dx_planes, int64_t ldp,
                             float* dbias_prev, int64_t M, int K, int N, void* workspace,
                             size_t workspace_bytes, void* stream);
int b200rec_tc_linear_bwd_dw(const void* a_planes, int64_t lda, const void* g_planes, int64_t ldg,
                             float* dW, int64_t M, int K, int N, void* workspace,
                             size_t workspace_bytes, void* stream);
/* The width-1 head of a CTR tower (last Linear of deepfm/net.py:169-174, K -> 1) as streaming
 * kernels (HBM-bound: a GEMM tile would waste 15/16 of the tensor core on it):
 *   tc_head_fwd  y[m] = sum_k a[m,k] w[k] + bias[0]          (a = planes [M,2*lda], w fp32 [K])
 *   tc_head_bwd  g = planes(dy[m] * w[k] * (a_hi[m,k] > 0)) [M,2*ldg],  dW[k] = sum_m a[m,k] dy[m],
 *                db[0] = sum_m dy[m]   (K % 8 == 0, K <= 2048; deterministic) */
int b200rec_tc_head_fwd(const void* a_planes, int64_t lda, int K, const float* w, const float* bias,
                        float* y, int64_t M, void* stream);
int b200rec_tc_head_bwd_workspace_bytes(int K, size_t* bytes_host);
int b200rec_tc_head_bwd(const void* a_planes, int64_t lda, int K, const float* w, const float* dy,
                        void* g_planes, int64_t ldg, float* dW, float* db, int64_t M,
                        void* workspace, size_t workspace_bytes, void* stream);
/* ESMM's two width-2 heads and the CTCVR product (models/multitask/esmm/net.py:85-111) on the
 * towers' last ReLU'd activations h_ctr, h_cvr fp32 [B,K] (contiguous, 16-byte aligned; K a multiple
 * of 4, K <= 256), W_t [K,2], b_t [2]:
 *   esmm_head_fwd  z_t = h_t W_t + b_t (fp32 FMAs); p1_t = 1/(1+expf(z0-z1)), p0_t = 1/(1+expf(z1-z0))
 *                  each on its own; writes ctr_out = p_ctr [B,2], ctr_one = p1_ctr [B,1], cvr_out,
 *                  cvr_one likewise, ctcvr_one = p1_ctr p1_cvr [B,1], ctcvr_prop = [1-ctcvr_one,
 *                  ctcvr_one] [B,2].
 *   esmm_head_bwd  from the gradients of the six outputs (each may be NULL: no contribution) and the
 *                  saved p_ctr = ctr_out, p_cvr = cvr_out: Gc = g_ctcvr_prop[:,1] + g_ctcvr_one -
 *                  g_ctcvr_prop[:,0]; G_t = g_t_out + [0, g_t_one], G_ctr1 += Gc p1_cvr, G_cvr1 +=
 *                  Gc p1_ctr; s_t = p0_t p1_t (G_t1 - G_t0), dz_t = [-s_t, s_t].  Writes dh_t = dz_t
 *                  W_t^T [B,K] (no ReLU mask: the tower's backward applies it), dW_t [K,2] and db_t
 *                  [2], summed in a fixed order (no float atomics: bit-identical across runs). */
int b200rec_esmm_head_fwd(const float* h_ctr, const float* h_cvr, int K, const float* W_ctr,
                          const float* b_ctr, const float* W_cvr, const float* b_cvr, float* ctr_out,
                          float* ctr_one, float* cvr_out, float* cvr_one, float* ctcvr_prop,
                          float* ctcvr_one, int64_t B, void* stream);
int b200rec_esmm_head_bwd_workspace_bytes(int64_t B, int K, size_t* bytes_host);
int b200rec_esmm_head_bwd(const float* g_ctr_out, const float* g_ctr_one, const float* g_cvr_out,
                          const float* g_cvr_one, const float* g_ctcvr_prop,
                          const float* g_ctcvr_one, const float* p_ctr, const float* p_cvr,
                          const float* h_ctr, const float* h_cvr, int K, const float* W_ctr,
                          const float* W_cvr, float* dh_ctr, float* dh_cvr, float* dW_ctr,
                          float* db_ctr, float* dW_cvr, float* db_cvr, int64_t B, void* workspace,
                          size_t workspace_bytes, void* stream);
/* ---- CTR head (csrc/ctr_head.cuh) ------------------------------------------ */
/* pred = sigmoid(a + b + c) (b, c may be NULL) and its backward dlogit = dpred * p (1-p)
 * (deepfm/net.py:47: sigmoid(y_first_order + y_second_order + y_dnn)); the mean of Paddle's
 * log_loss (eps inside both logs, deepfm/dygraph_model.py:53-58) as one deterministic reduction
 * and its backward dpred = dloss/n * (-y/(p+eps) + (1-y)/(1-p+eps)).  label: float32 or int64
 * [n].  The loss workspace must be zero before its first use. */
int b200rec_sum_sigmoid_fwd(const float* a, const float* b, const float* c, float* pred, int64_t n,
                            void* stream);
int b200rec_sum_sigmoid_bwd(const float* pred, const float* dpred, float* dlogit, int64_t n,
                            void* stream);
int b200rec_log_loss_workspace_bytes(size_t* bytes_host);
int b200rec_log_loss_mean_fwd(const float* pred, const void* label, int label_is_i64, double eps,
                              float* loss, int64_t n, void* workspace, size_t workspace_bytes,
                              void* stream);
int b200rec_log_loss_mean_bwd(const float* pred, const void* label, int label_is_i64, double eps,
                              const float* dloss, float* dpred, int64_t n, void* stream);
/* paddle.metric.Auc.update on the device: stat_pos / stat_neg [num_thresholds+1] int64 histograms,
 * bucket = clamp(int(pred * num_thresholds)).  One launch, no host sync. */
int b200rec_auc_update(const float* pred, const void* label, int label_is_i64, int64_t* stat_pos,
                       int64_t* stat_neg, int num_thresholds, int64_t n, void* stream);
/* tuning / bring-up knobs (key 0: force tile width BN; 1-3: descriptor overrides of the dW kernel;
 * 4: k-block of the K-major kernel, 32 = 64-byte swizzle (the default), 64 = 128-byte swizzle,
 * fewer stages) and the device word a pipeline watchdog writes before it traps. */
int b200rec_tc_debug(int key, int value);
int b200rec_tc_timeout_word(unsigned int* word_host);

/* Backward of b200rec_din_attn_fwd.  Inputs as forward plus the saved softmax `weights` and
 * dout [B,E].  Outputs: dhist [B,L,E]; dtseq [B,E] = the (h*t)-path part of d/dtseq; dtb [B,80] =
 * d/d(tb); dWac, dWd [E,80]; dW2 [80,40]; db2 [40]; dW3 [40]; da [B,L] scratch (d/d(pre-mask
 * score)).  The caller finishes the t-path with two small library GEMMs:
 *   dtseq += dtb (Wb-Wc)^T,  Gt = tseq^T dtb,  dW1 = [dWac ; Gt ; dWac-Gt ; dWd],  db1 = sum_b dtb.
 * dtseq/dtb are accumulated with float atomics (a few adds per element; not bit-reproducible);
 * the weight gradients are reduced in a fixed order (deterministic). */
int b200rec_din_attn_bwd_workspace_bytes(int64_t B, int L, int E, size_t* bytes_host);
int b200rec_din_attn_bwd(const float* hist, const float* tseq, const float* tb, const float* Wac,
                         const float* Wd, const float* W2, const float* b2, const float* W3,
                         const float* weights, const float* dout, float* da, float* dhist,
                         float* dtseq, float* dtb, float* dWac, float* dWd, float* dW2, float* db2,
                         float* dW3, int64_t B, int L, int E, float scale, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---- continuous_value_model (GPUBox branch) -------------------------------- */
/* models/rank/wide_deep/net.py:81-88: x [N,D+2] (cols 0,1 = show, click).
 * use_cvm=1: y [N,D+2], y0=log(x0+1), y1=log(x1+1)-y0, rest copied; use_cvm=0: y [N,D] = x[:,2:].
 * backward: dx[:,2:] = dy[:, (2|0):], dx[:,0:2] = show_click[:,0:2]. */
int b200rec_cvm_fwd(const float* x, float* y, int64_t N, int D, int use_cvm, void* stream);
int b200rec_cvm_bwd(const float* dy, const float* show_click, float* dx, int64_t N, int D,
                    int use_cvm, void* stream);

/* ---- K5: row-cyclic sharding helpers (owner = id mod world) --------------- */
/* Stable bucketing of n ids by owner rank (bucket order = owner-major, original order inside).
 *   send_ids[k]   local row (id div world) of the k-th id in bucket order; -1 if out of range
 *   perm[i]       slot of position i in bucket order: rows_back[perm[i]] is the row of ids[i],
 *                 so `perm` is the `ids` argument of embed_fm_fwd / gather over the received rows
 *   inv_perm[k]   position held by slot k: the `sorted_pos` argument (with seg_offsets = iota)
 *                 that makes embed_fm_bwd / segment_reduce emit gradients in bucket order
 *   counts[r]     number of ids owned by rank r (device int64[world])
 * The padding id travels to its natural owner (padding_idx mod world), whose gather zeroes it. */
int b200rec_shard_bucketize_workspace_bytes(int64_t n, int world, size_t* bytes_host);
int b200rec_shard_bucketize(const int64_t* ids, int64_t n, int world, int64_t V, int64_t* send_ids,
                            int64_t* perm, int32_t* inv_perm, int64_t* counts, void* workspace,
                            size_t workspace_bytes, void* stream);

/* ---- K6: DLRM dot interaction (models/rank/dlrm/net.py:97-115) -----------------------------------
 * T [B, N, d]: the num_field embedding rows followed by the bottom-MLP output x as the LAST row.
 * R [B, d + P]: R[:, :d] = x; R[:, d+p] = <T_i, T_j> over the upper triangle in row-major order,
 * P = N(N-1)/2, or N(N+1)/2 with self_interaction — whose diagonal entries are 0, as the
 * reference's triu(Z,1)+tril(MIN_FLOAT,-1)+masked_select evaluates (net.py:105-113).
 * Backward: dT from dR (includes dR[:, :d] flowing into the x row).  N*(d+1)+N*N floats of shared
 * memory per sample in flight must fit (N <= 128, d <= 256 checked). */
int b200rec_dot_interact_fwd(const float* T, float* R, int64_t B, int N, int d, int self_interaction,
                             void* stream);
int b200rec_dot_interact_bwd(const float* T, const float* dR, float* dT, int64_t B, int N, int d,
                             int self_interaction, void* stream);

/* ---- uint64 feasigns -> table rows ----------------------------------------------------------------
 * The PS / GPUBox path of the reference keys its sparse table by raw uint64 feasigns
 * (tools/static_gpubox_trainer.py:152-159; `sparse_embedding` ignores its nominal size,
 * models/rank/dnn/benchmark_gpubox.yaml); the dygraph path folds tokens into [0, V) on the host with
 * a per-slot salted hash (models/rank/dnn/benchmark_reader.py:50-52).  This is that fold on the
 * device, so a dense [V, D] HBM table can serve hashed keys with no host pass:
 *   z      = keys[i] ^ ((slot_of_key ? slot_of_key[i] + 1 : 0) * 0x9E3779B97F4A7C15)
 *   z      = splitmix64-finaliser(z)     (z ^= z>>30; z *= 0xBF58476D1CE4E5B9; z ^= z>>27;
 *                                          z *= 0x94D049BB133111EB; z ^= z>>31)
 *   rows[i]= reserve_zero ? (keys[i] == 0 ? 0 : 1 + z mod (V-1)) : z mod V
 * reserve_zero keeps row 0 for "no feature" (feasign 0 is the padding key of the readers,
 * models/rank/deepfm/criteo_reader.py:48,86-88).  Collisions share a row, exactly like the
 * reference's `% hash_dim`.  HBM-bound: 16 (+4) bytes per key. */
int b200rec_hash_keys(const uint64_t* keys, const int32_t* slot_of_key, int64_t n, int64_t V,
                      int reserve_zero, int64_t* rows, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200REC_H_ */
