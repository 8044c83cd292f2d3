/*
 * matchmaker_b200 -- C ABI of the H100-native (sm_90a) interaction-scoring library.
 *
 * This is the drop-in boundary for the query-document interaction hot path of
 * sebastian-hofstaetter/matchmaker.  The reference is pure Python/PyTorch and has no FFI of
 * its own; each entry point below replaces the *inline arithmetic* of one reference method
 * (cited as path:line relative to the reference repository root) and is what a binding for
 * that method calls.  The Python host layer (matchmaker_b200/) binds these symbols with
 * ctypes; INTEGRATION.md shows the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary;
 *   - every function returns 0 (MMB200_OK) or a negative MMB200_ERR_* code;
 *     mmb200_last_error() returns a thread-local human-readable message for the last failure;
 *   - pointers whose name does not end in `_host` are DEVICE pointers valid on the CURRENT
 *     CUDA device of the calling thread; `stream` is a cudaStream_t (0 = legacy default);
 *     launches are asynchronous with respect to the host and ordered on `stream`;
 *   - tensors are dense row-major ("contiguous" in PyTorch terms) unless a stride is given;
 *   - the library never falls back to a CPU implementation: on a device that is not
 *     compute capability 9.0 every compute entry point fails with MMB200_ERR_UNSUPPORTED.
 */
#ifndef MATCHMAKER_B200_H_
#define MATCHMAKER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMB200_VERSION 100 /* 0.1.0 */

#if defined(__GNUC__)
#define MMB200_API __attribute__((visibility("default")))
#else
#define MMB200_API
#endif

/* error codes */
#define MMB200_OK 0
#define MMB200_ERR_INVALID (-1)     /* bad argument (shape, dtype, alignment, null pointer) */
#define MMB200_ERR_CUDA (-2)        /* a CUDA runtime / driver call failed */
#define MMB200_ERR_UNSUPPORTED (-3) /* device is not sm_90, or shape outside kernel limits */

/* element types of embedding / vector tensors */
#define MMB200_F16 0
#define MMB200_BF16 1
#define MMB200_F32 2
#define MMB200_F32_SPLIT16 3 /* mmb200_flat_ip_topk only: fp32 vectors held as fp16 hi / lo halves (see there) */
/* OCP E4M3 "fn" (torch.float8_e4m3fn: max +-448, no infinity), one byte per value.  Accepted by mmb200_flat_ip_topk,
 * mmb200_ivf_search_gather (and mmb200_ivf_workspace_bytes) and mmb200_maxsim_store_fwd, with both operands in it and
 * 128 <= dim <= 1024, dim % 128 == 0.  The products run on the FP8 tensor cores with fp32 accumulation and the
 * results are the plain sums of products of the stored values: with values stored as e4m3(x * 2^s), the caller
 * multiplies a score by 2^-(s_query + s_store) to return to the unscaled domain (exact; void scores stay as they are). */
#define MMB200_F8E4M3 4

/* element types of mask tensors (nonzero = real token, zero = padding) */
#define MMB200_MASK_NONE 0
#define MMB200_MASK_U8 1  /* torch.bool / uint8 */
#define MMB200_MASK_I32 2
#define MMB200_MASK_I64 3 /* HF attention_mask */
#define MMB200_MASK_F32 4 /* matchmaker `(tokens > 0).float()` masks */

/* kernel selection for entry points that have more than one device implementation */
#define MMB200_IMPL_AUTO 0
#define MMB200_IMPL_SIMT 1    /* CUDA-core kernel, any shape/dtype */
#define MMB200_IMPL_TCGEN05 2 /* TMA + wgmma tensor-core kernel (fails if shape unsupported); the name is historical */
#define MMB200_IMPL_TCGEN05_DOCM 3 /* max-sim only: the "documents on M" tensor-core kernel */
#define MMB200_IMPL_TCGEN05_RAGGED 4 /* max-sim only: alias of MMB200_IMPL_TCGEN05, kept for ABI compatibility.  The
                                        tensor-core max-sim kernel always fetches each document only up to its last
                                        unmasked row (padding rows never leave HBM) */

MMB200_API int mmb200_version(void);
MMB200_API const char* mmb200_last_error(void);

/* Properties of CUDA device `device` (-1 = current). Any out pointer may be NULL. */
MMB200_API int mmb200_device_info(int device, int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------
 * ColBERT late-interaction max-sim
 *
 *   score[p] = sum_{i < Lq, q_mask[qi][i]} max_{j < Ld} ( d_mask[di][j] ? <q[qi][i], d[di][j]> : -1000 )
 *
 * Replaces: ColBERT.forward scoring            matchmaker/models/colbert.py:68-75   (masks given)
 *           ColBERT.forward_aggregation        matchmaker/models/colbert.py:100-112 (masks NULL)
 *           ColBERT.forward_inbatch_aggregation matchmaker/models/colbert.py:154-162
 *               (all pairs: n_pairs = n_q * n_d, pair_q[p] = p / n_d, pair_d[p] = p % n_d; its
 *                backward is mmb200_maxsim_allpairs_bwd below)
 *
 * q      [n_q, Lq, dim]  dtype `dtype`
 * d      [n_d, Ld, dim]  dtype `dtype`
 * q_mask [n_q, Lq] or NULL, d_mask [n_d, Ld] or NULL, element type `mask_dtype`
 * pair_q / pair_d [n_pairs] int32 or NULL.  With NULL: qi = p / docs_per_query, di = p
 *        (docs_per_query = 1 is the training/re-ranking case "pair p = query p x doc p";
 *         docs_per_query = 1000 is BASELINE config 3 "1 query x 1000 docs").
 * pair_dmask [n_pairs] int32 or NULL: row of d_mask applied to pair p (default di).  Exists only
 *        to reproduce colbert.py:158, which indexes the document mask by the QUERY position.
 * out    [n_pairs] float32
 * argmax [n_pairs, Lq] int32 or NULL: index j* of the max per query token (-1 when the query
 *        token is masked or every document position is masked) -- what backward needs.
 * A tensor with no elements may be passed as NULL: an empty batch (n_q = n_d = n_pairs = 0) returns 0 and launches
 * nothing.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_maxsim_fwd(const void* q, const void* d, const void* q_mask, const void* d_mask,
                      const int32_t* pair_q, const int32_t* pair_d, const int32_t* pair_dmask,
                      float* out, int32_t* argmax,
                      int64_t n_q, int64_t n_d, int64_t n_pairs, int32_t docs_per_query, int32_t Lq,
                      int32_t Ld, int32_t dim, int32_t dtype, int32_t mask_dtype, int32_t impl,
                      void* stream);

/* Backward of mmb200_maxsim_fwd (pairs mode with pair_q = pair_d = NULL, docs_per_query >= 1).
 * grad_out [n_pairs] f32; argmax from the forward; grad_q [n_q, Lq, dim] f32 and
 * grad_d [n_d, Ld, dim] f32 are OVERWRITTEN (zero-filled then accumulated).
 * Mirrors what autograd derives from colbert.py:68-75 (gradient flows only through the max
 * element; masked query tokens and fully masked documents get none).  A tensor with no elements may be NULL; with
 * n_q = n_d = 0 nothing is written. */
MMB200_API int mmb200_maxsim_bwd(const void* q, const void* d, const float* grad_out, const int32_t* argmax,
                      float* grad_q, float* grad_d, int64_t n_q, int64_t n_d, int64_t n_pairs,
                      int32_t docs_per_query, int32_t Lq, int32_t Ld, int32_t dim, int32_t dtype,
                      void* stream);

/* Backward of all-pairs scoring: mmb200_maxsim_fwd with n_pairs = n_q * n_d, pair_q[p] = p / n_d, pair_d[p] = p % n_d
 * (any pair_dmask), so pair p = a * n_d + b is query a against document b and every document is shared by all queries.
 * grad_out [n_q, n_d] f32; argmax [n_q * n_d, Lq] int32 from that forward (-1: no gradient);
 *   grad_q[a][i] = sum_b g[a,b] * d[b][argmax[a,b,i]]                       (ascending b)
 *   grad_d[b][r] = sum over (a, i) with argmax[a,b,i] = r of g[a,b] * q[a][i]  (ascending (a, i))
 * grad_q [n_q, Lq, dim] and grad_d [n_d, Ld, dim] f32 are OVERWRITTEN; a row no argmax points at is 0.  No atomics:
 * two runs give the same bits, and with n_q = 1 they are those of mmb200_maxsim_bwd(docs_per_query = n_d).
 * n_q * n_d < 2^31.  A tensor with no elements may be NULL; with n_q = 0 or n_d = 0 the other side's gradient is
 * zero-filled and no kernel runs. */
MMB200_API int mmb200_maxsim_allpairs_bwd(const void* q, const void* d, const float* grad_out, const int32_t* argmax,
                                          float* grad_q, float* grad_d, int64_t n_q, int64_t n_d, int32_t Lq,
                                          int32_t Ld, int32_t dim, int32_t dtype, void* stream);

/* Host-buffer variant (the end-to-end call): all pointers are HOST pointers (pinned memory
 * gives full PCIe bandwidth, pageable works).  Documents are streamed to the device in chunks
 * on internal streams, overlapped with the kernel; scores are copied back before returning.
 * Synchronous.  Same semantics as mmb200_maxsim_fwd with pair_q = pair_d = NULL.
 * chunk_pairs: documents per slab; 0 or -1 = default slab size (~96 MB). */
MMB200_API int mmb200_maxsim_fwd_host(const void* q_host, const void* d_host, const void* q_mask_host,
                           const void* d_mask_host, float* out_host, int64_t n_q, int64_t n_d,
                           int32_t docs_per_query, int32_t Lq, int32_t Ld, int32_t dim, int32_t dtype,
                           int32_t mask_dtype, int64_t chunk_pairs);

/* Store mode: max-sim against a ragged token store (passages keep only their real token rows, as the reference's
 * encode loop writes them, matchmaker/dense_retrieval.py:244), ColBERT.forward_aggregation semantics
 * (colbert.py:100-112, no masks):
 *
 *   out[p] = sum_{i < Lq} max_{off[d] <= r < off[d+1]} <q[pair_q[p]][i], store[r]>,   d = pair_d[p]
 *
 * store [n_rows, dim]; doc_offsets [n_docs + 1] int64, non-decreasing, doc_offsets[n_docs] <= n_rows (passage d is
 * rows [off[d], off[d+1]); empty ranges allowed; at most max_doc_len rows of a passage are read).
 * q [n_q, Lq, dim]; pair_q / pair_d [n_pairs] int32; pair_d[p] < 0 skips the pair (nothing is fetched) and, like a
 * passage without rows, scores -inf.  dtype / impl as mmb200_maxsim_fwd (AUTO picks the kernel it would pick for
 * the padded [n_docs, max_doc_len, dim] layout; scores are bit-identical to that layout with masks).  The tensor-core
 * kernels address the store with the passage's first row as the TMA row coordinate: n_rows < 2^31 - 1024.
 * dtype MMB200_F8E4M3 (q and store): the documents-on-M tensor-core kernel only (impl AUTO or
 * MMB200_IMPL_TCGEN05_DOCM; any other impl is MMB200_ERR_UNSUPPORTED), 1 <= Lq <= 128, dim % 128 == 0,
 * 128 <= dim <= 1024 (outside: MMB200_ERR_INVALID); scores in the scaled domain (see MMB200_F8E4M3). */
MMB200_API int mmb200_maxsim_store_fwd(const void* q, const void* store, const int64_t* doc_offsets,
                                       const int32_t* pair_q, const int32_t* pair_d, float* out, int64_t n_q,
                                       int64_t n_rows, int64_t n_docs, int64_t n_pairs, int32_t Lq, int32_t max_doc_len,
                                       int32_t dim, int32_t dtype, int32_t impl, void* stream);

/* ------------------------------------------------------------------------------------------
 * Cosine match matrix + RBF kernel pooling (KNRM / TK)
 *
 *   c_ij  = <q_i/(|q_i|+1e-13), d_j/(|d_j|+1e-13)>
 *   S_ik  = sum_j d_mask[j] * exp(-(c_ij - mu_k)^2 / (2 sigma_k^2))
 *   P_k   = sum_i q_mask[i] * log_scale * log(max(alpha_k * S_ik, 1e-10))
 *   score = sum_k weight_k * P_k
 *
 * Replaces: KNRM.forward        matchmaker/models/knrm.py:52-84        (alpha = NULL, log_scale = 0.01)
 *           ECAI20_TK.forward   matchmaker/models/published/ecai20_tk.py:105-124 (log_scale = 1)
 *           CosineMatrixAttention (allennlp 2.5.1, third party) at knrm.py:60, ecai20_tk.py:105
 *
 * q [B,Lq,D] f32, d [B,Ld,D] f32 (D % 4 == 0, 16-byte aligned); q_mask [B,Lq], d_mask [B,Ld] of
 * `mask_dtype` (matchmaker passes float masks: MMB200_MASK_F32); mu, sigma, weight [K] f32 device
 * arrays, alpha [K] or NULL (= 1); K <= 32.  B == 0 is valid (the per-pair pointers may then be NULL): nothing runs,
 * and every backward of this family sets grad_weight / grad_alpha to 0.
 * Outputs (any of per_kernel / per_kernel_query / cosine may be NULL):
 *   score [B]; per_kernel [B,K] (= P); per_kernel_query [B,Lq,K] (= S, what backward needs);
 *   cosine [B,Lq,Ld] = c_ij * q_mask[i] * d_mask[j] (the reference's secondary output).
 * impl: MMB200_IMPL_AUTO / _TCGEN05 take the tensor-core kernel for K <= 32, Lq <= 128, cosine == NULL (queries longer
 * than 32 terms: one pass per block of 32 query rows), _SIMT the FFMA kernel (any Lq).
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_kernel_pool_fwd(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                      const float* mu, const float* sigma, const float* alpha,
                                      const float* weight, float* score, float* per_kernel,
                                      float* per_kernel_query, float* cosine, int64_t B, int32_t Lq,
                                      int32_t Ld, int32_t D, int32_t K, float log_scale, int32_t mask_dtype,
                                      int32_t impl, void* stream);

/* Backward of mmb200_kernel_pool_fwd for d(loss)/d(score) = grad_score [B]:
 *   grad_q [B,Lq,D], grad_d [B,Ld,D] (overwritten), grad_alpha [K] or NULL, grad_weight [K]
 *   (overwritten; summed over the batch deterministically via `workspace` [2*B*K] f32).
 * per_kernel_query is S from the forward.  Matches autograd of the reference expression
 * (clamp passes gradient when alpha*S >= 1e-10; rows with |x| = 0 get no normalisation term). */
MMB200_API int mmb200_kernel_pool_bwd(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                      const float* mu, const float* sigma, const float* alpha,
                                      const float* weight, const float* per_kernel_query,
                                      const float* grad_score, float* grad_q, float* grad_d,
                                      float* grad_alpha, float* grad_weight, float* workspace, int64_t B,
                                      int32_t Lq, int32_t Ld, int32_t D, int32_t K, float log_scale,
                                      int32_t mask_dtype, void* stream);

/* Variants of the same pooling (SURVEY 8(f) row 3) -- mmb200_kernel_pool_fwd / _bwd are these with doc_gate = NULL,
 * clamp_min = 1e-10, score_bias = 0:
 *   doc_gate [B, Ld] f32 or NULL: multiplier of every activation of document term j (negative values count as 0),
 *            S_ik = sum_j d_mask[j] * doc_gate[j] * exp(...).  Replaces the `* document_stop_words` of
 *            CIKM20_TK_Sparse.forward, matchmaker/models/published/cikm20_tk_sparse.py:135.
 *   clamp_min: floor of alpha_k * S_ik before the log.  IDCM's ESM patch scorer uses 1e-4
 *            (matchmaker/models/published/sigir21_idcm.py:185).
 *   score_bias: added to the score (the bias of IDCM's `sampling_binweights` Linear(11, 1), sigir21_idcm.py:100,186).
 *   Conv-KNRM's n x n cross matches (matchmaker/models/conv_knrm.py:125-135) are n*n calls with log_scale = 0.01, each
 *   taking its K-slice of dense.weight (Linear over a concatenation = sum of per-block Linears).
 * Backward additionally returns grad_gate [B, Ld] (or NULL): d(loss)/d(doc_gate). */
MMB200_API int mmb200_kernel_pool_fwd_ex(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                         const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                         const float* weight, float* score, float* per_kernel, float* per_kernel_query,
                                         float* cosine, int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K,
                                         float log_scale, float clamp_min, float score_bias, int32_t mask_dtype,
                                         int32_t impl, void* stream);
/* Store mode of mmb200_kernel_pool_fwd_ex (inference only): documents are read from a store of live rows that was
 * encoded once (TK / TK-Sparse document contextualisation does not depend on the query):
 *
 *   score[p] = mmb200_kernel_pool_fwd_ex of query pair_q[p] against the rows doc_offsets[d] .. doc_offsets[d+1] - 1
 *              of `store` (at most max_doc_len of them), d = pair_d[p], every row unmasked
 *
 * store [n_rows, D] f32; doc_offsets [n_docs + 1] int64, non-decreasing, doc_offsets[n_docs] <= n_rows; q [n_q, Lq, D]
 * f32, q_mask [n_q, Lq] (mask_dtype) or NULL; pair_q / pair_d [n_pairs] int32, pairs of one query adjacent for L2 reuse
 * of its rows (any order is correct).  gate [n_rows] f32 in store order or NULL: the doc_gate of the row (TK-Sparse).
 * pair_d[p] < 0 and a passage without rows score -inf and fetch nothing.  impl as mmb200_kernel_pool_fwd_ex: AUTO
 * picks the kernel it would pick for the padded [n_docs, max_doc_len, D] layout, and scores are bit-identical to that
 * layout with the passages' rows unmasked and the rest masked.  The tensor-core kernel addresses the store with the
 * passage's first row as the TMA row coordinate: n_rows < 2^31 - 1024. */
MMB200_API int mmb200_kernel_pool_store_fwd(const float* q, const void* q_mask, const float* store,
                                            const int64_t* doc_offsets, const float* gate, const int32_t* pair_q,
                                            const int32_t* pair_d, const float* mu, const float* sigma,
                                            const float* alpha, const float* weight, float* score, int64_t n_q,
                                            int64_t n_rows, int64_t n_pairs, int32_t Lq, int32_t max_doc_len,
                                            int32_t D, int32_t K, float log_scale, float clamp_min, float score_bias,
                                            int32_t mask_dtype, int32_t impl, void* stream);
MMB200_API int mmb200_kernel_pool_bwd_ex(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                         const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                         const float* weight, const float* per_kernel_query, const float* grad_score,
                                         float* grad_q, float* grad_d, float* grad_gate, float* grad_alpha,
                                         float* grad_weight, float* workspace, int64_t B, int32_t Lq, int32_t Ld,
                                         int32_t D, int32_t K, float log_scale, float clamp_min, int32_t mask_dtype,
                                         void* stream);

/* Training pair on the tensor cores (the step of train.py:330-360 for KNRM / TK: forward, loss, backward).
 *   mmb200_kernel_pool_fwd_train = mmb200_kernel_pool_fwd_ex (tensor-core kernel; doc_gate as there, or NULL) that additionally leaves
 *   `saved` for the backward: mmb200_kernel_pool_saved_floats(B, Ld) = B * (33 * Ld + 32) floats, 16-byte aligned
 *   (cosines document-row-major [B][Ld][32], then 1 / (|d_j| + eps) [B][Ld], then 1 / (|q_i| + eps) [B][32]); the
 *   layout is private to the pair of calls.
 *   mmb200_kernel_pool_bwd_saved = mmb200_kernel_pool_bwd_ex (doc_gate / grad_gate as there, or NULL) computed from `saved` with both contractions
 *   (G q^ and G^T d^) as tf32 wgmma on the raw fp32 embeddings; gradients agree with the fp32 expression to a few
 *   1e-4 relative (tf32 operands; the reference trains under fp16 autocast).  grad_q / grad_d must be 16-byte aligned.
 *   Envelope: mmb200_kernel_pool_train_tc_supported(Lq, Ld, D, K) != 0  (Lq <= 32, K <= 32; D % 4 == 0 and D <= 320, or
 *   D % 64 == 0 and 512 < D <= 1024: the BERT-base / -large widths); outside it both calls return MMB200_ERR_UNSUPPORTED
 *   and the caller uses _fwd_ex / _bwd_ex (which stops at D <= 512).
 *   `workspace` of mmb200_kernel_pool_bwd_saved: mmb200_kernel_pool_bwd_saved_workspace_floats(B, Lq, Ld, D, K) floats,
 *   16-byte aligned.  That is 2 * B * K (as for _bwd_ex) up to D = 320; at 512 < D <= 1024 it also holds the backward's
 *   per-pair G matrices, B * (65 * Ldp + 32) floats more with Ldp = Ld rounded up to 64. */
MMB200_API int32_t mmb200_kernel_pool_train_tc_supported(int32_t Lq, int32_t Ld, int32_t D, int32_t K);
MMB200_API int64_t mmb200_kernel_pool_saved_floats(int64_t B, int32_t Ld);
MMB200_API int64_t mmb200_kernel_pool_bwd_saved_workspace_floats(int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K);
MMB200_API int mmb200_kernel_pool_fwd_train(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                            const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                            const float* weight, float* score, float* per_kernel, float* per_kernel_query, float* saved,
                                            int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K, float log_scale,
                                            float clamp_min, float score_bias, int32_t mask_dtype, void* stream);
MMB200_API int mmb200_kernel_pool_bwd_saved(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                            const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                            const float* weight, const float* per_kernel_query, const float* saved,
                                            const float* grad_score, float* grad_q, float* grad_d, float* grad_gate,
                                            float* grad_alpha, float* grad_weight,
                                            float* workspace, int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K,
                                            float log_scale, float clamp_min, int32_t mask_dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * BERT_DOT pair scoring: out[b] = <q[b], d[b]>, fp32 accumulate.
 * Replaces: BERT_Dot.forward   matchmaker/models/bert_dot.py:62  (bmm([B,1,dim],[B,dim,1]))
 * q, d [B, dim] of `dtype`; out [B] f32.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_dot_pairs(const void* q, const void* d, float* out, int64_t B, int32_t dim,
                                int32_t dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * TKL (long documents): per-chunk cosine + RBF kernels, sliding-window kernel pooling with learned
 * saturation, window scores; then the greedy top-3 window selection.
 *
 * Replaces: TKL_sigir20.forward   matchmaker/models/published/sigir20_tkl.py:180-252 (window scores)
 *                                 matchmaker/models/published/sigir20_tkl.py:254-286 (top hills)
 * Chunking / packing / contextualisation (:136-175) stay in PyTorch, as in the reference.
 *
 * q             [B, Lq, D] f32  contextualised, masked query embeddings (Lq <= 40)
 * q_mask        [B, Lq] (`mask_dtype`)
 * chunks        [Nc, 40, D] f32 contextualised packed chunks, overlap removed (:174)
 * chunk_mask    [Nc, 40]
 * slot_to_packed [B*C] int32: packed index of chunk slot (b, c), -1 where the reference's
 *               `packed_indices` (:159) dropped the chunk
 * mu, sigma, dense_w [K] (K <= 16)
 * saturation 0 ("embedding", :222-234): sat_red_w [D] = sat_emb_reduce1.weight, sat_params[13] =
 *               {sat_normer.weight[2], sat_normer.bias[2], saturation_linear.weight[2], .bias,
 *                saturation_linear2.weight[2], .bias, saturation_linear3.weight[2], .bias}
 * saturation 1 ("log", :245-246): sat_params[K] = kernel_mult[0]
 * window_score  [B, W] f32 out, W = (C*40 - 30)/2 + 1  (raw dense output, sentinel not yet applied)
 * n_chunks      Nc (rows of `chunks` / `chunk_mask`)
 * impl          MMB200_IMPL_AUTO: the TMA + wgmma kernel (Lq * K <= 512) when the kernel set activates on every cosine
 *               in [-1, 1] -- decided on the device, no host sync -- else the FFMA kernel; _TCGEN05 / _SIMT force one.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_tkl_window_scores(const float* q, const void* q_mask, const float* chunks,
                                        const void* chunk_mask, const int32_t* slot_to_packed,
                                        const float* mu, const float* sigma, const float* dense_w,
                                        const float* sat_red_w, const float* sat_params,
                                        float* window_score, int64_t B, int64_t n_chunks, int32_t Lq, int32_t D,
                                        int32_t C, int32_t K, int32_t saturation, int32_t mask_dtype, int32_t impl,
                                        void* stream);

/* Store mode of mmb200_tkl_window_scores (inference only): the chunks come from a store of passages that were chunked,
 * packed and contextualised once (TKL contextualises every packed chunk alone, so a chunk does not depend on the query
 * or on the rest of the batch):
 *
 *   window_score[p] = mmb200_tkl_window_scores of query pair_q[p] against the chunk slots doc_slots[pair_d[p], 0..C-1]
 *
 * q [n_q, Lq, D] f32, q_mask [n_q, Lq] (mask_dtype) or NULL; chunks [n_chunks, 40, D] f32, chunk_mask [n_chunks, 40]
 * (mask_dtype) or NULL; doc_slots [n_docs, C] int32: the store index of passage d's chunk in slot c, -1 where the
 * packing dropped the slot or the passage is shorter; pair_q / pair_d [n_pairs] int32, pair_d[p] < 0 = no slots (its
 * windows are all 0); window_score [n_pairs, W] out, W = (C*40 - 30)/2 + 1.  Everything else as
 * mmb200_tkl_window_scores, including the routing of impl; the windows are bit-identical to that entry's on the same
 * chunks gathered into the padded layout with q[pair_q] (same impl).  mmb200_tkl_top_hills selects on the result. */
MMB200_API int mmb200_tkl_store_window_scores(const float* q, const void* q_mask, const float* chunks,
                                              const void* chunk_mask, const int32_t* doc_slots, const int32_t* pair_q,
                                              const int32_t* pair_d, const float* mu, const float* sigma,
                                              const float* dense_w, const float* sat_red_w, const float* sat_params,
                                              float* window_score, int64_t n_q, int64_t n_chunks, int64_t n_docs,
                                              int64_t n_pairs, int32_t Lq, int32_t D, int32_t C, int32_t K,
                                              int32_t saturation, int32_t mask_dtype, int32_t impl, void* stream);

/* window_score [B,W] in; orig_score [B,W] out (may be the same buffer): the reference's "orig_score" (exact zeros ->
 * -9900 sentinel during selection, written back as 0).  chunk_scoring [15]; top_idx [B,3] int64;
 * top15 [B,15] ("top_k_non_overlapping"); score [B]. */
MMB200_API int mmb200_tkl_top_hills(const float* window_score, float* orig_score, const float* chunk_scoring,
                                    int64_t* top_idx, float* top15, float* score, int64_t B, int32_t W, void* stream);

/* slot_to_packed [n_slots] int32 from the reference's chunk packing mask `packed_indices` (sigir20_tkl.py:159, one
 * byte per chunk slot, n_slots = B*C): the packed index of the slot, -1 where the chunk was dropped. */
MMB200_API int mmb200_tkl_slot_map(const void* packed_mask, int32_t* slot_to_packed, int64_t n_slots, void* stream);

/* Backward of the TKL interaction stage (mmb200_tkl_window_scores + mmb200_tkl_top_hills) for
 * d(loss)/d(score) = grad_score [B]: what autograd derives from sigir20_tkl.py:180-286.  Only the <= 15
 * gathered windows per document carry gradient.
 * top_idx [B,3], orig_score [B,W]: outputs of mmb200_tkl_top_hills.
 * grad_q [B,Lq,D] and grad_chunks [n_chunks,40,D] are overwritten.
 * grad_params [K + 15 + (saturation == 0 ? 13 + D : K)]: d dense_w | d chunk_scoring | d sat_params |
 *   d sat_emb_reduce1.weight (embedding saturation only); summed over the batch in a fixed order.
 * workspace: B * (that length) floats. */
MMB200_API int mmb200_tkl_bwd(const float* q, const void* q_mask, const float* chunks, const void* chunk_mask,
                              const int32_t* slot_to_packed, const float* mu, const float* sigma,
                              const float* dense_w, const float* sat_red_w, const float* sat_params,
                              const float* chunk_scoring, const int64_t* top_idx, const float* orig_score,
                              const float* grad_score, float* grad_q, float* grad_chunks, float* grad_params,
                              float* workspace, int64_t B, int64_t n_chunks, int32_t Lq, int32_t D, int32_t C,
                              int32_t K, int32_t saturation, int32_t mask_dtype, void* stream);

/* The same backward with shared memory independent of D, for BERT-width embeddings (DESIGN 3.3c): same arguments and
 * outputs as mmb200_tkl_bwd; the work is split by 64-feature blocks over the union of the positions that the gathered
 * windows cover (<= 114 per document), with fp32 FFMA throughout.
 *   Envelope: 1 <= Lq <= 40, 1 <= K <= 16, D a multiple of 4 with 4 <= D <= 1024, C >= 1, either saturation; outside it
 *   the call returns MMB200_ERR_UNSUPPORTED before any launch.
 *   workspace: mmb200_tkl_bwd_wide_workspace_floats(B, D, K, saturation) floats (the per-document parameter partials,
 *   then the per-feature-block partial products and the per-document gradient coefficients).
 * No allocation and no synchronisation; every output has one writer and one summation order, so two runs give the same
 * bits and the call can be captured in a CUDA graph. */
MMB200_API int mmb200_tkl_bwd_wide(const float* q, const void* q_mask, const float* chunks, const void* chunk_mask,
                                   const int32_t* slot_to_packed, const float* mu, const float* sigma,
                                   const float* dense_w, const float* sat_red_w, const float* sat_params,
                                   const float* chunk_scoring, const int64_t* top_idx, const float* orig_score,
                                   const float* grad_score, float* grad_q, float* grad_chunks, float* grad_params,
                                   float* workspace, int64_t B, int64_t n_chunks, int32_t Lq, int32_t D, int32_t C,
                                   int32_t K, int32_t saturation, int32_t mask_dtype, void* stream);
MMB200_API int64_t mmb200_tkl_bwd_wide_workspace_floats(int64_t B, int32_t D, int32_t K, int32_t saturation);

/* Which TKL backward takes (Lq, D, K), on sm_90a's 227 KB of opt-in shared memory per block (a pure function of the
 * shape): 1 = mmb200_tkl_bwd (its one-CTA-per-document plan fits: D <= 356), 2 = mmb200_tkl_bwd_wide (up to D = 1024),
 * 0 = neither. */
MMB200_API int32_t mmb200_tkl_bwd_route(int32_t Lq, int32_t D, int32_t K);

/* ------------------------------------------------------------------------------------------
 * Exact maximum-inner-product search with fused per-query top-k (BERT_DOT dense retrieval scoring)
 *
 * Replaces: FaissIdIndexer / FaissBaseIndexer.search   matchmaker/retrieval/faiss_indices.py:27,34,49-74
 *           (faiss.IndexIDMap(IndexFlatIP), GPU-sharded, useFloat16), called from
 *           matchmaker/dense_retrieval.py:328 (index) and :391 (search).
 *
 * queries  [nq, dim], passages [n_pass, dim]: fp16 or bf16 (`dtype`), dim % 64 == 0, row-major,
 *          resident on the current device (one shard per GPU); fp32 accumulate on the tensor cores.
 *          dtype MMB200_F32_SPLIT16 (faiss without useFloat16, faiss_indices.py:65,72: fp32 storage): every fp32
 *          value x (pre-scaled by a power of two so that |x| < 2^15) is held as hi = fp16(x), lo = fp16(x - hi);
 *          passages [n_pass, 2*dim] = [hi | lo], queries [nq, 3*dim] = [hi | lo | hi]; the kernel runs 3*dim/64
 *          k-blocks pairing q_hi.p_hi + q_lo.p_hi + q_hi.p_lo (22 mantissa bits per operand, fp32 accumulate) and
 *          returns scores in the scaled domain (the caller multiplies by 2^-(sq+sp), exact).
 * ids      [n_pass] int64 user ids (add_with_ids) or NULL: id = id_base + row.
 * out_scores [nq, k] f32 descending; out_ids [nq, k] int64; ties ordered by id ascending (faiss leaves
 *          tie order unspecified); when n_pass < k the tail is (-3.4028235e38, -1) as in faiss.
 * workspace: device scratch of at least mmb200_flat_ip_workspace_bytes(nq, n_pass, k) bytes.
 * 1 <= k <= 1024 (k <= 256: 1024-entry candidate lists per query row; larger k: 2048-entry lists).
 * dtype MMB200_F8E4M3: queries and passages [., dim] e4m3, dim % 128 == 0, 128 <= dim <= 1024 (outside:
 *          MMB200_ERR_INVALID); scores in the scaled domain (see MMB200_F8E4M3).
 * ------------------------------------------------------------------------------------------ */
MMB200_API int64_t mmb200_flat_ip_workspace_bytes(int64_t nq, int64_t n_pass, int32_t k);
/* The work decomposition mmb200_flat_ip_topk uses on a device with `sm_count` SMs (pure host arithmetic, no device
 * needed): out[0] query blocks of 128, out[1] passage tiles of 256, out[2] passage ranges, out[3] tiles per range,
 * out[4] grid (CTAs, a multiple of the cluster size), out[5] cluster size, out[6..7] workspace bytes (low, high 32
 * bits).  Returns 0, or MMB200_ERR_INVALID for sizes mmb200_flat_ip_topk would reject. */
MMB200_API int mmb200_flat_ip_plan(int64_t nq, int64_t n_pass, int32_t k, int32_t sm_count, int32_t out[8]);
MMB200_API int mmb200_flat_ip_topk(const void* queries, const void* passages, const int64_t* ids,
                                   float* out_scores, int64_t* out_ids, void* workspace,
                                   int64_t workspace_bytes, int64_t nq, int64_t n_pass, int32_t dim, int32_t k,
                                   int32_t dtype, int64_t id_base, void* stream);

/* Merge candidate lists: cand_scores / cand_ids [nq, n_candidates] -> the k best per query under (score desc,
 * id asc).  A candidate is void when its SCORE is NaN, -inf or -FLT_MAX (faiss's "no result"); ids may be any int64,
 * negative user ids included (faiss IndexIDMap allows them).  Any n_candidates: more than 8192 per query are merged
 * in passes.  Used after the NCCL all-gather of per-rank top-k lists (the reference merges faiss IndexShards results on
 * the host). */
MMB200_API int mmb200_topk_merge(const float* cand_scores, const int64_t* cand_ids, float* out_scores,
                                 int64_t* out_ids, int64_t nq, int32_t n_candidates, int32_t k, void* stream);

/* Per-query de-duplication + top-k: the k best DISTINCT ids of cand_scores / cand_ids [nq, n_candidates], each id with
 * its highest score, ordered by (score desc, id asc).  Void candidates, any n_candidates (passes over groups of 8192)
 * and the (-FLT_MAX, -1) tail are as in mmb200_topk_merge.  1 <= k <= 4096; larger k returns MMB200_ERR_UNSUPPORTED.
 * Replaces the per-passage de-duplication loop of the maxP aggregation, matchmaker/dense_retrieval.py:414-427, and
 * builds the candidate passage lists of ColBERT end-to-end retrieval. */
MMB200_API int mmb200_topk_unique(const float* cand_scores, const int64_t* cand_ids, float* out_scores,
                                  int64_t* out_ids, int64_t nq, int32_t n_candidates, int32_t k, void* stream);

/* ------------------------------------------------------------------------------------------
 * Inverted-file (IVF) search: exact top-k over the rows of each query's probed lists
 *
 * Replaces: FaissIVFIndexer.search   matchmaker/retrieval/faiss_indices.py:106-145
 *           (faiss IndexIVFFlat / IndexIVFScalarQuantizer QT_fp16, METRIC_INNER_PRODUCT, GPU).
 *
 * rows     [n_rows, dim] (fp16 / bf16) or [n_rows, 2*dim] (MMB200_F32_SPLIT16, as for mmb200_flat_ip_topk): the
 *          index rows sorted by list; list l is rows [list_offsets[l], list_offsets[l+1]) (int64 [nlist + 1],
 *          non-decreasing, list_offsets[nlist] <= n_rows).  ids [n_rows] int64 user ids of those rows (any value).
 * queries  [nq, dim] in the rows' dtype ([nq, 3*dim] for MMB200_F32_SPLIT16; scores are then in the scaled domain).
 * probes   [nq, nprobe] int64 list ids, distinct within a row; an id outside [0, nlist) (the -1 filler of a coarse
 *          search over fewer than nprobe lists) probes nothing.
 * max_list_len: an upper bound of every list's length; a query's candidates from one list are kept in a slot of
 *          min(k, max_list_len) rounded up to 32 entries.  A list longer than the bound loses candidates (no fault).
 * out_scores / out_ids [nq, k]: the k best rows of the union of the probed lists under (score desc, id asc); fewer
 *          than k rows give the (-3.4028235e38, -1) tail.
 * The probe table is inverted on the device into per-list query sets; every (list, chunk of <= 128 probing queries) is
 * one work item of the flat-IP tensor-core kernel, which reads the list once per chunk.  No host synchronisation.
 * Envelope: 1 <= k <= 1024, 1 <= nprobe <= 1024, dim % 64 == 0, n_rows < 2^31 - 128, nq * nprobe < 2^31 - 128,
 * 16-byte aligned queries and rows.  Outside it: MMB200_ERR_INVALID.  Not sm_90: MMB200_ERR_UNSUPPORTED.
 * workspace: device scratch of at least mmb200_ivf_workspace_bytes(...) bytes, about nq * nprobe * (2 * qcols + 12 *
 * slot) bytes (qcols = dim, or 3 * dim for the split); 0 = sizes outside the envelope, -1 = no device.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int64_t mmb200_ivf_workspace_bytes(int64_t nq, int32_t nprobe, int64_t nlist, int64_t max_list_len,
                                              int32_t dim, int32_t k, int32_t dtype);
MMB200_API int mmb200_ivf_search(const void* queries, const void* rows, const int64_t* ids,
                                 const int64_t* list_offsets, const int64_t* probes, float* out_scores,
                                 int64_t* out_ids, void* workspace, int64_t workspace_bytes, int64_t nq,
                                 int32_t nprobe, int64_t nlist, int64_t n_rows, int64_t max_list_len, int32_t dim,
                                 int32_t k, int32_t dtype, void* stream);

/* The same search over rows that are NOT sorted by list: list position p (list l is positions
 * [list_offsets[l], list_offsets[l+1])) is row row_index[p] of `rows`.  row_index [list_offsets[nlist]] int64, each
 * entry in [0, n_rows); ids [n_rows] are indexed by row, not by list position.  Every other argument, the result and
 * the envelope are those of mmb200_ivf_search, including the workspace (mmb200_ivf_workspace_bytes).  This lets one
 * passage-ordered copy of the rows (ColBERT's token store) serve an inverted-file scan and per-passage scoring: the
 * scan gathers each tile's rows with 16-byte cp.async copies instead of one TMA box.
 * dtype MMB200_F8E4M3 (queries and rows e4m3, dim % 128 == 0, 128 <= dim <= 1024) is accepted here and by
 * mmb200_ivf_workspace_bytes, not by mmb200_ivf_search; scores in the scaled domain (see MMB200_F8E4M3). */
MMB200_API int mmb200_ivf_search_gather(const void* queries, const void* rows, const int64_t* ids,
                                        const int64_t* row_index, const int64_t* list_offsets, const int64_t* probes,
                                        float* out_scores, int64_t* out_ids, void* workspace, int64_t workspace_bytes,
                                        int64_t nq, int32_t nprobe, int64_t nlist, int64_t n_rows,
                                        int64_t max_list_len, int32_t dim, int32_t k, int32_t dtype, void* stream);

/* Spherical k-means centroid update: out[l] = normalised mean of rows perm[offsets[l] .. offsets[l+1]) of x
 * ([n, dim] fp16 / bf16 / fp32, `dtype`).  The sum runs in that order in fp64, so the result is bit-reproducible;
 * an empty list gives a zero row.  perm [offsets[nlist]] int64, out [nlist, dim] f32.  1 <= dim <= 4096, else
 * MMB200_ERR_INVALID. */
MMB200_API int mmb200_ivf_list_means(const void* x, const int64_t* perm, const int64_t* offsets, float* out,
                                     int64_t nlist, int32_t dim, int32_t dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Residual token codes (ColBERT IVF retrieval over a compressed store)
 *
 * Row r of list l = list_ids[r] is kept as `bits` (1 or 2) bits per dimension:
 *   code[d]  = #{i : cutoff[d][i] <= float(x[d]) - float(base[l][d])}     (fp32 arithmetic)
 *   value[d] = fp16_rn(float(base[l][d]) + float(weight[d][code[d]]))
 * base [nlist][dim] fp16, weight [dim][2^bits] fp16, cutoff [dim][2^bits - 1] fp32 ascending.  Dimension d is bits
 * [bits * (d % (8 / bits)), +bits) of byte d * bits / 8 of the row; codes [n_rows][dim * bits / 8] uint8.
 * dim % 64 == 0, 64 <= dim <= 1024; list_ids must lie in [0, nlist).  Every function decodes exactly `value`. */
MMB200_API int mmb200_residual_encode(const void* rows, const int32_t* list_ids, const void* base, const float* cutoff,
                                      uint8_t* codes, int64_t n_rows, int32_t dim, int32_t bits, void* stream);

/* out [n_rows][dim] fp16 = the decoded rows. */
MMB200_API int mmb200_residual_decode(const uint8_t* codes, const int32_t* list_ids, const void* base,
                                      const void* weight, void* out, int64_t n_rows, int32_t dim, int32_t bits,
                                      void* stream);

/* mmb200_ivf_search_gather (fp16) over the decoded rows of `codes` without materialising them: list position p is
 * code row row_index[p], which belongs to list l for every p in [list_offsets[l], list_offsets[l+1]).  The result is
 * bit-identical to mmb200_ivf_search_gather over mmb200_residual_decode(codes); workspace as mmb200_ivf_workspace_bytes
 * with dtype MMB200_F16. */
MMB200_API int mmb200_ivf_search_residual(const void* queries, const uint8_t* codes, const void* base,
                                          const void* weight, int32_t bits, const int64_t* ids,
                                          const int64_t* row_index, const int64_t* list_offsets, const int64_t* probes,
                                          float* out_scores, int64_t* out_ids, void* workspace,
                                          int64_t workspace_bytes, int64_t nq, int32_t nprobe, int64_t nlist,
                                          int64_t n_rows, int64_t max_list_len, int32_t dim, int32_t k, void* stream);

/* mmb200_maxsim_store_fwd with impl MMB200_IMPL_TCGEN05_DOCM over the decoded rows of `codes` (fp16 queries
 * [n_q, Lq, dim], 1 <= Lq <= 128), bit-identical to it over mmb200_residual_decode(codes). */
MMB200_API int mmb200_maxsim_store_residual_fwd(const void* q, const uint8_t* codes, const int32_t* list_ids,
                                                const void* base, const void* weight, int32_t bits,
                                                const int64_t* doc_offsets, const int32_t* pair_q,
                                                const int32_t* pair_d, float* out, int64_t n_q, int64_t n_rows,
                                                int64_t n_docs, int64_t n_pairs, int32_t Lq, int32_t max_doc_len,
                                                int32_t dim, void* stream);

/* ------------------------------------------------------------------------------------------
 * PLAID centroid interaction (Santhanam et al., "PLAID", CIKM 2022) over a ColBERT IVF token index: candidate passages
 * are scored from their rows' list (centroid) ids alone, with a query x centroid score table.
 *
 * mmb200_plaid_centroid_scores: queries [nq, Lq, dim] fp16 (all-zero rows are padding), centroids [nlist, dim] fp16.
 *          scores [nq, nlist, LQP] fp16, LQP = 32 * ceil(Lq / 32): scores[q][c][i] = fp16_rn(fp32 sum over d of
 *          q[i][d] * centroid[c][d]) (wgmma), 0 for i >= Lq.  keep [nq, ceil(nlist / 32)] uint32: bit c % 32 of word
 *          c / 32 is set when the max over the query's live tokens (a nonzero element) of float(scores[q][c][i]) is
 *          >= threshold; a query without live tokens keeps nothing.  threshold may be -inf, not NaN.
 * mmb200_plaid_candidates: probes [nq, n_probes] int64 list ids (outside [0, nlist): nothing); the passages of list l
 *          are plist_pids[plist_offsets[l] .. plist_offsets[l+1]) (int32 local ids in [0, n_docs)).  out_ids [nq, cap]
 *          int64: the union of the query's probed lists' passages as first_doc + pid, ascending, then -1.  A union
 *          larger than cap is truncated to its cap smallest ids.  bitmap: scratch of nq * max(1, ceil(n_docs / 32))
 *          uint32, cleared here.
 * mmb200_plaid_interaction: the scores and keep mask above, list_ids [n_rows] int32 (the list of every row),
 *          doc_offsets [n_docs + 1] int64 (passage d is rows [doc_offsets[d], doc_offsets[d+1])), cand_ids
 *          [nq, n_cand] int64 global ids (void: outside [first_doc, first_doc + n_docs), -1 included).  out [nq, n_cand]
 *          f32: sum over i < Lq of the max over the passage's rows r whose list is kept (prune != 0; every row when
 *          prune == 0) of float(scores[q][list_ids[r]][i]), summed in a fixed order; -inf when no row qualifies or the
 *          candidate is void.  keep may be NULL when prune == 0.
 * Envelope: 1 <= Lq <= 128, 1 <= nlist <= 2^18, dim % 64 == 0, 64 <= dim <= 1024, nq <= 65535 (scores, interaction),
 * 16-byte aligned queries, centroids and scores.  Outside it: MMB200_ERR_INVALID.  No host synchronisation.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_plaid_centroid_scores(const void* queries, const void* centroids, void* scores, uint32_t* keep,
                                            int64_t nq, int32_t Lq, int64_t nlist, int32_t dim, float threshold,
                                            void* stream);
MMB200_API int mmb200_plaid_candidates(const int64_t* probes, const int64_t* plist_offsets, const int32_t* plist_pids,
                                       uint32_t* bitmap, int64_t* out_ids, int64_t nq, int32_t n_probes, int64_t nlist,
                                       int64_t n_docs, int64_t cap, int64_t first_doc, void* stream);
MMB200_API int mmb200_plaid_interaction(const void* scores, const uint32_t* keep, const int32_t* list_ids,
                                        const int64_t* doc_offsets, const int64_t* cand_ids, float* out, int64_t nq,
                                        int32_t Lq, int64_t nlist, int64_t n_docs, int64_t n_cand, int64_t first_doc,
                                        int32_t prune, void* stream);

/* ------------------------------------------------------------------------------------------
 * Graph index: detour pruning of an exact k-NN graph, and a beam search over the graph
 *
 * Replaces: FaissHNSWIndexer   matchmaker/retrieval/faiss_indices.py:76-104 (faiss IndexHNSWFlat, CPU only), with one
 *           flat graph after CAGRA (Ootomo et al., ICDE 2024) instead of faiss's layers.
 *
 * mmb200_graph_prune: knn [n, K] int32, the k-NN list of every node in rank order (entries < 0 or >= n are void;
 *          valid entries of a row distinct).  out [n, R] int32: the R edges of each node with the fewest rank-based
 *          detours (edge u -> v at rank j has one through w = N(u)[i] when i < j and v = N(w)[p] with p < j), ties by
 *          rank, stored in rank order; fewer than R valid edges are padded with -1.  Integer work: bit-reproducible.
 *          1 <= K <= 1023, 1 <= R <= 1024, n < 2^31 - 1.  Outside: MMB200_ERR_INVALID.
 * mmb200_graph_hash_slots: slots of the search kernel's visited hash for list size L and degree R,
 *          next_pow2(4 * (L + R)) (0 outside 1 <= L, R <= 1024).  Pure host arithmetic.
 * mmb200_graph_search: beam search, one CTA per query.  rows [n, dim] fp16 or fp32 (`dtype`, 16-byte aligned), queries
 *          [nq, dim] in the same dtype, graph [n, R] int32 (-1 = no edge), entries [nq, n_entries] int64 row positions
 *          that start each query's list, ids [n] int64 user ids (NULL: the row position).  The list keeps the L best
 *          rows seen under (score desc, position asc); each step expands the best entry not yet expanded, scores its
 *          unvisited neighbours (fp32, fixed order) and merges them in.  It stops when every entry has been expanded or
 *          after 2 * L steps.  out_scores / out_ids [nq, k]: the first k entries, then (-3.4028235e38, -1).
 *          32 <= L <= 1024 (multiple of 32), 1 <= k <= L, 1 <= n_entries <= L, R <= 1024, dim <= 4096 and a multiple
 *          of 16 bytes.  No host synchronisation.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_graph_prune(const int32_t* knn, int32_t* out, int64_t n, int32_t K, int32_t R, void* stream);
MMB200_API int64_t mmb200_graph_hash_slots(int32_t L, int32_t R);
MMB200_API int mmb200_graph_search(const void* queries, const void* rows, const int64_t* ids, const int32_t* graph,
                                   const int64_t* entries, float* out_scores, int64_t* out_ids, int64_t nq, int64_t n,
                                   int32_t dim, int32_t R, int32_t n_entries, int32_t L, int32_t k, int32_t dtype,
                                   void* stream);

/* ------------------------------------------------------------------------------------------
 * Anisotropic-hashing (AH) index: a scan of 4-bit residual codes through per-query lookup tables, then exact reorder
 *
 * Replaces: ScaNNIndexer   matchmaker/retrieval/scann_index.py:10-53 (scann tree + score_ah(2, ...) + reorder, CPU only).
 *
 * mmb200_ah_search: the kr best rows by approximate score over each query's probed leaves.
 *          codes    [n_rows, dim / 4] uint8 sorted by leaf: leaf l is rows [list_offsets[l], list_offsets[l+1]) (int64
 *                   [nlist + 1], non-decreasing).  Byte j of a row holds the codeword of block 2j in its low nibble and
 *                   that of block 2j + 1 in its high nibble (M = dim / 2 blocks of 2 dimensions, 16 codewords each).
 *          luts     [nq, M, 16] fp32: luts[q][m][c] = <query q, codeword c of block m>.
 *          probes   [nq, nprobe] int64 leaf ids, distinct within a row; an id outside [0, nlist) probes nothing.
 *          bias     [nq, nprobe] fp32: <query, centroid of the probed leaf>.
 *          Approximate score of row r of leaf l for query q = bias + sum over m ascending of luts[q][m][code_m(r)], fp32.
 *          Each (query, probe) keeps its best min(kr, leaf length) rows in a slot of min(kr, max_list_len) rounded up
 *          to 32 entries (max_list_len should bound every leaf's length: a longer leaf keeps only its slot's worth of
 *          best rows, no fault), and the slots of a query are merged.
 *          out_scores / out_pos [nq, kr]: approximate scores and ROW POSITIONS under (score desc, position asc), with a
 *          (-3.4028235e38, -1) tail when the probed leaves hold fewer than kr rows.  Work items (leaf, chunk of <= 128
 *          probing queries) are built on the device; each reads the leaf's codes once per 8 resident lookup tables
 *          (fewer when the tables are large).  No host synchronisation.
 * mmb200_ah_workspace_bytes: device scratch of one mmb200_ah_search call, about nq * nprobe * 12 * slot bytes; 0 =
 *          sizes outside the envelope (checked without a device), -1 = no device.
 *          Envelope: 1 <= kr <= 1024, 1 <= nprobe <= 1024, dim % 64 == 0 with one lookup table (32 * dim bytes) and the
 *          code ring (32 * dim bytes) in 227 KB of shared memory (dim <= 3584), nq * nprobe < 2^31 - 128,
 *          n_rows < 2^31, 16-byte aligned luts and codes.  Outside it: MMB200_ERR_INVALID.  Not sm_90:
 *          MMB200_ERR_UNSUPPORTED.
 * mmb200_ah_reorder: exact re-scoring of a shortlist.  rows [n_rows, dim] fp16 or fp32 (`dtype`, 16-byte aligned),
 *          queries [nq, dim] in the same dtype, shortlist [nq, kr] int64 row positions (entries outside [0, n_rows) are
 *          void), ids [n_rows] int64 user ids (NULL: the position).  Every score is one fixed-order fp32 formula (lane
 *          teams over 16-byte chunks, xor butterfly).  out_scores / out_ids [nq, top_n]: the best top_n under (score
 *          desc, id asc), then (-3.4028235e38, -1).  1 <= top_n <= kr <= 1024, dim % 64 == 0, dim <= 4096.
 * ------------------------------------------------------------------------------------------ */
MMB200_API int64_t mmb200_ah_workspace_bytes(int64_t nq, int32_t nprobe, int64_t nlist, int64_t max_list_len,
                                             int32_t dim, int32_t kr);
MMB200_API int mmb200_ah_search(const float* luts, const uint8_t* codes, const int64_t* list_offsets,
                                const int64_t* probes, const float* bias, float* out_scores, int64_t* out_pos,
                                void* workspace, int64_t workspace_bytes, int64_t nq, int32_t nprobe, int64_t nlist,
                                int64_t n_rows, int64_t max_list_len, int32_t dim, int32_t kr, void* stream);
MMB200_API int mmb200_ah_reorder(const void* queries, const void* rows, const int64_t* ids, const int64_t* shortlist,
                                 float* out_scores, int64_t* out_ids, int64_t nq, int64_t n_rows, int32_t dim,
                                 int32_t kr, int32_t top_n, int32_t dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Storage block loader: byte ranges of files -> one contiguous DEVICE buffer.
 *
 * Replaces: the host path of the encoded collection between matchmaker/dense_retrieval.py:291-302
 *           (np.memmap of token_reps_<n>.npy cut to storage_filled_to_index) and :328
 *           (indexer.index(id_mapping, storage) -> faiss add_with_ids from host arrays).
 * Segment s = nbytes[s] bytes of file paths[s] starting at file_offsets[s]; segments land back to back at
 * dst_device.  pread() into two pinned staging buffers of staging_bytes (0 = 32 MiB) each, cudaMemcpyAsync on
 * `stream`, read of the next piece overlapped with the transfer of the previous one.  Returns after the last
 * piece has left the staging buffers (the device copies are complete on `stream` by then).
 * ------------------------------------------------------------------------------------------ */
MMB200_API int mmb200_storage_load(const char* const* paths, const int64_t* file_offsets, const int64_t* nbytes,
                                   int32_t n_segments, void* dst_device, int64_t staging_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MATCHMAKER_B200_H_ */
