// Parameter block shared by the kernel-pooling kernels (kernel_pool.cu: FFMA forward/backward;
// kernel_pool_ts.cu: tensor-core forward).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace mmb {

struct KpParams {
  const float* q;
  const float* d;
  const void* q_mask;
  const void* d_mask;
  const float* mu;
  const float* sigma;
  const float* alpha;
  const float* weight;
  int64_t B;
  int32_t Lq, Ld, D, K, mask_dtype;
  float log_scale;
  // variants of the same pooling (SURVEY 8(f) row 3): TK-Sparse gates every document term (cikm20_tk_sparse.py:135),
  // IDCM's ESM clamps at 1e-4 and adds the bias of its Linear(11, 1) (sigir21_idcm.py:185-186)
  const float* gate;     // [B, Ld] multiplier of the activations of document term j (values < 0 count as 0), or nullptr
  float clamp_min;       // floor of alpha_k * S_ik before the log (1e-10 in KNRM / TK / TK-Sparse / Conv-KNRM)
  float bias;            // added to the score
  float* grad_gate;      // [B, Ld] backward output, or nullptr
  // forward outputs
  float* score;
  float* per_kernel;
  float* per_kernel_query;
  float* cosine;
  // backward
  const float* S;
  const float* grad_score;
  float* grad_q;
  float* grad_d;
  float* ws_weight;  // [B,K]
  float* ws_alpha;   // [B,K]
  // state the tensor-core forward leaves for the tensor-core backward (kernel_pool_bwd_wg.cu), B * (33 Ld + 32) floats:
  // cosines document-row-major [B][Ld][32] (query term contiguous: one 128-byte row per document term, rows >= Lq
  // of a row are 0), then 1 / (|d_j| + eps) [B][Ld], then 1 / (|q_i| + eps) [B][32].  nullptr = do not save.
  float* saved;
  // tensor-core forward on a block of <= 32 query rows of a longer query (kernel_pool_ts.cu, Lq > 32): the kernel sees Lq =
  // rows of the block; the rows sit at q_row0 .. of Lq_total in q, q_mask and per_kernel_query.  0 / Lq otherwise.
  int32_t q_row0, Lq_total;
  float tf32_comp;   // backward: factor undoing the mean truncation of the raw fp32 operands to tf32 (1 + 2^-11), or 1
  // store mode (mmb200_kernel_pool_store_fwd, forward only): d is the store [n_rows, D] of live rows, B the number of
  // pairs; pair p scores query pair_q[p] of q [n_q, Lq_total, D] against passage pair_d[p], its rows
  // doc_offsets[pair_d[p]] .. (at most Ld of them).  The gate, if any, is [n_rows] in store order.  Null otherwise.
  const int64_t* doc_offsets;
  const int32_t* pair_q;
  const int32_t* pair_d;
  int64_t n_q, n_rows;
};

// store mode: the passage of pair p -- its first store row and its row count (0 for pair_d < 0 or an empty passage)
__device__ __forceinline__ int kp_store_rows(const KpParams& P, int64_t p, int64_t* row0) {
  const int64_t di = P.pair_d[p];
  if (di < 0) { *row0 = 0; return 0; }
  const int64_t a = P.doc_offsets[di], b = P.doc_offsets[di + 1];
  *row0 = a;
  return (int)max((int64_t)0, min(b - a, (int64_t)P.Ld));
}

__host__ __device__ inline int64_t kp_saved_floats(int64_t B, int Ld) { return B * ((int64_t)33 * Ld + 32); }
__host__ __device__ inline int64_t kp_saved_cos_off(int64_t p, int Ld) { return p * (int64_t)Ld * 32; }
__host__ __device__ inline int64_t kp_saved_rsd_off(int64_t B, int64_t p, int Ld) { return (B * 32 + p) * (int64_t)Ld; }
__host__ __device__ inline int64_t kp_saved_rsq_off(int64_t B, int64_t p, int Ld) { return B * (int64_t)Ld * 33 + p * 32; }

struct DeviceInfo;
// tensor-core forward (kernel_pool_ts.cu); *handled = false when the shape is
// outside the kernel's envelope
int kernel_pool_fwd_ts(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream, bool* handled);
// tensor-core backward from the state saved by the forward (kernel_pool_bwd_wg.cu); same convention
int kernel_pool_bwd_tc(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream, bool* handled);

// The wide backward's part of the workspace (kernel_pool_wide.cu), Ldp = Ld rounded up to 64 document rows, per pair:
// G1 [Ldp][32] and G2^T [32][Ldp] as tf32 bit patterns, the document terms prd [Ldp], the query terms prq [32].
struct KpWideWs {
  uint32_t* g1;
  uint32_t* g2t;
  float* prd;
  float* prq;
  int32_t Ldp;
};
// its envelope: 512 < D <= 1024, D % 64 == 0, Lq <= 32, K <= 32
bool kp_wide_shape_ok(int Lq, int Ld, int D, int K);
// floats of the wide part of the workspace, B * (65 Ldp + 32)
int64_t kp_wide_ws_floats(int64_t B, int Ld);
// saved-state backward at 512 < D <= 1024: the G pass then the gradient GEMMs; ws = the wide part of the workspace
int kernel_pool_bwd_wide(const KpParams& P, float* ws, const DeviceInfo& dev, cudaStream_t stream);

}  // namespace mmb
