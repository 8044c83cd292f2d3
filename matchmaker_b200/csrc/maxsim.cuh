// Internal interface of the max-sim kernels (shared by maxsim.cu and maxsim_host.cu).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/matchmaker_b200.h"

namespace mmb {

struct MaxsimParams {
  const void* q = nullptr;
  const void* d = nullptr;
  const void* q_mask = nullptr;
  const void* d_mask = nullptr;
  const int32_t* pair_q = nullptr;
  const int32_t* pair_d = nullptr;
  const int32_t* pair_dmask = nullptr;  // row of d_mask used for pair p (default: the document index)
  float* out = nullptr;
  int32_t* argmax = nullptr;
  int64_t n_q = 0, n_d = 0, n_pairs = 0;
  int64_t pair_base = 0;  // query of pair p (when pair_q == NULL) is (p + pair_base) / docs_per_query
  int32_t docs_per_query = 1, Lq = 0, Ld = 0, dim = 0, mask_dtype = MMB200_MASK_NONE;
  // Store mode (doc_offsets != NULL): d is a ragged token store [n_rows, dim]; document di is rows
  // [doc_offsets[di], doc_offsets[di + 1]), at most Ld of them are read.  No masks; pair_d < 0 and documents without
  // rows score -inf.  NULL: the padded [n_d, Ld, dim] layout above.
  const int64_t* doc_offsets = nullptr;
  int64_t n_rows = 0;
};

// Rows [*lo, *lo + return value) of document di in store mode; 0 rows for a skipped pair (di < 0).
__device__ __forceinline__ int store_doc_rows(const MaxsimParams& P, int64_t di, int64_t* lo) {
  if (di < 0) { *lo = 0; return 0; }
  const int64_t a = P.doc_offsets[di], b = P.doc_offsets[di + 1];
  *lo = a;
  return (int)max((int64_t)0, min(b - a, (int64_t)P.Ld));
}

struct DeviceInfo;
// maxsim_qm.cu: "queries on M" wgmma kernel (Lq <= 32, dim 64/128); *handled = false if out of envelope.
int maxsim_qm_launch(const MaxsimParams& P, int dtype, const DeviceInfo& dev, cudaStream_t stream, bool* handled);

// Validates, picks the SIMT or a tensor-core kernel and launches on `stream`.
int maxsim_fwd_device(const MaxsimParams& P, int dtype, int impl, cudaStream_t stream);

}  // namespace mmb
