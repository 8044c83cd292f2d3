// Parameter block shared by the TKL window-score kernels (tkl.cu: FFMA kernel, any activation pattern;
// tkl_ts.cu: TMA + wgmma kernel for kernel sets whose activations cover the whole cosine range).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace mmb {

struct TklParams {
  const float* q;            // [B, Lq, D] contextualised (masked) query embeddings
  const void* q_mask;        // [B, Lq]
  const float* chunks;       // [Nc, 40, D] contextualised packed chunks (overlap removed)
  const void* chunk_mask;    // [Nc, 40]
  const int32_t* slot_to_packed;  // [B*C], -1 = chunk slot skipped by the packing (all padding); [n_docs*C] in store mode
  const float* mu;
  const float* sigma;
  const float* dense_w;      // [K]
  const float* sat_red_w;    // [D]   ("embedding" saturation) or nullptr
  const float* sat_params;   // embedding: 13 floats (see host); log: kernel_mult0[K]
  float* window_score;       // [B, W]
  int64_t B, n_chunks;
  int32_t Lq, D, C, K, W, mask_dtype, saturation;  // saturation: 0 = embedding, 1 = log
  int32_t segs, chunks_per_seg;
  // plan written on the device by tkl_plan_kernel (tkl_ts.cu); nullptr when the tensor-core path is not in play
  const int32_t* plan;       // [0] = 1 when every cosine in [-1, 1] activates at least one kernel ("cover"),
                             // [1] = total tiles, [2 + b] = tiles before document b (B + 1 entries), then the cost prefix and the
                             // first tile of every CTA (layout in tkl_ts.cu:tkl_plan_kernel)
};

// Store mode (mmb200_tkl_store_window_scores): window row b belongs to pair b, which scores query row pair_q[b] of q
// against the chunk slots of passage pair_d[b], row pair_d[b] of slot_to_packed -- then the per-passage slot table
// [n_docs, C] of a document store (pair_d[b] < 0: every slot empty).  A kernel argument of its own, after the others,
// so that the padded instantiations (STORE = false, pair_q == nullptr) keep their parameter layout.
struct TklPairs {
  const int32_t* pair_q;     // [B]
  const int32_t* pair_d;     // [B]
  int64_t n_q;               // rows of q (the extent of the query tensor map)
};

// Row of q and row of slot_to_packed of window row b: b itself in the padded layout, the pair's entries in store mode.
template <bool STORE>
__device__ __forceinline__ int64_t tkl_q_row(const TklPairs& X, int64_t b) { return STORE ? (int64_t)X.pair_q[b] : b; }
template <bool STORE>
__device__ __forceinline__ int64_t tkl_slot_row(const TklPairs& X, int64_t b) { return STORE ? (int64_t)X.pair_d[b] : b; }

struct DeviceInfo;
// tkl_ts.cu: launches the plan kernel and the tensor-core kernel (which runs only if plan[0] == 1).  *handled = false
// when the shape is outside its envelope; *plan_out = device plan buffer (stream-ordered allocation, freed by the caller
// with cudaFreeAsync after the FFMA kernel -- which runs only if plan[0] == 0 -- has been enqueued).  X.pair_q != nullptr
// selects the store-mode instantiations.
int tkl_window_ts_launch(TklParams& P, const TklPairs& X, const DeviceInfo& dev, cudaStream_t stream, bool* handled,
                         int32_t** plan_out);

}  // namespace mmb
