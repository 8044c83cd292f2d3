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
  const int32_t* slot_to_packed;  // [B*C], -1 = chunk slot skipped by the packing (all padding)
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

struct DeviceInfo;
// tkl_ts.cu: launches the plan kernel and the tensor-core kernel (which runs only if plan[0] == 1).  *handled = false
// when the shape is outside its envelope; *plan_out = device plan buffer (stream-ordered allocation, freed by the caller
// with cudaFreeAsync after the FFMA kernel -- which runs only if plan[0] == 0 -- has been enqueued).
int tkl_window_ts_launch(TklParams& P, const DeviceInfo& dev, cudaStream_t stream, bool* handled, int32_t** plan_out);

}  // namespace mmb
