// BERT_DOT pair scoring: score[b] = <q[b], d[b]>  (matchmaker/models/bert_dot.py:62, a batched GEMM with
// M = N = 1 in the reference).  One warp per pair, 16-byte loads, fp32 accumulate.  HBM-bound and tiny.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "device_util.cuh"
#include "host_util.cuh"

namespace mmb {

template <typename T>
__global__ void __launch_bounds__(256) dot_pairs_kernel(const T* __restrict__ q, const T* __restrict__ d,
                                                        float* __restrict__ out, int64_t B, int dim) {
  constexpr int VEC = 16 / sizeof(T);
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec_ok = (dim % VEC == 0) &&
                      (((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(d)) & 15) == 0);
  for (int64_t b = warp; b < B; b += nwarps) {
    const T* qr = q + b * dim;
    const T* dr = d + b * dim;
    float acc = 0.f;
    if (vec_ok) {
      for (int c = lane; c < dim / VEC; c += 32) {
        const uint4 qa = *reinterpret_cast<const uint4*>(qr + (size_t)c * VEC);
        const uint4 da = *reinterpret_cast<const uint4*>(dr + (size_t)c * VEC);
        const T* qe = reinterpret_cast<const T*>(&qa);
        const T* de = reinterpret_cast<const T*>(&da);
#pragma unroll
        for (int e = 0; e < VEC; ++e) acc = fmaf(to_float(qe[e]), to_float(de[e]), acc);
      }
    } else {
      for (int c = lane; c < dim; c += 32) acc = fmaf(to_float(qr[c]), to_float(dr[c]), acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[b] = acc;
  }
}

}  // namespace mmb

extern "C" int mmb200_dot_pairs(const void* q, const void* d, float* out, int64_t B, int32_t dim, int32_t dtype,
                                void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(q && d && out, "null pointer");
  MMB_REQUIRE(B >= 0 && dim > 0, "bad shape");
  MMB_REQUIRE(dtype_size(dtype) != 0, "unknown dtype");
  if (B == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int grid = (int)std::min<int64_t>((B + 7) / 8, (int64_t)dev.sm_count * 8);
  return dispatch_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    dot_pairs_kernel<T><<<grid, 256, 0, stream>>>(static_cast<const T*>(q), static_cast<const T*>(d), out, B, dim);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  });
}
