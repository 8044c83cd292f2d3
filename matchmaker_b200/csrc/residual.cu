// Residual token codes (format in residual.cuh): encoding of fp16 rows and decoding back to fp16 rows.
//
// The hot paths decode inside the kernels that consume the rows (flat_ip_tc_residual_kernel in flat_ip.cu,
// maxsim_tc_residual_kernel in maxsim.cu); residual_decode_kernel materialises rows for tests and inspection.
#include <cuda_fp16.h>

#include <algorithm>

#include "host_util.cuh"
#include "residual.cuh"

namespace mmb {
namespace {

// One thread per code byte: the 8 / B dimensions it packs, each code the number of cutoffs <= the fp32 residual.
template <int B>
__global__ void __launch_bounds__(256) residual_encode_kernel(const __half* __restrict__ rows,
                                                              const int32_t* __restrict__ list_ids,
                                                              const __half* __restrict__ base,
                                                              const float* __restrict__ cutoff, int64_t n_rows, int dim,
                                                              uint8_t* __restrict__ codes) {
  constexpr int kPerByte = 8 / B, kCuts = (1 << B) - 1;
  const int pitch = dim * B / 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_rows * pitch; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / pitch;
    const int d0 = (int)(i % pitch) * kPerByte;
    const int64_t l = list_ids[r];
    uint32_t byte = 0;
#pragma unroll
    for (int j = 0; j < kPerByte; ++j) {
      const int d = d0 + j;
      const float res = __half2float(rows[r * dim + d]) - __half2float(base[l * dim + d]);
      uint32_t c = 0;
#pragma unroll
      for (int t = 0; t < kCuts; ++t) c += cutoff[d * kCuts + t] <= res ? 1u : 0u;
      byte |= c << (B * j);
    }
    codes[i] = (uint8_t)byte;
  }
}

// One thread per (row, 8 dimensions): one 16-byte store of decoded values.
template <int B>
__global__ void __launch_bounds__(256) residual_decode_kernel(const uint8_t* __restrict__ codes,
                                                              const int32_t* __restrict__ list_ids,
                                                              const __half* __restrict__ base,
                                                              const __half* __restrict__ weight, int64_t n_rows, int dim,
                                                              __half* __restrict__ out) {
  const int chunks = dim / 8, pitch = dim * B / 8;
  const uint16_t* w16 = reinterpret_cast<const uint16_t*>(weight);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_rows * chunks; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / chunks;
    const int c = (int)(i % chunks);
    const uint8_t* cb = codes + r * pitch + c * B;
    const uint32_t bits = B == 2 ? (uint32_t)cb[0] | ((uint32_t)cb[1] << 8) : (uint32_t)cb[0];
    const uint4 b8 = *reinterpret_cast<const uint4*>(base + (int64_t)list_ids[r] * dim + 8 * c);
    *reinterpret_cast<uint4*>(out + r * dim + 8 * c) = residual_chunk<B>(bits, b8, w16 + 8 * c * (1 << B));
  }
}

int check_residual_args(int64_t n_rows, int32_t dim, int32_t bits) {
  MMB_REQUIRE(n_rows >= 0, "n_rows must be >= 0");
  MMB_REQUIRE(bits == 1 || bits == 2, "residual codes have 1 or 2 bits per dimension");
  MMB_REQUIRE(dim % 64 == 0 && dim >= kResidualMinDim && dim <= kResidualMaxDim, "residual codes need dim % 64 == 0, 64 <= dim <= 1024");
  return MMB200_OK;
}

}  // namespace
}  // namespace mmb

extern "C" int mmb200_residual_encode(const void* rows, const int32_t* list_ids, const void* base, const float* cutoff,
                                      uint8_t* codes, int64_t n_rows, int32_t dim, int32_t bits, void* stream_) {
  using namespace mmb;
  if (int rc = check_residual_args(n_rows, dim, bits)) return rc;
  if (n_rows == 0) return MMB200_OK;
  MMB_REQUIRE(rows && list_ids && base && cutoff && codes, "null pointer");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int64_t work = n_rows * (dim * bits / 8);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)dev.sm_count * 16, (work + 255) / 256));
  const __half* x = static_cast<const __half*>(rows);
  const __half* b = static_cast<const __half*>(base);
  if (bits == 1) residual_encode_kernel<1><<<grid, 256, 0, stream>>>(x, list_ids, b, cutoff, n_rows, dim, codes);
  else residual_encode_kernel<2><<<grid, 256, 0, stream>>>(x, list_ids, b, cutoff, n_rows, dim, codes);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

extern "C" int mmb200_residual_decode(const uint8_t* codes, const int32_t* list_ids, const void* base, const void* weight,
                                      void* out, int64_t n_rows, int32_t dim, int32_t bits, void* stream_) {
  using namespace mmb;
  if (int rc = check_residual_args(n_rows, dim, bits)) return rc;
  if (n_rows == 0) return MMB200_OK;
  MMB_REQUIRE(codes && list_ids && base && weight && out, "null pointer");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(base) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int64_t work = n_rows * (dim / 8);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)dev.sm_count * 16, (work + 255) / 256));
  const __half* b = static_cast<const __half*>(base);
  const __half* w = static_cast<const __half*>(weight);
  __half* o = static_cast<__half*>(out);
  if (bits == 1) residual_decode_kernel<1><<<grid, 256, 0, stream>>>(codes, list_ids, b, w, n_rows, dim, o);
  else residual_decode_kernel<2><<<grid, 256, 0, stream>>>(codes, list_ids, b, w, n_rows, dim, o);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}
