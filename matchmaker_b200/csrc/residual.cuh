// Residual token codes of ColBERT IVF retrieval (DESIGN 3.4g): the format and its device decode helpers.
//
// A token row x of IVF list l is stored as b bits per dimension (b = 1 or 2) plus its list id:
//   code[d]  = #{i : cutoff[d][i] <= float(x[d]) - float(base[l][d])}      (2^b - 1 ascending fp32 cutoffs per dim)
//   value[d] = fp16_rn(float(base[l][d]) + float(weight[d][code[d]]))      (2^b fp16 weights per dim)
// Dimension d lives in bits [b * (d % (8 / b)), +b) of byte d * b / 8 of the row; a row is dim * b / 8 bytes.
// base [nlist][dim] fp16, weight [dim][2^b] fp16 (so weight index d * 2^b + c), cutoff [dim][2^b - 1] fp32.
// residual_value is the one definition of a decoded value: the encode/decode kernels, the IVF scan
// (flat_ip_tc_residual_kernel) and the max-sim (maxsim_tc_residual_kernel) all decode through it.
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

namespace mmb {

constexpr int kResidualMinDim = 64, kResidualMaxDim = 1024;

struct ResidualCodes {
  const uint8_t* codes;     // [n_rows][dim * bits / 8]
  const __half* base;       // [nlist][dim]
  const __half* weight;     // [dim][2^bits]
  int32_t bits;
};

__device__ __forceinline__ uint16_t residual_value(uint16_t base, uint16_t weight) {
  return __half_as_ushort(__float2half_rn(__half2float(__ushort_as_half(base)) + __half2float(__ushort_as_half(weight))));
}

// Eight consecutive dimensions d0 .. d0 + 7 (d0 % 8 == 0) of a row: `bits` holds their 8 * B code bits (byte d0 * B / 8
// in the low bits), `tab` the 8 * 2^B decoded values of those dimensions, dimension j's value of code c at j * 2^B + c.
// Returns the eight fp16 values in dimension order (16 bytes, one swizzle chunk of a wgmma tile row).
template <int B>
__device__ __forceinline__ uint4 residual_chunk_from_table(uint32_t bits, const uint16_t* tab) {
  constexpr uint32_t kMask = (1u << B) - 1u;
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t lo = tab[(2 * j) * (1 << B) + ((bits >> (B * 2 * j)) & kMask)];
    const uint32_t hi = tab[(2 * j + 1) * (1 << B) + ((bits >> (B * (2 * j + 1))) & kMask)];
    w[j] = lo | (hi << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// The same eight dimensions decoded against a row's own base: `base8` = base[l][d0 .. d0 + 7], `weight` the 8 * 2^B
// weights of those dimensions (layout of residual_chunk_from_table's table).
template <int B>
__device__ __forceinline__ uint4 residual_chunk(uint32_t bits, uint4 base8, const uint16_t* weight) {
  constexpr uint32_t kMask = (1u << B) - 1u;
  const uint32_t bw[4] = {base8.x, base8.y, base8.z, base8.w};
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t lo = residual_value((uint16_t)(bw[j] & 0xffffu),
                                       weight[(2 * j) * (1 << B) + ((bits >> (B * 2 * j)) & kMask)]);
    const uint32_t hi = residual_value((uint16_t)(bw[j] >> 16),
                                       weight[(2 * j + 1) * (1 << B) + ((bits >> (B * (2 * j + 1))) & kMask)]);
    w[j] = lo | (hi << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Code bits of the 64 dimensions of k-block kb of a row (8 * B bytes): a uint2 for B = 1, a uint4 for B = 2, returned as
// four 32-bit words of which the first 2 * B are used.  Chunk c (dims 8c .. 8c + 7) is residual_chunk_bits(words, c).
template <int B>
__device__ __forceinline__ uint4 residual_kblock_bits(const uint8_t* row, int kb) {
  if constexpr (B == 2) {
    return __ldg(reinterpret_cast<const uint4*>(row + kb * 16));
  } else {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(row + kb * 8));
    return make_uint4(v.x, v.y, 0u, 0u);
  }
}
template <int B>
__device__ __forceinline__ uint32_t residual_chunk_bits(const uint4& words, int c) {
  const uint32_t wd[4] = {words.x, words.y, words.z, words.w};
  if constexpr (B == 2) return (wd[c >> 1] >> (16 * (c & 1))) & 0xffffu;
  else return (wd[c >> 2] >> (8 * (c & 3))) & 0xffu;
}

}  // namespace mmb
