// Small device helpers shared by the kernels.  The RBF constants, the ex2 rounding and the norm epsilon live here once
// because the gradients are right only while the forward and backward kernels agree on them exactly.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace mmb {

// MUFU exp2 / log2 (approximate, denormals flushed to zero)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// L2 normalisation x / (|x| + kTinyNorm): allennlp's tiny_value_of_dtype(float32)
constexpr float kTinyNorm = 1e-13f;

// a = rbf_scale(sigma) turns the RBF kernel exp(-(c - mu)^2 / (2 sigma^2)) into ex2_approx(-((c - mu) a)^2)
__device__ __forceinline__ float rbf_scale(float sigma) { return sqrtf(0.5f * 1.4426950408889634f) / sigma; }

// x = hi + lo for fp32-grade products on the tf32 tensor cores: hi keeps the bits tf32 holds, lo = x - hi is exact
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}
__device__ __forceinline__ void split_tf32(const float4 v, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
  split_tf32(v.x, hi[0], lo[0]);
  split_tf32(v.y, hi[1], lo[1]);
  split_tf32(v.z, hi[2], lo[2]);
  split_tf32(v.w, hi[3], lo[3]);
}

// Shared-memory row stride (floats) of a [rows, D] fp32 tile read as float4: D rounded up to 4, then (stride / 4) made
// odd so that 8 consecutive rows hit 8 distinct 16-B bank groups.  The launchers size shared memory with it.
__host__ __device__ inline int padded_row_stride(int D) {
  int dp = (D + 3) & ~3;
  if (((dp >> 2) & 1) == 0) dp += 4;
  return dp;
}

template <typename T>
__device__ __forceinline__ float to_float(T v);
template <>
__device__ __forceinline__ float to_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// acc + <q[0..n), row chunk v> with one fma per element in element order: n = 8 fp16 (dot_chunk) or 4 fp32
// (dot_chunk_f32) values packed in 16 bytes.  The scoring loops of the graph search and the AH reorder use them.
__device__ __forceinline__ float dot_half2(uint32_t w, const float* q, float acc) {
  float lo, hi;
  asm("{\n\t.reg .f16 a, b;\n\tmov.b32 {a, b}, %2;\n\tcvt.f32.f16 %0, a;\n\tcvt.f32.f16 %1, b;\n\t}"
      : "=f"(lo), "=f"(hi)
      : "r"(w));
  acc = fmaf(q[0], lo, acc);
  return fmaf(q[1], hi, acc);
}
__device__ __forceinline__ float dot_chunk(const uint4 v, const float* q, float acc) {
  acc = dot_half2(v.x, q, acc);
  acc = dot_half2(v.y, q + 2, acc);
  acc = dot_half2(v.z, q + 4, acc);
  return dot_half2(v.w, q + 6, acc);
}
__device__ __forceinline__ float dot_chunk_f32(const uint4 v, const float* q, float acc) {
  acc = fmaf(q[0], __uint_as_float(v.x), acc);
  acc = fmaf(q[1], __uint_as_float(v.y), acc);
  acc = fmaf(q[2], __uint_as_float(v.z), acc);
  acc = fmaf(q[3], __uint_as_float(v.w), acc);
  return acc;
}

// Contiguous share [*begin, *end) of n items for this CTA of a persistent grid; the first n % gridDim.x CTAs take one more.
__device__ __forceinline__ void cta_share(int64_t n, int64_t* begin, int64_t* end) {
  const int64_t per = n / gridDim.x, rem = n % gridDim.x;
  *begin = (int64_t)blockIdx.x * per + min((int64_t)blockIdx.x, rem);
  *end = *begin + per + ((int64_t)blockIdx.x < rem ? 1 : 0);
}

}  // namespace mmb
