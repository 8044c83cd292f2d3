// Host-side helpers shared by the C-ABI entry points: error reporting, device properties,
// driver entry point for TMA tensor-map encoding (no link-time dependency on libcuda).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "../../include/matchmaker_b200.h"

namespace mmb {

void set_error(const std::string& msg);  // thread-local, readable via mmb200_last_error()

#define MMB_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::mmb::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" __FILE__ \
                       ":" + std::to_string(__LINE__) + ")");                                    \
      return MMB200_ERR_CUDA;                                                                     \
    }                                                                                             \
  } while (0)

#define MMB_REQUIRE(cond, msg)                         \
  do {                                                 \
    if (!(cond)) {                                     \
      ::mmb::set_error(std::string("invalid argument: ") + (msg)); \
      return MMB200_ERR_INVALID;                       \
    }                                                  \
  } while (0)

struct DeviceInfo {
  int device = -1;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  int max_smem_optin = 0;
};

// Properties of the current device (cached per device id).  Returns nonzero on failure.
int current_device_info(DeviceInfo* out);

// current_device_info, then MMB200_ERR_UNSUPPORTED unless the device can run the sm_90a wgmma / TMA kernels (sm_90a code
// loads on compute capability 9.0 only).
int require_sm90(DeviceInfo* dev);

// f(T{}) with T the element type of `dtype`: __half, __nv_bfloat16 or float (any other dtype).
template <class F>
int dispatch_dtype(int dtype, F&& f) {
  if (dtype == MMB200_F16) return f(__half{});
  if (dtype == MMB200_BF16) return f(__nv_bfloat16{});
  return f(float{});
}

// cuTensorMapEncodeTiled through cudaGetDriverEntryPoint; returns nonzero on failure.
int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2promo);

inline size_t dtype_size(int dtype) {
  switch (dtype) {
    case MMB200_F16:
    case MMB200_BF16:
      return 2;
    case MMB200_F32:
      return 4;
    default:
      return 0;
  }
}

inline size_t mask_dtype_size(int m) {
  switch (m) {
    case MMB200_MASK_U8:
      return 1;
    case MMB200_MASK_I32:
    case MMB200_MASK_F32:
      return 4;
    case MMB200_MASK_I64:
      return 8;
    default:
      return 0;
  }
}

}  // namespace mmb
