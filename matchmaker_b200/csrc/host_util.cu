// Error reporting, device properties and TMA tensor-map encoding for the C ABI.
#include "host_util.cuh"

#include <cudaTypedefs.h>

#include <mutex>
#include <vector>

namespace mmb {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }

int current_device_info(DeviceInfo* out) {
  static std::mutex mu;
  static std::vector<DeviceInfo> cache;
  int dev = -1;
  MMB_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if ((int)cache.size() <= dev) cache.resize(dev + 1);
  DeviceInfo& d = cache[dev];
  if (d.device != dev) {
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev));
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    d.device = dev;
  }
  *out = d;
  return MMB200_OK;
}

int require_sm90(DeviceInfo* dev) {
  if (int rc = current_device_info(dev)) return rc;
  if (!(dev->cc_major == 9 && dev->cc_minor == 0)) {
    set_error("matchmaker_b200 kernels are built for sm_90a only; device is sm_" + std::to_string(dev->cc_major) +
              std::to_string(dev->cc_minor));
    return MMB200_ERR_UNSUPPORTED;
  }
  return MMB200_OK;
}

int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2promo) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  static std::once_flag once;
  static cudaError_t lookup_err = cudaSuccess;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    lookup_err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (lookup_err == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  });
  if (!encode) {
    set_error(std::string("cuTensorMapEncodeTiled is not available from the driver: ") +
              cudaGetErrorString(lookup_err));
    return MMB200_ERR_CUDA;
  }
  cuuint64_t gdims[5];
  cuuint64_t gstrides[4];
  cuuint32_t gbox[5];
  cuuint32_t estrides[5];
  for (uint32_t i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estrides[i] = 1;
    if (i + 1 < rank) gstrides[i] = strides_bytes[i];
  }
  CUresult r = encode(map, dtype, rank, const_cast<void*>(base), gdims, gstrides, gbox, estrides,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, l2promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::string msg = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r) + " (rank " +
                      std::to_string(rank) + ", dims";
    for (uint32_t i = 0; i < rank; ++i) msg += " " + std::to_string(dims[i]);
    msg += ", box";
    for (uint32_t i = 0; i < rank; ++i) msg += " " + std::to_string(box[i]);
    msg += ")";
    set_error(msg);
    return MMB200_ERR_CUDA;
  }
  return MMB200_OK;
}

}  // namespace mmb

extern "C" int mmb200_version(void) { return MMB200_VERSION; }

extern "C" const char* mmb200_last_error(void) { return mmb::g_last_error.c_str(); }

extern "C" int mmb200_device_info(int device, int* sm_count, int* cc_major, int* cc_minor) {
  int dev = device;
  if (dev < 0) MMB_CHECK_CUDA(cudaGetDevice(&dev));
  int v = 0;
  if (sm_count) {
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    *sm_count = v;
  }
  if (cc_major) {
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev));
    *cc_major = v;
  }
  if (cc_minor) {
    MMB_CHECK_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev));
    *cc_minor = v;
  }
  return MMB200_OK;
}
