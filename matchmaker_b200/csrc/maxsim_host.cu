// Max-sim: backward kernel and the host-buffer (end-to-end) entry point.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "device_util.cuh"
#include "host_util.cuh"
#include "maxsim.cuh"

namespace mmb {

// Backward of score[p] = sum_i max_j <q_i, d_j> (autograd of matchmaker/models/colbert.py:68-75):
//   grad_q[qi][i]   = sum over the pairs p of query qi of  g[p] * d[p][j*(p, i)]
//   grad_d[p][j*]  += g[p] * q[qi][i]
// Two kernels, no atomics, every sum in a fixed order (round 1 added the docs_per_query contributions to grad_q with
// atomicAdd: run-to-run different low bits):
//   maxsim_bwd_d_kernel  one CTA per pair; thread k owns embedding element k (strided); query tokens are visited
//                        sequentially, so the adds into this pair's private document gradient are race-free and ordered
//   maxsim_bwd_q_kernel  one CTA per (query, token): walks the query's docs_per_query pairs in order
template <typename T>
__global__ void __launch_bounds__(128) maxsim_bwd_d_kernel(const T* __restrict__ q, const float* __restrict__ grad_out,
                                                           const int32_t* __restrict__ argmax, float* grad_d, int64_t n_pairs,
                                                           int docs_per_query, int Lq, int Ld, int dim) {
  for (int64_t p = blockIdx.x; p < n_pairs; p += gridDim.x) {
    const int64_t qi = p / docs_per_query;
    const float g = grad_out[p];
    const T* qp = q + qi * (int64_t)Lq * dim;
    float* gd = grad_d + p * (int64_t)Ld * dim;
    for (int i = 0; i < Lq; ++i) {
      const int a = argmax[p * Lq + i];
      if (a < 0) continue;  // uniform across the CTA
      for (int k = threadIdx.x; k < dim; k += blockDim.x) gd[(int64_t)a * dim + k] += g * to_float(qp[(int64_t)i * dim + k]);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(128) maxsim_bwd_q_kernel(const T* __restrict__ d, const float* __restrict__ grad_out,
                                                           const int32_t* __restrict__ argmax, float* grad_q, int64_t n_q,
                                                           int64_t n_pairs, int docs_per_query, int Lq, int Ld, int dim) {
  for (int64_t item = blockIdx.x; item < n_q * Lq; item += gridDim.x) {
    const int64_t qi = item / Lq;
    const int i = (int)(item % Lq);
    const int64_t p0 = qi * docs_per_query, p1 = min(n_pairs, p0 + docs_per_query);
    for (int k = threadIdx.x; k < dim; k += blockDim.x) {
      float acc = 0.f;
      for (int64_t p = p0; p < p1; ++p) {
        const int a = argmax[p * Lq + i];
        if (a >= 0) acc = fmaf(grad_out[p], to_float(d[(p * Ld + a) * (int64_t)dim + k]), acc);
      }
      grad_q[(qi * Lq + i) * (int64_t)dim + k] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Host-buffer pipeline: 3 device slabs, a copy stream and a compute stream per device.
// ---------------------------------------------------------------------------------------------
struct HostPipe {
  int device = -1;
  cudaStream_t copy = nullptr, compute = nullptr;
  cudaEvent_t filled[3] = {nullptr, nullptr, nullptr}, consumed[3] = {nullptr, nullptr, nullptr};
  void* slab[3] = {nullptr, nullptr, nullptr};
  size_t slab_bytes = 0;
  void* qbuf = nullptr;
  size_t q_bytes = 0;
  float* out = nullptr;
  size_t out_bytes = 0;
};

static std::mutex g_pipe_mu;
static std::vector<HostPipe> g_pipes;

static int ensure(void** p, size_t* have, size_t need) {
  if (*have >= need) return MMB200_OK;
  if (*p) MMB_CHECK_CUDA(cudaFree(*p));
  *p = nullptr;
  *have = 0;
  MMB_CHECK_CUDA(cudaMalloc(p, need));
  *have = need;
  return MMB200_OK;
}

static int get_pipe(HostPipe** out) {
  int dev = -1;
  MMB_CHECK_CUDA(cudaGetDevice(&dev));
  if ((int)g_pipes.size() <= dev) g_pipes.resize(dev + 1);
  HostPipe& hp = g_pipes[dev];
  if (hp.device != dev) {
    MMB_CHECK_CUDA(cudaStreamCreateWithFlags(&hp.copy, cudaStreamNonBlocking));
    MMB_CHECK_CUDA(cudaStreamCreateWithFlags(&hp.compute, cudaStreamNonBlocking));
    for (int i = 0; i < 3; ++i) {
      MMB_CHECK_CUDA(cudaEventCreateWithFlags(&hp.filled[i], cudaEventDisableTiming));
      MMB_CHECK_CUDA(cudaEventCreateWithFlags(&hp.consumed[i], cudaEventDisableTiming));
    }
    hp.device = dev;
  }
  *out = &hp;
  return MMB200_OK;
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace mmb

extern "C" int mmb200_maxsim_bwd(const void* q, const void* d, const float* grad_out, const int32_t* argmax,
                                 float* grad_q, float* grad_d, int64_t n_q, int64_t n_d, int64_t n_pairs,
                                 int32_t docs_per_query, int32_t Lq, int32_t Ld, int32_t dim, int32_t dtype,
                                 void* stream_) {
  using namespace mmb;
  // a tensor with no elements may come with a null pointer (torch hands one out for an empty tensor)
  MMB_REQUIRE((n_q == 0 || (q && grad_q)) && (n_d == 0 || (d && grad_d)) && (n_pairs == 0 || (grad_out && argmax)),
              "null pointer");
  MMB_REQUIRE(dtype_size(dtype) != 0, "unknown dtype");
  MMB_REQUIRE(n_q >= 0 && n_pairs >= 0 && docs_per_query >= 1 && n_pairs <= n_d &&
              (n_pairs + docs_per_query - 1) / docs_per_query <= n_q,
              "pair counts inconsistent");
  if (n_q == 0 && n_d == 0) return MMB200_OK;   // empty batch: no gradient to write
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MMB_CHECK_CUDA(cudaMemsetAsync(grad_d, 0, (size_t)n_d * Ld * dim * sizeof(float), stream));
  if (n_pairs == 0) {
    MMB_CHECK_CUDA(cudaMemsetAsync(grad_q, 0, (size_t)n_q * Lq * dim * sizeof(float), stream));
    return MMB200_OK;
  }
  const int grid_d = (int)std::min<int64_t>((int64_t)dev.sm_count * 16, n_pairs);
  const int grid_q = (int)std::min<int64_t>((int64_t)dev.sm_count * 16, n_q * Lq);
  return dispatch_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    maxsim_bwd_d_kernel<T><<<grid_d, 128, 0, stream>>>(static_cast<const T*>(q), grad_out, argmax, grad_d, n_pairs,
                                                       docs_per_query, Lq, Ld, dim);
    maxsim_bwd_q_kernel<T><<<grid_q, 128, 0, stream>>>(static_cast<const T*>(d), grad_out, argmax, grad_q, n_q, n_pairs,
                                                       docs_per_query, Lq, Ld, dim);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  });
}

extern "C" int mmb200_maxsim_fwd_host(const void* q_host, const void* d_host, const void* q_mask_host,
                                      const void* d_mask_host, float* out_host, int64_t n_q, int64_t n_d,
                                      int32_t docs_per_query, int32_t Lq, int32_t Ld, int32_t dim, int32_t dtype,
                                      int32_t mask_dtype, int64_t chunk_pairs) {
  using namespace mmb;
  MMB_REQUIRE(q_host && d_host && out_host, "null pointer");
  MMB_REQUIRE(dtype_size(dtype) != 0, "unknown dtype");
  MMB_REQUIRE(n_q > 0 && n_d >= 0 && Lq > 0 && Ld > 0 && dim > 0 && docs_per_query >= 1, "bad shape");
  if (q_mask_host || d_mask_host) MMB_REQUIRE(mask_dtype_size(mask_dtype) != 0, "unknown mask dtype");
  if (n_d == 0) return MMB200_OK;
  std::lock_guard<std::mutex> lock(g_pipe_mu);
  HostPipe* hp = nullptr;
  if (int rc = get_pipe(&hp)) return rc;

  // Documents are staged through device slabs by the copy engine, also when they sit in pinned host memory: the H100's
  // TMA unit does not fetch from mapped host memory (the kernel faults), so there is no zero-copy path on this GPU.
  if (chunk_pairs == -1) chunk_pairs = 0;

  const size_t es = dtype_size(dtype), ms = mask_dtype_size(mask_dtype);
  const size_t doc_bytes = (size_t)Ld * dim * es;
  const size_t dmask_bytes = d_mask_host ? (size_t)Ld * ms : 0;
  if (chunk_pairs <= 0) chunk_pairs = std::max<int64_t>(1, (int64_t)((96ull << 20) / doc_bytes));  // ~96 MB slabs
  chunk_pairs = std::min<int64_t>(chunk_pairs, n_d);
  const size_t slab_docs = align_up((size_t)chunk_pairs * doc_bytes, 256);
  const size_t slab_need = slab_docs + align_up((size_t)chunk_pairs * dmask_bytes, 256);
  if (hp->slab_bytes < slab_need) {
    for (int i = 0; i < 3; ++i) {
      size_t have = hp->slab_bytes;
      if (int rc = ensure(&hp->slab[i], &have, slab_need)) return rc;
    }
    hp->slab_bytes = slab_need;
  }
  const size_t q_bytes = (size_t)n_q * Lq * dim * es;
  const size_t qm_bytes = q_mask_host ? (size_t)n_q * Lq * ms : 0;
  if (int rc = ensure(&hp->qbuf, &hp->q_bytes, align_up(q_bytes, 256) + qm_bytes)) return rc;
  if (int rc = ensure(reinterpret_cast<void**>(&hp->out), &hp->out_bytes, (size_t)n_d * sizeof(float))) return rc;

  void* dq = hp->qbuf;
  void* dqm = q_mask_host ? static_cast<uint8_t*>(hp->qbuf) + align_up(q_bytes, 256) : nullptr;
  MMB_CHECK_CUDA(cudaMemcpyAsync(dq, q_host, q_bytes, cudaMemcpyHostToDevice, hp->compute));
  if (q_mask_host) MMB_CHECK_CUDA(cudaMemcpyAsync(dqm, q_mask_host, qm_bytes, cudaMemcpyHostToDevice, hp->compute));

  int64_t c = 0;
  for (int64_t lo = 0; lo < n_d; lo += chunk_pairs, ++c) {
    const int64_t n = std::min<int64_t>(chunk_pairs, n_d - lo);
    const int b = (int)(c % 3);
    if (c >= 3) MMB_CHECK_CUDA(cudaStreamWaitEvent(hp->copy, hp->consumed[b], 0));
    uint8_t* slab = static_cast<uint8_t*>(hp->slab[b]);
    MMB_CHECK_CUDA(cudaMemcpyAsync(slab, static_cast<const uint8_t*>(d_host) + (size_t)lo * doc_bytes,
                                   (size_t)n * doc_bytes, cudaMemcpyHostToDevice, hp->copy));
    if (d_mask_host)
      MMB_CHECK_CUDA(cudaMemcpyAsync(slab + slab_docs, static_cast<const uint8_t*>(d_mask_host) + (size_t)lo * dmask_bytes,
                                     (size_t)n * dmask_bytes, cudaMemcpyHostToDevice, hp->copy));
    MMB_CHECK_CUDA(cudaEventRecord(hp->filled[b], hp->copy));
    MMB_CHECK_CUDA(cudaStreamWaitEvent(hp->compute, hp->filled[b], 0));
    MaxsimParams P;
    P.q = dq; P.d = slab; P.q_mask = dqm; P.d_mask = d_mask_host ? slab + slab_docs : nullptr; P.out = hp->out + lo;
    P.n_q = n_q; P.n_d = n; P.n_pairs = n; P.pair_base = lo; P.docs_per_query = docs_per_query;
    P.Lq = Lq; P.Ld = Ld; P.dim = dim; P.mask_dtype = mask_dtype;
    if (int rc = maxsim_fwd_device(P, dtype, MMB200_IMPL_AUTO, hp->compute)) return rc;
    MMB_CHECK_CUDA(cudaEventRecord(hp->consumed[b], hp->compute));
  }
  MMB_CHECK_CUDA(cudaMemcpyAsync(out_host, hp->out, (size_t)n_d * sizeof(float), cudaMemcpyDeviceToHost, hp->compute));
  MMB_CHECK_CUDA(cudaStreamSynchronize(hp->compute));
  return MMB200_OK;
}
