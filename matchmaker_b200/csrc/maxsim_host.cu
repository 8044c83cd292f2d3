// Max-sim: backward kernels (pairs and in-batch all-pairs) and the host-buffer (end-to-end) entry point.
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

// Backward of all-pairs scoring (colbert.py:154-162): pair p = a * n_d + b is query a against document b, so every
// document is shared by all n_q queries and its gradient is a sum over them:
//   grad_q[a][i] = sum_b                          g[a,b] * d[b][argmax[a,b,i]]     (ascending b)
//   grad_d[b][r] = sum_{(a, i) : argmax[a,b,i] = r}  g[a,b] * q[a][i]              (ascending (a, i))
// Same rules as above: no atomics, each output element owned by one thread, fmaf from 0 in that order; with n_q = 1 the
// bits are those of maxsim_bwd_{d,q}_kernel with docs_per_query = n_d.
//   maxsim_allpairs_bwd_d_kernel  one CTA per (document, block of 64 rows, slice of 128 features): an in-batch call has
//                                 few documents (32 at TAS-B's batch), and this split still gives every SM a CTA.  Per
//                                 chunk of 1024 (a, i) the warps compact, in order, the entries whose argmax falls in
//                                 the CTA's rows; thread k then walks that list into its own column of a shared-memory
//                                 accumulator, and writes the column (zeros where no argmax points) at the end
//   maxsim_allpairs_bwd_q_kernel  one CTA per (query, token), like maxsim_bwd_q_kernel with document b = p % n_d; the
//                                 argmax and gradient of 1024 documents at a time are staged in shared memory so that
//                                 the document rows of four pairs are in flight at once
constexpr int kAllBwdThreads = 128;   // the feature slice of a grad_d CTA
constexpr int kAllBwdRows = 64;
constexpr int kAllBwdChunk = 1024;
constexpr int kAllBwdUnroll = 4;

template <typename T>
__global__ void __launch_bounds__(kAllBwdThreads)
maxsim_allpairs_bwd_d_kernel(const T* __restrict__ q, const float* __restrict__ grad_out, const int32_t* __restrict__ argmax,
                             float* __restrict__ grad_d, int64_t n_q, int64_t n_d, int Lq, int Ld, int dim) {
  constexpr int kPerWarp = kAllBwdChunk / (kAllBwdThreads / 32);
  __shared__ float acc[kAllBwdRows][kAllBwdThreads];   // column threadIdx.x belongs to thread threadIdx.x alone
  __shared__ int hit_e[kAllBwdChunk];                  // entry - chunk base | (row - r0) << 16
  __shared__ float hit_g[kAllBwdChunk];
  __shared__ int hit_n[kAllBwdThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rblocks = (Ld + kAllBwdRows - 1) / kAllBwdRows, slices = (dim + kAllBwdThreads - 1) / kAllBwdThreads;
  const int64_t n_items = n_d * rblocks * slices, n_e = n_q * Lq;
  for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int64_t b = item / (rblocks * slices);
    const int rem = (int)(item % (rblocks * slices));
    const int r0 = (rem / slices) * kAllBwdRows, nr = min(kAllBwdRows, Ld - r0);
    const int k = (rem % slices) * kAllBwdThreads + threadIdx.x;
    const bool kok = k < dim;
    for (int r = 0; r < kAllBwdRows; ++r) acc[r][threadIdx.x] = 0.f;
    for (int64_t c0 = 0; c0 < n_e; c0 += kAllBwdChunk) {
      int cnt = 0;
      for (int t = 0; t < kPerWarp; t += 32) {
        const int er = warp * kPerWarp + t + lane;
        const int64_t e = c0 + er;   // e = a * Lq + i
        int r = -1;
        float g = 0.f;
        if (e < n_e) {
          const int64_t a = e / Lq, p = a * n_d + b;
          r = argmax[p * Lq + (e - a * Lq)];
          if (r >= r0 && r < r0 + nr) g = grad_out[p];
        }
        const bool hit = r >= r0 && r < r0 + nr;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (hit) {
          const int slot = warp * kPerWarp + cnt + __popc(m & ((1u << lane) - 1u));
          hit_e[slot] = er | ((r - r0) << 16);
          hit_g[slot] = g;
        }
        cnt += __popc(m);
      }
      if (lane == 0) hit_n[warp] = cnt;
      __syncthreads();
      if (kok) {
        for (int w = 0; w < kAllBwdThreads / 32; ++w) {   // the warps' lists in order: ascending (a, i)
          const int n = hit_n[w];
          const int* he = hit_e + w * kPerWarp;
          const float* hg = hit_g + w * kPerWarp;
          for (int h = 0; h < n; h += kAllBwdUnroll) {
            float v[kAllBwdUnroll];
            int rr[kAllBwdUnroll];
#pragma unroll
            for (int u = 0; u < kAllBwdUnroll; ++u) {
              rr[u] = -1;
              v[u] = 0.f;
              if (h + u < n) {
                const int x = he[h + u];
                rr[u] = x >> 16;
                v[u] = to_float(q[(c0 + (x & 0xffff)) * dim + k]);   // q[a][i][k]
              }
            }
#pragma unroll
            for (int u = 0; u < kAllBwdUnroll; ++u)
              if (rr[u] >= 0) acc[rr[u]][threadIdx.x] = fmaf(hg[h + u], v[u], acc[rr[u]][threadIdx.x]);
          }
        }
      }
      __syncthreads();   // the hit lists are rewritten by the next chunk
    }
    if (kok)
      for (int r = 0; r < nr; ++r) grad_d[(b * Ld + r0 + r) * (int64_t)dim + k] = acc[r][threadIdx.x];
  }
}

template <typename T>
__global__ void __launch_bounds__(kAllBwdThreads)
maxsim_allpairs_bwd_q_kernel(const T* __restrict__ d, const float* __restrict__ grad_out, const int32_t* __restrict__ argmax,
                             float* __restrict__ grad_q, int64_t n_q, int64_t n_d, int Lq, int Ld, int dim) {
  __shared__ int s_r[kAllBwdChunk];
  __shared__ float s_g[kAllBwdChunk];
  for (int64_t item = blockIdx.x; item < n_q * Lq; item += gridDim.x) {
    const int64_t a = item / Lq;
    const int i = (int)(item % Lq);
    float* gq = grad_q + item * (int64_t)dim;
    for (int64_t b0 = 0; b0 < n_d; b0 += kAllBwdChunk) {
      const int nb = (int)min((int64_t)kAllBwdChunk, n_d - b0);
      __syncthreads();
      for (int j = threadIdx.x; j < nb; j += blockDim.x) {
        const int64_t p = a * n_d + b0 + j;
        s_r[j] = argmax[p * Lq + i];
        s_g[j] = grad_out[p];
      }
      __syncthreads();
      for (int k = threadIdx.x; k < dim; k += blockDim.x) {
        float acc = b0 == 0 ? 0.f : gq[k];   // a document count beyond one chunk continues the same chain
        for (int j = 0; j < nb; j += kAllBwdUnroll) {
          float v[kAllBwdUnroll];
          int rr[kAllBwdUnroll];
#pragma unroll
          for (int u = 0; u < kAllBwdUnroll; ++u) {
            rr[u] = j + u < nb ? s_r[j + u] : -1;
            v[u] = rr[u] >= 0 ? to_float(d[((b0 + j + u) * Ld + rr[u]) * (int64_t)dim + k]) : 0.f;
          }
#pragma unroll
          for (int u = 0; u < kAllBwdUnroll; ++u)
            if (rr[u] >= 0) acc = fmaf(s_g[j + u], v[u], acc);
        }
        gq[k] = acc;
      }
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

extern "C" int mmb200_maxsim_allpairs_bwd(const void* q, const void* d, const float* grad_out, const int32_t* argmax,
                                          float* grad_q, float* grad_d, int64_t n_q, int64_t n_d, int32_t Lq,
                                          int32_t Ld, int32_t dim, int32_t dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(n_q >= 0 && n_d >= 0 && Lq >= 1 && Ld >= 1 && dim >= 1, "bad shape");
  MMB_REQUIRE(n_d == 0 || n_q <= ((int64_t(1) << 31) - 1) / n_d,
              "n_q * n_d must be below 2^31 (the forward's pair indices are int32)");
  // a tensor with no elements may come with a null pointer (torch hands one out for an empty tensor)
  MMB_REQUIRE((n_q == 0 || (q && grad_q)) && (n_d == 0 || (d && grad_d)) && (n_q * n_d == 0 || (grad_out && argmax)),
              "null pointer");
  MMB_REQUIRE(dtype_size(dtype) != 0, "unknown dtype");
  if (n_q == 0 && n_d == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (n_q == 0 || n_d == 0) {   // no pairs: the side that has rows gets a zero gradient
    if (n_q) MMB_CHECK_CUDA(cudaMemsetAsync(grad_q, 0, (size_t)n_q * Lq * dim * sizeof(float), stream));
    if (n_d) MMB_CHECK_CUDA(cudaMemsetAsync(grad_d, 0, (size_t)n_d * Ld * dim * sizeof(float), stream));
    return MMB200_OK;
  }
  const int64_t d_items = n_d * ((Ld + kAllBwdRows - 1) / kAllBwdRows) * ((dim + kAllBwdThreads - 1) / kAllBwdThreads);
  const int grid_d = (int)std::min<int64_t>((int64_t)dev.sm_count * 16, d_items);
  const int grid_q = (int)std::min<int64_t>((int64_t)dev.sm_count * 16, n_q * Lq);
  return dispatch_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    maxsim_allpairs_bwd_d_kernel<T><<<grid_d, kAllBwdThreads, 0, stream>>>(static_cast<const T*>(q), grad_out, argmax,
                                                                           grad_d, n_q, n_d, Lq, Ld, dim);
    maxsim_allpairs_bwd_q_kernel<T><<<grid_q, kAllBwdThreads, 0, stream>>>(static_cast<const T*>(d), grad_out, argmax,
                                                                           grad_q, n_q, n_d, Lq, Ld, dim);
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
