// PLAID centroid interaction (Santhanam et al., CIKM 2022) for ColBERT IVF retrieval: the query x centroid score
// table with its keep mask, the candidate passages of the probed lists, and the per-passage interaction over the
// centroid ids of the passage's rows.
//
// - plaid_scores_kernel: S[q][c][i] = fp16_rn(sum_d q[i][d] * centroid[c][d]) on the tensor cores (wgmma, fp16 x fp16
//   -> fp32; centroids on M, query tokens on N), stored [nq, nlist, LQP] with LQP = 32 * ceil(Lq / 32); the epilogue
//   sets keep bit c of query q when the max over the query's live tokens of float(S) is >= the threshold.
// - plaid_mark_kernel + plaid_compact_kernel: the union of the passage lists of a query's probed lists, as a bitmap
//   over the rank's passages (atomicOr, order-free), then compacted to ascending global ids with a -1 tail.
// - plaid_interaction_kernel<NC, PRUNE>: a warp per (query, candidate) pair, lane j owning query tokens j + 32c; for
//   each row of the passage whose centroid is kept (PRUNE) or every row (!PRUNE), one fp16 S row gathered, a running
//   max per token, then a fixed-order sum.  No row of the token store is read.
#include <cuda_fp16.h>

#include <algorithm>

#include "host_util.cuh"
#include "ptx.cuh"

namespace mmb {
namespace {

constexpr int kPlaidMaxLq = 128;
constexpr int64_t kPlaidMaxNlist = int64_t(1) << 18;
constexpr int kScoreRows = 64;        // centroids per CTA of the score GEMM (the wgmma M)
constexpr int kPairsPerCta = 64;      // (query, candidate) pairs per CTA of the interaction
constexpr int kInteractionThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

template <int N>
__device__ __forceinline__ void plaid_wgmma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc);
template <>
__device__ __forceinline__ void plaid_wgmma<32>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n32k16_f16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void plaid_wgmma<64>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n64k16_f16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void plaid_wgmma<128>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n128k16_f16(d, a, b, acc);
}

// 16 bytes of row `r`, chunk `c` (8 fp16 along K) of a 128-byte-row operand tile, at its SWIZZLE_128B position: the
// layout make_wgmma_sw128_desc describes (chunk index XOR row % 8 inside each 1024-byte group of 8 rows).
__device__ __forceinline__ void put_sw128(uint8_t* tile, int r, int c, uint4 v) {
  *reinterpret_cast<uint4*>(tile + r * 128 + ((c ^ (r & 7)) << 4)) = v;
}

// One warpgroup per (64 centroids, query).  N = the wgmma N >= LQP (96 runs as 128 with zero columns).  Each 64-wide
// K block is copied into shared memory in the swizzled layout with plain loads, then 4 k16 steps.  A token is live when
// one of its fp16 elements is nonzero; padding tokens (all-zero rows) have S = 0 exactly and never set a keep bit.
template <int N>
__global__ void __launch_bounds__(128) plaid_scores_kernel(const __half* __restrict__ queries,
                                                           const __half* __restrict__ cents,
                                                           __half* __restrict__ scores, uint32_t* __restrict__ keep,
                                                           int Lq, int LQP, int64_t nlist, int dim, float threshold) {
  __shared__ __align__(1024) uint8_t sA[kScoreRows * 128];
  __shared__ __align__(1024) uint8_t sB[N * 128];
  __shared__ int live[N];
  __shared__ int any_live;
  __shared__ uint32_t kw[2];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t qi = blockIdx.y, c0 = (int64_t)blockIdx.x * kScoreRows;
  for (int i = tid; i < N; i += 128) live[i] = 0;
  if (tid < 2) kw[tid] = 0;
  if (tid == 0) any_live = 0;
  __syncthreads();

  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  const __half* qb = queries + qi * Lq * dim;
  for (int kb = 0; kb < dim; kb += 64) {
    for (int ch = tid; ch < kScoreRows * 8; ch += 128) {
      const int r = ch >> 3, c = ch & 7;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (c0 + r < nlist) v = *reinterpret_cast<const uint4*>(cents + (c0 + r) * dim + kb + 8 * c);
      put_sw128(sA, r, c, v);
    }
    for (int ch = tid; ch < N * 8; ch += 128) {
      const int r = ch >> 3, c = ch & 7;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (r < Lq) {
        v = *reinterpret_cast<const uint4*>(qb + (int64_t)r * dim + kb + 8 * c);
        if ((v.x | v.y | v.z | v.w) & 0x7fff7fffu) {   // a nonzero element (+-0 count as zero)
          live[r] = 1;
          any_live = 1;
        }
      }
      put_sw128(sB, r, c, v);
    }
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
    const uint64_t da = make_wgmma_sw128_desc(smem_u32(sA)), db = make_wgmma_sw128_desc(smem_u32(sB));
#pragma unroll
    for (int k = 0; k < 4; ++k) plaid_wgmma<N>(d, da + 2 * k, db + 2 * k, (kb | k) != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(d);
    __syncthreads();
  }

  // epilogue: thread (warp w, lane l) holds rows 16w + l/4 (+8), columns 8j + 2(l%4) + {0, 1}
  const int rr[2] = {16 * warp + (lane >> 2), 16 * warp + (lane >> 2) + 8};
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __half2 s = __floats2half2_rn(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
      const int64_t c = c0 + rr[h];
      if (col < LQP && c < nlist) *reinterpret_cast<__half2*>(scores + (qi * nlist + c) * LQP + col) = s;
      if (live[col]) mx[h] = fmaxf(mx[h], __low2float(s));
      if (live[col + 1]) mx[h] = fmaxf(mx[h], __high2float(s));
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(kFull, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(kFull, mx[h], 2));
    if ((lane & 3) == 0 && any_live && mx[h] >= threshold && c0 + rr[h] < nlist)
      atomicOr(&kw[rr[h] >> 5], 1u << (rr[h] & 31));
  }
  __syncthreads();
  const int64_t kwords = (nlist + 31) / 32, w = c0 / 32 + tid;
  if (tid < 2 && w < kwords) keep[qi * kwords + w] = kw[tid];
}

// A warp per (query, probe): every passage of the probed list sets its bit in the query's bitmap.
__global__ void __launch_bounds__(256) plaid_mark_kernel(const int64_t* __restrict__ probes,
                                                         const int64_t* __restrict__ plist_offsets,
                                                         const int32_t* __restrict__ plist_pids,
                                                         uint32_t* __restrict__ bitmap, int64_t nq, int n_probes,
                                                         int64_t nlist, int64_t words) {
  const int lane = threadIdx.x & 31;
  const int64_t n_items = nq * n_probes;
  for (int64_t it = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; it < n_items;
       it += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t l = probes[it];
    if (l < 0 || l >= nlist) continue;
    uint32_t* bm = bitmap + (it / n_probes) * words;
    for (int64_t p = plist_offsets[l] + lane; p < plist_offsets[l + 1]; p += 32) {
      const int32_t pid = plist_pids[p];
      atomicOr(&bm[pid >> 5], 1u << (pid & 31));
    }
  }
}

// One CTA per query: the set bits of its bitmap in ascending order, as global ids first_doc + pid, then -1 up to cap.
__global__ void __launch_bounds__(1024) plaid_compact_kernel(const uint32_t* __restrict__ bitmap,
                                                             int64_t* __restrict__ out, int64_t words, int64_t cap,
                                                             int64_t first_doc) {
  __shared__ int warp_sum[32];
  __shared__ int64_t base_s;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
  const uint32_t* bm = bitmap + blockIdx.x * words;
  int64_t* o = out + blockIdx.x * cap;
  if (tid == 0) base_s = 0;
  __syncthreads();
  for (int64_t w0 = 0; w0 < words; w0 += blockDim.x) {
    const int64_t w = w0 + tid;
    uint32_t bits = w < words ? bm[w] : 0u;
    const int cnt = __popc(bits);
    int incl = cnt;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int v = __shfl_up_sync(kFull, incl, s);
      if (lane >= s) incl += v;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
    for (int i = 0; i < nwarps; ++i) {
      before += i < warp ? warp_sum[i] : 0;
      total += warp_sum[i];
    }
    int64_t pos = base_s + before + incl - cnt;
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      if (pos < cap) o[pos] = first_doc + w * 32 + b;
      ++pos;
    }
    __syncthreads();
    if (tid == 0) base_s += total;
    __syncthreads();
  }
  for (int64_t p = base_s + tid; p < cap; p += blockDim.x) o[p] = -1;
}

// Grid (pair blocks, query): blocks of one query are adjacent in launch order, so the CTAs resident together read one
// query's S table out of L2.  The keep mask of the query sits in shared memory (PRUNE).
template <int NC, bool PRUNE>
__global__ void __launch_bounds__(kInteractionThreads) plaid_interaction_kernel(
    const __half* __restrict__ scores, const uint32_t* __restrict__ keep, const int32_t* __restrict__ list_ids,
    const int64_t* __restrict__ doc_offsets, const int64_t* __restrict__ cand, float* __restrict__ out, int Lq,
    int64_t nlist, int64_t n_docs, int64_t n_cand, int64_t first_doc) {
  extern __shared__ uint32_t smask[];
  constexpr int kLQP = 32 * NC, kWarps = kInteractionThreads / 32;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t q = blockIdx.y, p0 = (int64_t)blockIdx.x * kPairsPerCta;
  const int64_t* cq = cand + q * n_cand;
  float* oq = out + q * n_cand;
  bool mine = false;
  if (tid < kPairsPerCta && p0 + tid < n_cand) {
    const int64_t loc = cq[p0 + tid] - first_doc;
    mine = cq[p0 + tid] >= 0 && loc >= 0 && loc < n_docs;
  }
  if (!__syncthreads_or(mine)) {   // a block of void candidates (the -1 tail)
    if (tid < kPairsPerCta && p0 + tid < n_cand) oq[p0 + tid] = -INFINITY;
    return;
  }
  if (PRUNE) {
    const int64_t kwords = (nlist + 31) / 32;
    for (int64_t i = tid; i < kwords; i += kInteractionThreads) smask[i] = keep[q * kwords + i];
    __syncthreads();
  }
  const __half* sq = scores + q * nlist * kLQP;
  for (int k = 0; k < kPairsPerCta / kWarps; ++k) {
    const int64_t p = p0 + warp + kWarps * k;
    if (p >= n_cand) break;
    const int64_t id = cq[p], loc = id - first_doc;
    float result = -INFINITY;
    if (id >= 0 && loc >= 0 && loc < n_docs) {
      const int64_t r0 = doc_offsets[loc], r1 = doc_offsets[loc + 1];
      float m[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) m[c] = -INFINITY;
      bool kept = false;
      for (int64_t b = r0; b < r1; b += 32) {
        int lid = -1;
        if (b + lane < r1) {
          lid = list_ids[b + lane];
          if (lid < 0 || lid >= nlist || (PRUNE && !((smask[lid >> 5] >> (lid & 31)) & 1u))) lid = -1;
        }
        uint32_t bal = __ballot_sync(kFull, lid >= 0);
        kept |= bal != 0;
        while (bal) {   // two S rows in flight per step
          const int t0 = __ffs(bal) - 1;
          bal &= bal - 1;
          const int t1 = bal ? __ffs(bal) - 1 : t0;
          bal &= bal - 1;
          const int l0 = __shfl_sync(kFull, lid, t0), l1 = __shfl_sync(kFull, lid, t1);
          const __half* s0 = sq + (int64_t)l0 * kLQP;
          const __half* s1 = sq + (int64_t)l1 * kLQP;
          float v0[NC], v1[NC];
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            v0[c] = __half2float(s0[lane + 32 * c]);
            v1[c] = __half2float(s1[lane + 32 * c]);
          }
#pragma unroll
          for (int c = 0; c < NC; ++c) m[c] = fmaxf(m[c], fmaxf(v0[c], v1[c]));
        }
      }
      if (kept) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < NC; ++c)
          if (lane + 32 * c < Lq) s += m[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
        result = s;
      }
    }
    if (lane == 0) oq[p] = result;
  }
}

int check_plaid_table(int64_t nq, int32_t Lq, int64_t nlist) {
  MMB_REQUIRE(nq >= 0 && nq <= 65535, "0 <= nq <= 65535 queries per call");
  MMB_REQUIRE(Lq >= 1 && Lq <= kPlaidMaxLq, "PLAID needs 1 <= Lq <= 128");
  MMB_REQUIRE(nlist >= 1 && nlist <= kPlaidMaxNlist, "PLAID needs 1 <= nlist <= 2^18");
  return MMB200_OK;
}

}  // namespace
}  // namespace mmb

extern "C" int mmb200_plaid_centroid_scores(const void* queries, const void* centroids, void* scores, uint32_t* keep,
                                            int64_t nq, int32_t Lq, int64_t nlist, int32_t dim, float threshold,
                                            void* stream_) {
  using namespace mmb;
  if (int rc = check_plaid_table(nq, Lq, nlist)) return rc;
  MMB_REQUIRE(dim % 64 == 0 && dim >= 64 && dim <= 1024, "PLAID needs dim % 64 == 0, 64 <= dim <= 1024");
  MMB_REQUIRE(!(threshold != threshold), "the centroid score threshold is NaN");
  if (nq == 0) return MMB200_OK;
  MMB_REQUIRE(queries && centroids && scores && keep, "null pointer");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(queries) | reinterpret_cast<uintptr_t>(centroids) |
                reinterpret_cast<uintptr_t>(scores)) & 15) == 0, "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int nc = (Lq + 31) / 32, lqp = 32 * nc;
  const dim3 grid((unsigned)((nlist + kScoreRows - 1) / kScoreRows), (unsigned)nq);
  const __half* q = static_cast<const __half*>(queries);
  const __half* c = static_cast<const __half*>(centroids);
  __half* s = static_cast<__half*>(scores);
  if (nc == 1) plaid_scores_kernel<32><<<grid, 128, 0, stream>>>(q, c, s, keep, Lq, lqp, nlist, dim, threshold);
  else if (nc == 2) plaid_scores_kernel<64><<<grid, 128, 0, stream>>>(q, c, s, keep, Lq, lqp, nlist, dim, threshold);
  else plaid_scores_kernel<128><<<grid, 128, 0, stream>>>(q, c, s, keep, Lq, lqp, nlist, dim, threshold);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

extern "C" int mmb200_plaid_candidates(const int64_t* probes, const int64_t* plist_offsets, const int32_t* plist_pids,
                                       uint32_t* bitmap, int64_t* out_ids, int64_t nq, int32_t n_probes, int64_t nlist,
                                       int64_t n_docs, int64_t cap, int64_t first_doc, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(nq >= 0 && nq <= (int64_t(1) << 31) - 1, "0 <= nq < 2^31");
  MMB_REQUIRE(n_probes >= 1 && nlist >= 1 && n_docs >= 0 && n_docs < (int64_t(1) << 31), "bad sizes");
  MMB_REQUIRE(cap >= 1 && cap <= std::max<int64_t>(n_docs, 1), "1 <= cap <= max(n_docs, 1)");
  if (nq == 0) return MMB200_OK;
  MMB_REQUIRE(probes && plist_offsets && out_ids && bitmap && (plist_pids || n_docs == 0), "null pointer");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int64_t words = std::max<int64_t>(1, (n_docs + 31) / 32);
  MMB_CHECK_CUDA(cudaMemsetAsync(bitmap, 0, (size_t)(nq * words) * sizeof(uint32_t), stream));
  const int64_t warps = nq * n_probes;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)dev.sm_count * 16, (warps + 7) / 8));
  plaid_mark_kernel<<<grid, 256, 0, stream>>>(probes, plist_offsets, plist_pids, bitmap, nq, n_probes, nlist, words);
  MMB_CHECK_CUDA(cudaGetLastError());
  plaid_compact_kernel<<<(unsigned)nq, 1024, 0, stream>>>(bitmap, out_ids, words, cap, first_doc);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

extern "C" int mmb200_plaid_interaction(const void* scores, const uint32_t* keep, const int32_t* list_ids,
                                        const int64_t* doc_offsets, const int64_t* cand_ids, float* out, int64_t nq,
                                        int32_t Lq, int64_t nlist, int64_t n_docs, int64_t n_cand, int64_t first_doc,
                                        int32_t prune, void* stream_) {
  using namespace mmb;
  if (int rc = check_plaid_table(nq, Lq, nlist)) return rc;
  MMB_REQUIRE(n_docs >= 0 && n_cand >= 1, "bad sizes");
  if (nq == 0) return MMB200_OK;
  MMB_REQUIRE(scores && doc_offsets && cand_ids && out && (keep || !prune) && (list_ids || n_docs == 0),
              "null pointer");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int nc = (Lq + 31) / 32;
  const dim3 grid((unsigned)((n_cand + kPairsPerCta - 1) / kPairsPerCta), (unsigned)nq);
  const size_t smem = prune ? (size_t)((nlist + 31) / 32) * sizeof(uint32_t) : 0;
  const __half* s = static_cast<const __half*>(scores);
#define MMB_PLAID_LAUNCH(NC)                                                                                        \
  if (prune)                                                                                                      \
    plaid_interaction_kernel<NC, true><<<grid, kInteractionThreads, smem, stream>>>(s, keep, list_ids, doc_offsets, \
                                                                                    cand_ids, out, Lq, nlist, n_docs, \
                                                                                    n_cand, first_doc);            \
  else                                                                                                            \
    plaid_interaction_kernel<NC, false><<<grid, kInteractionThreads, 0, stream>>>(s, keep, list_ids, doc_offsets,   \
                                                                                  cand_ids, out, Lq, nlist, n_docs,  \
                                                                                  n_cand, first_doc);
  switch (nc) {
    case 1: MMB_PLAID_LAUNCH(1) break;
    case 2: MMB_PLAID_LAUNCH(2) break;
    case 3: MMB_PLAID_LAUNCH(3) break;
    default: MMB_PLAID_LAUNCH(4) break;
  }
#undef MMB_PLAID_LAUNCH
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}
