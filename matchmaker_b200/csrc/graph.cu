// Graph index (faiss_index_type "hnsw"): rank-based detour pruning of an exact k-NN graph, and a beam search with one
// CTA per query.  Both kernels are deterministic: the pruning is integer work, and the search orders every list under
// (score desc, id asc) with scores from one fixed-order fp32 formula.
#include <cuda_fp16.h>
#include <stdint.h>

#include <algorithm>

#include "device_util.cuh"
#include "host_util.cuh"

namespace mmb {
namespace {

constexpr int kPruneThreads = 256;
constexpr int kPruneMaxK = 1023;
constexpr int kPruneHash = 2048;       // open-addressing table of one node's k-NN list (K <= 1023: load <= 1/2)
constexpr int kSearchThreads = 128;
constexpr int kMaxDegree = 1024;
constexpr int kMaxList = 1024;
constexpr int kMaxDim = 4096;

__host__ __device__ inline int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

__device__ __forceinline__ uint32_t hash_slot(int32_t id, uint32_t mask) { return ((uint32_t)id * 2654435761u) & mask; }

// ---------------------------------------------------------------------------------------------------------------------
// Pruning.  Node u has its k-NN list N(u) (rank order).  The edge u -> v = N(u)[j] has a detour through w = N(u)[i] when
// i < j and v = N(w)[p] with p < j.  The R edges with the fewest detours are kept (ties by rank), in rank order.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPruneThreads) graph_prune_kernel(const int32_t* __restrict__ knn, int64_t n, int K,
                                                                    int R, int32_t* __restrict__ out) {
  __shared__ int32_t nbr[kPruneMaxK + 1];
  __shared__ int32_t cnt[kPruneMaxK + 1];
  __shared__ int32_t key[kPruneMaxK + 1];
  __shared__ int32_t hkey[kPruneHash];
  __shared__ int32_t hval[kPruneHash];
  __shared__ int32_t n_valid;
  constexpr uint32_t hmask = kPruneHash - 1;
  for (int64_t u = blockIdx.x; u < n; u += gridDim.x) {
    const int32_t* nu = knn + u * K;
    if (threadIdx.x == 0) n_valid = 0;
    for (int s = threadIdx.x; s < kPruneHash; s += blockDim.x) {
      hkey[s] = -1;
      hval[s] = INT32_MAX;
    }
    __syncthreads();
    int valid = 0;
    for (int j = threadIdx.x; j < K; j += blockDim.x) {
      int32_t v = nu[j];
      if (v < 0 || v >= n) v = -1;
      nbr[j] = v;
      cnt[j] = 0;
      if (v >= 0) {
        ++valid;
        uint32_t s = hash_slot(v, hmask);
        while (true) {
          const int32_t prev = atomicCAS(&hkey[s], -1, v);
          if (prev == -1 || prev == v) break;
          s = (s + 1) & hmask;
        }
        atomicMin(&hval[s], j);   // a repeated id keeps its first rank
      }
    }
    atomicAdd(&n_valid, valid);
    __syncthreads();
    if (n_valid > R) {   // otherwise every valid edge is kept and the counts are not needed
      const int kk = K * K;
      for (int idx = threadIdx.x; idx < kk; idx += blockDim.x) {
        const int i = idx / K, p = idx - i * K;
        const int32_t w = nbr[i];
        if (w < 0 || i >= K - 1 || p >= K - 1) continue;   // a detour needs i, p < j <= K - 1
        const int32_t v = knn[(int64_t)w * K + p];
        if (v < 0 || v >= n) continue;
        uint32_t s = hash_slot(v, hmask);
        int j = -1;
        while (true) {
          const int32_t h = hkey[s];
          if (h == v) {
            j = hval[s];
            break;
          }
          if (h == -1) break;
          s = (s + 1) & hmask;
        }
        if (j > i && j > p) atomicAdd(&cnt[j], 1);
      }
    }
    __syncthreads();
    // keys: detours (< 1024) above the rank (< 1024); an invalid edge is never kept
    for (int j = threadIdx.x; j < K; j += blockDim.x) key[j] = nbr[j] >= 0 ? (cnt[j] << 10) | j : INT32_MAX;
    __syncthreads();
    for (int j = threadIdx.x; j < K; j += blockDim.x) {
      const int32_t kj = key[j];
      int rank = 0;
      for (int t = 0; t < K; ++t) rank += key[t] < kj;
      cnt[j] = kj != INT32_MAX && rank < R;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < K; j += blockDim.x) {
      if (!cnt[j]) continue;
      int pos = 0;
      for (int t = 0; t < j; ++t) pos += cnt[t];
      out[u * R + pos] = nbr[j];
    }
    const int kept = min(n_valid, R);
    for (int r = kept + threadIdx.x; r < R; r += blockDim.x) out[u * R + r] = -1;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Search.  A list entry is one 64-bit key: the order-preserving bits of the fp32 score above (0x7fffffff - id) << 1 and
// the parent flag in bit 0.  Keys of distinct ids are distinct, so descending key order is (score desc, id asc) and the
// flag never decides it.  Key 0 is an empty slot.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t make_key(float s, int32_t id) {
  const uint32_t b = __float_as_uint(s + 0.0f);   // -0 -> +0
  const uint32_t o = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return ((uint64_t)o << 32) | ((uint64_t)(0x7fffffffu - (uint32_t)id) << 1);
}
__device__ __forceinline__ int32_t key_id(uint64_t k) { return (int32_t)(0x7fffffffu - (uint32_t)((k >> 1) & 0x7fffffffu)); }
__device__ __forceinline__ float key_score(uint64_t k) {
  const uint32_t o = (uint32_t)(k >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// keys[r] = key(<q, row ids[r]>, ids[r]) for r < c.  A team of `team` lanes (a power of two <= 32) scores one row with
// 16-byte loads: lane t sums chunks t, t + team, ... in order, then the team adds its lanes by an xor butterfly.
template <typename T>
__device__ void score_rows(const float* __restrict__ qs, const T* __restrict__ rows, int dim, int team,
                           const int32_t* ids, int c, uint64_t* keys) {
  constexpr int kEpc = 16 / sizeof(T);
  const int chunks = dim / kEpc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int per_warp = 32 / team, sub = lane / team, tl = lane & (team - 1);
  for (int r0 = warp * per_warp; r0 < c; r0 += nwarps * per_warp) {
    const int r = r0 + sub;
    float acc = 0.0f;
    int32_t id = -1;
    if (r < c) {
      id = ids[r];
      const uint4* src = reinterpret_cast<const uint4*>(rows + (int64_t)id * dim);
#pragma unroll 1   // unrolling makes the fp16 instantiation spill
      for (int ch = tl; ch < chunks; ch += team) {
        const uint4 v = __ldg(src + ch);
        if constexpr (sizeof(T) == 2)
          acc = dot_chunk(v, qs + ch * kEpc, acc);
        else
          acc = dot_chunk_f32(v, qs + ch * kEpc, acc);
      }
    }
    for (int o = team >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (r < c && tl == 0) keys[r] = make_key(acc, id);
  }
}

// Sorts a[0, N) descending, N a power of two.  Ends with a barrier.
__device__ void bitonic_sort_desc(uint64_t* a, int N) {
  for (int k = 2; k <= N; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int x = i ^ j;
        if (x > i) {
          const uint64_t ai = a[i], ax = a[x];
          if (((i & k) == 0) ? ai < ax : ai > ax) {
            a[i] = ax;
            a[x] = ai;
          }
        }
      }
      __syncthreads();
    }
}

// Sorts the bitonic sequence a[0, N) descending.  Ends with a barrier.
__device__ void bitonic_merge_desc(uint64_t* a, int N) {
  for (int j = N >> 1; j > 0; j >>= 1) {
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      const int x = i ^ j;
      if (x > i) {
        const uint64_t ai = a[i], ax = a[x];
        if (ai < ax) {
          a[i] = ax;
          a[x] = ai;
        }
      }
    }
    __syncthreads();
  }
}

// true when v was not in the table (and is now)
__device__ __forceinline__ bool hash_insert(int32_t* h, uint32_t mask, int32_t v) {
  uint32_t s = hash_slot(v, mask);
  while (true) {
    const int32_t prev = atomicCAS(&h[s], -1, v);
    if (prev == -1) return true;
    if (prev == v) return false;
    s = (s + 1) & mask;
  }
}

struct SearchLayout {
  int Lp, Rp, S, W, H;
  size_t bytes;
};

__host__ __device__ inline int graph_hash_slots(int L, int R) { return next_pow2(4 * (L + R)); }

__host__ __device__ inline SearchLayout search_layout(int L, int R, int dim) {
  SearchLayout s;
  s.Lp = next_pow2(L);
  s.Rp = next_pow2(R);
  s.S = s.Lp > s.Rp ? s.Lp : s.Rp;
  s.W = L > R ? L : R;
  s.H = graph_hash_slots(L, R);
  s.bytes = (size_t)dim * 4 + (size_t)(s.S + s.Rp) * 8 + (size_t)(s.W + s.H) * 4;
  return s;
}

// One CTA per query.  Shared memory: the query (fp32), the list (S keys: L entries and empty padding), the sorted
// candidates (Rp keys), the ids being scored (W), the visited hash (H slots).
template <typename T>
__global__ void __launch_bounds__(kSearchThreads) graph_search_kernel(
    const T* __restrict__ queries, const T* __restrict__ rows, const int64_t* __restrict__ ids,
    const int32_t* __restrict__ graph, const int64_t* __restrict__ entries, float* __restrict__ out_scores,
    int64_t* __restrict__ out_ids, int64_t n, int dim, int R, int m, int L, int k, int team) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int s_sel, s_fill, s_hcount;
  const SearchLayout lay = search_layout(L, R, dim);
  float* qs = reinterpret_cast<float*>(smem);
  uint64_t* list = reinterpret_cast<uint64_t*>(smem + (size_t)dim * 4);
  uint64_t* cand = list + lay.S;
  int32_t* work = reinterpret_cast<int32_t*>(cand + lay.Rp);
  int32_t* hash = work + lay.W;
  const uint32_t hmask = (uint32_t)lay.H - 1;
  const int64_t qi = blockIdx.x;
  const int tid = threadIdx.x, nt = blockDim.x;

  for (int c = tid; c < dim; c += nt) qs[c] = to_float(queries[qi * dim + c]);
  for (int s = tid; s < lay.H; s += nt) hash[s] = -1;
  for (int i = tid; i < lay.S; i += nt) list[i] = 0;
  if (tid == 0) s_fill = 0;
  __syncthreads();
  for (int i = tid; i < m; i += nt) {
    const int64_t e = entries[qi * m + i];
    if (e >= 0 && e < n && hash_insert(hash, hmask, (int32_t)e)) work[atomicAdd(&s_fill, 1)] = (int32_t)e;
  }
  __syncthreads();
  const int n_entry = s_fill;
  score_rows<T>(qs, rows, dim, team, work, n_entry, list);
  if (tid == 0) s_hcount = n_entry;
  __syncthreads();
  bitonic_sort_desc(list, lay.S);

  for (int it = 0; it < 2 * L; ++it) {
    if (tid == 0) {
      s_sel = L;
      s_fill = 0;
    }
    __syncthreads();
    int best = L;
    for (int i = tid; i < L; i += nt) {
      const uint64_t key = list[i];
      if (key != 0 && !(key & 1) && i < best) best = i;
    }
    if (best < L) atomicMin(&s_sel, best);
    __syncthreads();
    const int sel = s_sel;
    if (sel >= L) break;   // every entry of the list has been a parent
    const int32_t node = key_id(list[sel]);
    for (int r = tid; r < R; r += nt) {
      const int32_t v = graph[(int64_t)node * R + r];
      if (v >= 0 && v < n && hash_insert(hash, hmask, v)) work[atomicAdd(&s_fill, 1)] = v;
    }
    __syncthreads();
    if (tid == 0) list[sel] |= 1;
    const int c = s_fill;
    if (c > 0) {
      score_rows<T>(qs, rows, dim, team, work, c, cand);
      for (int i = c + tid; i < lay.Rp; i += nt) cand[i] = 0;
      __syncthreads();
      bitonic_sort_desc(cand, lay.Rp);
      // top S of (list, candidates): list[i] vs cand[S-1-i] gives a bitonic sequence holding the S best
      for (int i = tid; i < lay.Rp; i += nt) {
        const int li = lay.S - 1 - i;
        if (cand[i] > list[li]) list[li] = cand[i];
      }
      __syncthreads();
      bitonic_merge_desc(list, lay.S);
      for (int i = L + tid; i < lay.S; i += nt) list[i] = 0;   // the list keeps L entries
      if (tid == 0) s_hcount += c;
      __syncthreads();
      if (s_hcount > lay.H / 2) {
        // Forget every visited row but the list's.  A forgotten row scored below the list's L-th entry when it was
        // seen; that entry only rises, so scoring it again leaves the list as it is.
        for (int s = tid; s < lay.H; s += nt) hash[s] = -1;
        __syncthreads();
        for (int i = tid; i < L; i += nt) {
          const uint64_t key = list[i];
          if (key == 0) continue;
          hash_insert(hash, hmask, key_id(key));
          if (i + 1 == L || list[i + 1] == 0) s_hcount = i + 1;
        }
      }
    }
    __syncthreads();
  }

  for (int i = tid; i < k; i += nt) {
    const uint64_t key = list[i];
    float s = -3.4028234663852886e38f;
    int64_t id = -1;
    if (key != 0) {
      s = key_score(key);
      const int32_t pos = key_id(key);
      id = ids ? ids[pos] : (int64_t)pos;
    }
    out_scores[qi * k + i] = s;
    out_ids[qi * k + i] = id;
  }
}

}  // namespace
}  // namespace mmb

extern "C" int64_t mmb200_graph_hash_slots(int32_t L, int32_t R) {
  if (L < 1 || L > mmb::kMaxList || R < 1 || R > mmb::kMaxDegree) return 0;
  return mmb::graph_hash_slots(L, R);
}

extern "C" int mmb200_graph_prune(const int32_t* knn, int32_t* out, int64_t n, int32_t K, int32_t R, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(n >= 0 && n < INT32_MAX, "0 <= n < 2^31 - 1");
  MMB_REQUIRE(K >= 1 && K <= kPruneMaxK, "1 <= K <= 1023");
  MMB_REQUIRE(R >= 1 && R <= kMaxDegree, "1 <= R <= 1024");
  if (n == 0) return MMB200_OK;
  MMB_REQUIRE(knn && out, "null pointer");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int grid = (int)std::min<int64_t>(n, (int64_t)dev.sm_count * 4);
  graph_prune_kernel<<<grid, kPruneThreads, 0, stream>>>(knn, n, K, R, out);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

extern "C" int mmb200_graph_search(const void* queries, const void* rows, const int64_t* ids, const int32_t* graph,
                                   const int64_t* entries, float* out_scores, int64_t* out_ids, int64_t nq, int64_t n,
                                   int32_t dim, int32_t R, int32_t n_entries, int32_t L, int32_t k, int32_t dtype,
                                   void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(dtype == MMB200_F16 || dtype == MMB200_F32, "rows must be fp16 or fp32");
  const int epc = dtype == MMB200_F16 ? 8 : 4;
  MMB_REQUIRE(dim >= epc && dim <= kMaxDim && dim % epc == 0, "dim <= 4096, a multiple of 16 bytes of a row");
  MMB_REQUIRE(n >= 1 && n < INT32_MAX, "1 <= n < 2^31 - 1");
  MMB_REQUIRE(R >= 1 && R <= kMaxDegree, "1 <= R <= 1024");
  MMB_REQUIRE(L >= 32 && L <= kMaxList && L % 32 == 0, "32 <= L <= 1024, a multiple of 32");
  MMB_REQUIRE(k >= 1 && k <= L, "1 <= k <= L");
  MMB_REQUIRE(n_entries >= 1 && n_entries <= L, "1 <= n_entries <= L");
  MMB_REQUIRE(nq >= 0 && nq < INT32_MAX, "0 <= nq < 2^31 - 1");
  if (nq == 0) return MMB200_OK;
  MMB_REQUIRE(queries && rows && graph && entries && out_scores && out_ids, "null pointer");
  MMB_REQUIRE(((uintptr_t)rows & 15) == 0, "rows must be 16-byte aligned");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const SearchLayout lay = search_layout(L, R, dim);
  const int chunks = dim / epc;
  int team = 32;
  while (team > chunks) team >>= 1;
  auto launch = [&](auto t) -> int {
    using T = decltype(t);
    MMB_CHECK_CUDA(cudaFuncSetAttribute(graph_search_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)lay.bytes));
    graph_search_kernel<T><<<(unsigned)nq, kSearchThreads, lay.bytes, stream>>>(
        static_cast<const T*>(queries), static_cast<const T*>(rows), ids, graph, entries, out_scores, out_ids, n, dim,
        R, n_entries, L, k, team);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  };
  if (dtype == MMB200_F16) return launch(__half{});
  return launch(float{});
}
