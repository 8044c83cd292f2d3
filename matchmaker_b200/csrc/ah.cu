// Anisotropic-hashing (AH) index search, faiss_index_type "scann": a scan of 4-bit residual codes through per-query
// lookup tables, then an exact re-scoring of the shortlist.
//
//   ah_scan_kernel   persistent CTAs over work items (leaf, chunk of <= 128 probing queries), built on the device from
//       the probe table (ivf_items.cuh).  A leaf's codes are one contiguous byte range: warp 8 streams them into a ring
//       of 32-row tiles with bulk async copies (mbarrier full / empty ring).  Warps 0-7 each take one probing query of
//       the chunk at a time, with its [M, 16] fp32 lookup table staged in shared memory; lane l scores row l of every
//       tile: bias + sum_m T[m][code_m], m ascending.  The 16 entries of one block sit in 16 consecutive words, so the
//       table lookups of a warp never conflict.  Each warp keeps the best min(kr, leaf length) rows of its (query,
//       probe) pair: rows above its threshold are appended to a per-warp list in global memory, and a full list is cut
//       back to kr by bisection on 64-bit keys (score bits above the inverted position: all keys distinct, so the cut
//       is exact under (score desc, position asc)).  The survivors go to the pair's slot; topk_merge builds the
//       kr-entry shortlist of every query from its slots.
//   ah_reorder_kernel   one CTA per query: the exact inner product with each shortlisted row (lane teams, fixed-order
//       fp32, xor butterfly), a bitonic sort under (score desc, id asc), the first top_n out.
#include <cuda_fp16.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>

#include "device_util.cuh"
#include "host_util.cuh"
#include "ivf_items.cuh"
#include "ptx.cuh"

namespace mmb {
namespace {

constexpr int kAhWarps = 8;                       // consumer warps: one probing query each
constexpr int kAhThreads = 32 * (kAhWarps + 1);   // + the bulk-copy producer warp
constexpr int kAhTileRows = 32;                   // code rows per tile: one per lane
constexpr int kAhStages = 4;
constexpr int kAhMaxKr = 1024;
constexpr int kAhSmemBudget = 227 * 1024;         // opt-in shared memory per block on sm_90
constexpr int kAhSmemMisc = 1024;                 // barriers + alignment slack
constexpr int kReorderThreads = 128;

__host__ __device__ inline int ah_tile_bytes(int dim) { return kAhTileRows * (dim / 4); }
__host__ __device__ inline int ah_lut_bytes(int dim) { return (dim / 2) * 16 * (int)sizeof(float); }
// queries whose tables are resident at once (0: not even one fits next to the code ring)
inline int ah_group(int dim) {
  const int free_bytes = kAhSmemBudget - kAhSmemMisc - kAhStages * ah_tile_bytes(dim);
  return std::max(0, std::min(kAhWarps, free_bytes / ah_lut_bytes(dim)));
}
inline size_t ah_smem_bytes(int dim) {
  return (size_t)kAhStages * ah_tile_bytes(dim) + (size_t)ah_group(dim) * ah_lut_bytes(dim) + kAhSmemMisc;
}

__device__ __forceinline__ uint32_t score_key(float f) {
  const uint32_t b = __float_as_uint(f + 0.0f);   // -0 -> +0
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// (score desc, position asc) as one descending 64-bit key; 0 is below every real key
__device__ __forceinline__ uint64_t row_key(float s, uint32_t pos) {
  return ((uint64_t)score_key(s) << 32) | (uint64_t)(0xffffffffu - pos);
}

// Cuts the warp's list buf[0, cnt) (distinct keys) to its K largest keys, in place.  Returns the K-th key.
__device__ uint64_t cut_to_k(uint64_t* buf, int cnt, int K, int lane) {
  uint64_t lo = 0, hi = ~0ull;   // largest T with count(key >= T) >= K
  while (lo < hi) {
    const uint64_t mid = lo + ((hi - lo) >> 1) + 1;
    int c = 0;
    for (int e = lane; e < cnt; e += 32) c += buf[e] >= mid ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if (c >= K) lo = mid; else hi = mid - 1;
  }
  int out = 0;
  for (int base = 0; base < cnt; base += 32) {   // writes never pass the entries read in the same round
    const int e = base + lane;
    const uint64_t v = e < cnt ? buf[e] : 0;
    const bool keep = e < cnt && v >= lo;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    __syncwarp();
    if (keep) buf[out + __popc(b & ((1u << lane) - 1u))] = v;
    out += __popc(b);
  }
  __syncwarp();
  return lo;
}

struct AhParams {
  const float* luts;          // [nq][M][16]
  const uint8_t* codes;       // [n_rows][dim / 4]
  const int64_t* offsets;     // [nlist + 1]
  const float* bias;          // [nq * nprobe] <q, leaf centroid> of every (query, probe) pair
  const int4* items;          // (leaf, first pair row, pair rows, 0)
  const int32_t* n_items;
  const int32_t* pair_of_row; // pair row -> (query, probe) pair q * nprobe + j
  uint64_t* lists;            // [grid][kAhWarps][cap]
  float* cand_scores;         // [nq * nprobe][kslot]
  int64_t* cand_pos;
  int32_t nprobe, dim, kr, kslot, cap, group;
};

__global__ void __launch_bounds__(kAhThreads, 1) ah_scan_kernel(AhParams P) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int cb = P.dim / 4, M = P.dim / 2;
  const int tile_bytes = kAhTileRows * cb;
  uint8_t* ring = smem;
  float* luts = reinterpret_cast<float*>(smem + (size_t)kAhStages * tile_bytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(luts + (size_t)P.group * M * 16);
  uint64_t* empty = full + kAhStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_items = *P.n_items;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kAhStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kAhWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  int stage = 0;
  uint32_t phase = 0;
  if (warp == kAhWarps) {
    // producer: the leaf's tiles once per group of resident queries, in the consumers' order
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int4 it = P.items[item];
      const int64_t r0 = P.offsets[it.x];
      const int len = (int)(P.offsets[it.x + 1] - r0);
      const int n_tiles = (len + kAhTileRows - 1) / kAhTileRows;
      for (int g0 = 0; g0 < it.z; g0 += P.group)
        for (int t = 0; t < n_tiles; ++t) {
          mbar_wait(&empty[stage], phase ^ 1u);
          const uint32_t bytes = (uint32_t)(min(kAhTileRows, len - t * kAhTileRows) * cb);
          if (elect_one_sync()) {
            mbar_arrive_expect_tx(&full[stage], bytes);
            bulk_load(ring + (size_t)stage * tile_bytes, P.codes + (r0 + (int64_t)t * kAhTileRows) * cb, bytes, &full[stage]);
          }
          __syncwarp();
          if (++stage == kAhStages) { stage = 0; phase ^= 1u; }
        }
    }
    return;
  }
  uint64_t* list = P.lists + ((size_t)blockIdx.x * kAhWarps + warp) * P.cap;
  float* lut = luts + (size_t)warp * M * 16;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int4 it = P.items[item];
    const int64_t r0 = P.offsets[it.x];
    const int len = (int)(P.offsets[it.x + 1] - r0);
    const int n_tiles = (len + kAhTileRows - 1) / kAhTileRows;
    // rows kept per (query, probe).  kslot >= min(kr, len) whenever max_list_len bounds the leaf; a leaf longer than the
    // bound keeps its kslot best rows, so the list (capacity 2 * kslot + 32) never grows past its end.
    const int K = min(min(P.kr, len), P.kslot);
    for (int g0 = 0; g0 < it.z; g0 += P.group) {
      const bool active = warp < min(P.group, it.z - g0);
      int32_t pair = -1;
      float bias = 0.0f;
      if (active) {
        pair = P.pair_of_row[it.y + g0 + warp];
        bias = P.bias[pair];
        const float4* src = reinterpret_cast<const float4*>(P.luts + (size_t)(pair / P.nprobe) * M * 16);
        for (int v = lane; v < M * 4; v += 32) reinterpret_cast<float4*>(lut)[v] = src[v];
        __syncwarp();
      }
      int cnt = 0;
      uint64_t tau = 0;   // appends need key > tau
      for (int t = 0; t < n_tiles; ++t) {
        mbar_wait(&full[stage], phase);
        if (active) {
          const int row = t * kAhTileRows + lane;
          uint64_t key = 0;
          if (row < len) {
            const uint4* code = reinterpret_cast<const uint4*>(ring + (size_t)stage * tile_bytes + (size_t)lane * cb);
            float s = 0.0f;
            const float* tm = lut;
            for (int c = 0; c < cb / 16; ++c) {
              const uint4 v = code[c];
              const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
              for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int b = 0; b < 4; ++b) {   // byte = blocks 2j (low nibble) and 2j + 1 (high nibble)
                  const uint32_t byte = (w[i] >> (8 * b)) & 0xffu;
                  s += tm[byte & 15u];
                  s += tm[16 + (byte >> 4)];
                  tm += 32;
                }
            }
            key = row_key(bias + s, (uint32_t)(r0 + row));
          }
          const bool pass = key > tau;
          const unsigned b = __ballot_sync(0xffffffffu, pass);
          if (pass) list[cnt + __popc(b & ((1u << lane) - 1u))] = key;
          cnt += __popc(b);
          __syncwarp();
          if (cnt > P.cap - kAhTileRows) {   // room for one more tile is kept
            tau = cut_to_k(list, cnt, K, lane);
            cnt = K;
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == kAhStages) { stage = 0; phase ^= 1u; }
      }
      if (active) {
        if (cnt > K) {
          cut_to_k(list, cnt, K, lane);
          cnt = K;
        }
        float* cs = P.cand_scores + (size_t)pair * P.kslot;
        int64_t* cp = P.cand_pos + (size_t)pair * P.kslot;
        for (int e = lane; e < P.kslot; e += 32) {
          if (e < cnt) {
            const uint64_t k = list[e];
            cs[e] = key_score((uint32_t)(k >> 32));
            cp[e] = (int64_t)(0xffffffffu - (uint32_t)k);
          } else {
            cs[e] = -INFINITY;
            cp[e] = -1;
          }
        }
        __syncwarp();
      }
    }
  }
}

// One thread per (query, probe) pair: take the next row of the probed leaf's query set and record the pair there.  A
// pair whose leaf id is out of range (a -1 filler of the coarse search) probes nothing: its slot is filled as empty.
__global__ void ah_pairs_kernel(const int64_t* __restrict__ probes, int64_t n_pairs, int64_t nlist,
                                const int* __restrict__ row_base, int* __restrict__ fill, int32_t* __restrict__ pair_of_row,
                                float* __restrict__ cand_scores, int64_t* __restrict__ cand_pos, int kslot) {
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n_pairs; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = probes[p];
    if (l >= 0 && l < nlist) {
      pair_of_row[row_base[l] + atomicAdd(fill + l, 1)] = (int32_t)p;
    } else {
      for (int e = 0; e < kslot; ++e) {
        cand_scores[p * kslot + e] = -INFINITY;
        cand_pos[p * kslot + e] = -1;
      }
    }
  }
}

struct AhLayout {
  size_t cnt, fill, row_base, item_base, items, n_items, pair, cand_s, cand_p, lists, total;
  int kslot, cap, grid;
  int64_t n_pairs, max_items;
};

AhLayout ah_layout(int64_t nq, int nprobe, int64_t nlist, int64_t max_list_len, int kr, int sm_count) {
  AhLayout L{};
  L.grid = sm_count;
  L.n_pairs = nq * nprobe;
  L.kslot = (int)((std::min<int64_t>(kr, std::max<int64_t>(1, max_list_len)) + 31) / 32 * 32);
  L.cap = 2 * L.kslot + kAhTileRows;
  L.max_items = std::min<int64_t>(nlist, L.n_pairs) + (L.n_pairs + kIvfChunk - 1) / kIvfChunk;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  L.cnt = take((size_t)nlist * sizeof(int));
  L.fill = take((size_t)nlist * sizeof(int));
  L.row_base = take((size_t)nlist * sizeof(int));
  L.item_base = take((size_t)nlist * sizeof(int));
  L.items = take((size_t)L.max_items * sizeof(int4));
  L.n_items = take(sizeof(int));
  L.pair = take((size_t)L.n_pairs * sizeof(int32_t));
  L.cand_s = take((size_t)L.n_pairs * L.kslot * sizeof(float));
  L.cand_p = take((size_t)L.n_pairs * L.kslot * sizeof(int64_t));
  L.lists = take((size_t)L.grid * kAhWarps * L.cap * sizeof(uint64_t));
  L.total = off;
  return L;
}

bool ah_in_envelope(int64_t nq, int32_t nprobe, int64_t nlist, int32_t dim, int32_t kr) {
  return nq > 0 && nprobe >= 1 && nprobe <= kIvfMaxProbe && nlist >= 1 && kr >= 1 && kr <= kAhMaxKr && dim >= 64 &&
         dim % 64 == 0 && ah_group(dim) >= 1 && nq * nprobe < (1ll << 31) - kIvfChunk;
}

// ---------------------------------------------------------------------------------------------------------------------
// reorder
// ---------------------------------------------------------------------------------------------------------------------
struct RCand {
  float s;
  int32_t valid;
  int64_t id;
};
__device__ __forceinline__ bool rcand_before(const RCand& a, const RCand& b) {
  if (a.valid != b.valid) return a.valid > b.valid;
  if (a.s != b.s) return a.s > b.s;
  return a.id < b.id;
}

// One CTA per query.  Shared memory: the query (fp32 [dim]) and the candidates (Lp = next_pow2(kr)).
template <typename T>
__global__ void __launch_bounds__(kReorderThreads) ah_reorder_kernel(
    const T* __restrict__ queries, const T* __restrict__ rows, const int64_t* __restrict__ ids,
    const int64_t* __restrict__ shortlist, float* __restrict__ out_scores, int64_t* __restrict__ out_ids, int64_t n_rows,
    int dim, int kr, int Lp, int top_n, int team) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* qs = reinterpret_cast<float*>(smem);
  RCand* c = reinterpret_cast<RCand*>(smem + (size_t)dim * 4);
  const int64_t qi = blockIdx.x;
  for (int d = threadIdx.x; d < dim; d += blockDim.x) qs[d] = to_float(queries[qi * dim + d]);
  for (int i = threadIdx.x; i < Lp; i += blockDim.x) c[i] = RCand{-INFINITY, 0, -1};
  __syncthreads();
  // scores: a team of `team` lanes per row, lane t sums chunks t, t + team, ... in order, then an xor butterfly
  constexpr int kEpc = 16 / sizeof(T);
  const int chunks = dim / kEpc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int per_warp = 32 / team, sub = lane / team, tl = lane & (team - 1);
  for (int r0 = warp * per_warp; r0 < kr; r0 += nwarps * per_warp) {
    const int r = r0 + sub;
    float acc = 0.0f;
    int64_t pos = -1;
    if (r < kr) {
      pos = shortlist[qi * kr + r];
      if (pos >= 0 && pos < n_rows) {
        const uint4* src = reinterpret_cast<const uint4*>(rows + pos * dim);
#pragma unroll 1
        for (int ch = tl; ch < chunks; ch += team) {
          const uint4 v = __ldg(src + ch);
          if constexpr (sizeof(T) == 2)
            acc = dot_chunk(v, qs + ch * kEpc, acc);
          else
            acc = dot_chunk_f32(v, qs + ch * kEpc, acc);
        }
      } else {
        pos = -1;
      }
    }
    for (int o = team >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (r < kr && tl == 0 && pos >= 0) c[r] = RCand{acc, 1, ids ? ids[pos] : pos};
  }
  __syncthreads();
  for (int size = 2; size <= Lp; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int e = threadIdx.x; e < Lp / 2; e += blockDim.x) {
        const int i = 2 * e - (e & (stride - 1));
        const int j = i + stride;
        const bool up = (i & size) == 0;
        const RCand a = c[i], b = c[j];
        if (up ? rcand_before(b, a) : rcand_before(a, b)) { c[i] = b; c[j] = a; }
      }
      __syncthreads();
    }
  for (int e = threadIdx.x; e < top_n; e += blockDim.x) {
    const bool ok = e < Lp && c[e].valid;
    out_scores[qi * top_n + e] = ok ? c[e].s : -3.4028234663852886e38f;
    out_ids[qi * top_n + e] = ok ? c[e].id : -1;
  }
}

}  // namespace
}  // namespace mmb

extern "C" int64_t mmb200_ah_workspace_bytes(int64_t nq, int32_t nprobe, int64_t nlist, int64_t max_list_len, int32_t dim,
                                             int32_t kr) {
  using namespace mmb;
  if (!ah_in_envelope(nq, nprobe, nlist, dim, kr) || max_list_len < 0) return 0;
  DeviceInfo dev;
  if (current_device_info(&dev)) return -1;
  return (int64_t)ah_layout(nq, nprobe, nlist, max_list_len, kr, dev.sm_count).total;
}

extern "C" int mmb200_ah_search(const float* luts, const uint8_t* codes, const int64_t* list_offsets, const int64_t* probes,
                                const float* bias, float* out_scores, int64_t* out_pos, void* workspace,
                                int64_t workspace_bytes_given, int64_t nq, int32_t nprobe, int64_t nlist, int64_t n_rows,
                                int64_t max_list_len, int32_t dim, int32_t kr, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(luts && codes && list_offsets && probes && bias && out_scores && out_pos && workspace, "null pointer");
  MMB_REQUIRE(ah_in_envelope(nq, nprobe, nlist, dim, kr),
              "need nq >= 1, 1 <= nprobe <= 1024, 1 <= kr <= 1024, dim % 64 == 0 with the lookup table and the code "
              "ring in shared memory (dim <= 3584), nq * nprobe < 2^31 - 128");
  MMB_REQUIRE(n_rows >= 1 && n_rows < (1ll << 31), "1 <= n_rows < 2^31");
  MMB_REQUIRE(max_list_len >= 0 && max_list_len <= n_rows, "max_list_len must bound the leaf lengths");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(luts) | reinterpret_cast<uintptr_t>(codes)) & 15) == 0, "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const AhLayout L = ah_layout(nq, nprobe, nlist, max_list_len, kr, dev.sm_count);
  MMB_REQUIRE((size_t)workspace_bytes_given >= L.total, "workspace too small (see mmb200_ah_workspace_bytes)");
  uint8_t* w = static_cast<uint8_t*>(workspace);
  int* cnt = reinterpret_cast<int*>(w + L.cnt);
  int* fill = reinterpret_cast<int*>(w + L.fill);
  int* row_base = reinterpret_cast<int*>(w + L.row_base);
  int* item_base = reinterpret_cast<int*>(w + L.item_base);
  int4* items = reinterpret_cast<int4*>(w + L.items);
  int* n_items = reinterpret_cast<int*>(w + L.n_items);
  int32_t* pair_of_row = reinterpret_cast<int32_t*>(w + L.pair);
  float* cand_s = reinterpret_cast<float*>(w + L.cand_s);
  int64_t* cand_p = reinterpret_cast<int64_t*>(w + L.cand_p);

  // probe table -> per-leaf query sets -> work items
  MMB_CHECK_CUDA(cudaMemsetAsync(cnt, 0, L.row_base - L.cnt, stream));   // cnt and fill
  const int g = std::max(1, std::min(dev.sm_count * 8, (int)((L.n_pairs + 255) / 256)));
  ivf_count_kernel<<<g, 256, 0, stream>>>(probes, L.n_pairs, nlist, cnt);
  ivf_scan_kernel<<<1, 1024, 0, stream>>>(cnt, nlist, row_base, item_base, n_items);
  ah_pairs_kernel<<<g, 256, 0, stream>>>(probes, L.n_pairs, nlist, row_base, fill, pair_of_row, cand_s, cand_p, L.kslot);
  ivf_items_kernel<<<std::max(1, std::min(dev.sm_count * 4, (int)((nlist + 255) / 256))), 256, 0, stream>>>(
      cnt, nlist, row_base, item_base, items);
  MMB_CHECK_CUDA(cudaGetLastError());

  AhParams P{};
  P.luts = luts; P.codes = codes; P.offsets = list_offsets; P.bias = bias;
  P.items = items; P.n_items = n_items; P.pair_of_row = pair_of_row;
  P.lists = reinterpret_cast<uint64_t*>(w + L.lists);
  P.cand_scores = cand_s; P.cand_pos = cand_p;
  P.nprobe = nprobe; P.dim = dim; P.kr = kr; P.kslot = L.kslot; P.cap = L.cap; P.group = ah_group(dim);
  const size_t smem = ah_smem_bytes(dim);
  MMB_CHECK_CUDA(cudaFuncSetAttribute(ah_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ah_scan_kernel<<<L.grid, kAhThreads, smem, stream>>>(P);
  MMB_CHECK_CUDA(cudaGetLastError());
  return mmb200_topk_merge(cand_s, cand_p, out_scores, out_pos, nq, nprobe * L.kslot, kr, stream_);
}

extern "C" int mmb200_ah_reorder(const void* queries, const void* rows, const int64_t* ids, const int64_t* shortlist,
                                 float* out_scores, int64_t* out_ids, int64_t nq, int64_t n_rows, int32_t dim, int32_t kr,
                                 int32_t top_n, int32_t dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(dtype == MMB200_F16 || dtype == MMB200_F32, "rows must be fp16 or fp32");
  MMB_REQUIRE(dim >= 64 && dim % 64 == 0 && dim <= 4096, "64 <= dim <= 4096, a multiple of 64");
  MMB_REQUIRE(kr >= 1 && kr <= kAhMaxKr && top_n >= 1 && top_n <= kr, "1 <= top_n <= kr <= 1024");
  MMB_REQUIRE(n_rows >= 0 && nq >= 0 && nq < INT32_MAX, "0 <= nq < 2^31 - 1");
  if (nq == 0) return MMB200_OK;
  MMB_REQUIRE(queries && rows && shortlist && out_scores && out_ids, "null pointer");
  MMB_REQUIRE(((uintptr_t)rows & 15) == 0, "rows must be 16-byte aligned");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int Lp = 2;
  while (Lp < kr) Lp <<= 1;
  const size_t smem = (size_t)dim * 4 + (size_t)Lp * sizeof(RCand);
  const int chunks = dim / (dtype == MMB200_F16 ? 8 : 4);
  int team = 32;
  while (team > chunks) team >>= 1;
  auto launch = [&](auto t) -> int {
    using T = decltype(t);
    MMB_CHECK_CUDA(cudaFuncSetAttribute(ah_reorder_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ah_reorder_kernel<T><<<(unsigned)nq, kReorderThreads, smem, stream>>>(
        static_cast<const T*>(queries), static_cast<const T*>(rows), ids, shortlist, out_scores, out_ids, n_rows, dim, kr,
        Lp, top_n, team);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  };
  if (dtype == MMB200_F16) return launch(__half{});
  return launch(float{});
}
