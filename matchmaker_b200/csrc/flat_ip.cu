// Exact maximum-inner-product search with a fused per-query top-k (BERT_DOT dense retrieval scoring).
//
// Reference: `faiss.IndexIDMap(IndexFlatIP)` sharded over GPUs, called from
// matchmaker/retrieval/faiss_indices.py:27 (add_with_ids), :34 (search), :61-67 (shard=True, useFloat16),
// driven by matchmaker/dense_retrieval.py:328,391.  faiss tiles a cuBLAS GEMM into a score buffer and
// runs a k-selection kernel over it; here the [queries x passages] score matrix is never written:
//
//   flat_ip_tc_kernel   persistent CTAs over work items (block of 128 queries) x (range of passages); clusters of 2
//               CTAs take consecutive query blocks and share every passage tile by TMA multicast.
//       warp 8  TMA producer: per k-block one 16 KB query tile + this CTA's slice of the 16 KB passage tile
//       warpgroups 0, 1  wgmma m64n128k16: warpgroup c scores query rows 64c .. 64c + 63 against the 128 passages of a
//               tile (fp32 registers) and writes them to a shared-memory score tile; then its four warps filter them,
//               thread = query row, one 64-column half per warp: FMNMX tree -> maxima of 8-column sub-groups, compare
//               against the row's running threshold tau (the k-th best seen so far); sub-groups holding a candidate for
//               SOME row of the warp are scanned with warp-uniform control flow and a predicated shared-memory atomic +
//               global store into the row's candidate list (ONE list per row, capacity 1024, global memory).  The pair of
//               warps of a row quarter meets at a named barrier at the start of every tile; rows whose list could
//               overflow during the tile are compacted there (split between the two warps): 32-step bisection on the
//               order-preserving integer image of the scores finds the k-th largest, survivors are rewritten in place
//               and tau rises.  tau is also published per query (atomicMax) so items working on other passage ranges
//               of the same queries filter harder.  compact_row is __noinline__ to keep the per-tile loop small.
//   topk_merge_kernel   per query: bitonic sort of the candidate lists of all ranges (or, after the NCCL
//       all-gather, of all ranks) under the total order (score desc, id asc) -> [k] scores + ids.
//
// Tensor cores are used here because this is the one genuinely dense contraction of the hot path
// (arithmetic intensity ~ nq flops per passage byte).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include "device_util.cuh"
#include "host_util.cuh"
#include "ivf_items.cuh"
#include "ptx.cuh"
#include "residual.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 384;            // two consumer warpgroups (warps 0-7), TMA warp 8 (warps 9-11 idle)
constexpr int kRegsProducer = 40, kRegsConsumer = 232;  // setmaxnreg: 128 x 40 + 256 x 232 <= 384 x 168 (the launch)
// list entries per lane in a compaction: EPL = 32 -> capacity 1024 per row (k <= 256), EPL = 64 -> 2048 (k <= 1024)
constexpr int kMaxK = 1024;
__host__ __device__ constexpr int epl_for_k(int k) { return k <= 256 ? 32 : 64; }
constexpr int BM = 128;                 // queries per block (two wgmma M = 64 halves)
constexpr int BN = 128;                 // passages per tile (wgmma N)
constexpr int kABytes = BM * 128;       // one k-block (64 halfs) of the query tile
constexpr int kBBytes = BN * 128;
constexpr int kStageBytes = kABytes + kBBytes;  // 32 KB
constexpr int kStages = 4;
constexpr int kCsStride = BN + 4;       // floats per row of the score tile: 16-byte row reads by 8 threads hit 32 banks
constexpr int kMaxRanges = 32;

struct FipShared {
  uint64_t full[kStages];
  uint64_t empty[kStages];
  int cnt[BM];        // entries in each row's candidate list (appended to by both warps of the row's quarter)
  uint32_t tau[BM];   // order-preserving image of each row's threshold
};

struct FipParams {
  const int64_t* ids;       // [n_pass] user ids or nullptr (id = id_base + position)
  int64_t id_base;
  int64_t nq, n_pass;
  int32_t dim, k, kpad;             // kpad = k rounded up to 32 (list capacity per row is 32 * EPL)
  int32_t kblocks, kb_wrap;         // k-blocks of 64 along the QUERY rows; passage k-block = kb < kb_wrap ? kb : kb - kb_wrap
  int32_t n_qblocks, n_ranges, tiles_per_range, n_tiles;
  uint2* lists;             // [grid][BM][cap]  (score bits, position)
  uint32_t* tau_glob;       // [nq] order-preserving image of the per-query threshold
  float* cand_scores;       // [nq][n_ranges * kpad]; IVF mode: [n_pairs][kpad]
  int64_t* cand_ids;        // [nq][n_ranges * kpad]; IVF mode: [n_pairs][kpad]
};

// IVF mode only (flat_ip_tc_kernel<..., true>): a work item is (list, up to BM queries probing it).  A separate kernel
// parameter, so that the flat-IP instantiations keep their parameter block (compact_row takes FipParams by reference).
struct IvfParams {
  const int4* items;        // [*n_items] (list, first row of the gathered queries, query rows, 0)
  const int32_t* n_items;   // written on the device by ivf_scan_kernel
  const int64_t* offsets;   // [nlist + 1] row range of every list in the sorted layout
  const int32_t* pair;      // gathered query row -> its (query, probe) pair q * nprobe + j
  int32_t nprobe;
};

// Gather mode only (flat_ip_tc_gather_kernel): list position p of the layout is store row row_index[p].  The rows stay
// where they are (in the order stage 2 of ColBERT retrieval reads them); `FipParams::ids` is indexed by store row.
struct GatherParams {
  const uint8_t* rows;        // the store, rows `row_pitch` bytes apart (16-byte aligned)
  const int64_t* row_index;   // [list_offsets[nlist]] store row of every list position
  int64_t row_pitch;
};

// order-preserving map float -> uint32 (larger float <=> larger key)
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
constexpr uint32_t kKeyNegInf = 0x007fffffu;  // f2key(-inf)

__device__ __forceinline__ int64_t pos_to_id(const FipParams& P, uint32_t pos) {
  return P.ids ? P.ids[pos] : P.id_base + (int64_t)pos;
}

// Warp-cooperative compaction of one row's candidate list to its top-k under (score desc, id asc).
// `list` has `cnt` valid entries (cnt <= 32 * EPL).  Returns the new count (min(cnt, k)) and the key of
// the k-th best entry in *kth_key (kKeyNegInf if fewer than k entries).
// GATHER: a list entry's position is a list position, its id that of store row row_index[position].
template <int EPL, bool GATHER>
__device__ __forceinline__ int compact_row_impl(const FipParams& P, const int64_t* row_index, uint2* list, int cnt,
                                                int lane, uint32_t* kth_key) {
  uint32_t key[EPL], pos[EPL];
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const int e = lane + 32 * j;
    if (e < cnt) {
      const uint2 v = list[e];
      key[j] = f2key(__uint_as_float(v.x));
      pos[j] = v.y;
    } else {
      key[j] = 0u;  // below every real key (real keys are >= kKeyNegInf > 0 unless NaN; NaNs are not supported)
      pos[j] = 0xffffffffu;
    }
  }
  if (cnt <= P.k) {
    *kth_key = cnt == P.k ? 0u : kKeyNegInf;
    if (cnt == P.k) {  // exactly k: threshold = smallest key present
      uint32_t mn = 0xffffffffu;
#pragma unroll
      for (int j = 0; j < EPL; ++j)
        if (lane + 32 * j < cnt) mn = min(mn, key[j]);
      *kth_key = __reduce_min_sync(0xffffffffu, mn);
    }
    return cnt;
  }
  // largest T with count(key >= T) >= k
  uint32_t lo = 0u, hi = 0xffffffffu;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1) + 1u;  // upper mid
    int c = 0;
#pragma unroll
    for (int j = 0; j < EPL; ++j) c += (key[j] >= mid) ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if (c >= P.k) lo = mid; else hi = mid - 1u;
  }
  const uint32_t T = lo;
  int c_gt = 0, c_eq = 0;
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    c_gt += (key[j] > T) ? 1 : 0;
    c_eq += (key[j] == T) ? 1 : 0;
  }
  c_gt = __reduce_add_sync(0xffffffffu, c_gt);
  c_eq = __reduce_add_sync(0xffffffffu, c_eq);
  int need = P.k - c_gt;  // how many of the entries tied at T survive (1 <= need <= c_eq)
  uint64_t keep = 0u;     // bit j: entry j of this lane survives
#pragma unroll
  for (int j = 0; j < EPL; ++j)
    if (key[j] > T) keep |= 1ull << j;
  if (need == c_eq) {
#pragma unroll
    for (int j = 0; j < EPL; ++j)
      if (key[j] == T) keep |= 1ull << j;
  } else {
    // rare: more ties than room -> take the `need` smallest ids among them
    uint64_t taken = 0u;
    for (int n = 0; n < need; ++n) {
      unsigned long long best = ~0ull;
      int bj = -1;
#pragma unroll
      for (int j = 0; j < EPL; ++j)
        if (key[j] == T && !(taken & (1ull << j))) {
          const int64_t sid = GATHER ? P.ids[row_index[pos[j]]] : pos_to_id(P, pos[j]);
          const unsigned long long id = (unsigned long long)(sid ^ (1ll << 63));  // signed order
          if (id < best) { best = id; bj = j; }
        }
      unsigned long long wbest = best;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long ot = __shfl_xor_sync(0xffffffffu, wbest, o);
        wbest = ot < wbest ? ot : wbest;
      }
      const unsigned owner = __ballot_sync(0xffffffffu, best == wbest && bj >= 0);
      if (bj >= 0 && best == wbest && (int)(__ffs(owner) - 1) == lane) { taken |= 1ull << bj; keep |= 1ull << bj; }
    }
  }
  int base = 0;
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const bool kp = (keep >> j) & 1ull;
    const unsigned b = __ballot_sync(0xffffffffu, kp);
    if (kp) list[base + __popc(b & ((1u << lane) - 1u))] = make_uint2(__float_as_uint(key2f(key[j])), pos[j]);
    base += __popc(b);
  }
  __syncwarp();
  *kth_key = T;
  return P.k;
}

// __noinline__: the epilogue's per-tile loop has to stay inside the instruction cache.  With this routine inlined (and
// the column loop unrolled) the loop body streamed ~100 KB of code per tile and ran at IPC 0.03.
template <int EPL>
__device__ __noinline__ int compact_row(const FipParams& P, uint2* list, int cnt, int lane, uint32_t* kth_key) {
  return compact_row_impl<EPL, false>(P, nullptr, list, cnt, lane, kth_key);
}
template <int EPL>
__device__ __noinline__ int compact_row_gather(const FipParams& P, const int64_t* row_index, uint2* list, int cnt,
                                               int lane, uint32_t* kth_key) {
  return compact_row_impl<EPL, true>(P, row_index, list, cnt, lane, kth_key);
}

// CL = thread-block cluster size.  The CL CTAs of a cluster work on CL consecutive query blocks against the SAME passage
// tiles: each CTA fetches 1/CL of every passage tile and multicasts it to the whole cluster, so the L2 -> SM traffic per
// CTA drops from 32 KB to (16 + 16 / CL) KB per k-block.  A stage may be refilled only when EVERY CTA of the cluster has
// consumed it, hence the consumers arrive on the `empty` barriers of all CTAs (count 8 * CL).
template <typename T>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc);
template <>
__device__ __forceinline__ void wgmma_n128<__half>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n128k16_f16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void wgmma_n128<__nv_bfloat16>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n128k16_bf16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void wgmma_n128<__nv_fp8_e4m3>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n128k32_e4m3(d, a, b, acc);
}

// IVF = true: the probed-list scan of mmb200_ivf_search.  A work item is (list, chunk of <= BM probing queries) from
// V.items; the query tile is the chunk's rows of the pre-gathered queries (TMA cannot gather rows), the passage tiles
// are the list's row range, and rows past the list end are never candidates.  Each row of the chunk keeps its own list
// and publishes into its (query, probe) slot; tau_glob stays per query, since the k-th best score a query has in any of
// its lists bounds all of them.  Runs with CL = 1.  The mode only changes where an item's rows and tiles come from, so it
// is a template flag: with IVF = false every branch below folds away.
//
// GATHER = true (IVF mode, flat_ip_tc_gather_kernel): list position p is store row G.row_index[p], so the passage tile
// of an item is a gather that TMA cannot do.  The producer warp fills each stage's passage half with 16-byte cp.async
// copies in the SWIZZLE_128B layout TMA would write (rows past the list end zero-filled) and signals them on the stage's
// `full` barrier with one cp.async arrival per lane; the query half stays TMA.  List entries keep list positions, ids
// are P.ids[row_index[position]].  The consumers fence the async proxy before their wgmma reads the cp.async data.
//
// RB > 0 (gather mode over residual codes, flat_ip_tc_residual_kernel): the store holds RB-bit residual codes
// (residual.cuh) and the producer is the whole warpgroup 8-11.  An item is one list, so every value of a dimension
// depends only on its code: at the start of an item the producers build the list's table of decoded values
// ([dim][2^RB] fp16 behind the tile's store rows) and thread p then decodes row p of every passage tile with one table
// lookup per value, writing the same SWIZZLE_128B layout (zeros past the list end) with 16-byte shared stores.  Each
// producer thread fences the async proxy and arrives on `full` (1 + 128 arrivals); the query half stays TMA.
template <typename T, int CL, int EPL, bool IVF, bool GATHER, int RB = 0>
__device__ __forceinline__ void flat_ip_tc_body(const CUtensorMap& tmap_q, const CUtensorMap* tmap_p,
                                                FipParams P, IvfParams V, GatherParams G, ResidualCodes R = {}) {
  static_assert(!GATHER || (IVF && CL == 1), "the gather mode is a variant of the IVF scan");
  static_assert(RB == 0 || (GATHER && (RB == 1 || RB == 2)), "residual codes are read in gather mode, 1 or 2 bits");
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for SWIZZLE_128B tiles, derived by pointer arithmetic on the __shared__ array so the
  // compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  float* cs = reinterpret_cast<float*>(smem + (size_t)kStages * kStageBytes);     // [BM][kCsStride] score tile
  FipShared* S = reinterpret_cast<FipShared*>(cs + BM * kCsStride);
  constexpr int kCap = 32 * EPL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kblocks = P.kblocks;
  constexpr int kKbElems = 128 / (int)sizeof(T);   // elements of a k-block: one 128-byte swizzled row
  const int n_qgroups = (P.n_qblocks + CL - 1) / CL;   // CL consecutive query blocks per cluster work item
  const int n_items = IVF ? *V.n_items : n_qgroups * P.n_ranges;
  const int rank = CL > 1 ? (int)cluster_ctarank() : 0;
  const int cluster_id = blockIdx.x / CL, n_clusters = gridDim.x / CL;
  constexpr uint16_t kAllCtas = (uint16_t)((1u << CL) - 1u);

  int64_t* tile_rows = reinterpret_cast<int64_t*>(S + 1);   // GATHER: [BN] store rows of the producer's current tile
  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmap_q);
    if constexpr (!GATHER) prefetch_tensormap(tmap_p);
    // GATHER: the producer's expect_tx arrival + one cp.async arrival per lane
    // RB > 0: the expect_tx arrival + one arrival per producer thread
    for (int s = 0; s < kStages; ++s) { mbar_init(&S->full[s], RB ? 129 : GATHER ? 33 : 1); mbar_init(&S->empty[s], 8 * CL); }
    fence_barrier_init();
  }
  if (CL > 1) cluster_sync_all(); else __syncthreads();   // peers signal our barriers: their init must be visible cluster-wide

  if (warp >= 8) {
    setmaxnreg_dec<kRegsProducer>();
  }
  if (RB > 0 && warp >= 8) {
    if constexpr (RB > 0) {
      const int p = threadIdx.x - 256;   // tile row decoded by this thread
      uint16_t* rtab = reinterpret_cast<uint16_t*>(tile_rows + BN);
      const uint16_t* b16 = reinterpret_cast<const uint16_t*>(R.base);
      const uint16_t* w16 = reinterpret_cast<const uint16_t*>(R.weight);
      const int pitch = P.dim * RB / 8, ntab = P.dim << RB;
      uint32_t fill = 0;   // stages filled so far: stage fill % kStages, phase (fill / kStages) & 1
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {   // CL = 1: cluster_id = blockIdx.x
        const int4 it = V.items[item];
        const int64_t prow0 = V.offsets[it.x];
        const int len = (int)(V.offsets[it.x + 1] - prow0);
        const int64_t* ri = G.row_index + prow0 + p;
        named_bar_sync(7, 128);   // every producer thread is done with the previous item's table
        for (int e = p; e < ntab; e += 128) rtab[e] = residual_value(b16[(int64_t)it.x * P.dim + (e >> RB)], w16[e]);
        named_bar_sync(7, 128);
        for (int t0 = 0; t0 < len; t0 += BN) {
          const bool live = t0 + p < len;
          const uint8_t* crow = R.codes + (live ? ri[t0] : 0) * pitch;
          for (int kb = 0; kb < kblocks; ++kb, ++fill) {
            const uint32_t stage = fill % kStages, phase = (fill / kStages) & 1u;
            uint4 words = make_uint4(0u, 0u, 0u, 0u);
            if (live) words = residual_kblock_bits<RB>(crow, kb);   // in flight during the wait
            mbar_wait(&S->empty[stage], phase ^ 1u);
            uint8_t* st = smem + (size_t)stage * kStageBytes;
            if (warp == 8 && elect_one_sync()) {
              mbar_arrive_expect_tx(&S->full[stage], (uint32_t)kABytes);
              tma_load_2d(&tmap_q, st, &S->full[stage], kb * kKbElems, it.y, kEvictLast);
            }
            uint8_t* dst = st + kABytes + p * 128;
            const uint16_t* tab = rtab + ((kb * 64) << RB);
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              const uint4 v = live ? residual_chunk_from_table<RB>(residual_chunk_bits<RB>(words, c), tab + ((8 * c) << RB))
                                   : make_uint4(0u, 0u, 0u, 0u);
              *reinterpret_cast<uint4*>(dst + ((c ^ (p & 7)) << 4)) = v;   // SWIZZLE_128B: chunk c of row p
            }
            fence_proxy_async_smem();   // generic-proxy writes -> the consumers' wgmma (async proxy)
            mbar_arrive(&S->full[stage]);
          }
        }
      }
    }
  } else if (warp == 8) {
    // the whole warp walks the loop (uniform control flow and operands); one elected lane issues the TMA: inside an
    // `if (lane == 0)` region the compiler wraps every TMA in an ELECT / R2UR waterfall loop (ptx.cuh)
    int stage = 0;
    uint32_t phase = 0;
    for (int item = cluster_id; item < n_items; item += n_clusters) {
      int t0, t1, qrow0, prow0 = 0;
      int64_t prow_end = 0;
      if constexpr (IVF) {
        const int4 it = V.items[item];
        prow0 = (int)V.offsets[it.x];
        prow_end = V.offsets[it.x + 1];
        t0 = 0;
        t1 = (int)((prow_end - prow0 + BN - 1) / BN);
        qrow0 = it.y;
      } else {
        const int rg = item / n_qgroups, qb = (item % n_qgroups) * CL + rank;  // range-major: co-running CTAs share passages
        t0 = rg * P.tiles_per_range;
        t1 = min(P.n_tiles, t0 + P.tiles_per_range);
        qrow0 = qb * BM;
      }
      for (int t = t0; t < t1; ++t) {
        if constexpr (GATHER) {   // the tile's store rows, -1 past the list end (the previous tile's copies are issued)
          __syncwarp();
#pragma unroll
          for (int j = 0; j < BN / 32; ++j) {
            const int64_t p = prow0 + (int64_t)t * BN + lane + 32 * j;
            tile_rows[lane + 32 * j] = p < prow_end ? G.row_index[p] : -1;
          }
          __syncwarp();
        }
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&S->empty[stage], phase ^ 1u);
          uint8_t* st = smem + (size_t)stage * kStageBytes;
          if (elect_one_sync()) {
            mbar_arrive_expect_tx(&S->full[stage], (uint32_t)(GATHER ? kABytes : kStageBytes));
            const int kbp = kb < P.kb_wrap ? kb : kb - P.kb_wrap;   // fp32-split storage: [q_hi|q_lo|q_hi] x [p_hi|p_hi|p_lo]
            tma_load_2d(&tmap_q, st, &S->full[stage], kb * kKbElems, qrow0, kEvictLast);
            if constexpr (!GATHER) {
              if (CL == 1)
                tma_load_2d(tmap_p, st + kABytes, &S->full[stage], kbp * kKbElems, prow0 + t * BN, kEvictFirst);
              else  // this CTA's slice of the passage tile, written into every CTA of the cluster
                tma_load_2d_multicast(tmap_p, st + kABytes + rank * (kBBytes / CL), &S->full[stage], kbp * kKbElems,
                                      t * BN + rank * (BN / CL), kAllCtas, kEvictFirst);
            }
          }
          if constexpr (GATHER) {
            // lane = 16-byte chunk (lane & 7) of rows lane / 8 + 4 i: eight lanes read one row's 128 bytes of the k-block
            const int kbp = kb < P.kb_wrap ? kb : kb - P.kb_wrap;
            const int chunk = lane & 7;
            const uint8_t* src0 = G.rows + (size_t)kbp * 128 + chunk * 16;
            const uint32_t dst0 = smem_u32(st + kABytes);
#pragma unroll 8
            for (int i = 0; i < BN / 4; ++i) {
              const int r = (lane >> 3) + 4 * i;
              const int64_t row = tile_rows[r];
              const uint32_t dst = dst0 + r * 128 + ((chunk ^ (r & 7)) << 4);   // SWIZZLE_128B: chunk c of row r
              cp_async_16_zfill(dst, row >= 0 ? src0 + row * G.row_pitch : src0, row >= 0 ? 16u : 0u);
            }
            cp_async_mbar_arrive_noinc(&S->full[stage]);
          }
          __syncwarp();
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < 8) {
    // ------------------------------- consumers: wgmma, then filter + top-k lists ----------------------------
    // Warpgroup c computes the scores of query rows 64c .. 64c + 63 (wgmma m64n128k16, registers) and writes them to the
    // score tile; its four warps then filter them like this, thread = query row: warp (quarter, half) takes rows
    // [32 quarter, +32) and columns [64 half, +64) of every tile.  Both warps of a quarter append to the SAME per-row
    // list (shared-memory counter, atomicAdd) under the SAME threshold, so nothing about the selection changes.  The pair
    // meets at a named barrier at the start of every tile: counters are final there, both warps see the same set of
    // nearly-full rows and split their compaction.  A row gains at most BN entries per tile, so compacting when
    // cnt > cap - BN keeps every append in bounds.
    setmaxnreg_inc<kRegsConsumer>();
    const int c = warp >> 2;
    const int wq = warp & 3;
    const int quarter = 2 * c + (wq & 1);
    const int half = wq >> 1;
    const int row = quarter * 32 + lane;  // query row inside the block
    const uint32_t pair_bar = 1u + (uint32_t)quarter;
    const uint32_t wg_bar = 5u + (uint32_t)c;
    int stage = 0;
    uint32_t phase = 0;
    uint2* my_list = P.lists + ((size_t)blockIdx.x * BM + row) * kCap;
    uint2* warp_lists = P.lists + ((size_t)blockIdx.x * BM + quarter * 32) * kCap;
    int* cnt_s = S->cnt + quarter * 32;
    uint32_t* tau_s = S->tau + quarter * 32;
    const uint32_t my_cnt_addr = smem_u32(cnt_s + lane);
    const int fr0 = 64 * c + 16 * wq + (lane >> 2);   // score-tile rows of this thread's accumulator fragment: fr0, fr0 + 8
    const int fc0 = 2 * (lane & 3);
    for (int item = cluster_id; item < n_items; item += n_clusters) {
      int rg, qb, t0, t1;
      int64_t q, prow0 = 0, row_end = P.n_pass;   // rows [prow0, row_end) of the passages are candidates
      int32_t pair = -1;
      bool live;
      if constexpr (IVF) {
        const int4 it = V.items[item];
        rg = qb = 0;
        prow0 = V.offsets[it.x];
        row_end = V.offsets[it.x + 1];
        t0 = 0;
        t1 = (int)((row_end - prow0 + BN - 1) / BN);
        live = row < it.z;
        pair = live ? V.pair[it.y + row] : -1;
        q = live ? pair / V.nprobe : -1;
      } else {
        rg = item / n_qgroups;
        qb = (item % n_qgroups) * CL + rank;  // range-major: co-running CTAs share passages
        t0 = rg * P.tiles_per_range;
        t1 = min(P.n_tiles, t0 + P.tiles_per_range);
        q = (int64_t)qb * BM + row;
        live = q < P.nq;
      }
      uint32_t tau_seen = live ? P.tau_glob[q] : 0xffffffffu;  // dead rows accept nothing
      if (half == 0) { cnt_s[lane] = 0; tau_s[lane] = tau_seen; }
      for (int t = t0; t < t1; ++t) {
        {  // scores of the tile: 64 rows x 128 passages per warpgroup
          float acc[64];
#pragma unroll
          for (int j = 0; j < 64; ++j) acc[j] = 0.f;
          // one k-block's MMAs stay in flight while the next k-block is issued; a stage is released once its MMAs are done
          auto release = [&](int st) {
            __syncwarp();
            if (lane == 0) {
              if (CL == 1) mbar_arrive(&S->empty[st]);
              else
                for (int r = 0; r < CL; ++r) mbar_arrive_cluster(&S->empty[st], (uint32_t)r);
            }
          };
          int prev = -1;
          for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&S->full[stage], phase);
            if constexpr (GATHER) fence_proxy_async_smem();   // cp.async wrote the passage half: generic -> async proxy
            const uint32_t a = smem_u32(smem + (size_t)stage * kStageBytes);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)  // +32 bytes along K inside the 128-byte swizzle atom
              wgmma_n128<T>(acc, make_wgmma_sw128_desc(a + 64 * c * 128 + 32 * k), make_wgmma_sw128_desc(a + kABytes + 32 * k), 1u);
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0) release(prev);
            prev = stage;
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
          wgmma_wait<0>();
          release(prev);
          wgmma_fence_regs(acc);
          named_bar_sync(wg_bar, 128);     // every warp of the warpgroup has read the previous tile's scores
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            *reinterpret_cast<float2*>(cs + fr0 * kCsStride + 8 * j + fc0) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(cs + (fr0 + 8) * kCsStride + 8 * j + fc0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
          named_bar_sync(wg_bar, 128);
        }
        // this warp's 64 columns of its row into registers
        uint32_t r4[BN / 2 / 32][32];
#pragma unroll
        for (int cc = 0; cc < BN / 2 / 32; ++cc)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const uint4 v = *reinterpret_cast<const uint4*>(cs + row * kCsStride + half * (BN / 2) + cc * 32 + 4 * j);
            r4[cc][4 * j] = v.x; r4[cc][4 * j + 1] = v.y; r4[cc][4 * j + 2] = v.z; r4[cc][4 * j + 3] = v.w;
          }
        if (half == 0 && live) tau_s[lane] = max(tau_s[lane], tau_seen);   // other ranges' progress, fetched a tile ago
        named_bar_sync(pair_bar, 64);      // appends of the previous tile are complete, counters and thresholds final
        if (live) tau_seen = *reinterpret_cast<volatile const uint32_t*>(P.tau_glob + q);  // consumed one tile later
        const unsigned full_rows = __ballot_sync(0xffffffffu, cnt_s[lane] > kCap - BN);
        named_bar_sync(pair_bar, 64);      // both warps have read the counters before either appends to them again
        if (full_rows) {  // same value in both warps: rows are dealt alternately
          int idx = 0;
          for (unsigned m = full_rows; m; m &= m - 1, ++idx) {
            if ((idx & 1) != half) continue;
            const int rr = __ffs(m) - 1;
            uint32_t kth;
            int nc;
            if constexpr (GATHER) nc = compact_row_gather<EPL>(P, G.row_index, warp_lists + (size_t)rr * kCap, cnt_s[rr], lane, &kth);
            else nc = compact_row<EPL>(P, warp_lists + (size_t)rr * kCap, cnt_s[rr], lane, &kth);
            __syncwarp();
            int64_t q_rr = -1;   // IVF: the query of row rr
            if constexpr (IVF) q_rr = __shfl_sync(0xffffffffu, q, rr);
            if (lane == 0) {
              cnt_s[rr] = nc;
              tau_s[rr] = max(tau_s[rr], kth);
              const int64_t qq = IVF ? q_rr : (int64_t)qb * BM + quarter * 32 + rr;
              if (IVF ? qq >= 0 : qq < P.nq) atomicMax(P.tau_glob + qq, kth);
            }
          }
          named_bar_sync(pair_bar, 64);
        }
        const float tau = key2f(tau_s[lane]);
        const int64_t col0 = prow0 + (int64_t)t * BN + half * (BN / 2);
        const bool ragged = prow0 + (int64_t)t * BN + BN > row_end;
#pragma unroll
        for (int cc = 0; cc < BN / 2 / 32; ++cc) {
          uint32_t (&r)[32] = r4[cc];
          const uint32_t pbase = (uint32_t)(col0 + cc * 32);
          // A row sees a candidate in a few % of its 32-column groups, but SOME row of the warp does in most of them,
          // so the path behind the maxima has to be cheap for the idle lanes too: four sub-groups of 8 whose maxima
          // come out of one FMNMX tree, votes issued back to back, and only sub-groups with a candidate are scanned --
          // under warp-uniform control flow (per-lane branches cost a BSSY / BSYNC pair per element) with a
          // predicated atomic + store.
          float g4[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float m0 = fmaxf(fmaxf(__uint_as_float(r[8 * i]), __uint_as_float(r[8 * i + 1])), __uint_as_float(r[8 * i + 2]));
            const float m1 = fmaxf(fmaxf(__uint_as_float(r[8 * i + 3]), __uint_as_float(r[8 * i + 4])), __uint_as_float(r[8 * i + 5]));
            g4[i] = fmaxf(fmaxf(m0, m1), fmaxf(__uint_as_float(r[8 * i + 6]), __uint_as_float(r[8 * i + 7])));
          }
          const unsigned bal[4] = {__ballot_sync(0xffffffffu, g4[0] >= tau), __ballot_sync(0xffffffffu, g4[1] >= tau),
                                   __ballot_sync(0xffffffffu, g4[2] >= tau), __ballot_sync(0xffffffffu, g4[3] >= tau)};
          if ((bal[0] | bal[1]) | (bal[2] | bal[3])) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if (bal[i]) {
                uint32_t e[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  bool pass = __uint_as_float(r[8 * i + j]) >= tau;
                  if (ragged) pass = pass && (int64_t)(pbase + 8 * i + j) < row_end;
                  e[j] = pass ? (1u << j) : 0u;
                }
                uint32_t m = ((e[0] | e[1]) | (e[2] | e[3])) | ((e[4] | e[5]) | (e[6] | e[7]));
                while (__any_sync(0xffffffffu, m != 0)) {
                  const int j = (__ffs(m) - 1) & 7;  // 7 for lanes that are done (nothing stored)
                  const uint32_t a01 = (j & 1) ? r[8 * i + 1] : r[8 * i + 0], a23 = (j & 1) ? r[8 * i + 3] : r[8 * i + 2];
                  const uint32_t a45 = (j & 1) ? r[8 * i + 5] : r[8 * i + 4], a67 = (j & 1) ? r[8 * i + 7] : r[8 * i + 6];
                  const uint32_t a03 = (j & 2) ? a23 : a01, a47 = (j & 2) ? a67 : a45;
                  const uint32_t v = (j & 4) ? a47 : a03;
                  uint32_t slot;
                  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\tmov.u32 %0, 0;\n\t@p atom.shared.add.u32 %0, [%2], 1;\n\t}"
                               : "=r"(slot)
                               : "r"(m), "r"(my_cnt_addr)
                               : "memory");
                  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %0, 0;\n\t@p st.global.v2.u32 [%1], {%2, %3};\n\t}"
                               ::"r"(m), "l"(my_list + slot), "r"(v), "r"(pbase + 8 * i + j)
                               : "memory");
                  m &= m - 1;
                }
              }
            }
          }
        }
      }
      // item done: final compaction of every row (split between the two warps), then publish (score, id) candidates
      named_bar_sync(pair_bar, 64);
      for (int rr = half; rr < 32; rr += 2) {
        uint32_t kth;
        int nc;
        if constexpr (GATHER) nc = compact_row_gather<EPL>(P, G.row_index, warp_lists + (size_t)rr * kCap, cnt_s[rr], lane, &kth);
        else nc = compact_row<EPL>(P, warp_lists + (size_t)rr * kCap, cnt_s[rr], lane, &kth);
        int64_t q_rr = -1;   // IVF: the query of row rr and its output slot
        size_t slot_rr = 0;
        if constexpr (IVF) {
          q_rr = __shfl_sync(0xffffffffu, q, rr);
          slot_rr = (size_t)__shfl_sync(0xffffffffu, pair, rr) * P.kpad;
        }
        const int64_t qq = IVF ? q_rr : (int64_t)qb * BM + quarter * 32 + rr;
        if (IVF ? qq >= 0 : qq < P.nq) {
          if (lane == 0 && nc == P.k) atomicMax(P.tau_glob + qq, kth);
          const uint2* lst = warp_lists + (size_t)rr * kCap;
          float* cso = IVF ? P.cand_scores + slot_rr : P.cand_scores + (size_t)qq * P.n_ranges * P.kpad + (size_t)rg * P.kpad;
          int64_t* ci = IVF ? P.cand_ids + slot_rr : P.cand_ids + (size_t)qq * P.n_ranges * P.kpad + (size_t)rg * P.kpad;
          for (int e = lane; e < P.kpad; e += 32) {
            if (e < nc) {
              const uint2 v = lst[e];
              cso[e] = __uint_as_float(v.x);
              ci[e] = GATHER ? P.ids[G.row_index[v.y]] : pos_to_id(P, v.y);
            } else {
              cso[e] = -INFINITY;
              ci[e] = -1;
            }
          }
        }
        __syncwarp();
      }
      named_bar_sync(pair_bar, 64);   // the counters are reset by the next item only after both warps are done with them
    }
  }

  if (CL > 1) cluster_sync_all(); else __syncthreads();   // no CTA may exit while peers still multicast into it
}

template <typename T, int CL, int EPL = 32, bool IVF = false>
__global__ void __launch_bounds__(kThreads, 1)
flat_ip_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_p, FipParams P,
                  IvfParams V) {
  flat_ip_tc_body<T, CL, EPL, IVF, false>(tmap_q, &tmap_p, P, V, GatherParams{});
}

// A kernel of its own rather than one more flag on flat_ip_tc_kernel: the flat and IVF instantiations keep their names
// and parameter blocks, and this one takes no passage tensor map.
template <typename T, int EPL>
__global__ void __launch_bounds__(kThreads, 1)
flat_ip_tc_gather_kernel(const __grid_constant__ CUtensorMap tmap_q, FipParams P, IvfParams V, GatherParams G) {
  flat_ip_tc_body<T, 1, EPL, true, true>(tmap_q, nullptr, P, V, G);
}

// The gather mode over RB-bit residual codes (mmb200_ivf_search_residual): G.rows is unused, G.row_index as above.
template <int EPL, int RB>
__global__ void __launch_bounds__(kThreads, 1)
flat_ip_tc_residual_kernel(const __grid_constant__ CUtensorMap tmap_q, FipParams P, IvfParams V, GatherParams G,
                           ResidualCodes R) {
  flat_ip_tc_body<__half, 1, EPL, true, true, RB>(tmap_q, nullptr, P, V, G, R);
}

// E4M3 queries and rows (MMB200_F8E4M3): the same bodies, with 128-element k-blocks and wgmma m64n128k32.  Kernels of
// their own name, not instantiations of the two above: those names stand for the HGMMA (16-bit) kernels, while these
// emit QGMMA.
template <int CL, int EPL>
__global__ void __launch_bounds__(kThreads, 1)
flat_ip_tc_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_p, FipParams P,
                      IvfParams V) {
  flat_ip_tc_body<__nv_fp8_e4m3, CL, EPL, false, false>(tmap_q, &tmap_p, P, V, GatherParams{});
}

template <int EPL>
__global__ void __launch_bounds__(kThreads, 1)
flat_ip_tc_gather_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q, FipParams P, IvfParams V, GatherParams G) {
  flat_ip_tc_body<__nv_fp8_e4m3, 1, EPL, true, true>(tmap_q, nullptr, P, V, G);
}


// ---------------------------------------------------------------------------------------------
// merge: per query, sort L candidates by (score desc, id asc), emit the first k.
// ---------------------------------------------------------------------------------------------
struct Cand {
  float s;
  int32_t valid;
  int64_t id;
};
__device__ __forceinline__ bool cand_before(const Cand& a, const Cand& b) {
  if (a.valid != b.valid) return a.valid > b.valid;
  if (a.s != b.s) return a.s > b.s;
  return a.id < b.id;
}
// (valid desc, id asc, score desc): the order in which the first entry of every id is its best one
__device__ __forceinline__ bool cand_before_by_id(const Cand& a, const Cand& b) {
  if (a.valid != b.valid) return a.valid > b.valid;
  if (a.id != b.id) return a.id < b.id;
  return a.s > b.s;
}

// In-place bitonic sort of c[0, Lpow2) by the order `kById ? cand_before_by_id : cand_before`; ends with __syncthreads.
template <bool kById>
__device__ __forceinline__ void bitonic_sort(Cand* c, int Lpow2) {
  for (int size = 2; size <= Lpow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int e = threadIdx.x; e < Lpow2 / 2; e += blockDim.x) {
        const int i = 2 * e - (e & (stride - 1));
        const int j = i + stride;
        const bool up = ((i & size) == 0);
        const Cand a = c[i], b = c[j];
        const bool swap = kById ? (up ? cand_before_by_id(b, a) : cand_before_by_id(a, b))
                                : (up ? cand_before(b, a) : cand_before(a, b));
        if (swap) { c[i] = b; c[j] = a; }
      }
      __syncthreads();
    }
  }
}

// Block (q, grp) sorts candidates [grp * seg, min(L, (grp + 1) * seg)) of query q and writes its k best to row
// q * n_groups + grp of the output.  A candidate is void when its score is NaN, -inf or faiss's "no result" value
// (-FLT_MAX) -- NOT by the sign of its id: faiss IndexIDMap accepts negative user ids.  `final_pass` selects the
// filler for missing results: (-FLT_MAX, -1) as faiss returns them, or (-inf, -1) between passes.
// `unique` (mmb200_topk_unique): every id is kept once, with its highest score -- a first sort by (id, score desc)
// voids all but the first entry of each id, then the usual sort ranks the survivors.  Unique-with-max composes over
// groups, so the pass structure stays exact.
__global__ void __launch_bounds__(256) topk_merge_kernel(const float* __restrict__ cand_scores,
                                                         const int64_t* __restrict__ cand_ids, int64_t nq, int L, int seg,
                                                         int n_groups, int Lpow2, int k, int final_pass, int unique,
                                                         float* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
  extern __shared__ __align__(16) uint8_t msm[];
  Cand* c = reinterpret_cast<Cand*>(msm);
  for (int64_t item = blockIdx.x; item < nq * n_groups; item += gridDim.x) {
    const int64_t q = item / n_groups;
    const int grp = (int)(item % n_groups);
    const int lo = grp * seg, n = min(seg, L - lo);
    __syncthreads();
    for (int e = threadIdx.x; e < Lpow2; e += blockDim.x) {
      Cand v;
      if (e < n) {
        v.s = cand_scores[q * L + lo + e];
        v.id = cand_ids[q * L + lo + e];
        v.valid = (v.s == v.s && v.s > -3.4028234663852886e38f) ? 1 : 0;
      } else {
        v.s = -INFINITY; v.id = -1; v.valid = 0;
      }
      c[e] = v;
    }
    __syncthreads();
    if (unique) {
      bitonic_sort<true>(c, Lpow2);
      uint32_t dup = 0;   // bit b: element threadIdx.x + b * blockDim.x repeats the id before it (Lpow2 <= 32 * 256)
      for (int e = threadIdx.x, b = 0; e < Lpow2; e += blockDim.x, ++b)
        if (e > 0 && c[e].valid && c[e - 1].valid && c[e].id == c[e - 1].id) dup |= 1u << b;
      __syncthreads();
      for (int e = threadIdx.x, b = 0; e < Lpow2; e += blockDim.x, ++b)
        if ((dup >> b) & 1u) c[e].valid = 0;
      __syncthreads();
    }
    bitonic_sort<false>(c, Lpow2);
    for (int e = threadIdx.x; e < k; e += blockDim.x) {
      const bool ok = e < Lpow2 && c[e].valid;
      out_scores[item * k + e] = ok ? c[e].s : (final_pass ? -3.4028234663852886e38f : -INFINITY);
      out_ids[item * k + e] = ok ? c[e].id : -1;
    }
  }
}

struct Plan {
  int n_qblocks, n_tiles, n_ranges, tiles_per_range, grid, kpad, cl;
};

Plan make_plan(int64_t nq, int64_t n_pass, int k, int sm_count) {
  Plan pl;
  pl.n_qblocks = (int)((nq + BM - 1) / BM);
  pl.n_tiles = (int)((n_pass + BN - 1) / BN);
  pl.kpad = (k + 31) / 32 * 32;
  // cluster size: CTAs of a cluster take consecutive query blocks and share every passage tile by TMA multicast.  A
  // cluster slot without a query block still runs (its slice of the passage tile is needed by its peers), so only pair
  // up when little is wasted.  MMB200_FLATIP_CLUSTER overrides (1, 2 or 4).
  pl.cl = (pl.n_qblocks % 2 == 0 || pl.n_qblocks >= 9) ? 2 : 1;
  if (const char* env = getenv("MMB200_FLATIP_CLUSTER")) {
    const int c = atoi(env);
    if (c == 1 || c == 2 || c == 4) pl.cl = c;
  }
  const int n_qgroups = (pl.n_qblocks + pl.cl - 1) / pl.cl;
  const int max_clusters = std::max(1, sm_count / pl.cl);
  // number of passage ranges: every range restarts its threshold at -inf and pays ~log(range/k) list
  // compactions per query, so take the SMALLEST count whose item grid fills the SMs to >= 88 % (or the best
  // fill available).  MMB200_FLATIP_RANGES overrides it for experiments.
  int best_r = 1;
  double best_eff = -1.0;
  const int max_r = std::max(1, std::min(kMaxRanges, pl.n_tiles));
  double effs[kMaxRanges + 1];
  for (int r = 1; r <= max_r; ++r) {
    const int64_t items = (int64_t)n_qgroups * r;
    const int64_t g = std::min<int64_t>(max_clusters, items);
    const int64_t waves = (items + g - 1) / g;
    effs[r] = (double)items / (double)(waves * max_clusters);
    if (effs[r] > best_eff + 1e-9) { best_eff = effs[r]; best_r = r; }
  }
  for (int r = 1; r <= max_r; ++r)
    if (effs[r] >= 0.88 || effs[r] >= best_eff - 1e-9) { best_r = r; break; }
  if (const char* env = getenv("MMB200_FLATIP_RANGES")) {
    const int r = atoi(env);
    if (r >= 1 && r <= max_r) best_r = r;
  }
  pl.tiles_per_range = (pl.n_tiles + best_r - 1) / best_r;
  pl.n_ranges = (pl.n_tiles + pl.tiles_per_range - 1) / pl.tiles_per_range;
  pl.grid = pl.cl * (int)std::min<int64_t>(max_clusters, (int64_t)n_qgroups * pl.n_ranges);
  return pl;
}

inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

size_t workspace_bytes(const Plan& pl, int64_t nq, int k) {
  const size_t cap = 32 * (size_t)epl_for_k(k);
  return align256((size_t)nq * sizeof(uint32_t)) + align256((size_t)pl.grid * BM * cap * sizeof(uint2)) +
         align256((size_t)nq * pl.n_ranges * pl.kpad * sizeof(float)) +
         align256((size_t)nq * pl.n_ranges * pl.kpad * sizeof(int64_t));
}

size_t total_workspace_bytes(int64_t nq, int64_t n_pass, int k, int sm_count) {
  return workspace_bytes(make_plan(nq, n_pass, k, sm_count), nq, k);
}

__global__ void fill_u32(uint32_t* p, int64_t n, uint32_t v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// Largest candidate count one shared-memory sort takes (16 B per candidate).  More than that -- many passage ranges at
// k = 1024, or sharding.topk_all_gather_merge over a shard with thousands of local scores per query -- is merged in
// passes: groups of kMergeSeg candidates are cut to their k best, the survivors merged again.
constexpr int kMergeSeg = 8192;
constexpr int kMaxUniqueK = kMergeSeg / 2;

int launch_merge(const float* cand_scores, const int64_t* cand_ids, int64_t nq, int L, int k, float* out_scores,
                 int64_t* out_ids, const DeviceInfo& dev, cudaStream_t stream, bool unique = false) {
  MMB_CHECK_CUDA(cudaFuncSetAttribute(topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)(kMergeSeg * sizeof(Cand))));
  const float* in_s = cand_scores;
  const int64_t* in_i = cand_ids;
  float* tmp_s[2] = {nullptr, nullptr};
  int64_t* tmp_i[2] = {nullptr, nullptr};
  int cur = 0;
  int rc = MMB200_OK;
  while (true) {
    const bool last = L <= kMergeSeg;
    const int seg = last ? L : kMergeSeg;
    const int groups = (L + seg - 1) / seg;
    int lp = 2;
    while (lp < seg) lp <<= 1;
    const int k_out = last ? k : std::min(k, seg);
    float* o_s = out_scores;
    int64_t* o_i = out_ids;
    if (!last) {
      if (cudaMallocAsync(reinterpret_cast<void**>(&tmp_s[cur]), (size_t)nq * groups * k_out * sizeof(float), stream) != cudaSuccess ||
          cudaMallocAsync(reinterpret_cast<void**>(&tmp_i[cur]), (size_t)nq * groups * k_out * sizeof(int64_t), stream) != cudaSuccess) {
        set_error("topk merge: cannot allocate the intermediate candidate lists");
        rc = MMB200_ERR_CUDA;
        break;
      }
      o_s = tmp_s[cur];
      o_i = tmp_i[cur];
    }
    const int grid = (int)std::min<int64_t>(nq * groups, (int64_t)dev.sm_count * 4);
    topk_merge_kernel<<<grid, 256, (size_t)lp * sizeof(Cand), stream>>>(in_s, in_i, nq, L, seg, groups, lp, k_out, last ? 1 : 0,
                                                                        unique ? 1 : 0, o_s, o_i);
    if (cudaGetLastError() != cudaSuccess) {
      set_error("topk merge: kernel launch failed");
      rc = MMB200_ERR_CUDA;
      break;
    }
    if (last) break;
    in_s = o_s;
    in_i = o_i;
    L = groups * k_out;
    cur ^= 1;
    if (tmp_s[cur]) {  // the buffers of two passes ago are no longer read by anything enqueued after this point
      cudaFreeAsync(tmp_s[cur], stream);
      cudaFreeAsync(tmp_i[cur], stream);
      tmp_s[cur] = nullptr;
      tmp_i[cur] = nullptr;
    }
  }
  for (int i = 0; i < 2; ++i) {
    if (tmp_s[i]) cudaFreeAsync(tmp_s[i], stream);
    if (tmp_i[i]) cudaFreeAsync(tmp_i[i], stream);
  }
  return rc;
}

// ---------------------------------------------------------------------------------------------
// IVF probed-list scan: invert the probe table [nq, nprobe] into per-list query sets on the device, gather the probing
// queries list by list, scan every (list, chunk of <= BM queries) item with flat_ip_tc_kernel<..., IVF = true>, merge
// the per-(query, probe) slots.  Nothing is read back to the host: the item count stays in device memory.
// ---------------------------------------------------------------------------------------------
static_assert(BM == kIvfChunk, "an IVF work item is one query block");

// One warp per (query, probe) pair: take the next row of the probed list's query set and copy the query there.  A pair
// whose list id is out of range (a -1 filler of the coarse search) probes nothing: its slot is filled as empty.
__global__ void ivf_gather_kernel(const int64_t* __restrict__ probes, int64_t n_pairs, int64_t nlist, int nprobe,
                                  const int* __restrict__ row_base, int* __restrict__ fill, const uint4* __restrict__ queries,
                                  int row_vecs, uint4* __restrict__ gathered, int32_t* __restrict__ pair_of_row,
                                  float* __restrict__ cand_scores, int64_t* __restrict__ cand_ids, int kslot) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = warp0; p < n_pairs; p += n_warps) {
    const int64_t l = probes[p];
    const bool ok = l >= 0 && l < nlist;
    int r = 0;
    if (ok && lane == 0) r = row_base[l] + atomicAdd(fill + l, 1);
    r = __shfl_sync(0xffffffffu, r, 0);
    if (ok) {
      const uint4* src = queries + (p / nprobe) * row_vecs;
      uint4* dst = gathered + (int64_t)r * row_vecs;
      for (int v = lane; v < row_vecs; v += 32) dst[v] = src[v];
      if (lane == 0) pair_of_row[r] = (int32_t)p;
    } else {
      for (int e = lane; e < kslot; e += 32) {
        cand_scores[p * kslot + e] = -INFINITY;
        cand_ids[p * kslot + e] = -1;
      }
    }
  }
}

struct IvfLayout {
  size_t tau, lists, cand_s, cand_i, gathered, pair, cnt, fill, row_base, item_base, items, n_items, total;
  int kslot, grid;
  int64_t n_pairs, max_items;
};

// slot = per-(query, probe) candidates: a list of len rows yields at most min(k, len) of them
IvfLayout ivf_layout(int64_t nq, int nprobe, int64_t nlist, int64_t max_list_len, int qbytes, int k, int sm_count) {
  IvfLayout L{};
  L.grid = sm_count;
  L.n_pairs = nq * nprobe;
  L.kslot = (int)((std::min<int64_t>(k, std::max<int64_t>(1, max_list_len)) + 31) / 32 * 32);
  L.max_items = std::min<int64_t>(nlist, L.n_pairs) + (L.n_pairs + BM - 1) / BM;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
  L.tau = take((size_t)nq * sizeof(uint32_t));
  L.lists = take((size_t)L.grid * BM * 32 * epl_for_k(k) * sizeof(uint2));
  L.cand_s = take((size_t)L.n_pairs * L.kslot * sizeof(float));
  L.cand_i = take((size_t)L.n_pairs * L.kslot * sizeof(int64_t));
  L.gathered = take((size_t)L.n_pairs * qbytes);
  L.pair = take((size_t)L.n_pairs * sizeof(int32_t));
  L.cnt = take((size_t)nlist * sizeof(int));
  L.fill = take((size_t)nlist * sizeof(int));
  L.row_base = take((size_t)nlist * sizeof(int));
  L.item_base = take((size_t)nlist * sizeof(int));
  L.items = take((size_t)L.max_items * sizeof(int4));
  L.n_items = take(sizeof(int));
  L.total = off;
  return L;
}

}  // namespace

}  // namespace mmb

extern "C" int64_t mmb200_flat_ip_workspace_bytes(int64_t nq, int64_t n_pass, int32_t k) {
  using namespace mmb;
  if (nq <= 0 || n_pass <= 0 || k <= 0 || k > kMaxK) return 0;
  DeviceInfo dev;
  if (current_device_info(&dev)) return -1;
  return (int64_t)total_workspace_bytes(nq, n_pass, k, dev.sm_count);
}

extern "C" int mmb200_flat_ip_plan(int64_t nq, int64_t n_pass, int32_t k, int32_t sm_count, int32_t out[8]) {
  using namespace mmb;
  MMB_REQUIRE(out != nullptr, "null pointer");
  MMB_REQUIRE(nq > 0 && n_pass > 0 && k >= 1 && k <= kMaxK && sm_count >= 1, "bad sizes");
  MMB_REQUIRE(n_pass < (1ll << 32) - 512, "at most 2^32 passages per shard");
  const Plan pl = make_plan(nq, n_pass, k, sm_count);
  const uint64_t ws = (uint64_t)workspace_bytes(pl, nq, k);
  out[0] = pl.n_qblocks; out[1] = pl.n_tiles; out[2] = pl.n_ranges; out[3] = pl.tiles_per_range; out[4] = pl.grid; out[5] = pl.cl;
  out[6] = (int32_t)(uint32_t)(ws & 0xffffffffu); out[7] = (int32_t)(uint32_t)(ws >> 32);
  return MMB200_OK;
}

extern "C" int mmb200_flat_ip_topk(const void* queries, const void* passages, const int64_t* ids, float* out_scores,
                                   int64_t* out_ids, void* workspace, int64_t workspace_bytes_given, int64_t nq,
                                   int64_t n_pass, int32_t dim, int32_t k, int32_t dtype, int64_t id_base,
                                   void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(nq >= 0 && n_pass > 0, "need at least one passage");
  MMB_REQUIRE(k >= 1 && k <= kMaxK, "fused top-k supports 1 <= k <= 1024");
  MMB_REQUIRE(dtype == MMB200_F16 || dtype == MMB200_BF16 || dtype == MMB200_F32_SPLIT16 || dtype == MMB200_F8E4M3,
              "passage storage must be fp16, bf16, e4m3 or the fp16 hi/lo split of fp32 (MMB200_F32_SPLIT16)");
  MMB_REQUIRE(dim % 64 == 0 && dim >= 64, "vector dim must be a multiple of 64");
  const bool fp8 = dtype == MMB200_F8E4M3;
  MMB_REQUIRE(!fp8 || (dim % 128 == 0 && dim >= 128 && dim <= 1024), "e4m3 vectors need dim % 128 == 0, 128 <= dim <= 1024");
  MMB_REQUIRE(n_pass < (1ll << 32) - 512, "at most 2^32 passages per shard");
  if (nq == 0) return MMB200_OK;   // an empty batch: nothing to read or write (its tensors may be null), no device needed
  MMB_REQUIRE(queries && passages && out_scores && out_ids && workspace, "null pointer");
  const bool split = dtype == MMB200_F32_SPLIT16;
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(queries) | reinterpret_cast<uintptr_t>(passages)) & 15) == 0, "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const Plan pl = make_plan(nq, n_pass, k, dev.sm_count);
  MMB_REQUIRE((size_t)workspace_bytes_given >= total_workspace_bytes(nq, n_pass, k, dev.sm_count),
              "workspace too small (see mmb200_flat_ip_workspace_bytes)");
  const CUtensorMapDataType tdt = fp8                  ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                  : dtype == MMB200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                         : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const uint64_t q_cols = split ? 3ull * dim : (uint64_t)dim, p_cols = split ? 2ull * dim : (uint64_t)dim;
  const uint32_t esize = fp8 ? 1u : 2u, kbe = 128u / esize;   // bytes per element, elements per 128-byte k-block
  CUtensorMap tq;
  {
    const uint64_t dims[2] = {q_cols, (uint64_t)nq};
    const uint64_t strides[1] = {q_cols * esize};
    const uint32_t box[2] = {kbe, BM};
    if (int rc = encode_tensor_map(&tq, tdt, 2, queries, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  uint32_t* tau_glob = static_cast<uint32_t*>(workspace);
  fill_u32<<<64, 256, 0, stream>>>(tau_glob, nq, kKeyNegInf);
  MMB_CHECK_CUDA(cudaGetLastError());

  // one pass of flat_ip_tc_kernel over `n_rows` passages whose rows are `row_pitch` bytes apart
  auto run_pass = [&](const Plan& pp, int64_t n_rows, uint64_t row_pitch, const int64_t* pass_ids, int64_t pass_id_base,
                      FipParams* out_params) -> int {
    FipParams P{};
    uint8_t* w = static_cast<uint8_t*>(workspace) + align256((size_t)nq * sizeof(uint32_t));
    P.tau_glob = tau_glob;
    P.lists = reinterpret_cast<uint2*>(w);
    w += align256((size_t)pp.grid * BM * 32 * (size_t)epl_for_k(k) * sizeof(uint2));
    P.cand_scores = reinterpret_cast<float*>(w);
    w += align256((size_t)nq * pp.n_ranges * pp.kpad * sizeof(float));
    P.cand_ids = reinterpret_cast<int64_t*>(w);
    P.ids = pass_ids; P.id_base = pass_id_base; P.nq = nq; P.n_pass = n_rows; P.dim = dim; P.k = k; P.kpad = pp.kpad;
    P.n_qblocks = pp.n_qblocks; P.n_ranges = pp.n_ranges; P.tiles_per_range = pp.tiles_per_range; P.n_tiles = pp.n_tiles;
    P.kblocks = (int32_t)(q_cols / kbe);
    P.kb_wrap = split ? dim / 64 : P.kblocks;
    CUtensorMap tp;
    {
      const uint64_t dims[2] = {p_cols, (uint64_t)n_rows};
      const uint64_t strides[1] = {row_pitch};
      const uint32_t box[2] = {kbe, (uint32_t)(BN / pp.cl)};   // each CTA of a cluster fetches (and multicasts) its slice
      if (int rc = encode_tensor_map(&tp, tdt, 2, passages, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
        return rc;
    }
    const size_t smem = (size_t)kStages * kStageBytes + (size_t)BM * kCsStride * sizeof(float) + sizeof(FipShared) + 1024;
    auto launch = [&](auto kernel) -> int {
      MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      cudaLaunchConfig_t cfg{};
      cfg.gridDim = dim3((unsigned)pp.grid);
      cfg.blockDim = dim3(kThreads);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = stream;
      cudaLaunchAttribute attr{};
      attr.id = cudaLaunchAttributeClusterDimension;
      attr.val.clusterDim.x = (unsigned)pp.cl;
      attr.val.clusterDim.y = 1;
      attr.val.clusterDim.z = 1;
      cfg.attrs = &attr;
      cfg.numAttrs = 1;
      MMB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, tq, tp, P, IvfParams{}));
      return MMB200_OK;
    };
    if (out_params) *out_params = P;
    auto by_cluster = [&](auto t, auto epl) -> int {
      using T = decltype(t);
      constexpr int E = decltype(epl)::value;
      return pp.cl == 1   ? launch(flat_ip_tc_kernel<T, 1, E>)
             : pp.cl == 2 ? launch(flat_ip_tc_kernel<T, 2, E>)
                          : launch(flat_ip_tc_kernel<T, 4, E>);
    };
    auto fp8_by_cluster = [&](auto epl) -> int {
      constexpr int E = decltype(epl)::value;
      return pp.cl == 1   ? launch(flat_ip_tc_fp8_kernel<1, E>)
             : pp.cl == 2 ? launch(flat_ip_tc_fp8_kernel<2, E>)
                          : launch(flat_ip_tc_fp8_kernel<4, E>);
    };
    using E32 = std::integral_constant<int, 32>;
    using E64 = std::integral_constant<int, 64>;
    if (fp8) return epl_for_k(k) == 32 ? fp8_by_cluster(E32{}) : fp8_by_cluster(E64{});
    if (dtype == MMB200_BF16) return epl_for_k(k) == 32 ? by_cluster(__nv_bfloat16{}, E32{}) : by_cluster(__nv_bfloat16{}, E64{});
    return epl_for_k(k) == 32 ? by_cluster(__half{}, E32{}) : by_cluster(__half{}, E64{});
  };

  FipParams P{};
  if (int rc = run_pass(pl, n_pass, p_cols * esize, ids, id_base, &P)) return rc;
  return launch_merge(P.cand_scores, P.cand_ids, nq, pl.n_ranges * pl.kpad, k, out_scores, out_ids, dev, stream);
}

extern "C" int mmb200_topk_merge(const float* cand_scores, const int64_t* cand_ids, float* out_scores, int64_t* out_ids,
                                 int64_t nq, int32_t n_candidates, int32_t k, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(cand_scores && cand_ids && out_scores && out_ids, "null pointer");
  MMB_REQUIRE(nq >= 0 && n_candidates >= 1 && k >= 1, "bad sizes");
  if (nq == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  return launch_merge(cand_scores, cand_ids, nq, n_candidates, k, out_scores, out_ids, dev, static_cast<cudaStream_t>(stream_));
}

extern "C" int mmb200_topk_unique(const float* cand_scores, const int64_t* cand_ids, float* out_scores, int64_t* out_ids,
                                  int64_t nq, int32_t n_candidates, int32_t k, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(cand_scores && cand_ids && out_scores && out_ids, "null pointer");
  MMB_REQUIRE(nq >= 0 && n_candidates >= 1 && k >= 1, "bad sizes");
  if (k > kMaxUniqueK) {
    // a pass over groups of kMergeSeg candidates shrinks the list only while k <= kMergeSeg / 2
    set_error("topk_unique supports k <= 4096");
    return MMB200_ERR_UNSUPPORTED;
  }
  if (nq == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  return launch_merge(cand_scores, cand_ids, nq, n_candidates, k, out_scores, out_ids, dev, static_cast<cudaStream_t>(stream_),
                      true);
}

extern "C" int64_t mmb200_ivf_workspace_bytes(int64_t nq, int32_t nprobe, int64_t nlist, int64_t max_list_len, int32_t dim,
                                              int32_t k, int32_t dtype) {
  using namespace mmb;
  if (nq <= 0 || nprobe <= 0 || nprobe > kIvfMaxProbe || nlist <= 0 || k <= 0 || k > kMaxK || dim <= 0 || dim % 64 ||
      nq * nprobe >= (1ll << 31) - BM)
    return 0;
  if (dtype != MMB200_F16 && dtype != MMB200_BF16 && dtype != MMB200_F32_SPLIT16 && dtype != MMB200_F8E4M3) return 0;
  if (dtype == MMB200_F8E4M3 && (dim % 128 || dim < 128 || dim > 1024)) return 0;
  DeviceInfo dev;
  if (current_device_info(&dev)) return -1;
  const int qbytes = dtype == MMB200_F32_SPLIT16 ? 6 * dim : dtype == MMB200_F8E4M3 ? dim : 2 * dim;
  return (int64_t)ivf_layout(nq, nprobe, nlist, max_list_len, qbytes, k, dev.sm_count).total;
}

namespace mmb {
namespace {
// mmb200_ivf_search (row_index == nullptr: list position = row), mmb200_ivf_search_gather (list position p = row
// row_index[p] of the rows as given) and mmb200_ivf_search_residual (the same over residual codes R, rows = R->codes).
int ivf_search_impl(const void* queries, const void* rows, const int64_t* ids, const int64_t* row_index,
                    const int64_t* list_offsets, const int64_t* probes, float* out_scores, int64_t* out_ids, void* workspace,
                    int64_t workspace_bytes_given, int64_t nq, int32_t nprobe, int64_t nlist, int64_t n_rows,
                    int64_t max_list_len, int32_t dim, int32_t k, int32_t dtype, void* stream_,
                    const ResidualCodes* R = nullptr) {
  MMB_REQUIRE(queries && rows && ids && list_offsets && probes && out_scores && out_ids && workspace, "null pointer");
  MMB_REQUIRE(nq > 0 && nlist > 0 && n_rows > 0, "need at least one query, one list and one row");
  MMB_REQUIRE(k >= 1 && k <= kMaxK, "fused top-k supports 1 <= k <= 1024");
  MMB_REQUIRE(nprobe >= 1 && nprobe <= kIvfMaxProbe, "1 <= nprobe <= 1024");
  MMB_REQUIRE(dtype == MMB200_F16 || dtype == MMB200_BF16 || dtype == MMB200_F32_SPLIT16 ||
                  (dtype == MMB200_F8E4M3 && row_index && !R),
              "list storage must be fp16, bf16 or the fp16 hi/lo split of fp32 (MMB200_F32_SPLIT16); e4m3 rows are "
              "scanned in gather mode only");
  MMB_REQUIRE(dim % 64 == 0 && dim >= 64, "vector dim must be a multiple of 64");
  const bool fp8 = dtype == MMB200_F8E4M3;
  MMB_REQUIRE(!fp8 || (dim % 128 == 0 && dim >= 128 && dim <= 1024), "e4m3 vectors need dim % 128 == 0, 128 <= dim <= 1024");
  MMB_REQUIRE(n_rows < (1ll << 31) - BN, "at most 2^31 - 128 rows per shard");
  MMB_REQUIRE(max_list_len >= 0 && max_list_len <= n_rows, "max_list_len must bound the list lengths");
  MMB_REQUIRE(nq * nprobe < (1ll << 31) - BM, "nq * nprobe must stay below 2^31 (search the queries in batches)");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(queries) | reinterpret_cast<uintptr_t>(rows)) & 15) == 0, "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool split = dtype == MMB200_F32_SPLIT16;
  const int qcols = split ? 3 * dim : dim, pcols = split ? 2 * dim : dim;
  const int esize = fp8 ? 1 : 2, kbe = 128 / esize;   // bytes per element, elements per 128-byte k-block
  const IvfLayout L = ivf_layout(nq, nprobe, nlist, max_list_len, qcols * esize, k, dev.sm_count);
  MMB_REQUIRE((size_t)workspace_bytes_given >= L.total, "workspace too small (see mmb200_ivf_workspace_bytes)");
  uint8_t* w = static_cast<uint8_t*>(workspace);
  int* cnt = reinterpret_cast<int*>(w + L.cnt);
  int* fill = reinterpret_cast<int*>(w + L.fill);
  int* row_base = reinterpret_cast<int*>(w + L.row_base);
  int* item_base = reinterpret_cast<int*>(w + L.item_base);
  int4* items = reinterpret_cast<int4*>(w + L.items);
  int* n_items = reinterpret_cast<int*>(w + L.n_items);
  int32_t* pair_of_row = reinterpret_cast<int32_t*>(w + L.pair);
  uint4* gathered = reinterpret_cast<uint4*>(w + L.gathered);

  // probe table -> per-list query sets -> work items
  MMB_CHECK_CUDA(cudaMemsetAsync(cnt, 0, L.row_base - L.cnt, stream));   // cnt and fill
  const int g = std::max(1, std::min(dev.sm_count * 8, (int)((L.n_pairs + 255) / 256)));
  ivf_count_kernel<<<g, 256, 0, stream>>>(probes, L.n_pairs, nlist, cnt);
  ivf_scan_kernel<<<1, 1024, 0, stream>>>(cnt, nlist, row_base, item_base, n_items);
  ivf_gather_kernel<<<std::max(1, std::min(dev.sm_count * 8, (int)((L.n_pairs + 7) / 8))), 256, 0, stream>>>(
      probes, L.n_pairs, nlist, nprobe, row_base, fill, static_cast<const uint4*>(queries), qcols * esize / 16, gathered,
      pair_of_row, reinterpret_cast<float*>(w + L.cand_s), reinterpret_cast<int64_t*>(w + L.cand_i), L.kslot);
  ivf_items_kernel<<<std::max(1, std::min(dev.sm_count * 4, (int)((nlist + 255) / 256))), 256, 0, stream>>>(
      cnt, nlist, row_base, item_base, items);
  uint32_t* tau_glob = reinterpret_cast<uint32_t*>(w + L.tau);
  fill_u32<<<64, 256, 0, stream>>>(tau_glob, nq, kKeyNegInf);
  MMB_CHECK_CUDA(cudaGetLastError());

  const CUtensorMapDataType tdt = fp8                  ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                  : dtype == MMB200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                         : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const bool gather = row_index != nullptr;
  CUtensorMap tq, tp;
  {
    const uint64_t dims[2] = {(uint64_t)qcols, (uint64_t)L.n_pairs};
    const uint64_t strides[1] = {(uint64_t)qcols * esize};
    const uint32_t box[2] = {(uint32_t)kbe, BM};
    if (int rc = encode_tensor_map(&tq, tdt, 2, gathered, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  if (!gather) {
    const uint64_t dims[2] = {(uint64_t)pcols, (uint64_t)n_rows};
    const uint64_t strides[1] = {(uint64_t)pcols * 2};
    const uint32_t box[2] = {64, BN};
    if (int rc = encode_tensor_map(&tp, tdt, 2, rows, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  FipParams P{};
  P.ids = ids; P.id_base = 0; P.nq = nq; P.n_pass = n_rows; P.dim = dim; P.k = k; P.kpad = L.kslot;
  P.kblocks = qcols / kbe;
  P.kb_wrap = split ? dim / 64 : P.kblocks;
  P.n_qblocks = 0; P.n_ranges = 1; P.tiles_per_range = 0; P.n_tiles = 0;
  P.tau_glob = tau_glob;
  P.lists = reinterpret_cast<uint2*>(w + L.lists);
  P.cand_scores = reinterpret_cast<float*>(w + L.cand_s);
  P.cand_ids = reinterpret_cast<int64_t*>(w + L.cand_i);
  const IvfParams V{items, n_items, list_offsets, pair_of_row, nprobe};
  // the gather mode keeps its tile's store rows behind FipShared, the residual mode its list's decoded values after them
  const size_t smem = (size_t)kStages * kStageBytes + (size_t)BM * kCsStride * sizeof(float) + sizeof(FipShared) + 1024 +
                      (gather ? BN * sizeof(int64_t) : 0) + (R ? ((size_t)dim << R->bits) * sizeof(__half) : 0);
  auto launch = [&](auto kernel) -> int {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<L.grid, kThreads, smem, stream>>>(tq, tp, P, V);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  };
  const GatherParams G{static_cast<const uint8_t*>(rows), row_index, (int64_t)pcols * esize};
  auto launch_gather = [&](auto kernel) -> int {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<L.grid, kThreads, smem, stream>>>(tq, P, V, G);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  };
  int rc;
  const bool e32 = epl_for_k(k) == 32;
  if (R) {
    auto launch_residual = [&](auto kernel) -> int {
      MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      kernel<<<L.grid, kThreads, smem, stream>>>(tq, P, V, G, *R);
      MMB_CHECK_CUDA(cudaGetLastError());
      return MMB200_OK;
    };
    if (R->bits == 1)
      rc = e32 ? launch_residual(flat_ip_tc_residual_kernel<32, 1>) : launch_residual(flat_ip_tc_residual_kernel<64, 1>);
    else
      rc = e32 ? launch_residual(flat_ip_tc_residual_kernel<32, 2>) : launch_residual(flat_ip_tc_residual_kernel<64, 2>);
  } else if (gather) {
    if (fp8)
      rc = e32 ? launch_gather(flat_ip_tc_gather_fp8_kernel<32>) : launch_gather(flat_ip_tc_gather_fp8_kernel<64>);
    else if (dtype == MMB200_BF16)
      rc = e32 ? launch_gather(flat_ip_tc_gather_kernel<__nv_bfloat16, 32>) : launch_gather(flat_ip_tc_gather_kernel<__nv_bfloat16, 64>);
    else
      rc = e32 ? launch_gather(flat_ip_tc_gather_kernel<__half, 32>) : launch_gather(flat_ip_tc_gather_kernel<__half, 64>);
  } else if (dtype == MMB200_BF16) {
    rc = e32 ? launch(flat_ip_tc_kernel<__nv_bfloat16, 1, 32, true>) : launch(flat_ip_tc_kernel<__nv_bfloat16, 1, 64, true>);
  } else {
    rc = e32 ? launch(flat_ip_tc_kernel<__half, 1, 32, true>) : launch(flat_ip_tc_kernel<__half, 1, 64, true>);
  }
  if (rc) return rc;
  return launch_merge(P.cand_scores, P.cand_ids, nq, nprobe * L.kslot, k, out_scores, out_ids, dev, stream);
}
}  // namespace
}  // namespace mmb

extern "C" int mmb200_ivf_search(const void* queries, const void* rows, const int64_t* ids, const int64_t* list_offsets,
                                 const int64_t* probes, float* out_scores, int64_t* out_ids, void* workspace,
                                 int64_t workspace_bytes_given, int64_t nq, int32_t nprobe, int64_t nlist, int64_t n_rows,
                                 int64_t max_list_len, int32_t dim, int32_t k, int32_t dtype, void* stream_) {
  return mmb::ivf_search_impl(queries, rows, ids, nullptr, list_offsets, probes, out_scores, out_ids, workspace,
                              workspace_bytes_given, nq, nprobe, nlist, n_rows, max_list_len, dim, k, dtype, stream_);
}

extern "C" int mmb200_ivf_search_gather(const void* queries, const void* rows, const int64_t* ids, const int64_t* row_index,
                                        const int64_t* list_offsets, const int64_t* probes, float* out_scores,
                                        int64_t* out_ids, void* workspace, int64_t workspace_bytes_given, int64_t nq,
                                        int32_t nprobe, int64_t nlist, int64_t n_rows, int64_t max_list_len, int32_t dim,
                                        int32_t k, int32_t dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(row_index != nullptr, "null pointer");
  return ivf_search_impl(queries, rows, ids, row_index, list_offsets, probes, out_scores, out_ids, workspace,
                         workspace_bytes_given, nq, nprobe, nlist, n_rows, max_list_len, dim, k, dtype, stream_);
}

extern "C" int mmb200_ivf_search_residual(const void* queries, const uint8_t* codes, const void* base, const void* weight,
                                          int32_t bits, const int64_t* ids, const int64_t* row_index,
                                          const int64_t* list_offsets, const int64_t* probes, float* out_scores,
                                          int64_t* out_ids, void* workspace, int64_t workspace_bytes_given, int64_t nq,
                                          int32_t nprobe, int64_t nlist, int64_t n_rows, int64_t max_list_len,
                                          int32_t dim, int32_t k, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(codes && base && weight && row_index, "null pointer");
  MMB_REQUIRE(bits == 1 || bits == 2, "residual codes have 1 or 2 bits per dimension");
  MMB_REQUIRE(dim >= kResidualMinDim && dim <= kResidualMaxDim, "residual codes need 64 <= dim <= 1024");
  const ResidualCodes R{codes, static_cast<const __half*>(base), static_cast<const __half*>(weight), bits};
  return ivf_search_impl(queries, codes, ids, row_index, list_offsets, probes, out_scores, out_ids, workspace,
                         workspace_bytes_given, nq, nprobe, nlist, n_rows, max_list_len, dim, k, MMB200_F16, stream_, &R);
}

// Spherical k-means update: block l averages rows perm[offsets[l] .. offsets[l+1]) of x in that order (fp64
// accumulation), then divides by the norm.  One fixed order per list: the result is bit-reproducible.
namespace mmb {
namespace {
template <typename T>
__global__ void __launch_bounds__(256) ivf_list_means_kernel(const T* __restrict__ x, const int64_t* __restrict__ perm,
                                                             const int64_t* __restrict__ offsets, int64_t nlist, int dim,
                                                             float* __restrict__ out) {
  extern __shared__ double acc[];   // [dim]
  __shared__ double red[8];
  for (int64_t l = blockIdx.x; l < nlist; l += gridDim.x) {
    const int64_t lo = offsets[l], hi = offsets[l + 1];
    for (int c = threadIdx.x; c < dim; c += blockDim.x) {
      double s = 0.0;
      for (int64_t r = lo; r < hi; ++r) s += (double)to_float(x[perm[r] * dim + c]);
      acc[c] = s;
    }
    double ss = 0.0;
    for (int c = threadIdx.x; c < dim; c += blockDim.x) ss += acc[c] * acc[c];
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    double tot = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
    const double inv = tot > 0.0 ? 1.0 / sqrt(tot) : 0.0;   // an empty list gives a zero row
    for (int c = threadIdx.x; c < dim; c += blockDim.x) out[l * dim + c] = (float)(acc[c] * inv);
    __syncthreads();
  }
}
}  // namespace
}  // namespace mmb

extern "C" int mmb200_ivf_list_means(const void* x, const int64_t* perm, const int64_t* offsets, float* out, int64_t nlist,
                                     int32_t dim, int32_t dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(x && perm && offsets && out, "null pointer");
  MMB_REQUIRE(nlist >= 1 && dim >= 1 && dim <= 4096, "1 <= dim <= 4096, at least one list");
  MMB_REQUIRE(dtype == MMB200_F16 || dtype == MMB200_BF16 || dtype == MMB200_F32, "x must be fp16, bf16 or fp32");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int grid = (int)std::min<int64_t>(nlist, (int64_t)dev.sm_count * 16);
  const size_t smem = (size_t)dim * sizeof(double);
  auto launch = [&](auto t) -> int {
    using T = decltype(t);
    MMB_CHECK_CUDA(cudaFuncSetAttribute(ivf_list_means_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ivf_list_means_kernel<T><<<grid, 256, smem, stream>>>(static_cast<const T*>(x), perm, offsets, nlist, dim, out);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  };
  if (dtype == MMB200_F16) return launch(__half{});
  if (dtype == MMB200_BF16) return launch(__nv_bfloat16{});
  return launch(float{});
}
