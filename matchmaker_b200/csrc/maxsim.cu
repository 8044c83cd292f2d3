// ColBERT late-interaction max-sim for sm_90a.
//
//   score[p] = sum_i qmask[i] * max_j ( dmask[j] ? <q_i, d_j> : -1000 )
//
// Reference arithmetic: matchmaker/models/colbert.py:68-75 (forward), :100-112
// (forward_aggregation), :154-162 (forward_inbatch_aggregation).  Not a port: the reference
// materialises the [B, Lq, Ld] score tensor with cuBLAS bmm and runs four more eager kernels
// over it; here one persistent kernel streams the document token matrices through shared
// memory once and never writes the score matrix.
//
// Kernel `maxsim_tc_kernel` (documents on M; Lq <= 128, dim % 64 == 0, 64 <= dim <= 1024, and the query tile must leave
// room for two document stages: up to Lq 96 at dim 640 / 768 / 832 / 960, Lq 64 at dim 896 / 1024 on an H100; DESIGN 3.1):
//   * one CTA per SM, persistent over a contiguous range of pairs;
//   * warp 0 (one lane): TMA producer.  A document tile is 128 token rows x dim, fetched as
//     [KBS k-blocks][128 rows][64 halfs] with SWIZZLE_128B by ONE 4-D cp.async.bulk.tensor
//     per stage (rows past Ld are zero-filled by the TMA unit, no HBM traffic); the query
//     matrix ([NPAD rows][dim]) lives in a 2-slot ring (1 slot when two leave no room for two
//     stages) and is re-fetched only when the query of consecutive pairs changes;
//   * warpgroups 1 and 2: warpgroup c computes D[64 doc rows x NPAD query cols] (fp32,
//     registers) = Doc_tile[rows 64c..64c+63] * Q^T with wgmma m64n32k16 chunks, applies the
//     document mask (-1000) / tile padding (-inf) per row, and keeps a running column max over
//     the tiles of a pair (per thread over its two rows, then across the warp by shuffles);
//     the 8 warps combine through 8 KB of shared memory, query mask, warp-sum, one fp32 store
//     per pair.
//
// The hot path for Lq <= 32 is the transposed "queries on M" kernel in maxsim_qm.cu.
//
// Kernel `maxsim_simt_kernel`: CUDA-core version for any dtype / dim / length (fp32 inputs,
// dim % 64 != 0, argmax for backward); also the in-library cross-check of the tensor-core path.
//
// Store mode (MaxsimParams::doc_offsets, mmb200_maxsim_store_fwd): every kernel reads passage d
// as rows [off[d], off[d+1]) of a ragged [n_rows, dim] token store instead of a padded, masked
// [n_d, Ld, dim] tensor; rows past the passage's length are excluded like padding, without the
// -1000 fill (there is no mask).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "device_util.cuh"
#include "host_util.cuh"
#include "masks.cuh"
#include "maxsim.cuh"
#include "ptx.cuh"
#include "residual.cuh"

namespace mmb {

// ---------------------------------------------------------------------------------------------
// shared device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t pair_query(const MaxsimParams& P, int64_t p) {
  return P.pair_q ? static_cast<int64_t>(P.pair_q[p]) : (p + P.pair_base) / P.docs_per_query;
}
__device__ __forceinline__ int64_t pair_doc(const MaxsimParams& P, int64_t p) {
  return P.pair_d ? static_cast<int64_t>(P.pair_d[p]) : p;
}
__device__ __forceinline__ int64_t pair_dmask_row(const MaxsimParams& P, int64_t p) {
  return P.pair_dmask ? static_cast<int64_t>(P.pair_dmask[p]) : pair_doc(P, p);
}

constexpr float kMaskedScore = -1000.0f;  // colbert.py:69

// ---------------------------------------------------------------------------------------------
// SIMT kernel: one CTA (128 threads) per pair.  Q is staged in shared memory as fp32 with a
// padded row stride; warp w takes document rows w, w+4, ...; lane l owns query tokens l, l+32, ...
// ---------------------------------------------------------------------------------------------
constexpr int kSimtThreads = 128;
constexpr int kSimtMaxQPerLane = 4;  // Lq <= 128

template <typename T>
__global__ void __launch_bounds__(kSimtThreads) maxsim_simt_kernel(MaxsimParams P) {
  extern __shared__ float smem_f[];
  const int Lq = P.Lq, Ld = P.Ld, dim = P.dim;
  const int qstride = dim + 1;
  float* sq = smem_f;                          // [Lq][dim+1]
  float* smax = sq + (size_t)Lq * qstride;     // [4][Lq]
  int* sarg = reinterpret_cast<int*>(smax + 4 * Lq);  // [4][Lq]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  for (int64_t p = blockIdx.x; p < P.n_pairs; p += gridDim.x) {
    const int64_t qi = pair_query(P, p), di = pair_doc(P, p), dmi = pair_dmask_row(P, p);
    const T* qptr = static_cast<const T*>(P.q) + qi * (int64_t)Lq * dim;
    int64_t row0 = di * (int64_t)Ld;
    int nrows = Ld;
    if (P.doc_offsets) nrows = store_doc_rows(P, di, &row0);  // store mode: the passage's own rows, no mask
    const T* dptr = static_cast<const T*>(P.d) + row0 * dim;
    __syncthreads();
    for (int e = threadIdx.x; e < Lq * dim; e += kSimtThreads) {
      sq[(e / dim) * qstride + (e % dim)] = to_float(qptr[e]);
    }
    __syncthreads();
    float best[kSimtMaxQPerLane];
    int barg[kSimtMaxQPerLane];
#pragma unroll
    for (int t = 0; t < kSimtMaxQPerLane; ++t) { best[t] = -INFINITY; barg[t] = -1; }
    for (int j = warp; j < nrows; j += 4) {
      const bool ok = mask_at(P.d_mask, P.d_mask ? P.mask_dtype : MMB200_MASK_NONE, dmi * (int64_t)Ld + j);
      float acc[kSimtMaxQPerLane] = {0.f, 0.f, 0.f, 0.f};
      if (ok) {
        const T* drow = dptr + (int64_t)j * dim;
        for (int k = 0; k < dim; ++k) {
          const float dv = to_float(drow[k]);
#pragma unroll
          for (int t = 0; t < kSimtMaxQPerLane; ++t) {
            const int i = lane + 32 * t;
            if (i < Lq) acc[t] = fmaf(sq[i * qstride + k], dv, acc[t]);
          }
        }
      }
      // rows in ascending order: the first maximal real row wins, and a real row wins an exact tie against the -1000
      // fill of a masked row before it (the rule of the warp combine below and of the queries-on-M kernel)
#pragma unroll
      for (int t = 0; t < kSimtMaxQPerLane; ++t) {
        const float v = ok ? acc[t] : kMaskedScore;
        if (v > best[t] || (v == best[t] && ok && barg[t] < 0)) { best[t] = v; barg[t] = ok ? j : -1; }
      }
    }
#pragma unroll
    for (int t = 0; t < kSimtMaxQPerLane; ++t) {
      const int i = lane + 32 * t;
      if (i < Lq) { smax[warp * Lq + i] = best[t]; sarg[warp * Lq + i] = barg[t]; }
    }
    __syncthreads();
    if (warp == 0) {
      float total = 0.f;
      for (int i = lane; i < Lq; i += 32) {
        float m = smax[i];
        int a = sarg[i];
        for (int w = 1; w < 4; ++w) {
          const float v = smax[w * Lq + i];
          const int aw = sarg[w * Lq + i];
          // first occurrence of the max (lowest j) like a sequential scan
          if (v > m || (v == m && aw >= 0 && (a < 0 || aw < a))) { m = v; a = aw; }
        }
        const bool qok = mask_at(P.q_mask, P.q_mask ? P.mask_dtype : MMB200_MASK_NONE, qi * (int64_t)Lq + i);
        total += qok ? m : 0.f;
        if (P.argmax) P.argmax[p * Lq + i] = qok ? a : -1;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
      if (lane == 0) P.out[p] = total;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// wgmma kernel (documents on M)
// ---------------------------------------------------------------------------------------------
constexpr int kTcThreads = 384;        // warp 0 TMA (warps 1-3 idle), warpgroups 1 and 2: MMA + epilogue
constexpr int kTileRows = 128;         // document rows per stage: warpgroup c takes rows 64c .. 64c + 63
constexpr int kKBlockElems = 64;       // 64 x 16-bit = 128 B = one SWIZZLE_128B row
constexpr int kKBlockBytes = kTileRows * 128;  // 16 KB: [128 rows][128 B]
constexpr int kMaxStages = 12;
constexpr int kQSlots = 2;

struct TcShared {  // control block placed after the tile storage
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];   // 8 arrivals: every consumer warp
  uint64_t qfull[kQSlots];
  uint64_t qempty[kQSlots];     // 8 arrivals
  float colmax[2][8][128];      // [pair parity][consumer warp][query column]
};

struct TcLaunch {
  int32_t npad;        // query rows padded to a multiple of 32 (wgmma N)
  int32_t kblocks;     // dim / 64
  int32_t kbs;         // k-blocks per stage (1 or 2)
  int32_t stages;      // document stages in the ring
  int32_t tiles;       // ceil(Ld / 128)
  int32_t qslot_bytes; // kblocks * npad * 128
  int32_t qslots;      // query tiles in the ring: 2, or 1 when two do not leave room for two stages (dim 768, Lq > 32)
};

template <typename T>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc);
template <>
__device__ __forceinline__ void wgmma_n32<__half>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n32k16_f16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void wgmma_n32<__nv_bfloat16>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n32k16_bf16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void wgmma_n32<__nv_fp8_e4m3>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n32k32_e4m3(d, a, b, acc);
}

// NC = npad / 32 accumulator chunks of 16 registers per thread.
//
// RB > 0 (maxsim_tc_residual_kernel, store mode only): the store holds RB-bit residual codes (residual.cuh) with one
// list id per row, and warps 0-3 all produce: thread p decodes row p of every document tile (its codes from HBM, its
// list's base row from L2, the per-dimension weights from a shared-memory copy placed after TcShared) into the same
// SWIZZLE_128B layout the TMA writes, with 16-byte shared stores.  Rows past the passage are not written (the consumers
// exclude them).  Each producer thread fences the async proxy and arrives on `full` (128 arrivals); warp 0 still
// fetches the query tiles by TMA.
template <typename T, int KBS, int NC, int RB = 0>
__device__ __forceinline__ void maxsim_tc_body(const CUtensorMap& tmap_q, const CUtensorMap* tmap_d, MaxsimParams P,
                                               TcLaunch L, ResidualCodes R = {}, const int32_t* list_ids = nullptr) {
  static_assert(RB == 0 || RB == 1 || RB == 2, "residual codes have 1 or 2 bits");
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for SWIZZLE_128B tiles, derived by pointer arithmetic on the __shared__ array so the
  // compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int kStageBytes = KBS * kKBlockBytes;
  uint8_t* stage_base = smem;
  uint8_t* q_base = smem + (size_t)L.stages * kStageBytes;
  TcShared* S = reinterpret_cast<TcShared*>(q_base + (size_t)L.qslots * L.qslot_bytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  int64_t p_begin, p_end;
  cta_share(P.n_pairs, &p_begin, &p_end);

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmap_q);
    if constexpr (RB == 0) prefetch_tensormap(tmap_d);
    for (int s = 0; s < L.stages; ++s) { mbar_init(&S->full[s], RB ? 128 : 1); mbar_init(&S->empty[s], 8); }
    for (int s = 0; s < kQSlots; ++s) { mbar_init(&S->qfull[s], 1); mbar_init(&S->qempty[s], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  const int ksteps = L.kblocks / KBS;

  if (RB > 0 && warp < 4) {
    if constexpr (RB > 0) {
      const int p = threadIdx.x;   // tile row decoded by this thread
      const int dim = P.dim, pitch = dim * RB / 8;
      uint16_t* wtab = reinterpret_cast<uint16_t*>(S + 1);   // [dim][2^RB] weights
      const uint16_t* w16 = reinterpret_cast<const uint16_t*>(R.weight);
      for (int e = p; e < (dim << RB); e += 128) wtab[e] = w16[e];
      named_bar_sync(2, 128);
      int stage = 0;
      uint32_t phase = 0;
      int64_t prev_q = -1;
      uint32_t qcount = 0;
      for (int64_t pp = p_begin; pp < p_end; ++pp) {
        const int64_t qi = pair_query(P, pp), di = pair_doc(P, pp);
        if (qi != prev_q) {
          if (p == 0) {
            const uint32_t slot = L.qslots == 2 ? (qcount & 1u) : 0u, use = L.qslots == 2 ? (qcount >> 1) : qcount;
            mbar_wait(&S->qempty[slot], (use & 1u) ^ 1u);
            mbar_arrive_expect_tx(&S->qfull[slot], (uint32_t)L.qslot_bytes);
            tma_load_4d(&tmap_q, q_base + (size_t)slot * L.qslot_bytes, &S->qfull[slot], 0, 0, 0, (int)qi, kEvictLast);
          }
          ++qcount;
          prev_q = qi;
        }
        int64_t row0 = 0;
        const int nrows = store_doc_rows(P, di, &row0);
        for (int t = 0; t < L.tiles; ++t) {
          const bool mine = t * kTileRows + p < nrows;
          const int64_t row = row0 + t * kTileRows + p;
          const uint8_t* crow = R.codes + (mine ? row : 0) * pitch;
          const uint16_t* brow = reinterpret_cast<const uint16_t*>(R.base) + (mine ? (int64_t)list_ids[row] * dim : 0);
          for (int ks = 0; ks < ksteps; ++ks) {
            mbar_wait(&S->empty[stage], phase ^ 1u);
            if (mine) {
#pragma unroll
              for (int kb = 0; kb < KBS; ++kb) {
                const int kbi = ks * KBS + kb;
                const uint4 words = residual_kblock_bits<RB>(crow, kbi);
                uint4 b8[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) b8[c] = __ldg(reinterpret_cast<const uint4*>(brow + kbi * 64 + 8 * c));
                uint8_t* dst = stage_base + (size_t)stage * kStageBytes + kb * kKBlockBytes + p * 128;
#pragma unroll
                for (int c = 0; c < 8; ++c)
                  *reinterpret_cast<uint4*>(dst + ((c ^ (p & 7)) << 4)) =
                      residual_chunk<RB>(residual_chunk_bits<RB>(words, c), b8[c], wtab + ((kbi * 64 + 8 * c) << RB));
              }
              fence_proxy_async_smem();   // generic-proxy writes -> the consumers' wgmma (async proxy)
            }
            mbar_arrive(&S->full[stage]);
            if (++stage == L.stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else if (warp == 0) {
    // ------------------------------- TMA producer -------------------------------
    // The e4m3 kernel walks the loop with the whole warp and issues from one elected lane, so its TMA operands stay
    // uniform (no ELECT / R2UR waterfall loop around the loads, ptx.cuh); the 16-bit kernels keep their lane-0 loop.
    constexpr bool kWarpIssue = std::is_same<T, __nv_fp8_e4m3>::value;
    if (kWarpIssue || lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int64_t prev_q = -1;
      uint32_t qcount = 0;
      auto issuer = [&]() -> bool {
        if constexpr (kWarpIssue) return elect_one_sync();
        else return true;
      };
      for (int64_t p = p_begin; p < p_end; ++p) {
        const int64_t qi = pair_query(P, p), di = pair_doc(P, p);
        if (qi != prev_q) {
          const uint32_t slot = L.qslots == 2 ? (qcount & 1u) : 0u, use = L.qslots == 2 ? (qcount >> 1) : qcount;
          mbar_wait(&S->qempty[slot], (use & 1u) ^ 1u);
          if (issuer()) {
            mbar_arrive_expect_tx(&S->qfull[slot], (uint32_t)L.qslot_bytes);
            tma_load_4d(&tmap_q, q_base + (size_t)slot * L.qslot_bytes, &S->qfull[slot], 0, 0, 0, (int)qi,
                        kEvictLast);
          }
          if constexpr (kWarpIssue) __syncwarp();
          ++qcount;
          prev_q = qi;
        }
        // store mode: rows [row0, row0 + nrows) of the [n_rows, dim] store; tiles past the passage are not fetched
        int64_t row0 = 0;
        int nrows = P.Ld;
        if (P.doc_offsets) nrows = store_doc_rows(P, di, &row0);
        const int dcoord = P.doc_offsets ? 0 : (int)di;
        for (int t = 0; t < L.tiles; ++t) {
          for (int ks = 0; ks < ksteps; ++ks) {
            mbar_wait(&S->empty[stage], phase ^ 1u);
            if (issuer()) {
              if (t * kTileRows < nrows) {
                mbar_arrive_expect_tx(&S->full[stage], (uint32_t)kStageBytes);
                tma_load_4d(tmap_d, stage_base + (size_t)stage * kStageBytes, &S->full[stage], 0,
                            (int)row0 + t * kTileRows, ks * KBS, dcoord, kEvictFirst);
              } else {
                mbar_arrive(&S->full[stage]);
              }
            }
            if constexpr (kWarpIssue) __syncwarp();
            if (++stage == L.stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------- consumers: wgmma + masked column max -------------------
    const int c = (warp >> 2) - 1;     // warpgroup 0 / 1: document rows 64c .. 64c + 63 of every tile
    const int wq = warp & 3;
    const int ew = 4 * c + wq;         // 0..7
    const int cq = 2 * (lane & 3);     // first column of this thread inside an 8-column group
    const int dmt = P.d_mask ? P.mask_dtype : MMB200_MASK_NONE;
    const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
    int stage = 0;
    uint32_t phase = 0;
    int64_t prev_q = -1;
    uint32_t qcount = 0;
    int cur_slot = 0;
    for (int64_t p = p_begin; p < p_end; ++p) {
      const int64_t qi = pair_query(P, p);
      if (qi != prev_q) {
        if (prev_q >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&S->qempty[cur_slot]); }  // old Q no longer read
        cur_slot = L.qslots == 2 ? (int)(qcount & 1u) : 0;
        mbar_wait(&S->qfull[cur_slot], (L.qslots == 2 ? (qcount >> 1) : qcount) & 1u);
        ++qcount;
        prev_q = qi;
      }
      const uint32_t qaddr = smem_u32(q_base + (size_t)cur_slot * L.qslot_bytes);
      const int64_t dmrow = pair_dmask_row(P, p);
      int nrows = P.Ld;   // store mode: the passage's length (0 for a skipped pair)
      if (P.doc_offsets) {
        int64_t row0;
        nrows = store_doc_rows(P, pair_doc(P, p), &row0);
      }
      float colmax[NC][8];
#pragma unroll
      for (int h = 0; h < NC; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) colmax[h][j] = -INFINITY;
      for (int t = 0; t < L.tiles; ++t) {
        // this thread's two document rows; mask words fetched before the MMAs so their latency hides behind them
        const int g0 = t * kTileRows + 64 * c + 16 * wq + (lane >> 2), g1 = g0 + 8;
        const bool in0 = g0 < nrows, in1 = g1 < nrows;
        const uint64_t raw0 = (in0 && dmt != MMB200_MASK_NONE) ? mask_raw(P.d_mask, dmt, dmrow * (int64_t)P.Ld + g0) : 1;
        const uint64_t raw1 = (in1 && dmt != MMB200_MASK_NONE) ? mask_raw(P.d_mask, dmt, dmrow * (int64_t)P.Ld + g1) : 1;
        float acc[NC][16];
#pragma unroll
        for (int h = 0; h < NC; ++h)
#pragma unroll
          for (int j = 0; j < 16; ++j) acc[h][j] = 0.f;
        for (int ks = 0; ks < ksteps; ++ks) {
          mbar_wait(&S->full[stage], phase);
          const uint32_t aaddr = smem_u32(stage_base + (size_t)stage * kStageBytes) + 64 * c * 128;
          wgmma_fence();
#pragma unroll
          for (int kb = 0; kb < KBS; ++kb) {
            const uint32_t a_kb = aaddr + kb * kKBlockBytes;
            const uint32_t b_kb = qaddr + (uint32_t)((ks * KBS + kb) * L.npad * 128);
#pragma unroll
            for (int k = 0; k < 4; ++k) {  // 128 bytes / 32 bytes per wgmma K step (k16 of 16-bit, k32 of e4m3)
              const uint64_t adesc = make_wgmma_sw128_desc(a_kb + k * 32);
#pragma unroll
              for (int h = 0; h < NC; ++h)
                wgmma_n32<T>(acc[h], adesc, make_wgmma_sw128_desc(b_kb + h * 32 * 128 + k * 32), 1u);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&S->empty[stage]);  // smem stage free: these MMAs have completed
          if (++stage == L.stages) { stage = 0; phase ^= 1u; }
        }
#pragma unroll
        for (int h = 0; h < NC; ++h) wgmma_fence_regs(acc[h]);
        const float f0 = in0 ? (mask_test(raw0, dmt) ? 0.f : kMaskedScore) : -INFINITY;
        const float f1 = in1 ? (mask_test(raw1, dmt) ? 0.f : kMaskedScore) : -INFINITY;
        const bool keep0 = in0 && mask_test(raw0, dmt), keep1 = in1 && mask_test(raw1, dmt);
#pragma unroll
        for (int h = 0; h < NC; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v0 = keep0 ? acc[h][4 * j + e] : f0;
              const float v1 = keep1 ? acc[h][4 * j + 2 + e] : f1;
              colmax[h][2 * j + e] = fmaxf(colmax[h][2 * j + e], fmaxf(v0, v1));
            }
      }
      // max over the 8 row groups of the warp (lanes with the same lane % 4 hold the same columns)
#pragma unroll
      for (int h = 0; h < NC; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float v = colmax[h][j];
          v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
          v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
          v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
          colmax[h][j] = v;
        }
      const int buf = (int)((p - p_begin) & 1);
      if (lane < 4) {
#pragma unroll
        for (int h = 0; h < NC; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            *reinterpret_cast<float2*>(&S->colmax[buf][ew][h * 32 + 8 * j + cq]) = make_float2(colmax[h][2 * j], colmax[h][2 * j + 1]);
      }
      named_bar_sync(1, 256);
      if (ew == (int)((p - p_begin) & 7)) {  // rotate the final reduction over the 8 warps
        float total = 0.f;
#pragma unroll
        for (int h = 0; h < NC; ++h) {
          const int col = h * 32 + lane;
          float m = S->colmax[buf][0][col];
#pragma unroll
          for (int w = 1; w < 8; ++w) m = fmaxf(m, S->colmax[buf][w][col]);
          const bool qok = col < P.Lq && mask_test(qmt != MMB200_MASK_NONE ? mask_raw(P.q_mask, qmt, qi * (int64_t)P.Lq + col) : 1, qmt);
          total += qok ? m : 0.f;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
        if (lane == 0) P.out[p] = total;
      }
    }
  }
}

template <typename T, int KBS, int NC>
__global__ void __launch_bounds__(kTcThreads, 1)
maxsim_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                 MaxsimParams P, TcLaunch L) {
  maxsim_tc_body<T, KBS, NC>(tmap_q, &tmap_d, P, L);
}

// Store-mode max-sim over RB-bit residual codes (mmb200_maxsim_store_residual_fwd); row r belongs to list list_ids[r].
template <int KBS, int NC, int RB>
__global__ void __launch_bounds__(kTcThreads, 1)
maxsim_tc_residual_kernel(const __grid_constant__ CUtensorMap tmap_q, MaxsimParams P, TcLaunch L, ResidualCodes R,
                          const int32_t* list_ids) {
  maxsim_tc_body<__half, KBS, NC, RB>(tmap_q, nullptr, P, L, R, list_ids);
}

// Store-mode max-sim over an E4M3 store with E4M3 queries (mmb200_maxsim_store_fwd, MMB200_F8E4M3): the same body with
// 128-element k-blocks and wgmma m64n32k32.  A name of its own: maxsim_tc_kernel stands for the HGMMA (16-bit) kernel.
template <int KBS, int NC>
__global__ void __launch_bounds__(kTcThreads, 1)
maxsim_tc_fp8_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                     MaxsimParams P, TcLaunch L) {
  maxsim_tc_body<__nv_fp8_e4m3, KBS, NC>(tmap_q, &tmap_d, P, L);
}

template <typename T, int KBS, int NC>
struct TcKernel {
  static constexpr auto fn = maxsim_tc_kernel<T, KBS, NC>;
};
template <int KBS, int NC>
struct TcKernel<__nv_fp8_e4m3, KBS, NC> {
  static constexpr auto fn = maxsim_tc_fp8_kernel<KBS, NC>;
};

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static bool tc_supported(const MaxsimParams& P, int dtype, std::string* why) {
  if (dtype != MMB200_F16 && dtype != MMB200_BF16) { *why = "tensor-core path needs f16/bf16 inputs"; return false; }
  if (P.dim % 64 != 0 || P.dim < 64 || P.dim > 1024) { *why = "tensor-core path needs dim % 64 == 0, 64 <= dim <= 1024"; return false; }
  if (P.Lq < 1 || P.Lq > 128) { *why = "tensor-core path needs 1 <= Lq <= 128"; return false; }
  if (P.Ld < 1) { *why = "Ld < 1"; return false; }
  if (P.argmax) { *why = "argmax output is produced by the SIMT kernel"; return false; }
  if ((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d)) & 15) { *why = "q/d must be 16-byte aligned"; return false; }
  return true;
}

template <typename T, int KBS>
static int launch_tc_nc(int nc, int grid, size_t smem_bytes, cudaStream_t stream, const CUtensorMap& tq, const CUtensorMap& td,
                        const MaxsimParams& P, const TcLaunch& L) {
#define MMB_TC_CASE(N)                                                                                                  \
  case N:                                                                                                               \
    MMB_CHECK_CUDA(cudaFuncSetAttribute(TcKernel<T, KBS, N>::fn, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                                        (int)smem_bytes));                                                              \
    TcKernel<T, KBS, N>::fn<<<grid, kTcThreads, smem_bytes, stream>>>(tq, td, P, L);                                    \
    break;
  switch (nc) {
    MMB_TC_CASE(1)
    MMB_TC_CASE(2)
    MMB_TC_CASE(3)
    MMB_TC_CASE(4)
    default:
      set_error("maxsim documents-on-M: query tile out of range");
      return MMB200_ERR_INVALID;
  }
#undef MMB_TC_CASE
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

// Tile plan of the documents-on-M kernel over elements of `esize` bytes; `extra` bytes of shared memory follow TcShared.
static int plan_tc(const MaxsimParams& P, const DeviceInfo& dev, int extra, int esize, TcLaunch* out, size_t* smem_out) {
  TcLaunch L;
  L.npad = ((P.Lq + 31) / 32) * 32;
  L.kblocks = P.dim * esize / 128;
  L.kbs = (L.kblocks % 2 == 0) ? 2 : 1;
  L.tiles = (P.Ld + kTileRows - 1) / kTileRows;
  L.qslot_bytes = L.kblocks * L.npad * 128;
  const int stage_bytes = L.kbs * kKBlockBytes;
  // two query tiles when they leave room for at least two document stages; otherwise (large dim with Lq > 32) one,
  // re-fetched after the consumers release it
  int fixed = 0;
  for (L.qslots = kQSlots; L.qslots >= 1; --L.qslots) {
    fixed = L.qslots * L.qslot_bytes + (int)sizeof(TcShared) + extra + 1024 /* alignment slack */;
    L.stages = std::min(kMaxStages, (dev.max_smem_optin - fixed) / stage_bytes);
    if (L.stages >= 2) break;
  }
  if (L.qslots < 1 || L.stages < 2) {
    set_error("maxsim documents-on-M: query tile too large for shared memory");
    return MMB200_ERR_UNSUPPORTED;
  }
  *out = L;
  *smem_out = (size_t)L.stages * stage_bytes + fixed;
  return MMB200_OK;
}

// TMA map of the query tiles of the documents-on-M kernel: [NPAD rows][128 bytes] per k-block, all k-blocks of a query.
static int encode_tc_query_map(CUtensorMap* tq, const MaxsimParams& P, const TcLaunch& L, CUtensorMapDataType tdt,
                               int esize) {
  const uint32_t kbe = 128 / esize;
  const uint64_t dims[4] = {kbe, (uint64_t)P.Lq, (uint64_t)L.kblocks, (uint64_t)P.n_q};
  const uint64_t strides[3] = {(uint64_t)P.dim * esize, 128, (uint64_t)P.Lq * P.dim * esize};
  const uint32_t box[4] = {kbe, (uint32_t)L.npad, (uint32_t)L.kblocks, 1};
  return encode_tensor_map(tq, tdt, 4, P.q, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

static int launch_tc(const MaxsimParams& P, int dtype, const DeviceInfo& dev, cudaStream_t stream) {
  TcLaunch L;
  size_t smem_bytes;
  const int esize = dtype == MMB200_F8E4M3 ? 1 : 2;
  const uint32_t kbe = 128 / esize;
  if (int rc = plan_tc(P, dev, 0, esize, &L, &smem_bytes)) return rc;
  const CUtensorMapDataType tdt = dtype == MMB200_F16       ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                  : dtype == MMB200_F8E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                                           : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap tq, td;
  if (int rc = encode_tc_query_map(&tq, P, L, tdt, esize)) return rc;
  {
    // store mode: the [n_rows, dim] store is one "document"; a passage's tile starts at its first row
    const uint64_t d_rows = P.doc_offsets ? (uint64_t)P.n_rows : (uint64_t)P.Ld;
    const uint64_t d_count = P.doc_offsets ? 1 : (uint64_t)P.n_d;
    const uint64_t dims[4] = {kbe, d_rows, (uint64_t)L.kblocks, d_count};
    const uint64_t strides[3] = {(uint64_t)P.dim * esize, 128, d_rows * P.dim * esize};
    const uint32_t box[4] = {kbe, (uint32_t)kTileRows, (uint32_t)L.kbs, 1};
    if (int rc = encode_tensor_map(&td, tdt, 4, P.d, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  const int grid = (int)std::min<int64_t>(dev.sm_count, P.n_pairs);
  const int nc = L.npad / 32;
  if (dtype == MMB200_F8E4M3)
    return L.kbs == 2 ? launch_tc_nc<__nv_fp8_e4m3, 2>(nc, grid, smem_bytes, stream, tq, td, P, L)
                      : launch_tc_nc<__nv_fp8_e4m3, 1>(nc, grid, smem_bytes, stream, tq, td, P, L);
  if (dtype == MMB200_F16)
    return L.kbs == 2 ? launch_tc_nc<__half, 2>(nc, grid, smem_bytes, stream, tq, td, P, L)
                      : launch_tc_nc<__half, 1>(nc, grid, smem_bytes, stream, tq, td, P, L);
  return L.kbs == 2 ? launch_tc_nc<__nv_bfloat16, 2>(nc, grid, smem_bytes, stream, tq, td, P, L)
                    : launch_tc_nc<__nv_bfloat16, 1>(nc, grid, smem_bytes, stream, tq, td, P, L);
}

static int launch_simt(const MaxsimParams& P, int dtype, const DeviceInfo& dev, cudaStream_t stream) {
  MMB_REQUIRE(P.Lq <= 32 * kSimtMaxQPerLane, "SIMT max-sim kernel supports Lq <= 128");
  const size_t smem_bytes = ((size_t)P.Lq * (P.dim + 1) + 8 * (size_t)P.Lq) * sizeof(float);
  MMB_REQUIRE(smem_bytes <= (size_t)dev.max_smem_optin, "query tile does not fit in shared memory");
  const int grid = (int)std::min<int64_t>((int64_t)dev.sm_count * 8, P.n_pairs);
  return dispatch_dtype(dtype, [&](auto t) {
    using T = decltype(t);
    MMB_CHECK_CUDA(cudaFuncSetAttribute(maxsim_simt_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    maxsim_simt_kernel<T><<<grid, kSimtThreads, smem_bytes, stream>>>(P);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  });
}

// A tensor with no elements may come with a null pointer (torch hands one out for an empty tensor): an empty batch
// (n_q = n_d = n_pairs = 0) is valid and launches nothing.
int maxsim_fwd_device(const MaxsimParams& P, int dtype, int impl, cudaStream_t stream) {
  MMB_REQUIRE((P.q || P.n_q == 0) && (P.d || P.n_d == 0) && (P.out || P.n_pairs == 0), "null pointer: q, d, out must be non-null");
  MMB_REQUIRE(dtype_size(dtype) != 0, "unknown dtype");
  MMB_REQUIRE(P.n_pairs >= 0 && P.n_q >= 0 && P.n_d >= 0 && (P.n_pairs == 0 || (P.n_q > 0 && P.n_d > 0)), "bad counts");
  MMB_REQUIRE(P.Lq > 0 && P.Ld > 0 && P.dim > 0, "bad shape");
  MMB_REQUIRE(P.docs_per_query >= 1, "docs_per_query must be >= 1");
  if ((P.q_mask || P.d_mask)) MMB_REQUIRE(mask_dtype_size(P.mask_dtype) != 0, "unknown mask dtype");
  if (!P.pair_q) MMB_REQUIRE((P.pair_base + P.n_pairs + P.docs_per_query - 1) / P.docs_per_query <= P.n_q, "n_pairs / docs_per_query exceeds n_q");
  if (!P.pair_d) MMB_REQUIRE(P.n_pairs <= P.n_d, "n_pairs exceeds n_d");
  if (P.n_pairs == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  // the live-row fetch is the queries-on-M kernel's only path: the ragged name is an alias of the tensor-core one
  if (impl == MMB200_IMPL_TCGEN05_RAGGED) impl = MMB200_IMPL_TCGEN05;
  if (impl == MMB200_IMPL_AUTO || impl == MMB200_IMPL_TCGEN05) {
    bool handled = false;
    const int rc = maxsim_qm_launch(P, dtype, dev, stream, &handled);
    if (handled || rc != MMB200_OK) return rc;
  }
  std::string why;
  const bool tc_ok = tc_supported(P, dtype, &why);
  if ((impl == MMB200_IMPL_TCGEN05 || impl == MMB200_IMPL_TCGEN05_DOCM) && !tc_ok) {
    set_error(why);
    return MMB200_ERR_UNSUPPORTED;
  }
  if (impl == MMB200_IMPL_SIMT || !tc_ok) return launch_simt(P, dtype, dev, stream);
  return launch_tc(P, dtype, dev, stream);
}

// Store mode over an e4m3 store: only the documents-on-M kernel reads e4m3, so there is no kernel choice to make and
// no SIMT kernel to fall back to.
static int maxsim_store_fp8(const MaxsimParams& P, int impl, cudaStream_t stream) {
  if (impl != MMB200_IMPL_AUTO && impl != MMB200_IMPL_TCGEN05_DOCM) {
    set_error("e4m3 max-sim runs on the documents-on-M tensor-core kernel only (impl auto or tcgen05_docm)");
    return MMB200_ERR_UNSUPPORTED;
  }
  MMB_REQUIRE(P.n_pairs >= 0 && P.n_q >= 0, "bad counts");
  if (P.n_pairs == 0) return MMB200_OK;
  MMB_REQUIRE(P.q && P.d && P.out, "null pointer: q, store, out must be non-null");
  MMB_REQUIRE(P.n_q >= 1, "need at least one query");
  MMB_REQUIRE(P.Lq >= 1 && P.Lq <= 128, "e4m3 max-sim needs 1 <= Lq <= 128");
  MMB_REQUIRE(P.dim % 128 == 0 && P.dim >= 128 && P.dim <= 1024, "e4m3 max-sim needs dim % 128 == 0, 128 <= dim <= 1024");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d)) & 15) == 0, "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  return launch_tc(P, MMB200_F8E4M3, dev, stream);
}

}  // namespace mmb

extern "C" int mmb200_maxsim_fwd(const void* q, const void* d, const void* q_mask, const void* d_mask,
                                 const int32_t* pair_q, const int32_t* pair_d, const int32_t* pair_dmask,
                                 float* out, int32_t* argmax, int64_t n_q, int64_t n_d, int64_t n_pairs, int32_t docs_per_query, int32_t Lq,
                                 int32_t Ld, int32_t dim, int32_t dtype, int32_t mask_dtype, int32_t impl,
                                 void* stream) {
  mmb::MaxsimParams P;
  P.q = q; P.d = d; P.q_mask = q_mask; P.d_mask = d_mask; P.pair_q = pair_q; P.pair_d = pair_d; P.pair_dmask = pair_dmask;
  P.out = out; P.argmax = argmax; P.n_q = n_q; P.n_d = n_d; P.n_pairs = n_pairs;
  P.docs_per_query = docs_per_query; P.Lq = Lq; P.Ld = Ld; P.dim = dim; P.mask_dtype = mask_dtype;
  return mmb::maxsim_fwd_device(P, dtype, impl, static_cast<cudaStream_t>(stream));
}

extern "C" int mmb200_maxsim_store_fwd(const void* q, const void* store, const int64_t* doc_offsets,
                                       const int32_t* pair_q, const int32_t* pair_d, float* out, int64_t n_q,
                                       int64_t n_rows, int64_t n_docs, int64_t n_pairs, int32_t Lq, int32_t max_doc_len,
                                       int32_t dim, int32_t dtype, int32_t impl, void* stream) {
  MMB_REQUIRE(doc_offsets && pair_q && pair_d, "doc_offsets, pair_q and pair_d must be non-null");
  MMB_REQUIRE(n_rows >= 1 && n_docs >= 1 && max_doc_len >= 1, "the store needs at least one row, one passage, max_doc_len >= 1");
  MMB_REQUIRE(n_rows < (1ll << 31) - 1024, "at most 2^31 - 1024 store rows per device (TMA row coordinates are int32)");
  mmb::MaxsimParams P;
  P.q = q; P.d = store; P.pair_q = pair_q; P.pair_d = pair_d; P.out = out; P.n_q = n_q; P.n_d = n_docs;
  P.n_pairs = n_pairs; P.Lq = Lq; P.Ld = max_doc_len; P.dim = dim;
  P.doc_offsets = doc_offsets; P.n_rows = n_rows;
  if (dtype == MMB200_F8E4M3) return mmb::maxsim_store_fp8(P, impl, static_cast<cudaStream_t>(stream));
  return mmb::maxsim_fwd_device(P, dtype, impl, static_cast<cudaStream_t>(stream));
}

namespace mmb {
template <int KBS, int RB>
static int launch_tc_residual_nc(int nc, int grid, size_t smem_bytes, cudaStream_t stream, const CUtensorMap& tq,
                                 const MaxsimParams& P, const TcLaunch& L, const ResidualCodes& R,
                                 const int32_t* list_ids) {
#define MMB_TCR_CASE(N)                                                                                              \
  case N:                                                                                                            \
    MMB_CHECK_CUDA(cudaFuncSetAttribute(maxsim_tc_residual_kernel<KBS, N, RB>,                                        \
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));              \
    maxsim_tc_residual_kernel<KBS, N, RB><<<grid, kTcThreads, smem_bytes, stream>>>(tq, P, L, R, list_ids);          \
    break;
  switch (nc) {
    MMB_TCR_CASE(1)
    MMB_TCR_CASE(2)
    MMB_TCR_CASE(3)
    MMB_TCR_CASE(4)
    default:
      set_error("residual max-sim: query tile out of range");
      return MMB200_ERR_INVALID;
  }
#undef MMB_TCR_CASE
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}
}  // namespace mmb

extern "C" int mmb200_maxsim_store_residual_fwd(const void* q, const uint8_t* codes, const int32_t* list_ids,
                                                const void* base, const void* weight, int32_t bits,
                                                const int64_t* doc_offsets, const int32_t* pair_q, const int32_t* pair_d,
                                                float* out, int64_t n_q, int64_t n_rows, int64_t n_docs, int64_t n_pairs,
                                                int32_t Lq, int32_t max_doc_len, int32_t dim, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(n_pairs >= 0 && n_q >= 0, "bad counts");
  if (n_pairs == 0) return MMB200_OK;
  MMB_REQUIRE(q && codes && list_ids && base && weight && doc_offsets && pair_q && pair_d && out, "null pointer");
  MMB_REQUIRE(n_q >= 1 && n_rows >= 1 && n_docs >= 1 && max_doc_len >= 1,
              "need a query, one stored row, one passage and max_doc_len >= 1");
  MMB_REQUIRE(bits == 1 || bits == 2, "residual codes have 1 or 2 bits per dimension");
  MMB_REQUIRE(dim % 64 == 0 && dim >= kResidualMinDim && dim <= kResidualMaxDim, "residual codes need dim % 64 == 0, 64 <= dim <= 1024");
  MMB_REQUIRE(Lq >= 1 && Lq <= 128, "1 <= Lq <= 128");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(codes) | reinterpret_cast<uintptr_t>(base)) & 15) == 0,
              "16-byte alignment");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  MaxsimParams P;
  P.q = q; P.pair_q = pair_q; P.pair_d = pair_d; P.out = out; P.n_q = n_q; P.n_d = n_docs; P.n_pairs = n_pairs;
  P.Lq = Lq; P.Ld = max_doc_len; P.dim = dim; P.doc_offsets = doc_offsets; P.n_rows = n_rows;
  TcLaunch L;
  size_t smem_bytes;
  if (int rc = plan_tc(P, dev, (dim << bits) * (int)sizeof(__half), 2, &L, &smem_bytes)) return rc;
  CUtensorMap tq;
  if (int rc = encode_tc_query_map(&tq, P, L, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2)) return rc;
  const ResidualCodes R{codes, static_cast<const __half*>(base), static_cast<const __half*>(weight), bits};
  const int grid = (int)std::min<int64_t>(dev.sm_count, n_pairs);
  const int nc = L.npad / 32;
  if (bits == 1)
    return L.kbs == 2 ? launch_tc_residual_nc<2, 1>(nc, grid, smem_bytes, stream, tq, P, L, R, list_ids)
                      : launch_tc_residual_nc<1, 1>(nc, grid, smem_bytes, stream, tq, P, L, R, list_ids);
  return L.kbs == 2 ? launch_tc_residual_nc<2, 2>(nc, grid, smem_bytes, stream, tq, P, L, R, list_ids)
                    : launch_tc_residual_nc<1, 2>(nc, grid, smem_bytes, stream, tq, P, L, R, list_ids);
}
