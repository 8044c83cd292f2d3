// TKL (SIGIR'20) window scores on TMA + wgmma: the cosine of every (query row, document position) pair comes from
// the tensor cores with fp32-grade accuracy, the RBF activations, the sliding-window sums, the learned saturation
// and the dense layer are fused behind it; only [B, W] window scores are written.
//
// Reference arithmetic: matchmaker/models/published/sigir20_tkl.py:180-252 (the reference materialises
// [B, Lq, C*40, K] = 450 MB at BASELINE config 5 and re-reads it 30 times through two unfold reductions).
//
// Work decomposition.  A document is C chunk slots of 40 positions; slot c is either a packed chunk
// (slot_to_packed >= 0) or all padding.  Three slots = one TILE of 120 positions = 60 position pairs = 4 window
// BLOCKS of 15 pairs.  A window (30 positions, stride 2) is 15 consecutive pairs, so with blocks of 15 pairs every
// window is a block SUFFIX plus the next block's PREFIX: two running sums per (query row, kernel) instead of 15
// re-additions, and -- unlike prefix differences -- only additions of non-negative terms, so empty windows stay
// exactly empty (the -9900 sentinel of sigir20_tkl.py:257 keys on exact zeros).  tkl_plan_kernel counts the tiles of
// every document that can hold a non-zero window and prefix-sums them on the device; CTA x of the persistent grid
// takes the x-th equal share of that global tile sequence (documents are split where the share ends; a share that
// starts inside a document first replays the previous tile's last block -- its "halo" -- to rebuild the suffix sums).
// Windows outside every share are exactly 0 and come from one cudaMemsetAsync.
//
// Per CTA (768 threads = 6 warpgroups, registers re-dealt with setmaxnreg), same operand scheme as kernel_pool_ts.cu
// (x = hi + lo from split_tf32, the document operand split in registers):
//   warp 0      TMA producer: per 32-column k-chunk up to three [40 x 32] chunk boxes + one [40 x 32] query box
//   warps 2-3   query convert (Qhi / Qlo B operands, query norms)
//   warps 4-7   MMA warpgroup: A fragments of the tile's 120 positions (two 64-row halves) from the raw tile, hi / lo in
//               registers, wgmma m64n40k8 tf32 against Qhi and Qlo; then phase A: cosine tile to shared memory (masked
//               positions -> a sentinel whose activations are exactly 0) and the position flags
//   warps 8-23  epilogue, thread = (query row i, kernel k): walks the tile's 60 pairs in registers: activation pair sums,
//               block prefix / suffix, window sum, saturation (per-document table indexed by the window's token count),
//               w_k * T; a 16-value transposed butterfly per block reduces over the warp, 60 threads add the per-warp
//               partials in a fixed order.  Two cosine tiles travel between phase A and the epilogue through mbarriers.
//
// The window "length" of sigir20_tkl.py:210 counts positions whose K activations do not all vanish.  When every
// cosine in [-1, 1] activates at least one kernel (checked on the device by the plan kernel: true for every kernel
// set the reference ships) that is the count of unmasked positions, which is what this kernel uses; otherwise the
// plan says so and the FFMA kernel in tkl.cu, which tests the activations themselves, runs instead.
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "device_util.cuh"
#include "host_util.cuh"
#include "masks.cuh"
#include "ptx.cuh"
#include "tkl.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 768;
constexpr int kChunk = 40, kWindow = 30;
constexpr int kTileSlots = 3, kTileRows = kTileSlots * kChunk;   // 120 positions
constexpr int kTilePairs = kTileRows / 2;                       // 60
constexpr int kBlk = 15, kBlocks = kTilePairs / kBlk;           // 4 blocks of 15 pairs
constexpr int kMaxLq = 40;
constexpr int kMaxRaw = 6;
constexpr int kOps = 4;
constexpr int kNormRing = kOps + 2;
constexpr int kDxBytes = 128 * 128;       // [128 rows][32 fp32], rows 0..119 written
constexpr int kSlotBytes = kChunk * 128;  // one chunk's 40 rows of a k-chunk
constexpr int kQxBytes = kMaxLq * 128;
constexpr int kRawBytes = kDxBytes + kQxBytes;   // 21 KB
constexpr int kQopBytes = 2 * kMaxLq * 128;  // B operands: rows 0-39 Q hi, rows 40-79 Q lo
constexpr int kEpiWarps = 16, kEpiThreads = kEpiWarps * 32;
constexpr int kFirstDocWarp = 4, kFirstEpiWarp = 8;
constexpr int kReleaseArrivals = 4 + 64;   // lane 0 of each MMA warp + every lane of the two query warps
// The re-deal must fit the registers the CTA was LAUNCHED with (768 threads x 80 = 61 440), not the SM's 64 K: a
// setmaxnreg.inc beyond that pool never returns.  Only the light warpgroup gives registers back; the others keep 80.
constexpr int kRegsLight = 56, kRegsMma = 104;   // the MMA warpgroup takes what the light one gives back; epilogue keeps 80
constexpr int kDmRing = 512;     // position flags of the last tiles (a window reaches 29 positions into the previous tile)
constexpr int kCsStride = 122;            // floats per QUERY ROW of the cosine tile cs[i][position]: even (8-byte pair loads), 122 mod 32 = 26
                                          // puts the 3-4 query rows a warp reads at once on distinct bank pairs
constexpr int kSatStride = 33;            // table row stride (token counts 0..30)
constexpr float kSentinel = 1.0e6f;
constexpr float kClamp = 1e-10f;

struct TsShared {
  uint64_t raw_full[kMaxRaw];
  uint64_t raw_empty[kMaxRaw];
  uint64_t op_full[kOps];
  uint64_t op_empty[kOps];
  uint64_t cs_full[2];        // phase A (MMA warps) -> epilogue: cosine tile and position flags written
  uint64_t cs_empty[2];       // epilogue -> phase A: every epilogue warp is done with the cosine tile
  // query norms travel from the convert warps to phase A in their own ring: the convert warps run up to kOps k-chunks
  // ahead of the MMA warps -- kOps tiles when a tile is a single k-chunk (D <= 32)
  float rs_q[kNormRing][kMaxLq];
  float red[kMaxLq];          // sat_emb_reduce1(q_i)
  float qm[kMaxLq];
  float sp[16];
  alignas(16) uint16_t lenw[kBlocks][16]; // 16 x token count of the window ending at each pair of the tile (byte offset into a sat row),
                              // 15 per block in a 32-byte row: two 16-byte loads per block
  float dmring[kDmRing];      // unmasked flag of the positions, indexed by (tile sequence number * 120 + position) % kDmRing
  float part[kEpiWarps][64];  // per-warp partial window scores
  float4 sat[kMaxLq * kSatStride];   // (sat1 * gate, sat2, sat3 * gate, -) per (query row, token count)
};

// ---------------------------------------------------------------------------------------------------------------
// plan: tiles per document (prefix sums), the "cover" test of the kernel set, and the share of every CTA.  One block.
//   plan[0] = cover, plan[1] = total tiles, plan[2 + b] = tiles before document b (b = 0..B),
//   plan[3 + B + b] = cost before document b (b = 0..B), plan[4 + 2B + x] = first tile of CTA x (x = 0..grid).
// A tile's cost is counted in warp-tiles of epilogue work: kTileFixedCost for everything that does not depend on the
// query (convert, MMA, phase A, barriers; from the per-role profile) plus one per epilogue warp that holds an unmasked
// query row -- short queries leave most of phase B idle, so their documents' tiles are cheaper and a CTA takes more.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kTileFixedCost = 17;

// exclusive prefix sums of v[0..n) in place, v[n] = total; 1024 threads, 1024 elements per round: shuffles inside the
// warp, one shared-memory hop across warps (three barriers per round instead of twenty)
__device__ __forceinline__ void block_exclusive_scan_inplace(int32_t* v, int64_t n, int* wsum, int* carry, int32_t* total_out) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t == 0) *carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < n; base += 1024) {
    const int64_t i = base + t;
    const int x = i < n ? v[i] : 0;
    int incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += u;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    const int c0 = *carry;
    if (i < n) v[i] = c0 + incl - x + (warp > 0 ? wsum[warp - 1] : 0);
    __syncthreads();
    if (t == 0) *carry = c0 + wsum[31];
    __syncthreads();
  }
  if (t == 0) { *total_out = *carry; v[n] = *carry; }
  __syncthreads();
}

// STORE: document b is pair b, its slots are row pair_d[b] of slot_to_packed and its query mask row pair_q[b].
template <bool STORE>
__device__ __forceinline__ void tkl_plan_body(const int32_t* __restrict__ slot_to_packed, const void* __restrict__ q_mask,
                                              int mask_dtype, int64_t B, int C, int Lq, const float* __restrict__ mu,
                                              const float* __restrict__ sigma, int K, int grid, int force_cover,
                                              int32_t* __restrict__ plan, const TklPairs& X) {
  __shared__ int sums[1024];
  __shared__ int carry;
  __shared__ int total_tiles, total_cost;
  __shared__ float klo[32], khi[32];
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // tkl_ts_kernel may start its prologue now (it waits for this grid's completion before it reads the plan)
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t < K && t < 32) {
    const float h = 11.0f * sigma[t] / rbf_scale(1.0f);   // 11 / rbf_scale(sigma), rounded as 11 sigma / rbf_scale(1)
    klo[t] = mu[t] - h;
    khi[t] = mu[t] + h;
  }
  const int tiles_max = (C + kTileSlots - 1) / kTileSlots;
  // up to 1024 documents the two prefix arrays live in shared memory while they are built, scanned and searched (the global
  // round trips of the scans and of the 150 binary searches were a third of this kernel's 15 us); written out once at the end
  __shared__ int32_t s_tile[1025], s_cost[1025];
  const bool in_smem = B <= 1024;
  int32_t* tile_pre = in_smem ? s_tile : plan + 2;
  int32_t* cost_pre = in_smem ? s_cost : plan + 3 + B;
  int32_t* cta_start = plan + 4 + 2 * B;
  // pass 1: tiles and cost of every document: one warp per document, four documents per warp in flight (all of their slot
  // and mask words are requested before the first ballot -- one global-memory latency per batch, not four per document)
  const int qmt = q_mask ? mask_dtype : MMB200_MASK_NONE;
  const bool small = C <= 64 && Lq <= 64;
  for (int64_t b0 = (int64_t)warp * 4; b0 < B; b0 += 128) {
    bool pk0[4], pk1[4], lv0[4], lv1[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int64_t b = b0 + a;
      const bool ok = small && b < B;
      const int64_t sb = STORE ? (ok ? tkl_slot_row<true>(X, b) : -1) : b;
      const int64_t qb = STORE ? (ok ? tkl_q_row<true>(X, b) : 0) : b;
      const bool live = ok && (!STORE || sb >= 0);
      pk0[a] = live && lane < C && slot_to_packed[sb * C + lane] >= 0;
      pk1[a] = live && lane + 32 < C && slot_to_packed[sb * C + lane + 32] >= 0;
      lv0[a] = ok && lane < Lq && mask_at(q_mask, qmt, qb * Lq + lane);
      lv1[a] = ok && lane + 32 < Lq && mask_at(q_mask, qmt, qb * Lq + lane + 32);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int64_t b = b0 + a;
      if (b >= B) break;   // warp-uniform
      int c_last = -1, q_hi = 0;
      if (small) {
        const unsigned m0 = __ballot_sync(0xffffffffu, pk0[a]), m1 = __ballot_sync(0xffffffffu, pk1[a]);
        c_last = m1 ? 63 - __clz(m1) : (m0 ? 31 - __clz(m0) : -1);
        const unsigned q0 = __ballot_sync(0xffffffffu, lv0[a]), q1 = __ballot_sync(0xffffffffu, lv1[a]);
        q_hi = q1 ? 64 - __clz(q1) : (q0 ? 32 - __clz(q0) : 0);
      } else {
        const int64_t sb = tkl_slot_row<STORE>(X, b), qb = tkl_q_row<STORE>(X, b);
        for (int c0 = 0; c0 < C; c0 += 32) {
          const int c = c0 + lane;
          const unsigned m = __ballot_sync(0xffffffffu, (!STORE || sb >= 0) && c < C && slot_to_packed[sb * C + c] >= 0);
          if (m) c_last = c0 + 31 - __clz(m);
        }
        for (int i0 = 0; i0 < Lq; i0 += 32) {
          const int i = i0 + lane;
          const unsigned m = __ballot_sync(0xffffffffu, i < Lq && mask_at(q_mask, qmt, qb * Lq + i));
          if (m) q_hi = i0 + 32 - __clz(m);
        }
      }
      if (lane == 0) {
        // windows overlapping a packed chunk end at the latest in slot c_last + 1
        const int tiles = c_last < 0 ? 0 : min(tiles_max, (c_last + 1) / kTileSlots + 1);
        tile_pre[b] = tiles;
        cost_pre[b] = tiles * (kTileFixedCost + ((q_hi * K + 31) >> 5));
      }
    }
  }
  __syncthreads();
  block_exclusive_scan_inplace(tile_pre, B, sums, &carry, &total_tiles);
  block_exclusive_scan_inplace(cost_pre, B, sums, &carry, &total_cost);
  // pass 3: CTA x starts at the tile where the cumulative cost reaches x / grid of the total
  for (int x = t; x <= grid; x += 1024) {
    int start = total_tiles;
    if (x < grid && total_tiles > 0) {
      const long long target = (long long)total_cost * x / grid;
      int64_t lo = 0, hi = B - 1;   // last document whose cost prefix is <= target
      while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (cost_pre[mid] <= target) lo = mid; else hi = mid - 1;
      }
      const int tiles = tile_pre[lo + 1] - tile_pre[lo];
      const int dcost = cost_pre[lo + 1] - cost_pre[lo];
      const int per_tile = tiles > 0 ? dcost / tiles : 1;
      start = tile_pre[lo] + (tiles > 0 ? min(tiles, (int)((target - cost_pre[lo] + per_tile - 1) / per_tile)) : 0);
    }
    cta_start[x] = start;
  }
  if (in_smem)
    for (int64_t i = t; i <= B; i += 1024) { plan[2 + i] = s_tile[i]; plan[3 + B + i] = s_cost[i]; }
  // Cover: activation k is non-zero (ex2_approx) for |c - mu_k| * a_k <= sqrt(126); 11.0 leaves a margin.  The union of
  // the intervals [klo, khi) covers [-1.01, 1.01) iff the left end and every right end inside the range lie inside an
  // interval that extends beyond them -- one thread per end point instead of a serial sweep.  interaction.py's
  // tkl_kernel_set_covers restates this test in float32, rounding for rounding: where it says covered, impl="auto"
  // enqueues this kernel alone, so an answer of "not covered" here would leave the windows at the memset zeros.
  __shared__ int uncovered;
  if (t == 0) uncovered = 0;
  __syncthreads();
  if (t <= K && t <= 32) {
    const float x = t == 0 ? -1.01f : khi[t - 1];
    if (x >= -1.01f && x < 1.01f) {
      bool ok = false;
      for (int k = 0; k < K; ++k) ok = ok || (klo[k] <= x && khi[k] > x);
      if (!ok) atomicExch(&uncovered, 1);
    }
  }
  __syncthreads();
  if (t == 0) {
    plan[1] = total_tiles;
    plan[0] = (uncovered == 0 || force_cover == 1) && force_cover != -1 ? 1 : 0;
  }
}

__global__ void __launch_bounds__(1024) tkl_plan_kernel(const int32_t* __restrict__ slot_to_packed, const void* __restrict__ q_mask,
                                                        int mask_dtype, int64_t B, int C, int Lq, const float* __restrict__ mu,
                                                        const float* __restrict__ sigma, int K, int grid, int force_cover,
                                                        int32_t* __restrict__ plan) {
  tkl_plan_body<false>(slot_to_packed, q_mask, mask_dtype, B, C, Lq, mu, sigma, K, grid, force_cover, plan, TklPairs{});
}

// One CTA per SM at most (minBlocks 1): 64 registers, where the default bound spills the pair loads of the store mode.
__global__ void __launch_bounds__(1024, 1) tkl_plan_store_kernel(const int32_t* __restrict__ doc_slots, const void* __restrict__ q_mask,
                                                                 int mask_dtype, int64_t B, int C, int Lq, const float* __restrict__ mu,
                                                                 const float* __restrict__ sigma, int K, int grid, int force_cover,
                                                                 int32_t* __restrict__ plan, TklPairs X) {
  tkl_plan_body<true>(doc_slots, q_mask, mask_dtype, B, C, Lq, mu, sigma, K, grid, force_cover, plan, X);
}

// The tiles a CTA walks, identically in every role: [g_begin, g_end) of the global tile sequence, preceded by a halo
// tile when the share starts inside a document.
struct TileWalk {
  const int32_t* pre;   // plan + 2
  int g, g_end;
  int b;
  int t;                // tile inside document b
  int b_end_tile;       // tiles of document b
  bool halo;
  __device__ __forceinline__ bool init(const int32_t* plan, int B, int cta, int ncta) {
    pre = plan + 2;
    const int32_t* cta_start = plan + 4 + 2 * B;   // shares of equal COST (tkl_plan_kernel), monotone in the CTA index
    g = cta_start[cta];
    g_end = cta_start[cta + 1];
    if (g >= g_end) return false;
    int lo = 0, hi = B - 1;   // last document with pre[b] <= g ...
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (pre[mid] <= g) lo = mid; else hi = mid - 1;
    }
    b = lo;
    while (pre[b + 1] <= g) ++b;  // ... that has tiles (documents without tiles repeat the prefix value)
    t = g - pre[b];
    b_end_tile = pre[b + 1] - pre[b];
    halo = t > 0;
    if (halo) --t;
    return true;
  }
  __device__ __forceinline__ bool valid() const { return halo || g < g_end; }
  __device__ __forceinline__ void next() {
    if (halo) { halo = false; ++t; return; }
    ++g; ++t;
    if (g < g_end && t == b_end_tile) {
      ++b;
      while (pre[b + 1] == pre[b]) ++b;
      t = 0;
      b_end_tile = pre[b + 1] - pre[b];
    }
  }
};

// STORE: document b of the tile walk is pair b (TklPairs): its query box, query mask and saturation table come from query
// row pair_q[b], its chunk slots from row pair_d[b] of the passages' slot table.
template <int SAT, bool STORE>
__global__ void __launch_bounds__(kThreads, 1)
tkl_ts_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c, TklParams P,
              int n_raw, int fallback_available, TklPairs X) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* qring = smem;                                                    // [kOps][Qhi;Qlo]
  uint8_t* raws = smem + kOps * kQopBytes;                                  // [n_raw][Dx | Qx]
  float* cs = reinterpret_cast<float*>(raws + (size_t)n_raw * kRawBytes);   // [2][40 query rows][kCsStride] cosine tiles
  TsShared* S = reinterpret_cast<TsShared*>(cs + 2 * kMaxLq * kCsStride);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = (P.D + 31) / 32;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_c);
    for (int s = 0; s < n_raw; ++s) { mbar_init(&S->raw_full[s], 1); mbar_init(&S->raw_empty[s], kReleaseArrivals); }
    for (int s = 0; s < kOps; ++s) { mbar_init(&S->op_full[s], 64); mbar_init(&S->op_empty[s], 4); }
    for (int s = 0; s < 2; ++s) { mbar_init(&S->cs_full[s], 4); mbar_init(&S->cs_empty[s], kEpiWarps); }
    fence_barrier_init();
  }
  if (threadIdx.x < 16) S->sp[threadIdx.x] = (SAT == 0 && threadIdx.x < 13) ? P.sat_params[threadIdx.x] : 0.f;
  __syncthreads();

  // Programmatic dependent launch: this grid is launched while the plan kernel still runs (it triggers its dependents at
  // its first instruction), so the launch latency and the prologue above overlap with it; everything below reads the plan.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const bool covered = P.plan[0] == 1;
  // a kernel set without cover on a shape the FFMA kernel cannot run either: fail the launch (no printf here -- a
  // function call in the kernel would serialise its wgmma pipeline)
  if (!covered && !fallback_available && blockIdx.x == 0 && threadIdx.x == 0) __trap();

  // every role walks the same tile sequence with its own copy of the iterator (set up inside the role branch, after
  // setmaxnreg, so that it lives in that role's registers); without cover nobody has work and the FFMA kernel takes over
#define TKL_WALK() TileWalk tw; const bool have_work = covered && tw.init(P.plan, (int)P.B, (int)blockIdx.x, (int)gridDim.x)

  if (warp == 0) {
    // ------------------------------- TMA producer -------------------------------
    setmaxnreg_dec<kRegsLight>();
    TKL_WALK();
    if (lane == 0 && have_work) {
      int stage = 0;
      uint32_t phase = 0;
      for (; tw.valid(); tw.next()) {
        int pk[kTileSlots];
        int n_present = 0;
        const int64_t sb = tkl_slot_row<STORE>(X, tw.b);
#pragma unroll
        for (int s = 0; s < kTileSlots; ++s) {
          const int c = tw.t * kTileSlots + s;
          pk[s] = ((!STORE || sb >= 0) && c < P.C && !(tw.halo && s < kTileSlots - 1)) ? P.slot_to_packed[sb * P.C + c] : -1;
          n_present += pk[s] >= 0 ? 1 : 0;
        }
        const int qbox = (int)tkl_q_row<STORE>(X, tw.b);
        const uint32_t bytes = (uint32_t)(n_present * kSlotBytes + kQxBytes);
        for (int ck = 0; ck < nch; ++ck) {
          mbar_wait(&S->raw_empty[stage], phase ^ 1u);
          uint8_t* st = raws + (size_t)stage * kRawBytes;
          mbar_arrive_expect_tx(&S->raw_full[stage], bytes);
#pragma unroll
          for (int s = 0; s < kTileSlots; ++s)
            if (pk[s] >= 0) tma_load_3d(&tmap_c, st + s * kSlotBytes, &S->raw_full[stage], ck * 32, 0, pk[s], kEvictFirst);
          tma_load_3d(&tmap_q, st + kDxBytes, &S->raw_full[stage], ck * 32, 0, qbox, kEvictLast);
          if (++stage == n_raw) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp == 1) {
    setmaxnreg_dec<kRegsLight>();
  } else if (warp < 4) {
    // ------------------------------- query convert ------------------------------
    // 40 rows x 8 float4 per k-chunk = 320 float4 over 64 threads: thread qt owns 16-byte column c = qt & 7 of rows
    // (qt >> 3) + 8 j, j = 0..4
    setmaxnreg_dec<kRegsLight>();
    TKL_WALK();
    if (have_work) {
      const int qt = (warp - 2) * 32 + lane;
      const int c = qt & 7, r0 = qt >> 3;
      int rs_ = 0, os_ = 0, nr = 0;
      uint32_t rphase = 0, ophase = 0;
      for (; tw.valid(); tw.next()) {
        float ss[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
        for (int ck = 0; ck < nch; ++ck) {
          mbar_wait(&S->raw_full[rs_], rphase);
          const uint8_t* xq = raws + (size_t)rs_ * kRawBytes + kDxBytes;
          float4 x[5];
#pragma unroll
          for (int j = 0; j < 5; ++j) {
            const int row = r0 + 8 * j;
            x[j] = *reinterpret_cast<const float4*>(xq + row * 128 + ((c ^ (row & 7)) << 4));
            ss[j] = fmaf(x[j].x, x[j].x, fmaf(x[j].y, x[j].y, fmaf(x[j].z, x[j].z, fmaf(x[j].w, x[j].w, ss[j]))));
          }
          mbar_wait(&S->op_empty[os_], ophase ^ 1u);
          uint8_t* qo = qring + (size_t)os_ * kQopBytes;
#pragma unroll
          for (int j = 0; j < 5; ++j) {
            const int row = r0 + 8 * j;
            uint32_t hi[4], lo[4];
            split_tf32(x[j], hi, lo);
            const int off = row * 128 + ((c ^ (row & 7)) << 4);
            *reinterpret_cast<uint4*>(qo + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<uint4*>(qo + kMaxLq * 128 + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
          }
          if (ck == nch - 1) {
#pragma unroll
            for (int j = 0; j < 5; ++j) {
              float v = ss[j];
              v += __shfl_xor_sync(0xffffffffu, v, 1);
              v += __shfl_xor_sync(0xffffffffu, v, 2);
              v += __shfl_xor_sync(0xffffffffu, v, 4);
              if (c == 0) S->rs_q[nr][r0 + 8 * j] = 1.0f / (sqrtf(v) + kTinyNorm);
            }
          }
          fence_proxy_async_smem();
          mbar_arrive(&S->raw_empty[rs_]);
          mbar_arrive(&S->op_full[os_]);
          if (++rs_ == n_raw) { rs_ = 0; rphase ^= 1u; }
          if (++os_ == kOps) { os_ = 0; ophase ^= 1u; }
        }
        if (++nr == kNormRing) nr = 0;
      }
    }
  } else if (warp < kFirstEpiWarp) {
    // ------------------------------- MMA warpgroup: document operand, wgmma, cosine tile (phase A) -------------------
    // Thread (warp wq, lane) owns positions rb, rb + 8 (M-block 0) and 64 + rb, 72 + rb (M-block 1), rb = 16 wq + lane / 4.
    // Per 8-column K-step: the four positions' A fragments straight from the raw SWIZZLE_128B tile, split into hi / lo in
    // registers; D += Dhi Qhi^T + Dhi Qlo^T + Dlo Qhi^T + Dlo Qlo^T, wgmma m64n40k8 tf32 with A from registers.
    setmaxnreg_inc<kRegsMma>();
    TKL_WALK();
    if (have_work) {
      const int wq = warp & 3;
      const int tq = lane & 3;
      const int rb = 16 * wq + (lane >> 2);
      const int dmt = P.chunk_mask ? P.mask_dtype : MMB200_MASK_NONE;
      int rs_ = 0, os_ = 0, nr = 0;
      uint32_t rphase = 0, ophase = 0;
      int64_t tile_seq = 0;
      for (; tw.valid(); tw.next(), ++tile_seq) {
        const int t = tw.t;
        const int64_t sb = tkl_slot_row<STORE>(X, tw.b);
        uint64_t draw[4];
        bool present[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {   // the position's packed chunk, then its mask word: in flight during the MMAs
          const int row = rb + 8 * (e & 1) + 64 * (e >> 1);
          const int c = t * kTileSlots + row / kChunk;
          const int pk = ((!STORE || sb >= 0) && row < kTileRows && c < P.C) ? P.slot_to_packed[sb * P.C + c] : -1;
          present[e] = pk >= 0;
          draw[e] = pk < 0 ? 0 : dmt != MMB200_MASK_NONE ? mask_raw(P.chunk_mask, dmt, (int64_t)pk * kChunk + (row % kChunk)) : 1;
        }
        float acc0[20], acc1[20];
#pragma unroll
        for (int j = 0; j < 20; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }
        float ss[4] = {0.f, 0.f, 0.f, 0.f};
        for (int ck = 0; ck < nch; ++ck) {
          const int ksteps = (min(32, P.D - ck * 32) + 7) >> 3;   // 8 fp32 per wgmma K-step
          mbar_wait(&S->raw_full[rs_], rphase);
          mbar_wait(&S->op_full[os_], ophase);
          const float* x = reinterpret_cast<const float*>(raws + (size_t)rs_ * kRawBytes);
          const uint32_t qb = smem_u32(qring + (size_t)os_ * kQopBytes);
          const uint64_t bhi = make_wgmma_sw128_desc(qb), blo = make_wgmma_sw128_desc(qb + kMaxLq * 128);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (k < ksteps) {
              uint32_t ah[2][4], al[2][4];
#pragma unroll
              for (int mb = 0; mb < 2; ++mb) {
                const int ra = 64 * mb + rb, rc = ra + 8;   // rc & 7 == ra & 7
                const int ch0 = (2 * k) ^ (ra & 7), ch1 = (2 * k + 1) ^ (ra & 7);
                const float v[4] = {x[ra * 32 + ch0 * 4 + tq], x[rc * 32 + ch0 * 4 + tq], x[ra * 32 + ch1 * 4 + tq], x[rc * 32 + ch1 * 4 + tq]};
#pragma unroll
                for (int e = 0; e < 4; ++e) split_tf32(v[e], ah[mb][e], al[mb][e]);
                ss[2 * mb] = fmaf(v[0], v[0], fmaf(v[2], v[2], ss[2 * mb]));
                ss[2 * mb + 1] = fmaf(v[1], v[1], fmaf(v[3], v[3], ss[2 * mb + 1]));
              }
              const uint64_t kh = bhi + (uint64_t)(2 * k), kl = blo + (uint64_t)(2 * k);   // +32 bytes along K
              wgmma_fence();
              wgmma_m64n40k8_tf32_rs(acc0, ah[0], kh, 1u);
              wgmma_m64n40k8_tf32_rs(acc0, ah[0], kl, 1u);
              wgmma_m64n40k8_tf32_rs(acc0, al[0], kh, 1u);
              wgmma_m64n40k8_tf32_rs(acc0, al[0], kl, 1u);
              wgmma_m64n40k8_tf32_rs(acc1, ah[1], kh, 1u);
              wgmma_m64n40k8_tf32_rs(acc1, ah[1], kl, 1u);
              wgmma_m64n40k8_tf32_rs(acc1, al[1], kh, 1u);
              wgmma_m64n40k8_tf32_rs(acc1, al[1], kl, 1u);
              wgmma_commit();
              wgmma_wait<0>();
            }
          }
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&S->raw_empty[rs_]);
            mbar_arrive(&S->op_empty[os_]);
          }
          if (++rs_ == n_raw) { rs_ = 0; rphase ^= 1u; }
          if (++os_ == kOps) { os_ = 0; ophase ^= 1u; }
        }
        wgmma_fence_regs(acc0);
        wgmma_fence_regs(acc1);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          ss[e] += __shfl_xor_sync(0xffffffffu, ss[e], 1);
          ss[e] += __shfl_xor_sync(0xffffffffu, ss[e], 2);
        }
        const int buf = (int)(tile_seq & 1);
        float* cb = cs + buf * (kMaxLq * kCsStride);   // transposed: consecutive positions of one query row are adjacent
        mbar_wait(&S->cs_empty[buf], (uint32_t)((tile_seq >> 1) & 1) ^ 1u);
        const float* rq = S->rs_q[nr];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int row = rb + 8 * (e & 1) + 64 * (e >> 1);
          if (row < kTileRows) {
            const bool valid = present[e] && mask_test(draw[e], dmt);
            const float rsd = 1.0f / (sqrtf(ss[e]) + kTinyNorm);
            const float* a = (e >> 1) ? acc1 : acc0;
            const int ri = 2 * (e & 1);
#pragma unroll
            for (int j = 0; j < 5; ++j)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int col = 8 * j + 2 * tq + h;
                cb[col * kCsStride + row] = valid ? a[4 * j + ri + h] * rsd * rq[col] : kSentinel;
              }
            if (tq == 0) S->dmring[(tile_seq * kTileRows + row) & (kDmRing - 1)] = valid ? 1.f : 0.f;
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&S->cs_full[buf]);
        if (++nr == kNormRing) nr = 0;
      }
    }
  } else {
    // ------------------------------- epilogue ------------------------------------
    TKL_WALK();
    if (have_work) {
      const int ew = warp - kFirstEpiWarp;       // 0..15
      const int et = ew * 32 + lane;             // 0..511
      const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
      const int n_ik = P.Lq * P.K;
      const bool ik_live = et < n_ik;
      const int qi = ik_live ? et / P.K : 0;     // query row of this thread in phase B
      const int kk = ik_live ? et - qi * P.K : 0;
      const float a_k = rbf_scale(P.sigma[kk]);
      const float nma_k = -P.mu[kk] * a_k;        // x = (c - mu) a = c a + nma
      const float w_k = ik_live ? P.dense_w[kk] : 0.f;
      const float km_k = SAT == 1 ? P.sat_params[kk] : 1.f;
      float suf[kBlk];
#pragma unroll
      for (int r = 0; r < kBlk; ++r) suf[r] = 0.f;
      int64_t tile_seq = 0;
      int cur_doc = -1;
      int n_doc_warps = 0;   // epilogue warps holding an unmasked query row of the current document
      float qm_i = 0.f;

      for (; tw.valid(); tw.next(), ++tile_seq) {
        const int b = tw.b;
        const int t = tw.t;
        const int buf = (int)(tile_seq & 1);
        const float* cb = cs + buf * (kMaxLq * kCsStride);
        if (b != cur_doc) {
          // ---- new document: query mask, sat_emb_reduce1(q_i), saturation table indexed by (query row, token count)
          cur_doc = b;
          const int64_t qb = tkl_q_row<STORE>(X, b);
          named_bar_sync(1, kEpiThreads);   // nobody still reads the previous document's table / qm
          if (et < kMaxLq) S->qm[et] = (et < P.Lq && mask_at(P.q_mask, qmt, qb * P.Lq + et)) ? 1.f : 0.f;
          if (SAT == 0) {
            // the warp's rows ew, ew + 16, ew + 32 side by side: their loads are independent and in flight together (one
            // global-memory latency per document switch instead of one per row and 128-byte step)
            float rd[3] = {0.f, 0.f, 0.f};
            const float4* wr = reinterpret_cast<const float4*>(P.sat_red_w);
#pragma unroll 2
            for (int c4 = lane; c4 < (P.D >> 2); c4 += 32) {
              const float4 w = __ldg(wr + c4);
              float4 v[3];
#pragma unroll
              for (int a = 0; a < 3; ++a) {
                const int i = ew + kEpiWarps * a;
                v[a] = i < P.Lq ? __ldg(reinterpret_cast<const float4*>(P.q + (qb * P.Lq + i) * P.D) + c4)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
              }
#pragma unroll
              for (int a = 0; a < 3; ++a)
                rd[a] = fmaf(v[a].x, w.x, fmaf(v[a].y, w.y, fmaf(v[a].z, w.z, fmaf(v[a].w, w.w, rd[a]))));
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) {
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) rd[a] += __shfl_xor_sync(0xffffffffu, rd[a], o);
              if (lane == 0 && ew + kEpiWarps * a < kMaxLq) S->red[ew + kEpiWarps * a] = rd[a];
            }
          }
          named_bar_sync(1, kEpiThreads);
          if (SAT == 0) {
            const float* sp = S->sp;
            for (int e = et; e < kMaxLq * 31; e += kEpiThreads) {
              const int i = e / 31, len = e - i * 31;
              // LayerNorm over the pair (reduce(q_i), len), then three Linear(2,1) (sigir20_tkl.py:224-234); the gate
              // q_mask[i] * (len > 0) of :248 is folded into sat1 / sat3
              const float a0 = S->red[i], a1 = (float)len;
              const float mean = (a0 + a1) * 0.5f;
              const float d0 = a0 - mean, d1 = a1 - mean;
              const float rstd = rsqrtf((d0 * d0 + d1 * d1) * 0.5f + 1e-5f);
              const float y0 = d0 * rstd * sp[0] + sp[2], y1 = d1 * rstd * sp[1] + sp[3];
              const float gate = (S->qm[i] != 0.f && len > 0) ? 1.f : 0.f;
              S->sat[i * kSatStride + len] = make_float4((y0 * sp[4] + y1 * sp[5] + sp[6]) * gate,
                                                         1.0f / (y0 * sp[7] + y1 * sp[8] + sp[9]),
                                                         (y0 * sp[10] + y1 * sp[11] + sp[12]) * gate, 0.f);
            }
          }
          qm_i = S->qm[qi];   // written before the barrier above
          // query rows past the last unmasked one contribute exactly 0 to every window (the gate q_mask[i] of :248):
          // the warps that hold only such rows sit phase B out -- MSMARCO queries fill a fraction of the Lq slots
          int q_hi = 0;
          for (int i = kMaxLq - 1; i >= 0; --i)
            if (S->qm[i] != 0.f) { q_hi = i + 1; break; }
          n_doc_warps = (q_hi * P.K + 31) >> 5;
        }

        mbar_wait(&S->cs_full[buf], (uint32_t)((tile_seq >> 1) & 1));   // cosine tile and position flags of the tile
        // ---- token count of the window ending at each pair of this tile (sigir20_tkl.py:210 under "cover") ----
        if (et < 8 * kTilePairs) {   // eight threads per window, four positions each, three shuffle steps
          const int wl = et >> 3, sub = et & 7;
          const int last = t * kTileRows + 2 * wl + 1;   // last position of the window ending at pair wl
          float n = 0.f;
#pragma unroll
          for (int u = sub; u < kWindow; u += 8) {
            const int pos = last - u;
            if (pos >= 0) n += S->dmring[(tile_seq * kTileRows + 2 * wl + 1 - u) & (kDmRing - 1)];
          }
          n += __shfl_xor_sync(0xffffffffu, n, 1);
          n += __shfl_xor_sync(0xffffffffu, n, 2);
          n += __shfl_xor_sync(0xffffffffu, n, 4);
          if (sub == 0) S->lenw[wl / kBlk][wl % kBlk] = (uint16_t)(16 * (int)n);
        }
        named_bar_sync(3, kEpiThreads);
        // ---- phase B: activations, block prefix / suffix, windows ------------------------------------------------
        if (ew < n_doc_warps) {
          if (tw.halo) {
            // halo tile: only the suffix sums of its last block are wanted
            const float2* cblk = reinterpret_cast<const float2*>(cb + qi * kCsStride + 2 * kBlk * (kBlocks - 1));
#pragma unroll
            for (int r = 0; r < kBlk; ++r) {
              const float2 c = cblk[r];
              const float x0 = fmaf(c.x, a_k, nma_k), x1 = fmaf(c.y, a_k, nma_k);
              suf[r] = ex2_approx(-x0 * x0) + ex2_approx(-x1 * x1);
            }
#pragma unroll
            for (int r = kBlk - 2; r >= 0; --r) suf[r] += suf[r + 1];
          } else {
            // Windows that fall outside [0, W) (first block of a document, tail of the last tile) are computed like
            // the others -- from stale suffix sums or padding -- and dropped by the range check of the final write.
            const uint8_t* sat_row = reinterpret_cast<const uint8_t*>(S->sat + qi * kSatStride);
            for (int j = 0; j < kBlocks; ++j) {
              float tv[16];
              float pre = 0.f;
              const float2* cblk = reinterpret_cast<const float2*>(cb + qi * kCsStride + 2 * kBlk * j);
              uint32_t lw[8];   // the block's 15 window token counts: two 16-byte loads instead of 15 scalar ones
              {
                const uint4 la = *reinterpret_cast<const uint4*>(&S->lenw[j][0]), lb = *reinterpret_cast<const uint4*>(&S->lenw[j][8]);
                lw[0] = la.x; lw[1] = la.y; lw[2] = la.z; lw[3] = la.w; lw[4] = lb.x; lw[5] = lb.y; lw[6] = lb.z; lw[7] = lb.w;
              }
#pragma unroll
              for (int r = 0; r < kBlk; ++r) {
                const float2 c = cblk[r];
                const float x0 = fmaf(c.x, a_k, nma_k), x1 = fmaf(c.y, a_k, nma_k);
                const float u = ex2_approx(-x0 * x0) + ex2_approx(-x1 * x1);
                pre = r == 0 ? u : pre + u;
                const float Ssum = r < kBlk - 1 ? suf[r + 1] + pre : pre;
                suf[r] = u;   // suf[r] of the previous block was consumed by window r - 1
                const int lenb = (int)((lw[r >> 1] >> (16 * (r & 1))) & 0xffffu);
                if (SAT == 0) {
                  const float4 st = *reinterpret_cast<const float4*>(sat_row + lenb);
                  const float pw = ex2_approx(st.y * lg2_approx(fmaxf(Ssum, kClamp)));
                  tv[r] = w_k * fmaf(st.x, pw, -st.z);
                } else {
                  const float lg = 0.6931471805599453f * lg2_approx(fmaxf(Ssum * km_k, kClamp));
                  tv[r] = (lenb > 0 && qm_i != 0.f) ? w_k * lg : 0.f;
                }
              }
#pragma unroll
              for (int r = kBlk - 2; r >= 0; --r) suf[r] += suf[r + 1];
              tv[15] = 0.f;
              // transposed butterfly: 16 values x 32 lanes -> lane l holds the warp total of value l >> 1
#pragma unroll
              for (int jj = 0; jj < 8; ++jj) {
                const bool up = (lane & 16) != 0;
                const float send = up ? tv[jj] : tv[jj + 8];
                const float keep = up ? tv[jj + 8] : tv[jj];
                tv[jj] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
              }
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const bool up = (lane & 8) != 0;
                const float send = up ? tv[jj] : tv[jj + 4];
                const float keep = up ? tv[jj + 4] : tv[jj];
                tv[jj] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
              }
#pragma unroll
              for (int jj = 0; jj < 2; ++jj) {
                const bool up = (lane & 4) != 0;
                const float send = up ? tv[jj] : tv[jj + 2];
                const float keep = up ? tv[jj + 2] : tv[jj];
                tv[jj] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
              }
              {
                const bool up = (lane & 2) != 0;
                const float send = up ? tv[0] : tv[1];
                const float keep = up ? tv[1] : tv[0];
                tv[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
              }
              tv[0] += __shfl_xor_sync(0xffffffffu, tv[0], 1);
              const int vi = lane >> 1;   // = 8 b4 + 4 b3 + 2 b2 + b1
              if (!(lane & 1) && vi < kBlk) S->part[ew][kBlk * j + vi] = tv[0];
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&S->cs_empty[buf]);   // this warp is done with the cosine tile
        named_bar_sync(4, kEpiThreads);
        if (!tw.halo && et < kTilePairs) {
          const int w = t * kTilePairs - (kBlk - 1) + et;
          if (w >= 0 && w < P.W) {
            float pv[kEpiWarps];
#pragma unroll
            for (int ww = 0; ww < kEpiWarps; ++ww) pv[ww] = ww < n_doc_warps ? S->part[ww][et] : 0.f;   // loads in flight together
            float s = 0.f;
#pragma unroll
            for (int ww = 0; ww < kEpiWarps; ++ww) s += pv[ww];   // fixed order; the zeros of idle warps change nothing
            P.window_score[(int64_t)b * P.W + w] = s;
          }
        }
      }
    }
  }

}

#undef TKL_WALK

}  // namespace

int tkl_window_ts_launch(TklParams& P, const TklPairs& X, const DeviceInfo& dev, cudaStream_t stream, bool* handled,
                         int32_t** plan_out) {
  *handled = false;
  *plan_out = nullptr;
  const bool store = X.pair_q != nullptr;
  if (P.Lq > kMaxLq || P.K > 16 || P.Lq * P.K > kEpiThreads || P.D % 4 != 0) return MMB200_OK;
  if (P.B * (int64_t)P.C >= (1ll << 31) || P.B >= (1ll << 31) - 8) return MMB200_OK;
  const size_t fixed = (size_t)kOps * kQopBytes + 2 * (size_t)kMaxLq * kCsStride * sizeof(float) + sizeof(TsShared) + 1024;
  const int n_raw = std::min<int>(kMaxRaw, (int)(((size_t)dev.max_smem_optin - fixed) / kRawBytes));
  if (n_raw < 2) return MMB200_OK;
  const size_t smem = fixed + (size_t)n_raw * kRawBytes;
  CUtensorMap tq, tc;
  {
    const uint64_t dims[3] = {(uint64_t)P.D, (uint64_t)P.Lq, (uint64_t)(store ? X.n_q : P.B)};
    const uint64_t strides[2] = {(uint64_t)P.D * 4, (uint64_t)P.Lq * P.D * 4};
    const uint32_t box[3] = {32, (uint32_t)kMaxLq, 1};
    if (int rc = encode_tensor_map(&tq, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.q, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))
      return rc;
  }
  {
    // the packed chunk count is not part of the padded C ABI: every index the kernel uses comes from slot_to_packed, so
    // the outer extent only has to be an upper bound (B * C slots); the store entry passes its chunk count
    const uint64_t dims[3] = {(uint64_t)P.D, (uint64_t)kChunk, (uint64_t)(P.n_chunks > 0 ? P.n_chunks : P.B * P.C)};
    const uint64_t strides[2] = {(uint64_t)P.D * 4, (uint64_t)kChunk * P.D * 4};
    const uint32_t box[3] = {32, (uint32_t)kChunk, 1};
    if (int rc = encode_tensor_map(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.chunks, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  int32_t* plan = nullptr;
  const int grid = dev.sm_count;
  MMB_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&plan), (size_t)(2 * P.B + 6 + grid) * sizeof(int32_t), stream));
  int force = 0;
#ifdef MMB200_ENABLE_PROF
  if (const char* e = getenv("MMB200_TKL_COVER")) force = atoi(e);  // 1 / -1: force the answer of the cover test
#endif
  // the zero fill first: the window-score kernel is a programmatic dependent of the plan kernel (nothing may sit between them)
  MMB_CHECK_CUDA(cudaMemsetAsync(P.window_score, 0, (size_t)P.B * P.W * sizeof(float), stream));
  if (store)
    tkl_plan_store_kernel<<<1, 1024, 0, stream>>>(P.slot_to_packed, P.q_mask, P.mask_dtype, P.B, P.C, P.Lq, P.mu, P.sigma,
                                                  P.K, grid, force, plan, X);
  else
    tkl_plan_kernel<<<1, 1024, 0, stream>>>(P.slot_to_packed, P.q_mask, P.mask_dtype, P.B, P.C, P.Lq, P.mu, P.sigma, P.K, grid,
                                            force, plan);
  MMB_CHECK_CUDA(cudaGetLastError());
  P.plan = plan;
  *plan_out = plan;
  const int fallback = P.segs > 0 ? 1 : 0;
  auto launch_pdl = [&](auto kernel) -> cudaError_t {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, tq, tc, P, n_raw, fallback, X);
  };
  static bool attr_set[2][2][64] = {};
  const int di = dev.device & 63;
  auto launch = [&](auto kernel, bool& attr) -> cudaError_t {
    if (!attr) {
      if (cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dev.max_smem_optin))
        return e;
      attr = true;
    }
    return launch_pdl(kernel);
  };
  bool& attr = attr_set[P.saturation][store ? 1 : 0][di];
  if (P.saturation == 0)
    MMB_CHECK_CUDA(store ? launch(tkl_ts_kernel<0, true>, attr) : launch(tkl_ts_kernel<0, false>, attr));
  else
    MMB_CHECK_CUDA(store ? launch(tkl_ts_kernel<1, true>, attr) : launch(tkl_ts_kernel<1, false>, attr));
  MMB_CHECK_CUDA(cudaGetLastError());
  *handled = true;
  return MMB200_OK;
}

}  // namespace mmb
