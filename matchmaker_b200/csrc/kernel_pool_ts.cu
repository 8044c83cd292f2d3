// Cosine + RBF kernel pooling forward (KNRM / TK) on the tensor cores with fp32-grade accuracy.
//
// Arithmetic (x = hi + lo from split_tf32, [Qhi;Qlo] stacked along N):
//
//     D[128 doc rows x 64] = Dhi[128 x K] * [Qhi; Qlo]^T  +  Dlo[128 x K] * [Qhi; Qlo]^T
//
// The document operand never goes back to shared memory: the MMA warpgroups read the raw fp32 tile TMA delivered in the
// wgmma A-fragment layout, split it into hi / lo in registers and issue wgmma kind tf32 with A from registers; only the
// small query operand [Qhi;Qlo] is written to shared memory (K-major, SWIZZLE_128B) for the B descriptor.
//
// Padding is skipped instead of computed: the last document tile is fetched with a box of exactly
// round8(Ld mod 128) rows (rows past it hold stale, finite data whose results are masked), and the last K-chunk only
// multiplies the 8-column steps that hold data (D = 300 -> 2 of 4).
//
// Per CTA (persistent, one per SM, 640 threads = 5 warpgroups; registers are re-dealt with setmaxnreg):
//   warp 0      TMA producer: fp32 chunks [<=128 doc rows x 32] + [32 query rows x 32], SWIZZLE_128B, raw ring
//   warps 2-3   query convert, two threads per query row: hi / lo into the B-operand ring, query norms
//   warps 4-11  two MMA warpgroups, warpgroup c = document rows 64c .. 64c + 63: A fragments (hi, lo) from the raw
//               tile, wgmma m64n64k8 tf32 into registers, document norms by quad shuffles; then phase A: add the two
//               halves, scale by the norms, cosine tile to shared memory (masked rows -> sentinel), last live row
//               published
//   warps 12-19 epilogue, phase B: lane = query row, rows dealt round-robin to the warps two at a time, K activations
//               ex2(-((c-mu)a)^2) accumulated in registers; end of pair: log, per-kernel sums, score.
// The two cosine tiles are handed over between phase A and phase B through mbarriers (cs_full / cs_empty).
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "device_util.cuh"
#include "host_util.cuh"
#include "kernel_pool.cuh"
#include "masks.cuh"
#include "ptx.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 640;           // 20 warps, see the role table above
constexpr int kMaxRaw = 8;            // raw ring (TMA targets): 20 KB per slot
constexpr int kOps = 4;               // query-operand ring: B slot in shared memory (8 KB)
constexpr int kNormRing = kOps + 2;
constexpr int kDxBytes = 128 * 128;   // [128 rows][32 fp32]
constexpr int kQxBytes = 32 * 128;    // [32 query rows][32 fp32]
constexpr int kRawBytes = kDxBytes + kQxBytes;          // 20 KB
constexpr int kQ64Bytes = 64 * 128;   // rows 0-31 Q hi, rows 32-63 Q lo
constexpr int kEpiThreads = 256;
constexpr int kReleaseArrivals = 8 + 64;  // lane 0 of each MMA warp + every lane of the two query warps
constexpr int kFirstDocWarp = 4, kFirstEpiWarp = 12;
constexpr int kRegsLight = 56, kRegsMma = 88, kRegsEpilogue = 120;  // setmaxnreg budgets per warpgroup (<= 640 x 96)
constexpr float kSentinel = 1.0e6f;   // "cosine" of a masked row: ex2(-((1e6 - mu) a)^2) is exactly 0 for any sigma < 1e4

struct KpShared {
  uint64_t raw_full[kMaxRaw];    // TMA -> query convert, MMA warps
  uint64_t raw_empty[kMaxRaw];   // query convert, MMA warps -> TMA
  uint64_t op_full[kOps];        // query convert -> MMA warps
  uint64_t op_empty[kOps];       // MMA warps -> query convert
  uint64_t cs_full[2];           // phase A (MMA warps) -> phase B (epilogue warps)
  uint64_t cs_empty[2];          // phase B -> phase A
  // 1 / (|q| + eps) travels from the query convert warps to phase A in its own ring: the convert warps run up to kOps
  // k-chunks ahead of the MMA warps -- kOps tiles when a tile is a single k-chunk (D <= 32)
  float rs_q[kNormRing][32];
  float mu[32], a[32], alpha[32], w[32];
  float pk[32];
  float qm[32];
  float lg[2][128];              // per cosine tile: log2 of the document-term gate (0 without a gate)
  int live[2][8];                // per cosine tile: last unmasked document row + 1 of each MMA warp's 16 rows
};

// The body of both entry points below: the padded layout, or (STORE) the store mode, where pair p reads query
// pair_q[p] and its passage's rows from the store (KpParams::doc_offsets) with the passage's first row as the tile's
// TMA row coordinate
template <int KB, bool SAVE, bool STORE>
__device__ __forceinline__ void kernel_pool_ts_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_d,
                                                    const CUtensorMap& tmap_d_last, const KpParams& P, int n_raw,
                                                    int last_box_rows) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for SWIZZLE_128B tiles, derived by pointer arithmetic on the __shared__ array so the
  // compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* qring = smem;                                                        // [kOps][Qhi;Qlo]
  uint8_t* raws = smem + kOps * kQ64Bytes;                                      // [n_raw][Dx | Qx]
  float* cs = reinterpret_cast<float*>(raws + (size_t)n_raw * kRawBytes);       // [2][128][32] cosine tiles
  float* spart = cs + 2 * 128 * 32;                                            // [8][KB][32] end-of-pair scratch
  KpShared* S = reinterpret_cast<KpShared*>(spart + 8 * 32 * 32);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_padded = (P.Ld + 127) / 128;
  // store mode: the passage of pair p is rows row0 .. row0 + len of the store; its tiles start at row0
  auto pair_rows = [&](int64_t p, int64_t* row0) -> int {
    if constexpr (STORE) return kp_store_rows(P, p, row0);
    *row0 = 0;
    return P.Ld;
  };
  const int nch = (P.D + 31) / 32;
  int64_t p_begin, p_end;
  cta_share(P.B, &p_begin, &p_end);

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_d);
    prefetch_tensormap(&tmap_d_last);
    for (int s = 0; s < n_raw; ++s) { mbar_init(&S->raw_full[s], 1); mbar_init(&S->raw_empty[s], kReleaseArrivals); }
    for (int s = 0; s < kOps; ++s) { mbar_init(&S->op_full[s], 64); mbar_init(&S->op_empty[s], 8); }
    for (int s = 0; s < 2; ++s) { mbar_init(&S->cs_full[s], 8); mbar_init(&S->cs_empty[s], 8); }
    fence_barrier_init();
  }
  if (threadIdx.x < 32) {
    const int t = threadIdx.x;
    const bool ok = t < P.K;
    S->mu[t] = ok ? P.mu[t] : 0.f;
    S->a[t] = ok ? rbf_scale(P.sigma[t]) : 0.f;
    S->alpha[t] = ok ? (P.alpha ? P.alpha[t] : 1.f) : 1.f;
    S->w[t] = ok ? P.weight[t] : 0.f;
  }
  __syncthreads();

  // every role branch starts with its setmaxnreg so that ptxas allocates each branch against its own budget
  if (warp == 0) {
    // ------------------------------- TMA producer -------------------------------
    // The whole warp walks the loop (uniform control flow and operands); one elected lane issues: inside an
    // `if (lane == 0)` region the compiler wraps every TMA in an ELECT / R2UR waterfall loop (ptx.cuh)
    setmaxnreg_dec<kRegsLight>();
    int stage = 0;
    uint32_t phase = 0;
    const uint32_t last_bytes = (uint32_t)(last_box_rows * 128 + kQxBytes);
    for (int64_t p = p_begin; p < p_end; ++p) {
      int64_t row0;
      const int len = pair_rows(p, &row0);
      const int tiles = STORE ? (len + 127) / 128 : tiles_padded;
      const int qz = STORE ? P.pair_q[p] : (int)p;
      for (int t = 0; t < tiles; ++t) {
        const bool last = t == tiles - 1;
        // store mode: the tile's rows rounded up to 8, fetched as 32-row boxes (tmap_d) then 8-row boxes (tmap_d_last)
        const int rows8 = STORE ? (min(128, len - t * 128) + 7) & ~7 : 0;
        for (int ck = 0; ck < nch; ++ck) {
          mbar_wait(&S->raw_empty[stage], phase ^ 1u);
          uint8_t* st = raws + (size_t)stage * kRawBytes;
          if (elect_one_sync()) {
            if constexpr (STORE) {
              mbar_arrive_expect_tx(&S->raw_full[stage], (uint32_t)(rows8 * 128 + kQxBytes));
              const int y = (int)row0 + t * 128;
              int r = 0;
              for (; r + 32 <= rows8; r += 32) tma_load_3d(&tmap_d, st + r * 128, &S->raw_full[stage], ck * 32, y + r, 0, kEvictFirst);
              for (; r < rows8; r += 8) tma_load_3d(&tmap_d_last, st + r * 128, &S->raw_full[stage], ck * 32, y + r, 0, kEvictFirst);
            } else {
              mbar_arrive_expect_tx(&S->raw_full[stage], last ? last_bytes : (uint32_t)kRawBytes);
              tma_load_3d(last ? &tmap_d_last : &tmap_d, st, &S->raw_full[stage], ck * 32, t * 128, (int)p, kEvictFirst);
            }
            tma_load_3d(&tmap_q, st + kDxBytes, &S->raw_full[stage], ck * 32, P.q_row0, qz, kEvictLast);
          }
          __syncwarp();
          if (++stage == n_raw) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp == 1) {
    setmaxnreg_dec<kRegsLight>();
  } else if (warp < 4) {
    // ------------------------------- query convert: [Qhi;Qlo] B operand, norms ------
    setmaxnreg_dec<kRegsLight>();
    const int qt = (warp - 2) * 32 + lane;    // 0..63: (query row, column half)
    const int row = qt >> 1, half = qt & 1;
    const int sw = row & 7;
    int rs_ = 0, os_ = 0, nr = 0;
    uint32_t rphase = 0, ophase = 0;
    for (int64_t p = p_begin; p < p_end; ++p) {
      int64_t row0;
      const int tiles = STORE ? (pair_rows(p, &row0) + 127) / 128 : tiles_padded;
      for (int t = 0; t < tiles; ++t) {
        float4 ss4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int ck = 0; ck < nch; ++ck) {
          const bool have = half == 0 || P.D - ck * 32 > 16;  // this thread's 16 columns hold data
          mbar_wait(&S->raw_full[rs_], rphase);
          const uint8_t* xrow = raws + (size_t)rs_ * kRawBytes + kDxBytes + row * 128;
          float4 x[4];
#pragma unroll
          for (int c = 0; c < 4; ++c)
            x[c] = have ? *reinterpret_cast<const float4*>(xrow + (((4 * half + c) ^ sw) << 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float4 v = x[c];
            ss4.x = fmaf(v.x, v.x, ss4.x); ss4.y = fmaf(v.y, v.y, ss4.y); ss4.z = fmaf(v.z, v.z, ss4.z); ss4.w = fmaf(v.w, v.w, ss4.w);
          }
          mbar_wait(&S->op_empty[os_], ophase ^ 1u);
          uint8_t* hrow = qring + (size_t)os_ * kQ64Bytes + row * 128;
          uint8_t* lrow = hrow + 32 * 128;
          if (have) {
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              uint32_t hi[4], lo[4];
              split_tf32(x[c], hi, lo);
              const int off = (((4 * half + c) ^ sw) << 4);
              *reinterpret_cast<uint4*>(hrow + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
              *reinterpret_cast<uint4*>(lrow + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            }
          }
          if (ck == nch - 1) {
            float ss = (ss4.x + ss4.y) + (ss4.z + ss4.w);
            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
            if (half == 0) S->rs_q[nr][row] = 1.0f / (sqrtf(ss) + kTinyNorm);
          }
          // release the raw slot only after the stores that consumed the loaded values: an arrive placed right after
          // the LDS is hoisted above their completion by ptxas and the TMA overwrites rows that are still being read;
          // the operand stores are made visible to the tensor core's async proxy before the MMA warps are told
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
    // ------------------------------- document operand + wgmma + cosine tile (phase A) ------------------------------
    setmaxnreg_dec<kRegsMma>();
    const int c = (warp - kFirstDocWarp) >> 2;   // warpgroup: document rows 64c .. 64c + 63 of the tile
    const int wq = warp & 3;
    const int ew = 4 * c + wq;                   // 0..7
    const int r0 = 64 * c + 16 * wq + (lane >> 2), r1 = r0 + 8;   // this thread's two document rows
    const int tq = lane & 3;
    const int dmt = P.d_mask ? P.mask_dtype : MMB200_MASK_NONE;
    int rs_ = 0, os_ = 0, nr = 0;
    uint32_t rphase = 0, ophase = 0;
    int64_t tile_seq = 0;
    for (int64_t p = p_begin; p < p_end; ++p) {
      int64_t row0;
      const int len = pair_rows(p, &row0);
      const int tiles = STORE ? (len + 127) / 128 : tiles_padded;
      // first gate entry of the pair: the passage's first store row, or row p of the padded [B, Ld] gate
      const int64_t gate0 = STORE ? row0 : p * (int64_t)P.Ld;
      for (int t = 0; t < tiles; ++t, ++tile_seq) {
        const int g0 = t * 128 + r0, g1 = t * 128 + r1;
        const uint64_t draw0 = g0 < len ? (dmt != MMB200_MASK_NONE ? mask_raw(P.d_mask, dmt, p * (int64_t)P.Ld + g0) : 1) : 0;
        const uint64_t draw1 = g1 < len ? (dmt != MMB200_MASK_NONE ? mask_raw(P.d_mask, dmt, p * (int64_t)P.Ld + g1) : 1) : 0;
        float acc[32];   // columns 0..31: D . Qhi, 32..63: D . Qlo (rows r0 / r1)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = 0.f;
        float ss0 = 0.f, ss1 = 0.f;
        for (int ck = 0; ck < nch; ++ck) {
          const int ksteps = (min(32, P.D - ck * 32) + 7) >> 3;  // 8 fp32 per wgmma K-step
          mbar_wait(&S->raw_full[rs_], rphase);
          const float* x = reinterpret_cast<const float*>(raws + (size_t)rs_ * kRawBytes);
          // A fragments straight from the raw SWIZZLE_128B tile: element (row, col) sits in 16-byte chunk (col / 4) ^ (row & 7)
          uint32_t ahi[4][4], alo[4][4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int ch0 = (2 * k) ^ (r0 & 7), ch1 = (2 * k + 1) ^ (r0 & 7);   // r1 & 7 == r0 & 7
            const float v[4] = {x[r0 * 32 + ch0 * 4 + tq], x[r1 * 32 + ch0 * 4 + tq], x[r0 * 32 + ch1 * 4 + tq], x[r1 * 32 + ch1 * 4 + tq]};
#pragma unroll
            for (int e = 0; e < 4; ++e) split_tf32(v[e], ahi[k][e], alo[k][e]);
            ss0 = fmaf(v[0], v[0], fmaf(v[2], v[2], ss0));
            ss1 = fmaf(v[1], v[1], fmaf(v[3], v[3], ss1));
          }
          mbar_wait(&S->op_full[os_], ophase);
          const uint64_t b0 = make_wgmma_sw128_desc(smem_u32(qring + (size_t)os_ * kQ64Bytes));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (k < ksteps) {
              wgmma_m64n64k8_tf32_rs(acc, ahi[k], b0 + (uint64_t)(k * 2), 1u);   // +32 bytes along K
              wgmma_m64n64k8_tf32_rs(acc, alo[k], b0 + (uint64_t)(k * 2), 1u);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) {
            mbar_arrive(&S->raw_empty[rs_]);
            mbar_arrive(&S->op_empty[os_]);
          }
          if (++rs_ == n_raw) { rs_ = 0; rphase ^= 1u; }
          if (++os_ == kOps) { os_ = 0; ophase ^= 1u; }
        }
        wgmma_fence_regs(acc);
        ss0 += __shfl_xor_sync(0xffffffffu, ss0, 1); ss0 += __shfl_xor_sync(0xffffffffu, ss0, 2);
        ss1 += __shfl_xor_sync(0xffffffffu, ss1, 1); ss1 += __shfl_xor_sync(0xffffffffu, ss1, 2);
        const float rsd0 = 1.0f / (sqrtf(ss0) + kTinyNorm), rsd1 = 1.0f / (sqrtf(ss1) + kTinyNorm);
        const bool valid0 = g0 < len && mask_test(draw0, dmt), valid1 = g1 < len && mask_test(draw1, dmt);
        const int buf = (int)(tile_seq & 1);
        float* cbuf = cs + buf * (128 * 32);
        mbar_wait(&S->cs_empty[buf], (uint32_t)((tile_seq >> 1) & 1) ^ 1u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = 8 * j + 2 * tq;   // query columns col, col + 1
          const float q0 = S->rs_q[nr][col], q1 = S->rs_q[nr][col + 1];
          const float c00 = (acc[4 * j + 0] + acc[4 * (j + 4) + 0]) * rsd0 * q0;
          const float c01 = (acc[4 * j + 1] + acc[4 * (j + 4) + 1]) * rsd0 * q1;
          const float c10 = (acc[4 * j + 2] + acc[4 * (j + 4) + 2]) * rsd1 * q0;
          const float c11 = (acc[4 * j + 3] + acc[4 * (j + 4) + 3]) * rsd1 * q1;
          *reinterpret_cast<float2*>(cbuf + r0 * 32 + ((((col >> 2) ^ (r0 & 7))) << 2) + (col & 3)) =
              make_float2(valid0 ? c00 : kSentinel, valid0 ? c01 : kSentinel);
          *reinterpret_cast<float2*>(cbuf + r1 * 32 + ((((col >> 2) ^ (r1 & 7))) << 2) + (col & 3)) =
              make_float2(valid1 ? c10 : kSentinel, valid1 ? c11 : kSentinel);
          if constexpr (SAVE) {  // training: leave the unmasked cosines and the norms for the tensor-core backward
            if (g0 < P.Ld) *reinterpret_cast<float2*>(P.saved + kp_saved_cos_off(p, P.Ld) + (int64_t)g0 * 32 + col) = make_float2(c00, c01);
            if (g1 < P.Ld) *reinterpret_cast<float2*>(P.saved + kp_saved_cos_off(p, P.Ld) + (int64_t)g1 * 32 + col) = make_float2(c10, c11);
          }
        }
        if constexpr (SAVE) {
          if (tq == 0) {
            if (g0 < P.Ld) P.saved[kp_saved_rsd_off(P.B, p, P.Ld) + g0] = rsd0;
            if (g1 < P.Ld) P.saved[kp_saved_rsd_off(P.B, p, P.Ld) + g1] = rsd1;
          }
          if (t == 0 && ew == 0) P.saved[kp_saved_rsq_off(P.B, p, P.Ld) + lane] = S->rs_q[nr][lane];
        }
        // last live row + 1 of this warp's 16 rows: phase B stops there instead of testing every row
        const int live = __reduce_max_sync(0xffffffffu, valid1 ? r1 + 1 : valid0 ? r0 + 1 : 0);
        if (lane == 0) S->live[buf][ew] = live;
        if (tq == 0) {
          // gate g_j * exp(-x^2) = 2^(-u^2 + log2 g_j): one exponent term per document row, no extra multiply
          S->lg[buf][r0] = (P.gate && g0 < len) ? __log2f(fmaxf(P.gate[gate0 + g0], 0.f)) : 0.f;
          S->lg[buf][r1] = (P.gate && g1 < len) ? __log2f(fmaxf(P.gate[gate0 + g1], 0.f)) : 0.f;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&S->cs_full[buf]);
        if (++nr == kNormRing) nr = 0;
      }
    }
  } else {
    // ------------------------------- epilogue (phase B) ------------------------------------
    setmaxnreg_inc<kRegsEpilogue>();
    const int ew = warp - kFirstEpiWarp;  // 0..7
    const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
    int64_t tile_seq = 0;
    // kernel centres / widths in registers when they fit (the reference's 11- and 21-kernel models); otherwise they are
    // re-read from shared memory inside the activation loop
    constexpr bool kRegConst = KB <= 21;
    float mu_r[kRegConst ? KB : 1], a_r[kRegConst ? KB : 1];
    if constexpr (kRegConst) {
#pragma unroll
      for (int k = 0; k < KB; ++k) { mu_r[k] = S->mu[k]; a_r[k] = S->a[k]; }
    }
    for (int64_t p = p_begin; p < p_end; ++p) {
      float acc[KB];
#pragma unroll
      for (int k = 0; k < KB; ++k) acc[k] = 0.f;
      int64_t row0;
      const int len = pair_rows(p, &row0);
      const int tiles = STORE ? (len + 127) / 128 : tiles_padded;
      const int64_t qz = STORE ? P.pair_q[p] : p;
      uint64_t qraw = 0;
      if (lane < P.Lq) qraw = qmt != MMB200_MASK_NONE ? mask_raw(P.q_mask, qmt, qz * P.Lq_total + P.q_row0 + lane) : 1;
      // Short queries: phase B has lane = query row, so a 6-token query would leave 26 lanes of every MUFU instruction
      // idle.  With q_hi = 1 + last unmasked query row, the warp's lanes are dealt as 32 / qp sub-streams of qp query rows
      // (qp = 4, 8, 16 or 32 >= q_hi); sub-stream s takes the document rows r + 16 s, and the sub-streams are added at
      // the end of the pair.  Rows >= qp are masked query rows: their S is not needed (it is reported as 0).
      int qp = 32;
      if (qmt != MMB200_MASK_NONE) {
        const unsigned qm_bits = __ballot_sync(0xffffffffu, lane < P.Lq && mask_test(qraw, qmt));
        const int q_hi = qm_bits ? 32 - __clz(qm_bits) : 0;
        qp = q_hi <= 4 ? 4 : q_hi <= 8 ? 8 : q_hi <= 16 ? 16 : 32;
      }
      const int qi = lane & (qp - 1);            // query row of this lane in phase B
      const int sub16 = 16 * (lane / qp);        // document-row offset of this lane's sub-stream
      const int rstep = 16 * (32 / qp);          // document rows one warp iteration advances by
      for (int t = 0; t < tiles; ++t, ++tile_seq) {
        const int buf = (int)(tile_seq & 1);
        const float* cbuf = cs + buf * (128 * 32);
        mbar_wait(&S->cs_full[buf], (uint32_t)((tile_seq >> 1) & 1));
        {  // phase B: lane = query row; document rows are dealt round-robin to the 8 warps, two at a time (rows r and
           // r + 8 give the MUFU two independent streams).  Masked rows below the last live row carry the sentinel
           // and contribute exactly 0; rows above it are not visited.  The next pair of cosines is loaded before the
           // current one is consumed so that the MUFU stream does not drain at every iteration.
          const int* lv = S->live[buf];
          const int rows_live = max(max(max(lv[0], lv[1]), max(lv[2], lv[3])), max(max(lv[4], lv[5]), max(lv[6], lv[7])));
          auto cos_at = [&](int r) -> float {
            return r < rows_live ? cbuf[r * 32 + (((qi >> 2) ^ (r & 7)) << 2) + (qi & 3)] : kSentinel;
          };
          const float* lgs = S->lg[buf];
          float c0 = cos_at(ew + sub16), c1 = cos_at(ew + sub16 + 8);
          float l0 = lgs[(ew + sub16) & 127], l1 = lgs[(ew + sub16 + 8) & 127];
          for (int r0 = ew; r0 < rows_live; r0 += rstep) {   // uniform trip count: rows past rows_live read the sentinel
            const int r = r0 + sub16 + rstep;
            const float n0 = cos_at(r), n1 = cos_at(r + 8);
            const float m0 = lgs[r & 127], m1 = lgs[(r + 8) & 127];
#pragma unroll
            for (int k = 0; k < KB; ++k) {
              const float m = kRegConst ? mu_r[k] : S->mu[k], a = kRegConst ? a_r[k] : S->a[k];
              const float u0 = (c0 - m) * a, u1 = (c1 - m) * a;
              acc[k] += ex2_approx(fmaf(-u0, u0, l0)) + ex2_approx(fmaf(-u1, u1, l1));
            }
            c0 = n0; c1 = n1;
            l0 = m0; l1 = m1;
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&S->cs_empty[buf]);
      }
      // ---- end of pair: S_ik = sum over the 8 warps, log, mask, per-kernel sums, score ----
      if (qp < 32) {   // warp-uniform: add the sub-streams; afterwards every lane holds the total of its query row
#pragma unroll
        for (int k = 0; k < KB; ++k) {
          float v = acc[k];
          for (int o = qp; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          acc[k] = lane < qp ? v : 0.f;
        }
      }
#pragma unroll
      for (int k = 0; k < KB; ++k) spart[(ew * KB + k) * 32 + lane] = acc[k];
      if (ew == 0) S->qm[lane] = (lane < P.Lq && mask_test(qraw, qmt)) ? 1.f : 0.f;   // qraw = 0 for lanes >= Lq
      named_bar_sync(2, kEpiThreads);
      {
        const bool q_live = S->qm[lane] != 0.f;
        for (int k = ew; k < KB; k += 8) {  // warp = kernel, lane = query term
          float Ssum = 0.f;
#pragma unroll
          for (int w8 = 0; w8 < 8; ++w8) Ssum += spart[(w8 * KB + k) * 32 + lane];
          float L = 0.f;
          if (k < P.K && lane < P.Lq) {
            if (P.per_kernel_query) P.per_kernel_query[(p * P.Lq_total + P.q_row0 + lane) * (int64_t)P.K + k] = Ssum;
            if (q_live) L = P.log_scale * logf(fmaxf(Ssum * S->alpha[k], P.clamp_min));
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) L += __shfl_xor_sync(0xffffffffu, L, o);
          if (lane == 0) S->pk[k] = L;
        }
      }
      named_bar_sync(4, kEpiThreads);
      if (ew == 7) {  // Linear(K, 1): lane = kernel (K <= 32; w is 0 beyond K)
        const float v = lane < P.K ? S->pk[lane] : 0.f;
        if (lane < P.K && P.per_kernel) P.per_kernel[p * P.K + lane] = v;
        float sc = v * S->w[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
        // store mode: a pair without rows (pair_d < 0 or an empty passage) scores -inf
        if (lane == 0) P.score[p] = STORE && len == 0 ? -INFINITY : sc + P.bias;
      }
    }
  }
}

template <int KB, bool SAVE>
__global__ void __launch_bounds__(kThreads, 1)
kernel_pool_ts_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                      const __grid_constant__ CUtensorMap tmap_d_last, KpParams P, int n_raw, int last_box_rows) {
  kernel_pool_ts_body<KB, SAVE, false>(tmap_q, tmap_d, tmap_d_last, P, n_raw, last_box_rows);
}

// store mode (mmb200_kernel_pool_store_fwd): tmap_d / tmap_d_last are 32- / 8-row boxes over the whole store
template <int KB>
__global__ void __launch_bounds__(kThreads, 1)
kernel_pool_ts_store_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                            const __grid_constant__ CUtensorMap tmap_d_last, KpParams P, int n_raw) {
  kernel_pool_ts_body<KB, false, true>(tmap_q, tmap_d, tmap_d_last, P, n_raw, 0);
}

template <int KB>
int launch(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream, const CUtensorMap& tq, const CUtensorMap& td,
           const CUtensorMap& td_last, int last_box_rows) {
  static_assert(KB <= 32, "end-of-pair scratch holds 32 kernels");
  const size_t fixed = (size_t)(2 * 128 * 32 + 8 * 32 * 32) * sizeof(float) + sizeof(KpShared) + 1024 + (size_t)kOps * kQ64Bytes;
  const int n_raw = std::min<int>(kMaxRaw, (int)(((size_t)dev.max_smem_optin - fixed) / kRawBytes));
  const size_t smem = fixed + (size_t)n_raw * kRawBytes;
  if (n_raw < 2 || smem > (size_t)dev.max_smem_optin) {
    set_error("kernel_pool tensor-core forward: shared-memory plan does not fit");
    return MMB200_ERR_UNSUPPORTED;
  }
  const int grid = (int)std::min<int64_t>(dev.sm_count, P.B);
  if (P.saved) {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_ts_kernel<KB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel_pool_ts_kernel<KB, true><<<grid, kThreads, smem, stream>>>(tq, td, td_last, P, n_raw, last_box_rows);
  } else if (P.doc_offsets) {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_ts_store_kernel<KB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel_pool_ts_store_kernel<KB><<<grid, kThreads, smem, stream>>>(tq, td, td_last, P, n_raw);
  } else {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_ts_kernel<KB, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel_pool_ts_kernel<KB, false><<<grid, kThreads, smem, stream>>>(tq, td, td_last, P, n_raw, last_box_rows);
  }
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

// score[b] = sum over query blocks + bias, per_kernel[b, k] = sum over query blocks (fixed order: deterministic)
__global__ void kp_combine_query_blocks(const float* __restrict__ score_blk, const float* __restrict__ pk_blk, int nblk, int64_t B,
                                        int K, float bias, float* __restrict__ score, float* __restrict__ per_kernel) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < B) {
    float s = 0.f;
    for (int x = 0; x < nblk; ++x) s += score_blk[x * B + i];
    score[i] = s + bias;
  }
  if (per_kernel && i < B * K) {
    float s = 0.f;
    for (int x = 0; x < nblk; ++x) s += pk_blk[x * B * K + i];
    per_kernel[i] = s;
  }
}

static int kernel_pool_fwd_ts_block(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream) {
  CUtensorMap tq, td, td_last;
  {
    const uint64_t dims[3] = {(uint64_t)P.D, (uint64_t)P.Lq_total, (uint64_t)(P.doc_offsets ? P.n_q : P.B)};
    const uint64_t strides[2] = {(uint64_t)P.D * 4, (uint64_t)P.Lq_total * P.D * 4};
    const uint32_t box[3] = {32, 32, 1};
    if (int rc = encode_tensor_map(&tq, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.q, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))
      return rc;
  }
  const int last_rows = P.Ld - ((P.Ld + 127) / 128 - 1) * 128;       // rows of the last document tile, 1..128
  const int last_box_rows = std::min(128, (last_rows + 7) & ~7);
  if (P.doc_offsets) {
    // store mode: one map over the whole store, row coordinate = the passage's first row + the tile's; each tile is
    // fetched as 32-row boxes (td) and then 8-row boxes (td_last), so at most 7 rows past a passage are read
    const uint64_t dims[3] = {(uint64_t)P.D, (uint64_t)P.n_rows, 1};
    const uint64_t strides[2] = {(uint64_t)P.D * 4, (uint64_t)P.n_rows * P.D * 4};
    const uint32_t box[3] = {32, 32, 1}, box8[3] = {32, 8, 1};
    if (int rc = encode_tensor_map(&td, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.d, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
    if (int rc = encode_tensor_map(&td_last, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.d, dims, strides, box8,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  } else {
    const uint64_t dims[3] = {(uint64_t)P.D, (uint64_t)P.Ld, (uint64_t)P.B};
    const uint64_t strides[2] = {(uint64_t)P.D * 4, (uint64_t)P.Ld * P.D * 4};
    const uint32_t box[3] = {32, 128, 1};
    if (int rc = encode_tensor_map(&td, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.d, dims, strides, box,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
    const uint32_t box_last[3] = {32, (uint32_t)last_box_rows, 1};
    if (int rc = encode_tensor_map(&td_last, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, P.d, dims, strides, box_last,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  // exact instantiations for the reference's kernel counts (KNRM: 11, TK / TKL: 11 or 21 -- no padded activations)
  if (P.K == 11) return launch<11>(P, dev, stream, tq, td, td_last, last_box_rows);
  if (P.K == 21) return launch<21>(P, dev, stream, tq, td, td_last, last_box_rows);
  if (P.K <= 12) return launch<12>(P, dev, stream, tq, td, td_last, last_box_rows);
  if (P.K <= 24) return launch<24>(P, dev, stream, tq, td, td_last, last_box_rows);
  return launch<32>(P, dev, stream, tq, td, td_last, last_box_rows);
}

}  // namespace

int kernel_pool_fwd_ts(const KpParams& P0, const DeviceInfo& dev, cudaStream_t stream, bool* handled) {
  *handled = false;
  constexpr int kMaxBlocks = 4;   // queries up to 128 terms
  if (P0.Lq > 32 * kMaxBlocks || P0.K > 32 || P0.cosine != nullptr || P0.D % 4 != 0) return MMB200_OK;
  if (P0.Lq > 32 && P0.saved != nullptr) return MMB200_OK;   // the saved-state layout holds 32 query rows
  KpParams P = P0;
  P.q_row0 = 0;
  P.Lq_total = P0.Lq;
  *handled = true;
  if (P0.Lq <= 32) return kernel_pool_fwd_ts_block(P, dev, stream);
  // Longer queries: one pass of the same kernel per block of 32 query rows (the document tiles are streamed once per
  // block -- still several times faster than the FFMA kernel), per-block scores and per-kernel sums added afterwards.
  const int nblk = (P0.Lq + 31) / 32;
  float* tmp = nullptr;
  const size_t n_tmp = (size_t)nblk * P0.B * (1 + P0.K);
  MMB_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&tmp), n_tmp * sizeof(float), stream));
  int rc = MMB200_OK;
  for (int x = 0; x < nblk && rc == MMB200_OK; ++x) {
    P.q_row0 = 32 * x;
    P.Lq = std::min(32, P0.Lq - 32 * x);
    P.score = tmp + (size_t)x * P0.B;
    P.per_kernel = tmp + (size_t)nblk * P0.B + (size_t)x * P0.B * P0.K;
    P.bias = 0.f;
    rc = kernel_pool_fwd_ts_block(P, dev, stream);
  }
  if (rc == MMB200_OK) {
    const int64_t n = std::max<int64_t>(P0.B * (P0.per_kernel ? P0.K : 1), P0.B);
    kp_combine_query_blocks<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(tmp, tmp + (size_t)nblk * P0.B, nblk, P0.B, P0.K, P0.bias,
                                                                              P0.score, P0.per_kernel);
    if (cudaGetLastError() != cudaSuccess) { set_error("kp_combine_query_blocks launch failed"); rc = MMB200_ERR_CUDA; }
  }
  MMB_CHECK_CUDA(cudaFreeAsync(tmp, stream));
  return rc;
}

}  // namespace mmb
