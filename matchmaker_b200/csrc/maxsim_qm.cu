// ColBERT max-sim, "queries on M" wgmma kernel: the hot path for Lq <= 32.
//
// Why this orientation: with documents on M (maxsim.cu) the max over document rows is a reduction across the rows of
// the accumulator, i.e. across threads.  Here the accumulator is transposed:
//
//     D[64 x TN] = Qrep[64 x dim] * Doc[TN x dim]^T        (one wgmma chain per document tile)
//
// row = query token, column = document row, so the max over a document is a per-thread FMNMX chain over the
// accumulator registers plus two quad shuffles.  Rows 0..31 of Qrep are the query; rows 32..63 of the instruction read
// whatever follows the query in shared memory and are never looked at.
//
// The document mask is applied in the epilogue as an fp32 penalty per document row, added to every query's score of
// that row: 0 for real tokens, -inf for padding and for the tile's rows past Ld, so masked rows can never win the max.
// The reference's -1000 fill (matchmaker/models/colbert.py:69) only matters when it IS the max; that is reproduced
// exactly by one "virtual" document row (the last row of the last tile, index >= Ld, zero data from TMA out-of-bounds
// fill) whose penalty is -1000 when the document has at least one masked position and -inf otherwise.  Two helper warps
// write the penalty row per document tile while TMA streams the token vectors.
//
// Nothing on a warp's per-document path waits for a global load: the per-pair indices and lengths arrive 32 pairs at a
// time, a batch ahead (PairStream; the consumers, which only need the query, keep just a batch of pair_q), and the
// penalty writers keep the mask words of their next two tiles in flight.  setmaxnreg moves registers from the helper
// warpgroup to the consumers, whose accumulators are the kernel's register peak.
//
// Per CTA (persistent, one per SM, 384 threads = 3 warpgroups):
//   warp 0        TMA producer: query tile (2-slot ring, re-fetched when the query changes), document tiles
//   warps 1, 2    penalty writers, warp 1 + c for consumer warpgroup c's documents
//   warpgroups 1, 2  consumers: warpgroup c takes the CTA's documents c, c + 2, ...; per tile 4 * dim / 64 * TN / 64
//                 wgmma m64n64k16 into registers, then the masked max over the tile in the same registers.  While one
//                 warpgroup reduces, the other one's MMAs run.  Each warpgroup has its own half of the stage ring, so
//                 every stage barrier has one consumer that waits for its phases in order.
// HBM-bound by design: per document one TMA box, one fp32 store.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "device_util.cuh"
#include "host_util.cuh"
#include "masks.cuh"
#include "maxsim.cuh"
#include "ptx.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 384;
constexpr int kMaxStages = 8;                // even: half of the ring per consumer warpgroup
constexpr int kQSlots = 2;
constexpr int kQRows = 32;
constexpr int kQBlockBytes = kQRows * 128;   // one k-block of the query tile (4 KB)
// setmaxnreg budgets: the helper warpgroup (producer, penalty writers) gives registers to the two consumer warpgroups, whose
// NCH x 32 accumulators are the kernel's register peak.  128 x 104 + 256 x 200 = 384 x 168 (the launch).
constexpr int kRegsHelper = 104, kRegsConsumer = 200;

struct QmShared {
  uint64_t full[kMaxStages];   // 2 arrivals: TMA producer (with tx bytes) + penalty writer
  uint64_t empty[kMaxStages];  // 4 arrivals: the warps of the warpgroup that owns the stage
  uint64_t qfull[kQSlots];
  uint64_t qempty[kQSlots];    // 8 arrivals: every warp of both consumer warpgroups
  float part[2][2];            // [consumer][pair parity]: row sum of query rows 16..31
};

struct QmLaunch {
  int32_t kblocks;      // dim / 64 (1 or 2)
  int32_t tn;           // document rows per tile (multiple of 64, <= 256)
  int32_t tiles;        // tiles per document; tiles * tn >= Ld + 1
  int32_t stages;       // even: stages [0, stages / 2) serve warpgroup 0, the rest warpgroup 1
  int32_t doc_bytes;    // kblocks * tn * 128
  int32_t stage_bytes;  // doc_bytes + penalty row (tn fp32, rounded to 1 KB)
};

// One warp's own sequence of pairs p = first, first + step, ... < end and what the warp needs of each: its query, its
// document, its document-mask row, and (ragged fetch, store mode) its first row and the rows worth fetching.  Lane l
// holds element l of a batch of 32.  A batch's index arrays are read with one coalesced load per array two batches
// ahead of use, store mode's doc_offsets of those documents one batch ahead, and elements are handed out by
// __shfl_sync: the warp never waits on a per-pair global load.  Every lane of the warp calls next() and the accessors
// together.
template <bool kStore>
struct PairStream {
  // Indices are int32 like the pair arrays of the C ABI; the implicit document index p (< n_pairs <= n_d) is one too:
  // it becomes the TMA box's int32 document coordinate, and the mask row index is widened to int64 before it is scaled.
  struct Batch {
    int32_t q, d, dm, rows;
    int64_t row0, row_end;   // store mode: [doc_offsets[d], doc_offsets[d + 1])
  };
  const MaxsimParams& P;
  int64_t first, end, step;
  int64_t pre_batch;   // batch index held in `pre`
  int k;               // current element of `cur` (-1 before the first next())
  int lane;
  Batch cur, nxt, pre;   // cur: resolved; nxt: second-level loads in flight; pre: first-level loads in flight

  __device__ __forceinline__ PairStream(const MaxsimParams& P_, int64_t first_, int64_t end_, int64_t step_, int lane_)
      : P(P_), first(first_), end(end_), step(step_), lane(lane_) {
    load1(cur, 0);
    load1(nxt, 1);
    load2(cur);
    load2(nxt);
    resolve(cur);
    pre_batch = 2;
    load1(pre, pre_batch);
    k = -1;
  }
  // indices: pair_q / pair_d / pair_dmask / rows_needed of this lane's pair
  __device__ __forceinline__ void load1(Batch& b, int64_t bi) {
    const int64_t p = first + (bi * 32 + lane) * step;
    b.q = 0; b.d = -1; b.dm = 0; b.rows = 0; b.row0 = 0; b.row_end = 0;
    if (p >= end) return;
    b.q = P.pair_q ? P.pair_q[p] : (int32_t)((p + P.pair_base) / P.docs_per_query);
    b.d = P.pair_d ? P.pair_d[p] : (int32_t)p;
    if (P.pair_dmask) b.dm = P.pair_dmask[p];
    if (!kStore && P.rows_needed) b.rows = P.rows_needed[p];   // ragged fetch has no pair_d: the document is p
  }
  // what depends on the indices (waits for load1's results)
  __device__ __forceinline__ void load2(Batch& b) {
    if (!P.pair_dmask) b.dm = b.d;
    if constexpr (kStore) {
      if (b.d >= 0) { b.row0 = P.doc_offsets[b.d]; b.row_end = P.doc_offsets[b.d + 1]; }
    }
  }
  __device__ __forceinline__ void resolve(Batch& b) {
    if constexpr (kStore) b.rows = (int)max((int64_t)0, min(b.row_end - b.row0, (int64_t)P.Ld));   // 0 for d < 0
  }
  // moves to the next pair of the sequence; the accessors below read the current one (a shuffle each: a role shuffles
  // only what it uses, so the loads of the rest are dead code)
  __device__ __forceinline__ void next() {
    if (++k == 32) {   // the loads waited for here were issued one batch ago
      cur = nxt;
      resolve(cur);
      nxt = pre;
      load2(nxt);
      load1(pre, ++pre_batch);
      k = 0;
    }
  }
  __device__ __forceinline__ int64_t q() const { return __shfl_sync(0xffffffffu, cur.q, k); }
  __device__ __forceinline__ int64_t d() const { return __shfl_sync(0xffffffffu, cur.d, k); }
  __device__ __forceinline__ int64_t dm() const { return __shfl_sync(0xffffffffu, cur.dm, k); }
  __device__ __forceinline__ int rows() const { return __shfl_sync(0xffffffffu, cur.rows, k); }
  __device__ __forceinline__ int64_t row0() const { return __shfl_sync(0xffffffffu, cur.row0, k); }
};

template <typename T>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc);
template <>
__device__ __forceinline__ void wgmma_n64<__half>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n64k16_f16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void wgmma_n64<__nv_bfloat16>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n64k16_bf16(d, a, b, acc);
}

// running maximum of (v, column) in column order; ties keep the first column
template <bool kArgmax>
__device__ __forceinline__ void take(float v, int col, float& m, int& am) {
  if constexpr (kArgmax) {
    const bool gt = v > m;
    m = gt ? v : m;
    am = gt ? col : am;
  } else {
    m = fmaxf(m, v);
  }
}

// kArgmax: the training instantiation also tracks WHICH document row won each query token's max (what backward needs,
// matchmaker/models/colbert.py:71 through autograd).  NCH = tn / 64 accumulator chunks of 32 registers.
// kStore: store mode (P.doc_offsets != NULL) -- a template parameter so that the padded instantiations compile as before.
template <typename T, int NCH, bool kArgmax, bool kStore>
__global__ void __launch_bounds__(kThreads, 1)
maxsim_qm_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_d,
                 const __grid_constant__ CUtensorMap tmap_d16, MaxsimParams P, QmLaunch L) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for SWIZZLE_128B tiles, derived by pointer arithmetic on the __shared__ array so the
  // compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int qslot_bytes = L.kblocks * kQBlockBytes;
  uint8_t* q_base = smem;                                            // [kQSlots][kblocks][32 rows][128 B]
  uint8_t* stage_base = q_base + kQSlots * qslot_bytes;              // [stages][doc tile | penalty row]
  QmShared* S = reinterpret_cast<QmShared*>(stage_base + (size_t)L.stages * L.stage_bytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  int64_t p_begin, p_end;
  cta_share(P.n_pairs, &p_begin, &p_end);

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmap_q);
    prefetch_tensormap(&tmap_d);
    for (int s = 0; s < L.stages; ++s) { mbar_init(&S->full[s], 2); mbar_init(&S->empty[s], 4); }
    for (int s = 0; s < kQSlots; ++s) { mbar_init(&S->qfull[s], 1); mbar_init(&S->qempty[s], 8); }
    fence_barrier_init();
  }
  if (P.rows_needed || kStore) {
    // ragged fetch (and store mode) leaves rows of a stage untouched: start from zeros so that stale rows are always
    // finite and the virtual row (index >= Ld, only ever written by TMA zero fill) is zero
    for (int s = 0; s < L.stages; ++s) {
      uint4* z = reinterpret_cast<uint4*>(stage_base + (size_t)s * L.stage_bytes);
      for (int e = threadIdx.x; e < L.doc_bytes / 16; e += kThreads) z[e] = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async_smem();
  }
  __syncthreads();

  // every role branch starts with its setmaxnreg so that ptxas allocates each branch against its own budget
  if (warp == 0) {
    setmaxnreg_dec<kRegsHelper>();
    // ------------------------------- TMA producer -------------------------------
    // the whole warp walks the pairs (it shares out their metadata); lane 0 waits on the barriers and issues the TMA
    PairStream<kStore> meta(P, p_begin, p_end, 1, lane);
    const int ring = L.stages >> 1;
    int64_t seq0 = 0, seq1 = 0;   // tiles filled so far into each warpgroup's half of the ring
    int64_t prev_q = -1;
    uint32_t qcount = 0;
    for (int64_t p = p_begin; p < p_end; ++p) {
      meta.next();
      const int64_t qi = meta.q();
      const int64_t di = meta.d();
      // store mode: the passage's rows start at row `row0` of the [n_rows, dim] store (tensor-map dim 3 has extent 1)
      const int64_t row0 = kStore ? meta.row0() : 0;
      const int need_rows = meta.rows();
      if (lane == 0) {
        if (qi != prev_q) {
          const uint32_t slot = qcount & 1u, use = qcount >> 1;
          mbar_wait(&S->qempty[slot], (use & 1u) ^ 1u);
          mbar_arrive_expect_tx(&S->qfull[slot], (uint32_t)(L.kblocks * kQBlockBytes));
          for (int kb = 0; kb < L.kblocks; ++kb)
            tma_load_4d(&tmap_q, q_base + (size_t)slot * qslot_bytes + kb * kQBlockBytes, &S->qfull[slot], 0, 0, kb, (int)qi,
                        kEvictLast);
          ++qcount;
          prev_q = qi;
        }
        const int dcoord = kStore ? 0 : (int)di;
        const int c = (int)((p - p_begin) & 1);
        for (int t = 0; t < L.tiles; ++t) {
          const int64_t j = c ? seq1++ : seq0++;
          const int stage = c * ring + (int)(j % ring);
          const uint32_t phase = (uint32_t)((j / ring) & 1);
          mbar_wait(&S->empty[stage], phase ^ 1u);
          uint8_t* dst = stage_base + (size_t)stage * L.stage_bytes;
          if (!P.rows_needed && !kStore) {
            mbar_arrive_expect_tx(&S->full[stage], (uint32_t)L.doc_bytes);
            tma_load_4d(&tmap_d, dst, &S->full[stage], 0, t * L.tn, 0, (int)di, kEvictFirst);
          } else {
            // 16-row blocks up to the document's last unmasked row (store mode: its last row); the rest of the stage
            // keeps stale (finite) rows, which the penalty row masks with -inf
            const int rows_here = min(max(need_rows - t * L.tn, 0), L.tn);
            const int nb = (rows_here + 15) >> 4;
            if (nb == 0) {
              mbar_arrive(&S->full[stage]);
            } else {
              mbar_arrive_expect_tx(&S->full[stage], (uint32_t)(nb * L.kblocks * 2048));
              for (int kb = 0; kb < L.kblocks; ++kb)
                for (int b16 = 0; b16 < nb; ++b16)
                  tma_load_4d(&tmap_d16, dst + kb * L.tn * 128 + b16 * 2048, &S->full[stage], 0,
                              (int)row0 + t * L.tn + b16 * 16, kb, dcoord, kEvictFirst);
            }
          }
        }
      }
      __syncwarp();
    }
  } else if (warp == 1 || warp == 2) {
    setmaxnreg_dec<kRegsHelper>();
    // ------------------------------- penalty writers -----------------------------
    // writer c fills the penalty rows of consumer warpgroup c's half of the ring (pairs p_begin + c, + 2, ...), so every
    // stage has one writer that sees its uses in order (a second writer could pass a parity wait one phase early).  The
    // mask words of the writer's next two tiles (four documents of the CTA at one tile per document) are in flight in
    // two register sets that take turns; a copy between them would wait for the load.
    constexpr int kW = 2 * NCH;          // rows of a tile per lane (TN = 64 NCH)
    const int c = warp - 1;
    const int dmt = P.d_mask ? P.mask_dtype : MMB200_MASK_NONE;
    const int ring = L.stages >> 1;
    PairStream<kStore> meta(P, p_begin + c, p_end, 2, lane);
    int64_t seq = 0;                    // tiles written into this half of the ring
    int64_t wp = p_begin + c;           // pair and tile being written
    int wt = 0;
    bool any_masked = false;
    int64_t fp = wp;                    // pair and tile being fetched
    int ft = 0;
    int64_t f_dm = 0;                   // mask row and row limit of pair fp
    int f_lim = 0;
    auto fetch = [&](uint64_t (&raw)[kW], int& lim) {
      if (fp < p_end && ft == 0) {
        meta.next();
        f_dm = meta.dm();
        f_lim = kStore ? meta.rows() : P.Ld;   // store mode: the passage's length, 0 for a skipped pair
      }
#pragma unroll
      for (int k = 0; k < kW; ++k) {
        const int r = lane + 32 * k, g = ft * L.tn + r;
        raw[k] = 1;
        if (dmt != MMB200_MASK_NONE && fp < p_end && r < L.tn && g < P.Ld)
          raw[k] = mask_raw(P.d_mask, dmt, f_dm * (int64_t)P.Ld + g);
      }
      lim = f_lim;
      if (++ft == L.tiles) { ft = 0; fp += 2; }
    };
    auto write = [&](const uint64_t (&raw)[kW], int lim) {
      float pen[kW];
      bool masked_here = false;
#pragma unroll
      for (int k = 0; k < kW; ++k) {
        const int r = lane + 32 * k, g = wt * L.tn + r;
        const bool in_doc = r < L.tn && g < lim;
        const bool ok = in_doc && mask_test(raw[k], dmt);
        masked_here |= in_doc && !ok;
        pen[k] = ok ? 0.f : -INFINITY;
      }
      any_masked |= __any_sync(0xffffffffu, masked_here);
      const int stage = c * ring + (int)(seq % ring);
      const uint32_t phase = (uint32_t)((seq / ring) & 1);
      ++seq;
      mbar_wait(&S->empty[stage], phase ^ 1u);
      float* pt = reinterpret_cast<float*>(stage_base + (size_t)stage * L.stage_bytes + L.doc_bytes);
#pragma unroll
      for (int k = 0; k < kW; ++k) {
        const int r = lane + 32 * k, g = wt * L.tn + r;
        // the virtual -1000 row exists only in the masked (padded) layout
        if (r < L.tn) pt[r] = (!kStore && g == L.tiles * L.tn - 1) ? (any_masked ? -1000.f : -INFINITY) : pen[k];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&S->full[stage]);
      if (++wt == L.tiles) { wt = 0; wp += 2; any_masked = false; }
    };
    uint64_t ra[kW], rb[kW];
    int la, lb;
    fetch(ra, la);
    fetch(rb, lb);
    while (wp < p_end) {
      write(ra, la);
      fetch(ra, la);
      if (wp >= p_end) break;
      write(rb, lb);
      fetch(rb, lb);
    }
  } else if (warp == 3) {
    setmaxnreg_dec<kRegsHelper>();   // idle: its registers go to the consumers
  } else {
    setmaxnreg_inc<kRegsConsumer>();
    // ------------------------------- consumers: wgmma + masked max ------------------------
    const int c = (warp >> 2) - 1;        // consumer warpgroup 0 / 1
    const int wq = warp & 3;              // warp inside the warpgroup: rows 16 wq .. 16 wq + 15
    const int r0 = 16 * wq + (lane >> 2), r1 = r0 + 8;   // this thread's query rows (< 32 for wq < 2)
    const int cq = 2 * (lane & 3);        // this thread's first column inside an 8-column group
    const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
    const int ring = L.stages >> 1;
    int64_t seq = 0;   // tiles consumed from this warpgroup's half of the ring
    int64_t prev_q = -1;
    uint32_t qcount = 0;
    int cur_slot = 0;
    // pair_q mode: pair_q of this lane's pair in the current and the next batch of 32 pairs (one coalesced load per batch,
    // a batch ahead of use); the consumers need nothing else per pair, so they carry no PairStream (register budget)
    auto load_q = [&](int64_t n0) -> int32_t { return p_begin + n0 + lane < p_end ? P.pair_q[p_begin + n0 + lane] : 0; };
    int32_t qb_cur = 0, qb_nxt = 0;
    if (P.pair_q) { qb_cur = load_q(0); qb_nxt = load_q(32); }
    for (int64_t n = 0; p_begin + n < p_end; ++n) {
      const int64_t p = p_begin + n;
      int64_t qi;
      if (P.pair_q) {
        if ((n & 31) == 0 && n > 0) { qb_cur = qb_nxt; qb_nxt = load_q(n + 32); }
        qi = __shfl_sync(0xffffffffu, qb_cur, (int)(n & 31));
      } else {
        qi = (p + P.pair_base) / P.docs_per_query;
      }
      if (qi != prev_q) {
        // every MMA of this warpgroup that read the old query tile has completed (wgmma_wait below)
        if (prev_q >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&S->qempty[cur_slot]); }
        cur_slot = (int)(qcount & 1u);
        mbar_wait(&S->qfull[cur_slot], (qcount >> 1) & 1u);
        ++qcount;
        prev_q = qi;
      }
      if ((int)(n & 1) != c) continue;
      const uint32_t qaddr = smem_u32(q_base + (size_t)cur_slot * qslot_bytes);
      // query-mask words: first needed in the epilogue, after this document's MMAs (L1 hits after the query's first pair)
      uint64_t qraw0 = 0, qraw1 = 0;
      if (wq < 2) {
        if (r0 < P.Lq) qraw0 = (qmt != MMB200_MASK_NONE) ? mask_raw(P.q_mask, qmt, qi * (int64_t)P.Lq + r0) : 1;
        if (r1 < P.Lq) qraw1 = (qmt != MMB200_MASK_NONE) ? mask_raw(P.q_mask, qmt, qi * (int64_t)P.Lq + r1) : 1;
      }
      float m0 = -INFINITY, m1 = -INFINITY;
      int a0 = -1, a1 = -1;   // row of the running maximum (first one on ties); stays -1 when nothing beats -inf
      for (int t = 0; t < L.tiles; ++t) {
        const int stage = c * ring + (int)(seq % ring);
        mbar_wait(&S->full[stage], (uint32_t)((seq / ring) & 1));
        ++seq;
        const uint32_t daddr = smem_u32(stage_base + (size_t)stage * L.stage_bytes);
        float acc[NCH][32];   // the first K-step overwrites (scale-d = 0): no zeroing inside the wgmma pipeline
        wgmma_fence();
        for (int kb = 0; kb < L.kblocks; ++kb) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t adesc = make_wgmma_sw128_desc(qaddr + kb * kQBlockBytes + k * 32);
#pragma unroll
            for (int h = 0; h < NCH; ++h)
              wgmma_n64<T>(acc[h], adesc, make_wgmma_sw128_desc(daddr + kb * L.tn * 128 + h * 64 * 128 + k * 32), (kb | k) != 0);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < NCH; ++h) wgmma_fence_regs(acc[h]);
        if (wq < 2) {
          const float* pen = reinterpret_cast<const float*>(stage_base + (size_t)stage * L.stage_bytes + L.doc_bytes);
#pragma unroll
          for (int h = 0; h < NCH; ++h) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int col = h * 64 + 8 * j + cq;
              const float2 pv = *reinterpret_cast<const float2*>(pen + col);
              const int gcol = t * L.tn + col;
              take<kArgmax>(acc[h][4 * j + 0] + pv.x, gcol, m0, a0);
              take<kArgmax>(acc[h][4 * j + 1] + pv.y, gcol + 1, m0, a0);
              take<kArgmax>(acc[h][4 * j + 2] + pv.x, gcol, m1, a1);
              take<kArgmax>(acc[h][4 * j + 3] + pv.y, gcol + 1, m1, a1);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&S->empty[stage]);
      }
      if (wq < 2) {
        // the four threads of a quad hold the same two rows: combine (larger value, then first column)
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float om0 = __shfl_xor_sync(0xffffffffu, m0, o), om1 = __shfl_xor_sync(0xffffffffu, m1, o);
          if constexpr (kArgmax) {
            const int oa0 = __shfl_xor_sync(0xffffffffu, a0, o), oa1 = __shfl_xor_sync(0xffffffffu, a1, o);
            if (om0 > m0 || (om0 == m0 && (unsigned)oa0 < (unsigned)a0)) { m0 = om0; a0 = oa0; }
            if (om1 > m1 || (om1 == m1 && (unsigned)oa1 < (unsigned)a1)) { m1 = om1; a1 = oa1; }
          } else {
            m0 = fmaxf(m0, om0);
            m1 = fmaxf(m1, om1);
          }
        }
        const bool ok0 = mask_test(qraw0, qmt), ok1 = mask_test(qraw1, qmt);   // qraw = 0 for rows >= Lq
        if constexpr (kArgmax) {
          // rows >= Ld are the -inf padding and the virtual -1000 row: a max taken there carries no gradient (-1), like a
          // masked query token
          if ((lane & 3) == 0) {
            if (r0 < P.Lq) P.argmax[p * (int64_t)P.Lq + r0] = (ok0 && a0 < P.Ld) ? a0 : -1;
            if (r1 < P.Lq) P.argmax[p * (int64_t)P.Lq + r1] = (ok1 && a1 < P.Ld) ? a1 : -1;
          }
        }
        float total = (lane & 3) == 0 ? (ok0 ? m0 : 0.f) + (ok1 ? m1 : 0.f) : 0.f;
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
        const int buf = (int)((n >> 1) & 1);
        if (wq == 1 && lane == 0) S->part[c][buf] = total;
        named_bar_sync(1 + c, 64);
        if (wq == 0 && lane == 0) P.out[p] = total + S->part[c][buf];
      }
    }
  }
}

template <typename T, bool kArgmax, bool kStore>
int launch_qm(int nch, int grid, size_t smem_bytes, cudaStream_t stream, const CUtensorMap& tq, const CUtensorMap& td,
              const CUtensorMap& td16, const MaxsimParams& P, const QmLaunch& L) {
#define MMB_QM_CASE(N)                                                                                                  \
  case N:                                                                                                               \
    MMB_CHECK_CUDA(cudaFuncSetAttribute(maxsim_qm_kernel<T, N, kArgmax, kStore>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                        (int)smem_bytes));                                                              \
    maxsim_qm_kernel<T, N, kArgmax, kStore><<<grid, kThreads, smem_bytes, stream>>>(tq, td, td16, P, L);                \
    break;
  switch (nch) {
    MMB_QM_CASE(1)
    MMB_QM_CASE(2)
    MMB_QM_CASE(3)
    MMB_QM_CASE(4)
    default:
      set_error("maxsim queries-on-M: tile width out of range");
      return MMB200_ERR_INVALID;
  }
#undef MMB_QM_CASE
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

}  // namespace

// rows_needed[di] = 1 + last unmasked row (one warp per document)
__global__ void __launch_bounds__(256) rows_needed_kernel(const void* __restrict__ d_mask, int mask_dtype,
                                                          int32_t* __restrict__ rows_needed, int64_t n_d, int Ld) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= n_d) return;
  int last = 0;
  if (!d_mask) last = Ld;
  else
    for (int j = lane; j < Ld; j += 32)
      if (mask_at(d_mask, mask_dtype, w * Ld + j)) last = j + 1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  if (lane == 0) rows_needed[w] = last;
}

int maxsim_rows_needed_launch(const void* d_mask, int mask_dtype, int32_t* rows_needed, int64_t n_d, int Ld,
                              cudaStream_t stream) {
  if (n_d == 0) return MMB200_OK;
  rows_needed_kernel<<<(unsigned)((n_d + 7) / 8), 256, 0, stream>>>(d_mask, d_mask ? mask_dtype : MMB200_MASK_NONE, rows_needed, n_d, Ld);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

// Returns MMB200_OK with *handled = false when the shape is outside this kernel's envelope.
int maxsim_qm_launch(const MaxsimParams& P, int dtype, const DeviceInfo& dev, cudaStream_t stream, bool* handled) {
  *handled = false;
  if (dtype != MMB200_F16 && dtype != MMB200_BF16) return MMB200_OK;
  if (P.Lq > kQRows || (P.dim != 64 && P.dim != 128)) return MMB200_OK;
  if (P.rows_needed && (P.pair_d || P.pair_dmask)) return MMB200_OK;  // rows_needed is indexed by the implicit doc id
  if ((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d)) & 15) return MMB200_OK;
  QmLaunch L;
  L.kblocks = P.dim / 64;
  const int rows = P.Ld + (P.doc_offsets ? 0 : 1);  // + the virtual row that carries the reference's -1000 fill
  L.tiles = (rows + 255) / 256;
  L.tn = (((rows + L.tiles - 1) / L.tiles) + 63) / 64 * 64;
  L.doc_bytes = L.kblocks * L.tn * 128;
  L.stage_bytes = L.doc_bytes + (L.tn * 4 + 1023) / 1024 * 1024;
  const int fixed = kQSlots * L.kblocks * kQBlockBytes + (int)sizeof(QmShared) + 1024;
  L.stages = std::min(kMaxStages, (dev.max_smem_optin - fixed) / L.stage_bytes) & ~1;
  if (L.stages < 2) return MMB200_OK;
  const size_t smem_bytes = (size_t)L.stages * L.stage_bytes + fixed;

  const CUtensorMapDataType tdt = dtype == MMB200_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  CUtensorMap tq, td;
  {
    const uint64_t dims[4] = {64, (uint64_t)P.Lq, (uint64_t)L.kblocks, (uint64_t)P.n_q};
    const uint64_t strides[3] = {(uint64_t)P.dim * 2, 128, (uint64_t)P.Lq * P.dim * 2};
    const uint32_t box[4] = {64, (uint32_t)kQRows, 1, 1};
    if (int rc = encode_tensor_map(&tq, tdt, 4, P.q, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B))
      return rc;
  }
  // documents: [n_d][Ld rows][kblocks][64], or in store mode the [n_rows][kblocks][64] store as one "document" whose
  // row coordinate is the passage's first row (rows past n_rows are zero-filled by TMA)
  const uint64_t d_rows = P.doc_offsets ? (uint64_t)P.n_rows : (uint64_t)P.Ld;
  const uint64_t d_count = P.doc_offsets ? 1 : (uint64_t)P.n_d;
  {
    const uint64_t dims[4] = {64, d_rows, (uint64_t)L.kblocks, d_count};
    const uint64_t strides[3] = {(uint64_t)P.dim * 2, 128, d_rows * P.dim * 2};
    const uint32_t box[4] = {64, (uint32_t)L.tn, (uint32_t)L.kblocks, 1};
    if (int rc = encode_tensor_map(&td, tdt, 4, P.d, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  CUtensorMap td16;
  {
    const uint64_t dims[4] = {64, d_rows, (uint64_t)L.kblocks, d_count};
    const uint64_t strides[3] = {(uint64_t)P.dim * 2, 128, d_rows * P.dim * 2};
    const uint32_t box[4] = {64, 16, 1, 1};
    if (int rc = encode_tensor_map(&td16, tdt, 4, P.d, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
  }
  *handled = true;
  const int grid = (int)std::min<int64_t>(dev.sm_count, P.n_pairs);
  const int nch = L.tn / 64;
  if (P.doc_offsets) {   // store mode never asks for argmax
    if (P.argmax) { *handled = false; return MMB200_OK; }
    return dtype == MMB200_F16 ? launch_qm<__half, false, true>(nch, grid, smem_bytes, stream, tq, td, td16, P, L)
                               : launch_qm<__nv_bfloat16, false, true>(nch, grid, smem_bytes, stream, tq, td, td16, P, L);
  }
  if (dtype == MMB200_F16)
    return P.argmax ? launch_qm<__half, true, false>(nch, grid, smem_bytes, stream, tq, td, td16, P, L)
                    : launch_qm<__half, false, false>(nch, grid, smem_bytes, stream, tq, td, td16, P, L);
  return P.argmax ? launch_qm<__nv_bfloat16, true, false>(nch, grid, smem_bytes, stream, tq, td, td16, P, L)
                  : launch_qm<__nv_bfloat16, false, false>(nch, grid, smem_bytes, stream, tq, td, td16, P, L);
}

}  // namespace mmb
