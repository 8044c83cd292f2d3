// ColBERT max-sim, the headline wgmma kernel: the hot path for Lq <= 32.  ("qm", queries on M, is its historical name:
// the MMA once put the query on M and the documents on N.)
//
// Orientation: document rows on M, query tokens on N.  Per 64-row chunk of a document
//
//     D[64 x 32] = Chunk[64 x dim] * Q[32 x dim]^T        (4 * dim / 64 wgmma m64n32k16)
//
// A is the chunk in its stage, B the 32-row query tile: nothing is padded (N = 32 is Lq's ceiling), where a query on
// M = 64 wasted half of every instruction.  Thread (warp w, lane l) of a consumer warpgroup holds chunk rows
// 16 w + l / 4 and that + 8 for query tokens 8 j + 2 (l % 4) + {0, 1}, j < 4: 16 accumulators, 2 rows x 8 tokens.  The
// max over a document's rows crosses threads, so it is deferred: each thread keeps a running maximum per token over
// its rows of every chunk of the document (per chunk 2 penalties and 8 independent 2-deep chains, in every warp), and
// the rows meet once per document, after its last chunk: shuffles over lane bits 2..4, then the four warps through
// shared memory, where warp 0 finishes the document while warps 1-3 go on to the next one.
//
// Only live rows are fetched.  A document's live rows are [0, live) with live = 1 + its last unmasked row (Ld without a
// mask; the passage's length in store mode); it takes nch = max(1, ceil(live / 64)) chunks of the stage ring.  In the
// padded layout the chunks are END-aligned: chunk ch starts at row live - 64 (nch - ch), so the first one may start
// below row 0, where TMA zero-fills without reading HBM, and no padding row is read.  A first chunk whose lower half
// lies wholly below row 0 loads only its upper half (a 32-row box per k-block): skipping the zero fill measured
// faster.  Store mode stays start-aligned
// (below a passage's first row lie the previous passage's rows), so its last chunk holds rows past `live`.  A document
// with no live row takes one chunk that is not fetched (the stage holds whatever it held before).  The mask is applied
// in the reduction as an fp32 penalty per row, 0 for live unmasked rows and -inf for every other row (rows below 0
// included), so no such row can win the max whatever its data.  The reference's -1000 fill (matchmaker/models/colbert.py:69) only
// matters when it IS the max; it is one more candidate taken after the whole document, value -1000 at row Ld (so ties
// go to real rows and the argmax reports -1), when the document has a masked position anywhere in its Ld rows --
// live < Ld, or a hole before its last live row.
//
// Everything a document's chunks need from its mask is summed up in a per-document RECORD in shared memory, written by
// scout warps up to a ring's depth of documents ahead: the live-row count, the fill flag and one bit per row (1 = live
// and unmasked).  The producer takes the chunk count from it and the consumers take the penalty of every row from its
// bits, so the mask loads' latency sits entirely in the scouts, which wait on nothing but a free record slot.  Nothing
// on a warp's per-document path waits for a global load: the per-pair indices and lengths arrive 32 pairs at a time, a
// batch ahead (PairStream; the consumers, which only need the query, keep just a batch of pair_q).  setmaxnreg moves
// registers from the helper warpgroup to the consumers.
//
// Per CTA (persistent, one per SM, 384 threads = 3 warpgroups):
//   warp 0        TMA producer: query tile (2-slot ring, re-fetched when the query changes), document chunks: one
//                 {64, 64 rows, dim / 64} box per chunk, or one 32-row box per k-block for the upper half of a first
//                 chunk whose lower half is below row 0 (rows below 0 and past Ld are zero-filled by TMA and cost no HBM
//                 traffic), issued by one elected lane of the converged warp
//   warps 1-3     mask scouts: scout s takes the CTA's documents s, s + 3, ...; per document it ballots the mask words
//                 of its rows (keeping its next two documents' words in flight) and fills the document's record
//   warpgroups 1, 2  consumers: warpgroup c takes the CTA's documents c, c + 2, ...; per chunk 4 * dim / 64 wgmma
//                 m64n32k16 into registers, then the masked running maxima of the chunk's rows, and the stage goes
//                 back at once; per document one combine of the rows.  While one warpgroup reduces, the other one's
//                 MMAs run.  Each warpgroup has its own half of the stage ring, so every stage barrier has one consumer
//                 that waits for its phases in order.
// Record slot n % records holds the CTA's document n; the slot count is a multiple of 6, so every slot has one scout
// and one consumer warpgroup, and each of them (and the producer) passes through the slot's phases in order.
// HBM-bound by design: per chunk one TMA box, per document one fp32 store.
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
constexpr int kChunkRows = 64;
constexpr int kChunkKBlockBytes = kChunkRows * 128;   // one k-block of a chunk (8 KB)
constexpr int kMaxStages = 32;               // even: half of the ring per consumer warpgroup (12 at dim 128, 24 at dim 64)
constexpr int kMaxLd = 4096;
constexpr int kScouts = 3;                   // warps 1..3 (one scout falls behind the documents; two or three keep up)
constexpr int kRecordStep = 6;               // record slots come in multiples of kScouts and of the 2 consumer warpgroups
constexpr int kMaxRecords = 48;
constexpr int kRecordReserve = 12 * 1024;    // shared memory kept for records before the stage count is chosen
constexpr int kQSlots = 2;
constexpr int kQRows = 32;
constexpr int kQBlockBytes = kQRows * 128;   // one k-block of the query tile (4 KB)
// record word 0: live rows | kFill; word 1 unused (keeps the bit words 8-byte aligned); words 2, 3: zero, the bits of
// rows [-64, 0) (an end-aligned first chunk reads them: rows below 0 are never live); words 4 + 2 k, 5 + 2 k: the bits
// of rows [64 k, 64 k + 32) and [64 k + 32, 64 k + 64)
constexpr uint32_t kFill = 1u << 16, kLiveMask = kFill - 1;
constexpr int kRecBits = 4;   // first word of row 0's bits
// setmaxnreg budgets: the helper warpgroup (producer, scouts) gives registers to the two consumer warpgroups, whose
// accumulator, running maxima and epilogue are the kernel's register peak.  128 x 120 + 256 x 192 = 384 x 168 (the
// launch).
constexpr int kRegsHelper = 120, kRegsConsumer = 192;

// Debugging build only (-DMMB200_ENABLE_PROF, MMB200_MAXSIM_PROF=1): clock64 cycles of each role and of each of its
// waits, summed over the CTAs into g_qm_prof and printed by the host after the launch.  The product build compiles
// every QM_PROF statement out.
#ifdef MMB200_ENABLE_PROF
enum QmProf {
  kPrTotal, kPrQEmpty, kPrRFull, kPrEmpty, kPrTma, kPrChunks,                 // producer (warp 0, lane 0)
  kCoTotal, kCoRFull, kCoFull, kCoIssue, kCoMma, kCoReduce, kCoEpilogue, kCoDocs,   // consumers (lane 0 of warps 4, 8)
  kScTotal, kScREmpty,                                                        // scouts (lane 0 of warps 1..3)
  kProfCount
};
__device__ unsigned long long g_qm_prof[kProfCount];
#define QM_PROF(...) __VA_ARGS__
#else
#define QM_PROF(...)
#endif

struct QmShared {
  uint64_t full[kMaxStages];   // 1 arrival: TMA producer (with tx bytes)
  uint64_t empty[kMaxStages];  // 4 arrivals: the warps of the warpgroup that owns the stage
  uint64_t qfull[kQSlots];
  uint64_t qempty[kQSlots];    // 8 arrivals: every warp of both consumer warpgroups
  uint64_t rfull[kMaxRecords];    // 1 arrival: the scout that filled the record
  uint64_t rempty[kMaxRecords];   // 5 arrivals: the producer and the 4 warps of the consuming warpgroup
  // [consumer][document parity][warp][query token]: each warp's maxima over its rows of the document, and their rows
  float xm[2][2][4][32];
  int32_t xa[2][2][4][32];
};

struct QmLaunch {
  int32_t kblocks;      // dim / 64 (1 or 2)
  int32_t stages;       // even: stages [0, stages / 2) serve warpgroup 0, the rest warpgroup 1
  int32_t chunk_bytes;  // kblocks * 8 KB
  int32_t records;      // record slots, a multiple of kRecordStep
  int32_t rec_words;    // record stride: 4 + 2 * ceil(Ld / 64) words
};

// Slot and phase parity of one role's walk through the record ring: every step-th document from the role's first one.
struct RecCursor {
  int slot;
  uint32_t phase;
  __device__ __forceinline__ void advance(int step, int records) {
    slot += step;
    if (slot >= records) { slot -= records; phase ^= 1u; }
  }
};

// Tensor maps of the query tile and of the document chunks: {64, 64 rows, kblocks, 1} boxes, and {64, 32 rows, 1, 1}
// boxes for the upper half of one k-block of a padded first chunk whose lower half lies wholly below row 0.
struct QmMaps {
  CUtensorMap q;
  CUtensorMap d;
  CUtensorMap dh;
};

// One warp's own sequence of pairs p = first, first + step, ... < end and what the warp needs of each: its query, its
// document, its document-mask row, and (store mode) its first row and length.  Lane l holds element l of a batch of 32.
// A batch's index arrays are read with one coalesced load per array two batches ahead of use, store mode's doc_offsets
// of those documents one batch ahead, and elements are handed out by __shfl_sync: the warp never waits on a per-pair
// global load.  Every lane of the warp calls next() and the accessors together.
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
  // indices: pair_q / pair_d / pair_dmask of this lane's pair
  __device__ __forceinline__ void load1(Batch& b, int64_t bi) {
    const int64_t p = first + (bi * 32 + lane) * step;
    b.q = 0; b.d = -1; b.dm = 0; b.rows = 0; b.row0 = 0; b.row_end = 0;
    if (p >= end) return;
    b.q = P.pair_q ? P.pair_q[p] : (int32_t)((p + P.pair_base) / P.docs_per_query);
    b.d = P.pair_d ? P.pair_d[p] : (int32_t)p;
    if (P.pair_dmask) b.dm = P.pair_dmask[p];
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
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc);
template <>
__device__ __forceinline__ void wgmma_n32<__half>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n32k16_f16(d, a, b, acc);
}
template <>
__device__ __forceinline__ void wgmma_n32<__nv_bfloat16>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  wgmma_m64n32k16_bf16(d, a, b, acc);
}

// running maximum of (v, row) in row order; ties keep the first row
template <bool kArgmax>
__device__ __forceinline__ void take(float v, int row, float& m, int& am) {
  if constexpr (kArgmax) {
    const bool gt = v > m;
    m = gt ? v : m;
    am = gt ? row : am;
  } else {
    m = fmaxf(m, v);
  }
}

// kArgmax: the training instantiation also tracks WHICH document row won each query token's max (what backward needs,
// matchmaker/models/colbert.py:71 through autograd).
// kStore: store mode (P.doc_offsets != NULL) -- a template parameter so that the padded instantiations carry no
// doc_offsets loads.
template <typename T, bool kArgmax, bool kStore>
__global__ void __launch_bounds__(kThreads, 1)
maxsim_qm_kernel(const __grid_constant__ QmMaps M, MaxsimParams P, QmLaunch L) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-B alignment for SWIZZLE_128B tiles, derived by pointer arithmetic on the __shared__ array so the
  // compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int qslot_bytes = L.kblocks * kQBlockBytes;
  uint8_t* q_base = smem;                                            // [kQSlots][kblocks][32 rows][128 B]
  uint8_t* stage_base = q_base + kQSlots * qslot_bytes;              // [stages][chunk]
  uint32_t* rec_base = reinterpret_cast<uint32_t*>(stage_base + (size_t)L.stages * L.chunk_bytes);   // [records][rec_words]
  QmShared* S = reinterpret_cast<QmShared*>(rec_base + (size_t)L.records * L.rec_words);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  int64_t p_begin, p_end;
  cta_share(P.n_pairs, &p_begin, &p_end);

  if (threadIdx.x == 0) {
    prefetch_tensormap(&M.q);
    prefetch_tensormap(&M.d);
    if (!kStore) prefetch_tensormap(&M.dh);
    for (int s = 0; s < L.stages; ++s) { mbar_init(&S->full[s], 1); mbar_init(&S->empty[s], 4); }
    for (int s = 0; s < kQSlots; ++s) { mbar_init(&S->qfull[s], 1); mbar_init(&S->qempty[s], 8); }
    for (int r = 0; r < L.records; ++r) {
      mbar_init(&S->rfull[r], 1);
      mbar_init(&S->rempty[r], 5);
      rec_base[(size_t)r * L.rec_words + kRecBits - 2] = 0;
      rec_base[(size_t)r * L.rec_words + kRecBits - 1] = 0;
    }
    fence_barrier_init();
  }
  __syncthreads();

  // every role branch starts with its setmaxnreg so that ptxas allocates each branch against its own budget
  if (warp == 0) {
    setmaxnreg_dec<kRegsHelper>();
    // ------------------------------- TMA producer -------------------------------
    // The whole warp walks the pairs (it shares out their metadata) and waits on the barriers; one elected lane
    // arrives and issues the TMA, so every coordinate stays warp-uniform and the issue needs no per-lane loop.  Each
    // warpgroup's half of the stage ring is walked with a running stage index and phase (no division per chunk).
    PairStream<kStore> meta(P, p_begin, p_end, 1, lane);
    const int ring = L.stages >> 1;
    int st_cur = 0, st_oth = 0;            // next stage inside the half of the current / the other document's warpgroup
    uint32_t ph_cur = 0, ph_oth = 0;       // and its phase parity
    int64_t prev_q = -1;
    uint32_t qcount = 0;
    RecCursor rc{0, 0};
    QM_PROF(unsigned long long prof[kProfCount] = {}; const long long t_start = clock64(); long long t_;)
    for (int64_t p = p_begin; p < p_end; ++p) {
      meta.next();
      const int64_t qi = meta.q();
      const int64_t di = meta.d();
      // store mode: the passage's rows start at row `row0` of the [n_rows, dim] store (tensor-map dim 3 has extent 1)
      const int64_t row0 = kStore ? meta.row0() : 0;
      if (qi != prev_q) {
        const uint32_t slot = qcount & 1u, use = qcount >> 1;
        QM_PROF(t_ = clock64();)
        mbar_wait(&S->qempty[slot], (use & 1u) ^ 1u);
        QM_PROF(prof[kPrQEmpty] += clock64() - t_;)
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&S->qfull[slot], (uint32_t)(L.kblocks * kQBlockBytes));
          for (int kb = 0; kb < L.kblocks; ++kb)
            tma_load_4d(&M.q, q_base + (size_t)slot * qslot_bytes + kb * kQBlockBytes, &S->qfull[slot], 0, 0, kb, (int)qi,
                        kEvictLast);
        }
        __syncwarp();
        ++qcount;
        prev_q = qi;
      }
      const int c = (int)((p - p_begin) & 1);
      // live rows of this document, from its record (filled by its scout long before)
      QM_PROF(t_ = clock64();)
      mbar_wait(&S->rfull[rc.slot], rc.phase);
      QM_PROF(prof[kPrRFull] += clock64() - t_;)
      const int live = (int)(rec_base[(size_t)rc.slot * L.rec_words] & kLiveMask);
      __syncwarp();
      if (lane == 0) mbar_arrive(&S->rempty[rc.slot]);
      rc.advance(1, L.records);
      const int dcoord = kStore ? 0 : (int)di;
      const int nch = max(1, (live + kChunkRows - 1) / kChunkRows);
      // padded layout: the chunks are END-aligned, chunk ch starts at row live - 64 (nch - ch), so they cover exactly
      // [live - 64 nch, live); rows below 0 are outside the tensor map's row extent and TMA zero-fills them without
      // reading HBM.  Store mode stays start-aligned: a negative offset there would read the previous passage's rows.
      int row = kStore ? (int)row0 : live - kChunkRows * nch;
      for (int ch = 0; ch < nch; ++ch, row += kChunkRows) {
        const int stage = c * ring + st_cur;
        QM_PROF(t_ = clock64();)
        mbar_wait(&S->empty[stage], ph_cur ^ 1u);
        QM_PROF(prof[kPrEmpty] += clock64() - t_; t_ = clock64(); ++prof[kPrChunks];)
        if (elect_one_sync()) {
          uint8_t* dst = stage_base + (size_t)stage * L.chunk_bytes;
          if (live == 0) {
            mbar_arrive(&S->full[stage]);
          } else if (!kStore && row + kChunkRows / 2 <= 0) {
            // a first chunk with at most 32 rows at or above row 0: only the upper half of each k-block is loaded.
            // The lower half keeps whatever the stage held; those rows are below 0, so their penalty is -inf and no
            // value there (NaN and inf included) can win a max.
            mbar_arrive_expect_tx(&S->full[stage], (uint32_t)(L.chunk_bytes / 2));
            for (int kb = 0; kb < L.kblocks; ++kb)
              tma_load_4d(&M.dh, dst + kb * kChunkKBlockBytes + kChunkKBlockBytes / 2, &S->full[stage], 0,
                          row + kChunkRows / 2, kb, dcoord, kEvictFirst);
          } else {
            // one full box per chunk: the zero fill below row 0 and past Ld costs no HBM traffic, and short boxes
            // cost more TMA issues and handshakes than they save
            mbar_arrive_expect_tx(&S->full[stage], (uint32_t)L.chunk_bytes);
            tma_load_4d(&M.d, dst, &S->full[stage], 0, row, 0, dcoord, kEvictFirst);
          }
        }
        __syncwarp();
        QM_PROF(prof[kPrTma] += clock64() - t_;)
        if (++st_cur == ring) { st_cur = 0; ph_cur ^= 1u; }
      }
      // the next document belongs to the other warpgroup
      const int st = st_cur; st_cur = st_oth; st_oth = st;
      const uint32_t ph = ph_cur; ph_cur = ph_oth; ph_oth = ph;
    }
    QM_PROF(prof[kPrTotal] = clock64() - t_start;
            if (lane == 0) for (int i = kPrTotal; i <= kPrChunks; ++i) atomicAdd(&g_qm_prof[i], prof[i]);)
  } else if (warp <= kScouts) {
    setmaxnreg_dec<kRegsHelper>();
    // ------------------------------- mask scouts -----------------------------
    // scout s fills the records of the CTA's documents s, s + kScouts, ...  Per document: ballot the mask words of its
    // rows (lane l loads the words of rows l, l + 32, ...), which gives the row bits, the live count and the fill flag.
    // The first 256 rows' words of the scout's next two documents are in flight in registers while one is scanned, and
    // the only wait is for the document's record slot to come free.
    constexpr int kW = 8;                // mask words per lane prefetched: rows [0, 256) of a document
    const int s = warp - 1;
    const int dmt = P.d_mask ? P.mask_dtype : MMB200_MASK_NONE;
    const int nwin = (P.Ld + 32 * kW - 1) / (32 * kW);
    const int bit_words = L.rec_words - kRecBits;
    PairStream<kStore> meta(P, p_begin + s, p_end, kScouts, lane);
    RecCursor rc{s, 0};
    int64_t fp = p_begin + s;           // next pair whose mask words are loaded
    // mask words as loaded: nothing reads them before the document is scanned, so the loads stay in flight until then
    auto load_win = [&](uint64_t (&raw)[kW], int64_t dm, int w) {
#pragma unroll
      for (int k = 0; k < kW; ++k) {
        const int g = w * 32 * kW + 32 * k + lane;
        raw[k] = (dmt != MMB200_MASK_NONE && g < P.Ld) ? mask_raw(P.d_mask, dmt, dm * (int64_t)P.Ld + g) : 1;
      }
    };
    auto fetch = [&](uint64_t (&raw)[kW], int64_t& dm, int& lim) {
      if (fp < p_end) {
        meta.next();
        dm = meta.dm();
        lim = kStore ? meta.rows() : P.Ld;   // store mode: the passage's length, 0 for a skipped pair
        load_win(raw, dm, 0);
      }
      fp += kScouts;
    };
    // one document: wait for its record slot, scan its mask into the record, prefetch the scout's document after next
    // into `raw`, hand the record over
    QM_PROF(unsigned long long prof_re = 0; const long long t_start = clock64();)
    auto doc = [&](uint64_t (&raw)[kW], int64_t& dm, int& lim) {
      QM_PROF(const long long t_ = clock64();)
      mbar_wait(&S->rempty[rc.slot], rc.phase ^ 1u);
      QM_PROF(prof_re += clock64() - t_;)
      uint32_t* rec = rec_base + (size_t)rc.slot * L.rec_words;
      int live = 0;
      bool masked = false;
      for (int w = 0; w < nwin; ++w) {
        if (w > 0) load_win(raw, dm, w);   // documents longer than 256 rows: the later words are loaded here
#pragma unroll
        for (int k = 0; k < kW; ++k) {
          const int g = w * 32 * kW + 32 * k + lane;
          const bool in_doc = g < lim;
          const bool ok = in_doc && mask_test(raw[k], dmt);
          masked |= in_doc && !ok;
          const uint32_t b = __ballot_sync(0xffffffffu, ok);
          const int wi = w * kW + k;       // ballot word of rows [32 wi, 32 wi + 32)
          if (b) live = 32 * wi + 32 - __clz(b);
          if (lane == 0 && wi < bit_words) rec[kRecBits + wi] = b;
        }
      }
      // the reference fills every masked position with -1000, including the trailing ones that are never visited
      const bool fill = !kStore && __any_sync(0xffffffffu, masked);
      fetch(raw, dm, lim);
      if (lane == 0) {
        rec[0] = (uint32_t)live | (fill ? kFill : 0u);
        mbar_arrive(&S->rfull[rc.slot]);
      }
      rc.advance(kScouts, L.records);
    };
    uint64_t ra[kW], rb[kW];
    int64_t dma = 0, dmb = 0;
    int la = 0, lb = 0;
    fetch(ra, dma, la);
    fetch(rb, dmb, lb);
    for (int64_t sp = p_begin + s; sp < p_end;) {
      doc(ra, dma, la);
      if ((sp += kScouts) >= p_end) break;
      doc(rb, dmb, lb);
      sp += kScouts;
    }
    QM_PROF(if (lane == 0) {
      atomicAdd(&g_qm_prof[kScTotal], (unsigned long long)(clock64() - t_start));
      atomicAdd(&g_qm_prof[kScREmpty], prof_re);
    })
  } else {
    setmaxnreg_inc<kRegsConsumer>();
    // ------------------------------- consumers: wgmma + masked max ------------------------
    const int c = (warp >> 2) - 1;        // consumer warpgroup 0 / 1
    const int wq = warp & 3;              // warp inside the warpgroup: chunk rows 16 wq .. 16 wq + 15
    const int r0 = 16 * wq + (lane >> 2); // this thread's chunk rows: r0 and r0 + 8
    const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
    const int ring = L.stages >> 1;
    int64_t prev_q = -1;
    uint32_t qcount = 0;
    int cur_slot = 0;
    RecCursor rc{c, 0};   // records of this warpgroup's documents
    // pair_q mode: pair_q of this lane's pair in the current and the next batch of 32 pairs (one coalesced load per batch,
    // a batch ahead of use); the consumers need nothing else per pair, so they carry no PairStream (register budget)
    auto load_q = [&](int64_t n0) -> int32_t { return p_begin + n0 + lane < p_end ? P.pair_q[p_begin + n0 + lane] : 0; };
    int32_t qb_cur = 0, qb_nxt = 0;
    if (P.pair_q) { qb_cur = load_q(0); qb_nxt = load_q(32); }
    // implicit queries: (p + pair_base) / docs_per_query, divided once and then counted along
    int64_t q_run = 0;
    int32_t q_rem = 0;
    if (!P.pair_q) {
      q_run = (p_begin + P.pair_base) / P.docs_per_query;
      q_rem = (int32_t)((p_begin + P.pair_base) - q_run * P.docs_per_query);
    }
    QM_PROF(unsigned long long prof[kProfCount] = {}; const long long t_start = clock64(); long long t_;)
    // Query tiles: walks the CTA's pairs up to pair n (every warp of both warpgroups passes through every query change,
    // so each query slot's empty barrier gets its 8 arrivals in order).  A slot goes back after every MMA of this
    // warpgroup that read it has completed (each chunk's MMAs are waited for before it is reduced).
    int64_t n_walk = 0;
    auto walk_to = [&](int64_t n) {
      for (; n_walk <= n; ++n_walk) {
        int64_t qi;
        if (P.pair_q) {
          if ((n_walk & 31) == 0 && n_walk > 0) { qb_cur = qb_nxt; qb_nxt = load_q(n_walk + 32); }
          qi = __shfl_sync(0xffffffffu, qb_cur, (int)(n_walk & 31));
        } else {
          qi = q_run;
          if (++q_rem == P.docs_per_query) { q_rem = 0; ++q_run; }
        }
        if (qi != prev_q) {
          if (prev_q >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&S->qempty[cur_slot]); }
          cur_slot = (int)(qcount & 1u);
          mbar_wait(&S->qfull[cur_slot], (qcount >> 1) & 1u);
          ++qcount;
          prev_q = qi;
        }
      }
      return prev_q;
    };
    // what a document's chunks and epilogue need
    struct Doc {
      int64_t n;              // pair p_begin + n
      uint32_t qlo;           // low word of its query tile's B descriptor
      uint64_t qraw;          // warp 0: query-mask word of token `lane` (0 for tokens >= Lq)
      int slot;               // its record slot
      uint32_t head;          // record word 0
      int live, nch;
    };
    auto begin = [&](Doc& D, int64_t n) {
      const int64_t qi = walk_to(n);
      D.n = n;
      D.qlo = (uint32_t)make_wgmma_sw128_desc(smem_u32(q_base + (size_t)cur_slot * qslot_bytes));
      // query-mask word: first needed in warp 0's epilogue (L1 hits after the query's first pair)
      D.qraw = 0;
      if (wq == 0 && lane < P.Lq)
        D.qraw = (qmt != MMB200_MASK_NONE) ? mask_raw(P.q_mask, qmt, qi * (int64_t)P.Lq + lane) : 1;
      // the document's record: live rows, fill flag, row bits (filled by its scout long before)
      QM_PROF(t_ = clock64();)
      mbar_wait(&S->rfull[rc.slot], rc.phase);
      QM_PROF(prof[kCoRFull] += clock64() - t_; ++prof[kCoDocs];)
      D.slot = rc.slot;
      rc.advance(2, L.records);
      D.head = rec_base[(size_t)D.slot * L.rec_words];
      D.live = (int)(D.head & kLiveMask);
      D.nch = max(1, (D.live + kChunkRows - 1) / kChunkRows);
    };
    // waits for the next chunk of this warpgroup's ring and starts its MMAs, D[64 rows x 32 tokens] = Chunk * Q^T (the
    // first K-step overwrites: scale-d = 0); returns the stage.  A descriptor's high word is the same for every SW128
    // tile; its low word is built once, from a warp-uniform (shuffled) address so that it stays in a uniform register,
    // and stepped by immediates: +2 (32 B) per K-step, one k-block of the chunk / of the query tile per k-block.
    int st_next = 0;
    uint32_t ph_next = 0;
    constexpr uint64_t kDescHi = (uint64_t)(1024 >> 4) << 32 | (uint64_t)1 << 62;   // make_wgmma_sw128_desc's
    auto issue = [&](float (&acc)[16], uint32_t qlo_doc) -> int {
      const int stage = c * ring + st_next;
      QM_PROF(t_ = clock64();)
      mbar_wait(&S->full[stage], ph_next);
      QM_PROF(prof[kCoFull] += clock64() - t_; t_ = clock64();)
      if (++st_next == ring) { st_next = 0; ph_next ^= 1u; }
      const uint32_t daddr = smem_u32(stage_base + (size_t)stage * L.chunk_bytes);
      const uint32_t dlo = (uint32_t)make_wgmma_sw128_desc(__shfl_sync(0xffffffffu, daddr, 0));
      const uint32_t qlo = __shfl_sync(0xffffffffu, qlo_doc, 0);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_n32<T>(acc, kDescHi | (dlo + 2 * k), kDescHi | (qlo + 2 * k), k != 0);
      if (L.kblocks > 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_n32<T>(acc, kDescHi | (dlo + (kChunkKBlockBytes >> 4) + 2 * k),
                       kDescHi | (qlo + (kQBlockBytes >> 4) + 2 * k), 1);
      }
      wgmma_commit();
      wgmma_fence_regs(acc);
      QM_PROF(prof[kCoIssue] += clock64() - t_;)
      return stage;
    };
    // Running maxima of this thread's 8 query tokens 8 j + 2 (lane % 4) + {0, 1} (e = 2 j + {0, 1}) over the rows it
    // holds of every chunk of the document so far, and with kArgmax the row of each (the first one on ties: a thread
    // visits its rows in increasing order); -1 while nothing beats -inf.
    float mx[8];
    int ax[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { mx[e] = -INFINITY; ax[e] = -1; }
    // masked max over chunk ch of document D (finished MMAs in acc), then the stage goes back to the producer.  Row r
    // of the chunk is document row col0 + r: col0 = 64 ch in store mode, live - 64 (nch - ch) for the end-aligned padded
    // layout (only the first chunk can start below row 0, whose bits are the record's zero guard words).  The penalty
    // of a row is 0 for a live unmasked row and -inf otherwise, ADDED to the product (not a select), so that scores and
    // argmax are those of the full-tile kernel also for NaN / inf padding.
    auto reduce = [&](float (&acc)[16], int stage, const Doc& D, int ch) {
      wgmma_fence_regs(acc);
      const int col0 = kStore ? kChunkRows * ch : D.live - kChunkRows * (D.nch - ch);
      const int x0 = col0 + r0, x1 = x0 + 8;   // >= -64
      const uint32_t* bits = rec_base + (size_t)D.slot * L.rec_words + kRecBits;
      const float p0 = (bits[x0 >> 5] >> (x0 & 31)) & 1u ? 0.f : -INFINITY;
      const float p1 = (bits[x1 >> 5] >> (x1 & 31)) & 1u ? 0.f : -INFINITY;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int i = 4 * (e >> 1) + (e & 1);
        take<kArgmax>(acc[i] + p0, x0, mx[e], ax[e]);
        take<kArgmax>(acc[i + 2] + p1, x1, mx[e], ax[e]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&S->empty[stage]);
    };
    // (value, row) pairs: the larger value, then the first row (a row index -1 goes with -inf and loses every tie)
    auto combine = [&](float om, int oa, float& m, int& a) {
      if constexpr (kArgmax) {
        if (om > m || (om == m && (unsigned)oa < (unsigned)a)) { m = om; a = oa; }
      } else {
        m = fmaxf(m, om);
      }
    };
    // after document D's last chunk: the maxima over the warpgroup's rows, the -1000 fill, the query mask, the row sum
    // and the store; the record goes back
    auto epilogue = [&](const Doc& D) {
      QM_PROF(t_ = clock64();)
      if (lane == 0) mbar_arrive(&S->rempty[D.slot]);   // every read of the record is above
      // the 8 lanes of a warp that share lane % 4 hold the same tokens for different rows (lane bits 2..4)
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float om = __shfl_xor_sync(0xffffffffu, mx[e], o);
          const int oa = kArgmax ? __shfl_xor_sync(0xffffffffu, ax[e], o) : 0;
          combine(om, oa, mx[e], ax[e]);
        }
      }
      // the four warps' maxima meet in shared memory, [warp][token]; warp 0 finishes the document while warps 1-3 go
      // on.  The warpgroup's next document writes the other buffer; the one after writes this one again only once
      // the MMAs of the document between have completed, and warp 0 issues its part of them after reading this one.
      const int buf = (int)((D.n >> 1) & 1);
      float* xm = S->xm[c][buf][0];
      int32_t* xa = S->xa[c][buf][0];
      if (lane < 4) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int t = 8 * (e >> 1) + 2 * lane + (e & 1);
          xm[32 * wq + t] = mx[e];
          if constexpr (kArgmax) xa[32 * wq + t] = ax[e];
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) { mx[e] = -INFINITY; ax[e] = -1; }
      if (wq != 0) {
        named_bar_arrive(1 + c, 128);
      } else {
        named_bar_sync(1 + c, 128);
        // lane t: query token t
        float m = xm[lane];
        int a = kArgmax ? xa[lane] : -1;
#pragma unroll
        for (int w = 1; w < 4; ++w) combine(xm[32 * w + lane], kArgmax ? xa[32 * w + lane] : 0, m, a);
        // the reference's -1000 fill, after every real row (ties keep the real row); row Ld reports -1 below
        if (D.head & kFill) take<kArgmax>(-1000.f, P.Ld, m, a);
        const bool ok = mask_test(D.qraw, qmt);   // qraw = 0 for tokens >= Lq
        const int64_t p = p_begin + D.n;
        if constexpr (kArgmax) {
          // rows >= Ld are the -inf padding and the -1000 fill: a max taken there carries no gradient (-1), like a
          // masked query token
          if (lane < P.Lq) P.argmax[p * (int64_t)P.Lq + lane] = (ok && a < P.Ld) ? a : -1;
        }
        // the score sums the tokens as ((t0 + t1) + (t2 + t3)) + ((t4 + t5) + (t6 + t7)) over t_i = q[i] + q[i + 8]
        // for tokens 0..15, the same over tokens 16..31, and then the two halves: a fixed association, so that the
        // score does not depend on how the rows were split among threads
        float s = ok ? m : 0.f;
        s += __shfl_down_sync(0xffffffffu, s, 8);
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float hi = __shfl_sync(0xffffffffu, s, 16);
        if (lane == 0) P.out[p] = s + hi;
      }
      QM_PROF(prof[kCoEpilogue] += clock64() - t_;)
    };
    // one chunk at a time: its stage goes back to the producer as soon as it is reduced, and the other warpgroup's
    // MMAs fill the tensor cores meanwhile
    const int64_t n_pairs = p_end - p_begin;
    float acc[16];
    for (int64_t n = c; n < n_pairs; n += 2) {
      Doc D;
      begin(D, n);
      for (int ch = 0; ch < D.nch; ++ch) {
        const int st = issue(acc, D.qlo);
        QM_PROF(t_ = clock64();)
        wgmma_wait<0>();
        QM_PROF(prof[kCoMma] += clock64() - t_; t_ = clock64();)
        reduce(acc, st, D, ch);
        QM_PROF(prof[kCoReduce] += clock64() - t_;)
      }
      epilogue(D);
    }
    QM_PROF(prof[kCoTotal] = clock64() - t_start;
            if (wq == 0 && lane == 0) for (int i = kCoTotal; i <= kCoDocs; ++i) atomicAdd(&g_qm_prof[i], prof[i]);)
  }
}

template <typename T, bool kArgmax, bool kStore>
int launch_qm(int grid, size_t smem_bytes, cudaStream_t stream, const QmMaps& M, const MaxsimParams& P,
              const QmLaunch& L) {
  MMB_CHECK_CUDA(cudaFuncSetAttribute(maxsim_qm_kernel<T, kArgmax, kStore>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem_bytes));
  maxsim_qm_kernel<T, kArgmax, kStore><<<grid, kThreads, smem_bytes, stream>>>(M, P, L);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

int launch_qm_dispatch(int grid, size_t smem_bytes, cudaStream_t stream, const QmMaps& M, const MaxsimParams& P,
                       const QmLaunch& L, int dtype) {
  if (P.doc_offsets)
    return dtype == MMB200_F16 ? launch_qm<__half, false, true>(grid, smem_bytes, stream, M, P, L)
                               : launch_qm<__nv_bfloat16, false, true>(grid, smem_bytes, stream, M, P, L);
  if (dtype == MMB200_F16)
    return P.argmax ? launch_qm<__half, true, false>(grid, smem_bytes, stream, M, P, L)
                    : launch_qm<__half, false, false>(grid, smem_bytes, stream, M, P, L);
  return P.argmax ? launch_qm<__nv_bfloat16, true, false>(grid, smem_bytes, stream, M, P, L)
                  : launch_qm<__nv_bfloat16, false, false>(grid, smem_bytes, stream, M, P, L);
}

}  // namespace

// Returns MMB200_OK with *handled = false when the shape is outside this kernel's envelope.
int maxsim_qm_launch(const MaxsimParams& P, int dtype, const DeviceInfo& dev, cudaStream_t stream, bool* handled) {
  *handled = false;
  if (dtype != MMB200_F16 && dtype != MMB200_BF16) return MMB200_OK;
  if (P.Lq > kQRows || (P.dim != 64 && P.dim != 128) || P.Ld > kMaxLd) return MMB200_OK;
  if ((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d)) & 15) return MMB200_OK;
  if (P.doc_offsets && P.argmax) return MMB200_OK;   // store mode never asks for argmax
  QmLaunch L;
  L.kblocks = P.dim / 64;
  L.chunk_bytes = L.kblocks * kChunkKBlockBytes;
  L.rec_words = kRecBits + 2 * ((P.Ld + kChunkRows - 1) / kChunkRows);
  const int fixed = kQSlots * L.kblocks * kQBlockBytes + (int)sizeof(QmShared) + 1024;
  L.stages = std::min(kMaxStages, (dev.max_smem_optin - fixed - kRecordReserve) / L.chunk_bytes) & ~1;
  // the records take what is left: 48 slots up to Ld 256 or so, 24 at dim 128 and Ld 4096
  const int rec_bytes = L.rec_words * 4;
  L.records = std::min(kMaxRecords, (dev.max_smem_optin - fixed - L.stages * L.chunk_bytes) / rec_bytes);
  L.records -= L.records % kRecordStep;
  // at least two stages per half of the ring, so that a chunk loads while the previous one is reduced
  if (L.stages < 4 || L.records < kRecordStep) return MMB200_OK;
  const size_t smem_bytes = (size_t)L.stages * L.chunk_bytes + (size_t)L.records * rec_bytes + fixed;

  const CUtensorMapDataType tdt = dtype == MMB200_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  QmMaps M;
  {
    const uint64_t dims[4] = {64, (uint64_t)P.Lq, (uint64_t)L.kblocks, (uint64_t)P.n_q};
    const uint64_t strides[3] = {(uint64_t)P.dim * 2, 128, (uint64_t)P.Lq * P.dim * 2};
    const uint32_t box[4] = {64, (uint32_t)kQRows, 1, 1};
    if (int rc = encode_tensor_map(&M.q, tdt, 4, P.q, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
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
    const uint32_t box[4] = {64, (uint32_t)kChunkRows, (uint32_t)L.kblocks, 1};
    if (int rc = encode_tensor_map(&M.d, tdt, 4, P.d, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
      return rc;
    const uint32_t half[4] = {64, (uint32_t)kChunkRows / 2, 1, 1};
    if (!P.doc_offsets)   // store mode never takes half boxes
      if (int rc = encode_tensor_map(&M.dh, tdt, 4, P.d, dims, strides, half, CU_TENSOR_MAP_SWIZZLE_128B,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B))
        return rc;
  }
  *handled = true;
  const int grid = (int)std::min<int64_t>(dev.sm_count, P.n_pairs);
#ifdef MMB200_ENABLE_PROF
  const bool prof = getenv("MMB200_MAXSIM_PROF") != nullptr;
  if (prof) {
    const unsigned long long zero[kProfCount] = {};
    MMB_CHECK_CUDA(cudaMemcpyToSymbolAsync(g_qm_prof, zero, sizeof(zero), 0, cudaMemcpyHostToDevice, stream));
  }
  const int rc = launch_qm_dispatch(grid, smem_bytes, stream, M, P, L, dtype);
  if (prof && rc == MMB200_OK) {
    unsigned long long h[kProfCount];
    MMB_CHECK_CUDA(cudaMemcpyFromSymbolAsync(h, g_qm_prof, sizeof(h), 0, cudaMemcpyDeviceToHost, stream));
    MMB_CHECK_CUDA(cudaStreamSynchronize(stream));
    // per CTA (producer), per consumer warpgroup, per scout; cycles, and cycles per chunk / per document
    const double ctas = grid, wgs = 2.0 * grid, scouts = (double)kScouts * grid;
    const double chunks = (double)h[kPrChunks], docs = (double)h[kCoDocs];
    fprintf(stderr,
            "maxsim_prof pairs %lld Ld %d chunks %.0f | cycles per CTA: producer total %.0f qempty %.0f rfull %.0f "
            "empty %.0f tma %.0f | per consumer warpgroup: total %.0f rfull %.0f full %.0f issue %.0f mma %.0f "
            "reduce %.0f epilogue %.0f | per scout: total %.0f rempty %.0f | per chunk: producer %.0f (empty %.0f, "
            "tma %.0f), warpgroup full %.0f issue %.0f mma %.0f reduce %.0f | per document per warpgroup: total %.0f "
            "epilogue %.0f rfull %.0f\n",
            (long long)P.n_pairs, P.Ld, chunks, h[kPrTotal] / ctas, h[kPrQEmpty] / ctas, h[kPrRFull] / ctas,
            h[kPrEmpty] / ctas, h[kPrTma] / ctas, h[kCoTotal] / wgs, h[kCoRFull] / wgs, h[kCoFull] / wgs,
            h[kCoIssue] / wgs, h[kCoMma] / wgs, h[kCoReduce] / wgs, h[kCoEpilogue] / wgs, h[kScTotal] / scouts,
            h[kScREmpty] / scouts, h[kPrTotal] / chunks, h[kPrEmpty] / chunks, h[kPrTma] / chunks, h[kCoFull] / chunks,
            h[kCoIssue] / chunks, h[kCoMma] / chunks, h[kCoReduce] / chunks, h[kCoTotal] / docs, h[kCoEpilogue] / docs,
            h[kCoRFull] / docs);
  }
  return rc;
#else
  return launch_qm_dispatch(grid, smem_bytes, stream, M, P, L, dtype);
#endif
}

}  // namespace mmb
