// TKL (SIGIR'20) interaction stage: per-chunk cosine + RBF kernels, sliding-window (30, stride 2) kernel
// pooling with learned saturation, window scores, and the greedy top-3 "hills" selection.
//
// Reference arithmetic: matchmaker/models/published/sigir20_tkl.py:180-286.  The reference scatters the
// per-chunk activations into a zero tensor [B*C, Lq, 40, K], re-assembles [B, Lq, C*40, K] (450 MB at
// BASELINE config 5) and runs two strided window reductions that each re-read it 15 times.  Here one CTA
// walks a document segment chunk by chunk, keeps the activations of the last 40 position PAIRS in a
// shared-memory ring (a window of 30 positions at stride 2 is exactly 15 consecutive pairs), finishes
// every window as soon as its last pair is known, and writes only the window score [B, W].
//
// Exact-zero semantics the reference depends on are preserved: a position counts towards the window
// "length" iff the sum of its K activations is != 0 (sigir20_tkl.py:210), windows whose score is exactly
// 0 become the -9900 sentinel (:257), and window sums are formed directly from the activations (no
// prefix-difference tricks that would leave round-off residue in empty windows).
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "device_util.cuh"
#include "host_util.cuh"
#include "masks.cuh"
#include "tkl.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 40;      // sigir20_tkl.py:52
constexpr int kWindow = 30;     // :56
constexpr int kPairsPerChunk = kChunk / 2;
constexpr int kWinPairs = kWindow / 2;  // 15
constexpr int kRing = 2 * kPairsPerChunk;  // pairs kept: previous + current chunk
constexpr int kZStride = kRing + 1;        // odd strides: the window phase walks query rows across lanes
constexpr int kMaxLq = 40;
constexpr float kClamp = 1e-10f;

// rows -> smem, L2-normalised; one warp per row.  Optionally dots the RAW row with `red_w`.
__device__ __forceinline__ void load_rows_norm(const float* __restrict__ src, int nrows_valid, int nrows, int D, int dp,
                                               float* __restrict__ dst, const float* __restrict__ red_w,
                                               float* __restrict__ red_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int d4 = D >> 2;
  for (int r = warp; r < nrows; r += nw) {
    float* drow = dst + (size_t)r * dp;
    if (r < nrows_valid) {
      const float4* srow = reinterpret_cast<const float4*>(src + (size_t)r * D);
      float ss = 0.f, rd = 0.f;
      for (int c = lane; c < d4; c += 32) {
        const float4 v = __ldg(srow + c);
        ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
        if (red_w) {
          const float4 w = __ldg(reinterpret_cast<const float4*>(red_w) + c);
          rd = fmaf(v.x, w.x, rd); rd = fmaf(v.y, w.y, rd); rd = fmaf(v.z, w.z, rd); rd = fmaf(v.w, w.w, rd);
        }
        *reinterpret_cast<float4*>(drow + 4 * c) = v;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
        rd += __shfl_xor_sync(0xffffffffu, rd, o);
      }
      const float inv = 1.0f / (sqrtf(ss) + kTinyNorm);
      __syncwarp();
      for (int c = lane; c < d4; c += 32) {
        float4 v = *reinterpret_cast<float4*>(drow + 4 * c);
        v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
        *reinterpret_cast<float4*>(drow + 4 * c) = v;
      }
      if (lane == 0 && red_out) red_out[r] = rd;
    } else {
      for (int c = lane; c < d4; c += 32) *reinterpret_cast<float4*>(drow + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (lane == 0 && red_out) red_out[r] = 0.f;
    }
  }
}

// cos[40 x 40]: 200 threads, each 4 query rows (ti + 10 r) x 2 chunk rows (tj + 20 s).
__device__ __forceinline__ void cos_40x40(const float* __restrict__ qs, const float* __restrict__ ds, int D, int dp,
                                          float* __restrict__ cs /* [40][41] */) {
  const int t = threadIdx.x;
  if (t >= 200) return;
  const int ti = t % 10, tj = t / 10;
  float acc[4][2] = {};
  const int d4 = D >> 2;
  for (int c = 0; c < d4; ++c) {
    float4 qv[4], dv[2];
#pragma unroll
    for (int r = 0; r < 4; ++r) qv[r] = *reinterpret_cast<const float4*>(qs + (size_t)(ti + 10 * r) * dp + 4 * c);
#pragma unroll
    for (int s = 0; s < 2; ++s) dv[s] = *reinterpret_cast<const float4*>(ds + (size_t)(tj + 20 * s) * dp + 4 * c);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        acc[r][s] = fmaf(qv[r].x, dv[s].x, acc[r][s]);
        acc[r][s] = fmaf(qv[r].y, dv[s].y, acc[r][s]);
        acc[r][s] = fmaf(qv[r].z, dv[s].z, acc[r][s]);
        acc[r][s] = fmaf(qv[r].w, dv[s].w, acc[r][s]);
      }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 2; ++s) cs[(ti + 10 * r) * 41 + tj + 20 * s] = acc[r][s];
}

// PROF (MMB200_TKL_PROF=1): debugging aid, thread 0 of CTA 0 accumulates the cycles of each phase of the chunk loop.
// STORE: document b is pair b (TklPairs): query row pair_q[b], chunk slots from row pair_d[b] of the passages' slot table.
template <int KB, bool PROF, bool STORE>
__global__ void __launch_bounds__(kThreads) tkl_window_kernel(TklParams P, long long* prof, TklPairs X) {
  long long pc[5] = {0, 0, 0, 0, 0};
  long long t_mark = PROF ? clock64() : 0;
  auto lap = [&](int slot) {
    if constexpr (PROF) {
      const long long now = clock64();
      pc[slot] += now - t_mark;
      t_mark = now;
    }
  };
  extern __shared__ __align__(16) float sm[];
  const int D = P.D, dp = padded_row_stride(D), Lq = P.Lq, K = P.K;
  float* qs = sm;                                   // [40][dp]  normalised query rows
  float* ds = qs + (size_t)kMaxLq * dp;             // [40][dp]  normalised chunk rows
  float* cs = ds + (size_t)kChunk * dp;             // [40][41]
  constexpr int UST = kRing * KB + 1;               // row stride of U (odd -> no bank conflicts across query rows)
  float* U = cs + kMaxLq * 41;                      // [40 i][kRing][KB] pair sums of activations
  float* Z = U + (size_t)kMaxLq * UST;              // [40 i][kRing] non-zero position counts per pair
  float* red = Z + kMaxLq * kZStride;               // [40] sat_emb_reduce1(q_i)
  float* qm_s = red + kMaxLq;                       // [40]
  float* dm_s = qm_s + kMaxLq;                      // [40]
  float* mu_s = dm_s + kChunk;                      // [KB]
  float* a_s = mu_s + KB;
  float* w_s = a_s + KB;
  float* km_s = w_s + KB;                           // kernel_mult0 (log saturation)
  float* sp = km_s + KB;                            // [16] saturation scalars
  float* pk = sp + 16;                              // [20][KB] per-kernel sums over query rows
  float* T = pk + 20 * KB;                          // [20 windows][40][KB] saturated activations
  const int t = threadIdx.x;
  if (P.plan && P.plan[0] == 1) return;  // the tensor-core kernel (tkl_ts.cu) took this call

  if (t < KB) {
    const bool ok = t < K;
    mu_s[t] = ok ? P.mu[t] : 0.f;
    a_s[t] = ok ? rbf_scale(P.sigma[t]) : 0.f;
    w_s[t] = ok ? P.dense_w[t] : 0.f;
    km_s[t] = (ok && P.saturation == 1) ? P.sat_params[t] : 1.f;
  }
  if (t < 16) sp[t] = (P.saturation == 0 && t < 13) ? P.sat_params[t] : 0.f;

  const int64_t n_items = P.B * P.segs;
  for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int64_t b = item / P.segs;
    const int seg = (int)(item % P.segs);
    const int c_first = seg * P.chunks_per_seg;
    const int c_last = min(P.C, c_first + P.chunks_per_seg);
    if (c_first >= c_last) continue;
    const int64_t qb = tkl_q_row<STORE>(X, b);
    __syncthreads();
    load_rows_norm(P.q + qb * (int64_t)Lq * D, Lq, kMaxLq, D, dp, qs, P.saturation == 0 ? P.sat_red_w : nullptr, red);
    if (t < kMaxLq) qm_s[t] = (t < Lq && mask_at(P.q_mask, P.q_mask ? P.mask_dtype : 0, qb * (int64_t)Lq + t)) ? 1.f : 0.f;
    // one halo chunk in front supplies the 14 pairs that windows ending in this segment reach back to
    for (int c = max(0, c_first - 1); c < c_last; ++c) {
      // store mode reads the pair's passage again per chunk (an L1 hit) rather than holding it across the loop
      const int64_t sb = tkl_slot_row<STORE>(X, b);
      const int pk_idx = (STORE && sb < 0) ? -1 : P.slot_to_packed[sb * P.C + c];
      __syncthreads();
      lap(4);
      if (pk_idx >= 0) {
        load_rows_norm(P.chunks + (int64_t)pk_idx * kChunk * D, kChunk, kChunk, D, dp, ds, nullptr, nullptr);
        if (t < kChunk) dm_s[t] = mask_at(P.chunk_mask, P.chunk_mask ? P.mask_dtype : 0, (int64_t)pk_idx * kChunk + t) ? 1.f : 0.f;
        __syncthreads();
        lap(0);
        cos_40x40(qs, ds, D, dp, cs);
        __syncthreads();
        lap(1);
      }
      // activations of this chunk's 20 position pairs -> ring
      for (int e = t; e < kMaxLq * kPairsPerChunk; e += kThreads) {
        const int i = e / kPairsPerChunk, ul = e % kPairsPerChunk;
        const int slot = (c * kPairsPerChunk + ul) % kRing;
        float* u = U + (size_t)i * UST + slot * KB;
        float nz = 0.f;
        if (pk_idx >= 0 && i < Lq) {
          const int p0 = 2 * ul, p1 = p0 + 1;
          const float c0 = cs[i * 41 + p0], c1 = cs[i * 41 + p1];
          const bool m0 = dm_s[p0] != 0.f, m1 = dm_s[p1] != 0.f;
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int k = 0; k < KB; ++k) {
            const float x0 = (c0 - mu_s[k]) * a_s[k], x1 = (c1 - mu_s[k]) * a_s[k];
            const float v0 = (m0 && k < K) ? ex2_approx(-x0 * x0) : 0.f;
            const float v1 = (m1 && k < K) ? ex2_approx(-x1 * x1) : 0.f;
            s0 += v0; s1 += v1;
            u[k] = v0 + v1;
          }
          nz = (s0 != 0.f ? 1.f : 0.f) + (s1 != 0.f ? 1.f : 0.f);  // sigir20_tkl.py:210
        } else {
#pragma unroll
          for (int k = 0; k < KB; ++k) u[k] = 0.f;
        }
        Z[i * kZStride + slot] = nz;
      }
      __syncthreads();
      lap(2);
      if (c < c_first) continue;  // halo chunk: nothing to finish
      // windows whose last pair lies in this chunk: w + 14 in [20c, 20c+20)
      const int w_lo = max(0, c * kPairsPerChunk - (kWinPairs - 1));
      const int w_hi = min(P.W, c * kPairsPerChunk + kPairsPerChunk - (kWinPairs - 1));
      const int nw = w_hi - w_lo;
      if (nw <= 0) continue;
      for (int e = t; e < nw * kMaxLq; e += kThreads) {
        const int wl = e / kMaxLq, i = e % kMaxLq;
        const int w = w_lo + wl;
        float S[KB];
#pragma unroll
        for (int k = 0; k < KB; ++k) S[k] = 0.f;
        float len = 0.f;
        for (int u = 0; u < kWinPairs; ++u) {
          const int slot = (w + u) % kRing;
          const float* up = U + (size_t)i * UST + slot * KB;
#pragma unroll
          for (int k = 0; k < KB; ++k) S[k] += up[k];
          len += Z[i * kZStride + slot];
        }
        const float gate = (i < Lq && qm_s[i] != 0.f && len > 0.f) ? 1.f : 0.f;  // :248
        float* Tp = T + ((size_t)wl * kMaxLq + i) * KB;
        if (P.saturation == 0) {
          // LayerNorm over the pair (reduce(q_i), len), then three Linear(2,1) (:224-234)
          const float a0 = red[i], a1 = len;
          const float mean = (a0 + a1) * 0.5f;
          const float d0 = a0 - mean, d1 = a1 - mean;
          const float rstd = rsqrtf((d0 * d0 + d1 * d1) * 0.5f + 1e-5f);
          const float y0 = d0 * rstd * sp[0] + sp[2], y1 = d1 * rstd * sp[1] + sp[3];
          const float sat1 = y0 * sp[4] + y1 * sp[5] + sp[6];
          const float sat2 = 1.0f / (y0 * sp[7] + y1 * sp[8] + sp[9]);
          const float sat3 = y0 * sp[10] + y1 * sp[11] + sp[12];
#pragma unroll
          for (int k = 0; k < KB; ++k) {
            const float pw = ex2_approx(sat2 * lg2_approx(fmaxf(S[k], kClamp)));
            Tp[k] = (k < K) ? (sat1 * pw - sat3) * gate : 0.f;
          }
        } else {
#pragma unroll
          for (int k = 0; k < KB; ++k) Tp[k] = (k < K) ? logf(fmaxf(S[k] * km_s[k], kClamp)) * gate : 0.f;  // :246
        }
      }
      __syncthreads();
      for (int e = t; e < nw * KB; e += kThreads) {  // per_kernel = sum over query rows (:249)
        const int wl = e / KB, k = e % KB;
        float s = 0.f;
        for (int i = 0; i < Lq; ++i) s += T[((size_t)wl * kMaxLq + i) * KB + k];
        pk[wl * KB + k] = s;
      }
      __syncthreads();
      if (t < nw) {  // dense (:251-252)
        float s = 0.f;
        for (int k = 0; k < K; ++k) s = fmaf(pk[t * KB + k], w_s[k], s);
        P.window_score[b * P.W + w_lo + t] = s;
      }
      lap(3);
    }
  }
  if (PROF && blockIdx.x == 0 && t == 0) {
    for (int i = 0; i < 5; ++i) prof[i] = pc[i];
  }
}

// One block per document: sentinel, 3 greedy hills, neighbours, weighted sum (sigir20_tkl.py:254-286).  The window
// scores live in shared memory for the whole selection (round 1 walked them in global memory with one warp per document:
// 31 dependent global round trips per pass, 26 us for 128 documents; this version is bound by one read and one write).
constexpr int kHillThreads = 256;

__global__ void __launch_bounds__(kHillThreads) tkl_hills_kernel(const float* window_score, float* orig_score,
                                                                const float* __restrict__ chunk_scoring,
                                                                int64_t* __restrict__ top_idx, float* __restrict__ top15,
                                                                float* __restrict__ score, int64_t B, int W) {
  extern __shared__ float hsm[];
  float* orig = hsm;            // [W] scores with the -9900 sentinel (what the reference indexes for the neighbours)
  float* wk = hsm + W;          // [W] working copy, suppressed regions overwritten
  __shared__ float red_v[kHillThreads / 32];
  __shared__ int red_i[kHillThreads / 32];
  __shared__ int best_s[3];
  __shared__ float t15[15];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    const float* win = window_score + b * W;   // may alias orig_score (in-place use): read completely before any write
    __syncthreads();
    for (int w = t; w < W; w += kHillThreads) {
      float v = win[w];
      if (v == 0.f) v = -9900.f;  // :257
      orig[w] = v;
      wk[w] = v;
    }
    __syncthreads();
    for (int c = 0; c < 3; ++c) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int w = t; w < W; w += kHillThreads) {
        const float v = wk[w];
        if (v > bv) { bv = v; bi = w; }  // ascending scan keeps the first maximum
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
      __syncthreads();
      if (t == 0) {
        float fv = red_v[0];
        int fi = red_i[0];
        for (int x = 1; x < kHillThreads / 32; ++x)
          if (red_v[x] > fv || (red_v[x] == fv && red_i[x] < fi)) { fv = red_v[x]; fi = red_i[x]; }
        best_s[c] = fi;
      }
      __syncthreads();
      const int bi_all = best_s[c];
      for (int w = t; w < W; w += kHillThreads)
        if (fabsf((float)(w - bi_all)) < 15.0f) wk[w] = -10001.f - (float)c;  // |r - best| < window/2 (:270-271)
      __syncthreads();
    }
    if (t < 15) {
      const int c = t % 3, off_sel = t / 3;  // cat([idx, idx-1, idx+1, idx-2, idx+2], dim=1) (:274)
      const int off = off_sel == 0 ? 0 : (off_sel == 1 ? -1 : (off_sel == 2 ? 1 : (off_sel == 3 ? -2 : 2)));
      int idx = best_s[c] + off;
      idx = idx < 0 ? 0 : (idx >= W ? W - 1 : idx);
      float v = orig[idx];
      if (v <= -9900.f) v = 0.f;  // :281
      top15[b * 15 + t] = v;
      t15[t] = v * chunk_scoring[t];
    }
    if (t < 3) top_idx[b * 3 + t] = best_s[t];
    __syncthreads();
    if (t == 0) {  // fixed-order sum over the 15 terms
      float tot = 0.f;
      for (int l = 0; l < 15; ++l) tot += t15[l];
      score[b] = tot;
    }
    for (int w = t; w < W; w += kHillThreads) {
      const float v = orig[w];
      orig_score[b * W + w] = v <= -9900.f ? 0.f : v;  // :284 (the reference's returned "orig_score")
    }
  }
}

// slot_to_packed[s] = (number of packed slots before s) if packed[s] else -1.  One block; n = B * C is small.
__global__ void __launch_bounds__(1024) tkl_slot_map_kernel(const uint8_t* __restrict__ packed, int64_t n,
                                                            int32_t* __restrict__ slot_to_packed) {
  __shared__ int wsum[32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t per = (n + 1023) / 1024;
  const int64_t lo = min(n, (int64_t)t * per), hi = min(n, lo + per);
  int local = 0;
  for (int64_t i = lo; i < hi; ++i) local += packed[i] ? 1 : 0;
  int incl = local;   // inclusive scan over the block: shuffles inside the warp, one shared-memory hop across warps
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
  int run = incl - local + (warp > 0 ? wsum[warp - 1] : 0);
  for (int64_t i = lo; i < hi; ++i) slot_to_packed[i] = packed[i] ? run++ : -1;
}

// The routing both window-score entries share: the tensor-core kernel where its envelope and the device-side cover test
// allow, the FFMA kernel otherwise.  X.pair_q != nullptr selects the store-mode instantiations.
template <bool STORE>
int tkl_window_scores_run(TklParams& P, const TklPairs& X, const DeviceInfo& dev, int impl, cudaStream_t stream) {
  const int64_t B = P.B;
  const int C = P.C, K = P.K, D = P.D;
  // split long documents over several CTAs when there are fewer documents than SMs
  int segs = 1;
  if (B < dev.sm_count) segs = std::min<int>(C, std::max<int>(1, (int)((2 * dev.sm_count + B - 1) / B)));
  P.chunks_per_seg = (C + segs - 1) / segs;
  P.segs = (C + P.chunks_per_seg - 1) / P.chunks_per_seg;
  const int KB = K <= 12 ? 12 : 16;
  const int dp = padded_row_stride(D);
  const size_t need = ((size_t)2 * kMaxLq * dp + kMaxLq * 41 + (size_t)kMaxLq * (kRing * KB + 1) + kMaxLq * kZStride + 3 * kMaxLq +
                       4 * KB + 16 + 20 * KB + (size_t)20 * kMaxLq * KB) * sizeof(float);
  const bool ffma_fits = need <= (size_t)dev.max_smem_optin;
  // Tensor-core kernel first (tkl_ts.cu).  Its plan kernel decides ON THE DEVICE whether the kernel set lets it run
  // ("cover", see there); the FFMA kernel below is enqueued as well and returns at once when the plan says the
  // tensor-core kernel took the call -- no host synchronisation either way.
  int32_t* plan = nullptr;
  if (impl != MMB200_IMPL_SIMT) {
    if (!ffma_fits) P.segs = 0;   // tells the tensor-core kernel that nothing can take over
    bool handled = false;
    if (int rc = tkl_window_ts_launch(P, X, dev, stream, &handled, &plan)) return rc;
    if (impl == MMB200_IMPL_TCGEN05 && !handled) {
      set_error("tkl_window_scores: shape outside the tensor-core kernel's envelope (Lq <= 40, K <= 16, Lq * K <= 512)");
      return MMB200_ERR_UNSUPPORTED;
    }
    if (handled && (impl == MMB200_IMPL_TCGEN05 || !ffma_fits)) {
      MMB_CHECK_CUDA(cudaFreeAsync(plan, stream));
      return MMB200_OK;
    }
  }
  if (!ffma_fits) {
    set_error("TKL kernel: embedding dim / kernel count too large for the shared-memory plan (D=300 fits with K <= 12)");
    return MMB200_ERR_UNSUPPORTED;
  }
  const int grid = (int)std::min<int64_t>(B * P.segs, (int64_t)dev.sm_count * 2);
#ifdef MMB200_ENABLE_PROF
  if (!STORE && KB == 12 && getenv("MMB200_TKL_PROF")) {
    long long* prof = nullptr;
    long long h[5] = {0};
    MMB_CHECK_CUDA(cudaMalloc(&prof, sizeof(h)));
    MMB_CHECK_CUDA(cudaMemset(prof, 0, sizeof(h)));
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_window_kernel<12, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    tkl_window_kernel<12, true, false><<<grid, kThreads, need, stream>>>(P, prof, X);
    MMB_CHECK_CUDA(cudaStreamSynchronize(stream));
    MMB_CHECK_CUDA(cudaMemcpy(h, prof, sizeof(h), cudaMemcpyDeviceToHost));
    MMB_CHECK_CUDA(cudaFree(prof));
    fprintf(stderr, "tkl_prof cycles (CTA 0): load+norm %lld | cosine %lld | activations %lld | windows %lld | other %lld\n", h[0], h[1],
            h[2], h[3], h[4]);
    return MMB200_OK;
  }
#endif
  if (KB == 12) {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_window_kernel<12, false, STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    tkl_window_kernel<12, false, STORE><<<grid, kThreads, need, stream>>>(P, nullptr, X);
  } else {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_window_kernel<16, false, STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    tkl_window_kernel<16, false, STORE><<<grid, kThreads, need, stream>>>(P, nullptr, X);
  }
  MMB_CHECK_CUDA(cudaGetLastError());
  if (plan) MMB_CHECK_CUDA(cudaFreeAsync(plan, stream));
  return MMB200_OK;
}

// Argument checks both window-score entries share.
int tkl_window_scores_check(const float* q, const float* chunks, const int32_t* slots, const float* mu, const float* sigma,
                            const float* dense_w, const float* sat_red_w, const float* sat_params, float* window_score,
                            const void* q_mask, const void* chunk_mask, int32_t Lq, int32_t D, int32_t C, int32_t K,
                            int32_t saturation, int32_t mask_dtype, int32_t impl) {
  MMB_REQUIRE(q && chunks && slots && mu && sigma && dense_w && sat_params && window_score, "null pointer");
  MMB_REQUIRE(impl == MMB200_IMPL_AUTO || impl == MMB200_IMPL_SIMT || impl == MMB200_IMPL_TCGEN05, "impl: auto, simt or tcgen05");
  MMB_REQUIRE(Lq >= 1 && Lq <= kMaxLq, "TKL kernel supports 1 <= Lq <= 40");
  MMB_REQUIRE(D > 0 && D % 4 == 0, "embedding dim must be a multiple of 4");
  MMB_REQUIRE(C >= 1 && K >= 1 && K <= 16, "need C >= 1 and K <= 16");
  MMB_REQUIRE(saturation == 0 || saturation == 1, "saturation: 0 = embedding, 1 = log");
  MMB_REQUIRE(saturation == 1 || sat_red_w != nullptr, "embedding saturation needs sat_emb_reduce1 weights");
  if (q_mask || chunk_mask) MMB_REQUIRE(mask_dtype_size(mask_dtype) != 0, "unknown mask dtype");
  return MMB200_OK;
}

}  // namespace

}  // namespace mmb

extern "C" int mmb200_tkl_slot_map(const void* packed_mask, int32_t* slot_to_packed, int64_t n_slots, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(packed_mask && slot_to_packed && n_slots >= 0, "bad arguments");
  if (n_slots == 0) return MMB200_OK;
  tkl_slot_map_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream_)>>>(static_cast<const uint8_t*>(packed_mask), n_slots,
                                                                         slot_to_packed);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

extern "C" int mmb200_tkl_window_scores(const float* q, const void* q_mask, const float* chunks, const void* chunk_mask,
                                        const int32_t* slot_to_packed, const float* mu, const float* sigma,
                                        const float* dense_w, const float* sat_red_w, const float* sat_params,
                                        float* window_score, int64_t B, int64_t n_chunks, int32_t Lq, int32_t D,
                                        int32_t C, int32_t K, int32_t saturation, int32_t mask_dtype, int32_t impl,
                                        void* stream_) {
  using namespace mmb;
  if (int rc = tkl_window_scores_check(q, chunks, slot_to_packed, mu, sigma, dense_w, sat_red_w, sat_params, window_score,
                                       q_mask, chunk_mask, Lq, D, C, K, saturation, mask_dtype, impl))
    return rc;
  MMB_REQUIRE(B >= 0, "B >= 0");
  if (B == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  TklParams P{};
  P.q = q; P.q_mask = q_mask; P.chunks = chunks; P.chunk_mask = chunk_mask; P.slot_to_packed = slot_to_packed;
  P.mu = mu; P.sigma = sigma; P.dense_w = dense_w; P.sat_red_w = sat_red_w; P.sat_params = sat_params;
  P.window_score = window_score; P.B = B; P.n_chunks = n_chunks; P.Lq = Lq; P.D = D; P.C = C; P.K = K;
  P.mask_dtype = mask_dtype;
  P.saturation = saturation;
  P.W = (C * kChunk - kWindow) / 2 + 1;
  return tkl_window_scores_run<false>(P, TklPairs{nullptr, nullptr, B}, dev, impl, static_cast<cudaStream_t>(stream_));
}

extern "C" int mmb200_tkl_store_window_scores(const float* q, const void* q_mask, const float* chunks,
                                              const void* chunk_mask, const int32_t* doc_slots, const int32_t* pair_q,
                                              const int32_t* pair_d, const float* mu, const float* sigma,
                                              const float* dense_w, const float* sat_red_w, const float* sat_params,
                                              float* window_score, int64_t n_q, int64_t n_chunks, int64_t n_docs,
                                              int64_t n_pairs, int32_t Lq, int32_t D, int32_t C, int32_t K,
                                              int32_t saturation, int32_t mask_dtype, int32_t impl, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(n_pairs >= 0, "n_pairs >= 0");
  if (n_pairs == 0) return MMB200_OK;   // nothing to write: the empty outputs may be null
  if (int rc = tkl_window_scores_check(q, chunks, doc_slots, mu, sigma, dense_w, sat_red_w, sat_params, window_score,
                                       q_mask, chunk_mask, Lq, D, C, K, saturation, mask_dtype, impl))
    return rc;
  MMB_REQUIRE(pair_q && pair_d, "null pointer");
  MMB_REQUIRE(n_q >= 1 && n_q < (1ll << 31) && n_docs >= 1, "need 1 <= n_q < 2^31 and n_docs >= 1");
  // chunk indices are int32 TMA coordinates
  MMB_REQUIRE(n_chunks >= 1 && n_chunks < (1ll << 31), "need 1 <= n_chunks < 2^31");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  TklParams P{};
  P.q = q; P.q_mask = q_mask; P.chunks = chunks; P.chunk_mask = chunk_mask; P.slot_to_packed = doc_slots;
  P.mu = mu; P.sigma = sigma; P.dense_w = dense_w; P.sat_red_w = sat_red_w; P.sat_params = sat_params;
  P.window_score = window_score; P.B = n_pairs; P.n_chunks = n_chunks; P.Lq = Lq; P.D = D; P.C = C; P.K = K;
  P.mask_dtype = mask_dtype;
  P.saturation = saturation;
  P.W = (C * kChunk - kWindow) / 2 + 1;
  return tkl_window_scores_run<true>(P, TklPairs{pair_q, pair_d, n_q}, dev, impl, static_cast<cudaStream_t>(stream_));
}

extern "C" int mmb200_tkl_top_hills(const float* window_score, float* orig_score, const float* chunk_scoring,
                                    int64_t* top_idx, float* top15, float* score, int64_t B, int32_t W, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(window_score && orig_score && chunk_scoring && top_idx && top15 && score, "null pointer");
  MMB_REQUIRE(W >= 3, "need at least 3 windows");
  if (B == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  const size_t smem = (size_t)2 * W * sizeof(float);
  MMB_REQUIRE(smem <= (size_t)dev.max_smem_optin, "too many windows for the hills kernel");
  MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_hills_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tkl_hills_kernel<<<(unsigned)std::min<int64_t>(B, (int64_t)dev.sm_count * 8), kHillThreads, smem, static_cast<cudaStream_t>(stream_)>>>(
      window_score, orig_score, chunk_scoring, top_idx, top15, score, B, W);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}
