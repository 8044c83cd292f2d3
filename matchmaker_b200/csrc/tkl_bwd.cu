// TKL interaction stage, backward (what torch autograd derives from sigir20_tkl.py:180-286).
//
// Only the <= 15 windows that the top-3 "hills" selection gathered (sigir20_tkl.py:274-286) receive
// gradient, so the backward is sparse: per document at most 15 windows x 30 positions are revisited.  One
// CTA per document walks its selected windows; for each it re-derives the cosine tile [Lq x 30], the kernel
// activations, the window sums and the saturation exactly as the forward does, then pushes the gradient
// through  score_w -> dense -> saturation (pow / LayerNorm(2) / three Linear(2,1), or log) -> window sums ->
// RBF kernels -> cosine -> L2 normalisation  to the contextualised query / chunk embeddings, and accumulates
// the parameter gradients per document (reduced over the batch in a fixed order afterwards: deterministic).
//
// The discrete parts (window "length" counts, the -9900 sentinel, argmax) carry no gradient, as in autograd.
//
// tkl_bwd_kernel keeps [rows x D] tiles in shared memory (D <= 356 on an H100).  The wide backward below
// (mmb200_tkl_bwd_wide) computes the same gradients with shared memory independent of D, for BERT-width embeddings.
#include <algorithm>

#include "device_util.cuh"
#include "host_util.cuh"
#include "masks.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 40, kWindow = 30, kMaxLq = 40, kRows = 32;  // 30 window rows padded to 32
constexpr float kClamp = 1e-10f;
constexpr int kNSat = 13;

struct TklBwdParams {
  const float* q; const void* q_mask; const float* chunks; const void* chunk_mask; const int32_t* slot_to_packed;
  const float* mu; const float* sigma; const float* dense_w; const float* sat_red_w; const float* sat_params;
  const float* chunk_scoring; const int64_t* top_idx; const float* orig_score; const float* grad_score;
  float* grad_q; float* grad_chunks;
  float* ws;  // [B][ws_stride]: dense_w[K] | chunk_scoring[15] | sat[13 or K] | red_w[D]
  int64_t B;
  int32_t Lq, D, C, K, W, mask_dtype, saturation, ws_stride;
};

// ---- per-window math shared by tkl_bwd_kernel and the wide backward (tkl_bwd_wide_g_kernel); independent of D ----

// Window sums S[k] of one query row over the 30 positions of one window (cosines c_row[0..30), position masks dm) and
// the window's token count (positions where some kernel fires, sigir20_tkl.py:210); returns the count.
template <int KB>
__device__ __forceinline__ float tkl_window_sums(const float* c_row, const float* dm, const float* mu_s, const float* a_s,
                                                 int K, float (&S)[KB]) {
#pragma unroll
  for (int k = 0; k < KB; ++k) S[k] = 0.f;
  float len = 0.f;
  for (int r = 0; r < kWindow; ++r) {
    if (dm[r] == 0.f) continue;
    const float c = c_row[r];
    float any = 0.f;
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      const float u = (c - mu_s[k]) * a_s[k];
      const float v = k < K ? ex2_approx(-u * u) : 0.f;
      S[k] += v; any += v;
    }
    len += any != 0.f ? 1.f : 0.f;
  }
  return len;
}

// Saturation forward + backward of one (query row, window) for the window gradient gw: writes the saturated, gated T
// (for d dense_w) to Tm[KB], d S to dS[KB] and the row's parameter-gradient pieces to pp[kNSat + KB]; adds the
// row's d (red_w . q_raw) to da0 (embedding saturation).  row_live: the query row exists and is unmasked; a0 = red_w . q_raw.
template <int KB>
__device__ __forceinline__ void tkl_window_sat_bwd(const float (&S)[KB], float len, bool row_live, float a0_in, float gw,
                                                   int K, int saturation, const float* sp, const float* w_s,
                                                   const float* km_s, float* Tm, float* dS, float* pp, float& da0) {
  const float gate = (row_live && len > 0.f) ? 1.f : 0.f;
#pragma unroll
  for (int x = 0; x < kNSat + KB; ++x) pp[x] = 0.f;
  if (saturation == 0) {
    const float a0 = a0_in, a1 = len;
    const float mean = (a0 + a1) * 0.5f, d0 = a0 - mean, d1 = a1 - mean;
    const float rstd = rsqrtf((d0 * d0 + d1 * d1) * 0.5f + 1e-5f);
    const float n0 = d0 * rstd, n1 = d1 * rstd;
    const float y0 = n0 * sp[0] + sp[2], y1 = n1 * sp[1] + sp[3];
    const float sat1 = y0 * sp[4] + y1 * sp[5] + sp[6];
    const float z2 = y0 * sp[7] + y1 * sp[8] + sp[9];
    const float sat2 = 1.f / z2;
    const float sat3 = y0 * sp[10] + y1 * sp[11] + sp[12];
    float dsat1 = 0.f, dsat2 = 0.f, dsat3 = 0.f;
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      const float Sc = fmaxf(S[k], kClamp);
      const float lnS = logf(Sc);
      const float Pw = expf(sat2 * lnS);
      const float dT = (k < K) ? gw * w_s[k] * gate : 0.f;
      Tm[k] = (k < K) ? (sat1 * Pw - sat3) * gate : 0.f;
      dsat1 += dT * Pw; dsat3 -= dT;
      const float dP = dT * sat1;
      dsat2 += dP * Pw * lnS;
      dS[k] = (S[k] >= kClamp) ? dP * sat2 * Pw / Sc : 0.f;
    }
    const float dz2 = -dsat2 * sat2 * sat2;
    const float dy0 = dsat1 * sp[4] + dz2 * sp[7] + dsat3 * sp[10];
    const float dy1 = dsat1 * sp[5] + dz2 * sp[8] + dsat3 * sp[11];
    const float dn0 = dy0 * sp[0], dn1 = dy1 * sp[1];
    // LayerNorm over two values: n1 = -n0, so d a0 = rstd (dn0 - dn1) / 2 (1 - n0^2) with 1 - n0^2 = eps rstd^2.  The
    // last form keeps full precision when |a0 - a1| >> sqrt(eps), where 1 - n0 * n0 is fp32 rounding noise.
    da0 += rstd * (dn0 - dn1) * 0.5f * (1e-5f * rstd * rstd);  // the length input (index 1) is a count: no gradient
    pp[0] = dy0 * n0; pp[1] = dy1 * n1; pp[2] = dy0; pp[3] = dy1;            // sat_normer weight, bias
    pp[4] = dsat1 * y0; pp[5] = dsat1 * y1; pp[6] = dsat1;                   // saturation_linear
    pp[7] = dz2 * y0; pp[8] = dz2 * y1; pp[9] = dz2;                         // saturation_linear2
    pp[10] = dsat3 * y0; pp[11] = dsat3 * y1; pp[12] = dsat3;                // saturation_linear3
  } else {
#pragma unroll
    for (int k = 0; k < KB; ++k) {
      const float x = S[k] * km_s[k];
      const bool on = (k < K) && x >= kClamp;
      const float dT = (k < K) ? gw * w_s[k] * gate : 0.f;
      Tm[k] = (k < K) ? logf(fmaxf(x, kClamp)) * gate : 0.f;
      dS[k] = on ? dT / S[k] : 0.f;
      pp[kNSat + k] = on ? dT / km_s[k] : 0.f;  // d kernel_mult[0][k]
    }
  }
}

// d loss / d cosine c from the window-sum gradients dS[KB] through the RBF kernels
template <int KB>
__device__ __forceinline__ float tkl_dcos(float c, const float* dS, const float* mu_s, const float* a_s,
                                          const float* is2_s) {
  float G = 0.f;
#pragma unroll
  for (int k = 0; k < KB; ++k) {
    const float diff = c - mu_s[k], u = diff * a_s[k];
    G = fmaf(dS[k] * ex2_approx(-u * u), -diff * is2_s[k], G);
  }
  return G;
}

template <int KB>
__global__ void __launch_bounds__(kThreads) tkl_bwd_kernel(TklBwdParams P) {
  extern __shared__ __align__(16) float sm[];
  const int D = P.D, dp = padded_row_stride(D), Lq = P.Lq, K = P.K;
  const float** rowptr = reinterpret_cast<const float**>(sm);          // [32] source row of each window position
  float** growptr = reinterpret_cast<float**>(sm) + kRows;             // [32] gradient row
  float* qs = sm + 4 * kRows;                  // [40][dp] normalised query rows (after 64 pointers = 512 B)
  float* ds = qs + (size_t)kMaxLq * dp;        // [32][dp] normalised window rows
  float* gq = ds + (size_t)kRows * dp;         // [40][dp] d(q^) accumulated over the windows
  float* gd = gq + (size_t)kMaxLq * dp;        // [32][dp] d(d^) of the current window
  float* cs = gd + (size_t)kRows * dp;         // [40][33] cosine
  float* dc = cs + kMaxLq * 33;                // [40][33] d cosine
  float* Ss = dc + kMaxLq * 33;                // [40][KB] window sums S
  float* dS = Ss + kMaxLq * KB;                // [40][KB]
  float* Tm = dS + kMaxLq * KB;                // [40][KB] saturated, gated T (for d dense_w)
  float* parts = Tm + kMaxLq * KB;             // [40][kNSat + KB] per-query-row parameter-gradient pieces
  float* nq = parts + kMaxLq * (kNSat + KB);   // [40] |q|
  float* sq = nq + kMaxLq;                     // [40] |q| + eps
  float* red = sq + kMaxLq;                    // [40] red_w . q_raw
  float* da0 = red + kMaxLq;                   // [40] accumulated d r_i
  float* qm_s = da0 + kMaxLq;                  // [40]
  float* len_s = qm_s + kMaxLq;                // [40]
  float* nd = len_s + kMaxLq;                  // [32]
  float* sd = nd + kRows;                      // [32]
  float* dm_s = sd + kRows;                    // [32]
  float* mu_s = dm_s + kRows;                  // [KB]
  float* a_s = mu_s + KB;
  float* is2_s = a_s + KB;
  float* w_s = is2_s + KB;
  float* km_s = w_s + KB;
  float* sp = km_s + KB;                       // [16]
  float* acc_w = sp + 16;                      // [KB] d dense_w
  float* acc_sat = acc_w + KB;                 // [kNSat + KB] d sat params (embedding: 13; log: K)
  float* gwin = acc_sat + kNSat + KB;          // [16] gradient per gathered slot
  int* win = reinterpret_cast<int*>(gwin + 16);  // [16] window index per slot
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;

  if (t < KB) {
    const bool ok = t < K;
    const float sg = ok ? P.sigma[t] : 1.f;
    mu_s[t] = ok ? P.mu[t] : 0.f;
    a_s[t] = ok ? rbf_scale(sg) : 0.f;
    is2_s[t] = ok ? 1.f / (sg * sg) : 0.f;
    w_s[t] = ok ? P.dense_w[t] : 0.f;
    km_s[t] = (ok && P.saturation == 1) ? P.sat_params[t] : 1.f;
  }
  if (t < 16) sp[t] = (P.saturation == 0 && t < kNSat) ? P.sat_params[t] : 0.f;

  for (int64_t b = blockIdx.x; b < P.B; b += gridDim.x) {
    __syncthreads();
    const float g = P.grad_score[b];
    // ---- query rows: normalise, keep |q|, |q|+eps and red_w . q_raw ----
    for (int r = warp; r < kMaxLq; r += kThreads / 32) {
      float* drow = qs + (size_t)r * dp;
      float ss = 0.f, rd = 0.f;
      if (r < Lq) {
        const float* src = P.q + (b * Lq + r) * (int64_t)D;
        for (int c = lane; c < D; c += 32) {
          const float v = src[c];
          ss = fmaf(v, v, ss);
          if (P.saturation == 0) rd = fmaf(v, P.sat_red_w[c], rd);
          drow[c] = v;
        }
      } else {
        for (int c = lane; c < D; c += 32) drow[c] = 0.f;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) { ss += __shfl_xor_sync(0xffffffffu, ss, o); rd += __shfl_xor_sync(0xffffffffu, rd, o); }
      const float n = sqrtf(ss), s = n + kTinyNorm;
      __syncwarp();
      for (int c = lane; c < D; c += 32) { drow[c] *= 1.f / s; gq[(size_t)r * dp + c] = 0.f; }
      if (lane == 0) { nq[r] = n; sq[r] = s; red[r] = rd; da0[r] = 0.f; }
    }
    if (t < kMaxLq) qm_s[t] = (t < Lq && mask_at(P.q_mask, P.q_mask ? P.mask_dtype : 0, b * (int64_t)Lq + t)) ? 1.f : 0.f;
    if (t < KB) acc_w[t] = 0.f;
    if (t < kNSat + KB) acc_sat[t] = 0.f;
    if (t < 15) {
      // slot s gathers window clamp(best[c] + off) (sigir20_tkl.py:274-278); a sentinel/zero window passes nothing (:281)
      const int c = t % 3, sel = t / 3;
      const int off = sel == 0 ? 0 : (sel == 1 ? -1 : (sel == 2 ? 1 : (sel == 3 ? -2 : 2)));
      int w = (int)P.top_idx[b * 3 + c] + off;
      w = w < 0 ? 0 : (w >= P.W ? P.W - 1 : w);
      const float v = P.orig_score[b * P.W + w];
      win[t] = w;
      gwin[t] = (v != 0.f) ? g * P.chunk_scoring[t] : 0.f;
      P.ws[b * P.ws_stride + K + t] = g * v;  // d chunk_scoring[s] = g * top15[s]
    }
    __syncthreads();
    if (t == 0) {  // merge slots that point at the same window
      for (int a = 0; a < 15; ++a)
        for (int c = a + 1; c < 15; ++c)
          if (win[c] == win[a] && gwin[c] != 0.f) { gwin[a] += gwin[c]; gwin[c] = 0.f; }
    }
    __syncthreads();

    for (int slot = 0; slot < 15; ++slot) {
      const float gw = gwin[slot];
      if (gw == 0.f) continue;  // uniform
      const int w = win[slot];
      __syncthreads();
      // ---- the 30 positions of window w -> source rows ----
      if (t < kRows) {
        const int p = 2 * w + t;
        const float* src = nullptr;
        float* gdst = nullptr;
        float m = 0.f;
        if (t < kWindow && p < P.C * kChunk) {
          const int pk = P.slot_to_packed[b * P.C + p / kChunk];
          if (pk >= 0) {
            const int64_t row = (int64_t)pk * kChunk + p % kChunk;
            src = P.chunks + row * D;
            gdst = P.grad_chunks + row * D;
            m = mask_at(P.chunk_mask, P.chunk_mask ? P.mask_dtype : 0, row) ? 1.f : 0.f;
          }
        }
        rowptr[t] = src; growptr[t] = gdst; dm_s[t] = m;
      }
      __syncthreads();
      for (int r = warp; r < kRows; r += kThreads / 32) {
        float* drow = ds + (size_t)r * dp;
        const float* src = rowptr[r];
        float ss = 0.f;
        if (src) for (int c = lane; c < D; c += 32) { const float v = src[c]; ss = fmaf(v, v, ss); drow[c] = v; }
        else for (int c = lane; c < D; c += 32) drow[c] = 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        const float n = sqrtf(ss), s = n + kTinyNorm;
        __syncwarp();
        for (int c = lane; c < D; c += 32) drow[c] *= 1.f / s;
        if (lane == 0) { nd[r] = n; sd[r] = s; }
      }
      __syncthreads();
      for (int e = t; e < kMaxLq * kRows; e += kThreads) {  // cosine [40 x 32]
        const int i = e / kRows, r = e % kRows;
        float acc = 0.f;
        const float4* a = reinterpret_cast<const float4*>(qs + (size_t)i * dp);
        const float4* c4 = reinterpret_cast<const float4*>(ds + (size_t)r * dp);
        for (int c = 0; c < (D >> 2); ++c) {
          const float4 x = a[c], y = c4[c];
          acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
        }
        cs[i * 33 + r] = acc;
      }
      __syncthreads();
      if (t < kMaxLq) {  // window sums, length, saturation forward + backward for query row t
        const int i = t;
        float S[KB];
        const float len = tkl_window_sums<KB>(cs + i * 33, dm_s, mu_s, a_s, K, S);
        tkl_window_sat_bwd<KB>(S, len, i < Lq && qm_s[i] != 0.f, red[i], gw, K, P.saturation, sp, w_s, km_s,
                               Tm + i * KB, dS + i * KB, parts + i * (kNSat + KB), da0[i]);
      }
      __syncthreads();
      if (t < K) {  // d dense_w[k] += gw * sum_i T[i][k]
        float s = 0.f;
        for (int i = 0; i < Lq; ++i) s += Tm[i * KB + t];
        acc_w[t] += gw * s;
      }
      if (t >= 32 && t < 32 + kNSat + KB) {  // parameter pieces summed over query rows in a fixed order
        const int x = t - 32;
        float s = 0.f;
        for (int i = 0; i < Lq; ++i) s += parts[i * (kNSat + KB) + x];
        acc_sat[x] += s;
      }
      for (int e = t; e < kMaxLq * kRows; e += kThreads) {  // d cosine
        const int i = e / kRows, r = e % kRows;
        dc[i * 33 + r] = (r < kWindow && dm_s[r] != 0.f) ? tkl_dcos<KB>(cs[i * 33 + r], dS + i * KB, mu_s, a_s, is2_s) : 0.f;
      }
      __syncthreads();
      for (int col = t; col < D; col += kThreads) {  // d q^ += dc d^ ; d d^ = dc^T q^
        float qcol[kMaxLq];
#pragma unroll
        for (int i = 0; i < kMaxLq; ++i) qcol[i] = qs[(size_t)i * dp + col];
        float gacc[kMaxLq];
#pragma unroll
        for (int i = 0; i < kMaxLq; ++i) gacc[i] = 0.f;
        for (int r = 0; r < kWindow; ++r) {
          const float dv = ds[(size_t)r * dp + col];
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < kMaxLq; ++i) {
            const float G = dc[i * 33 + r];
            s = fmaf(G, qcol[i], s);
            gacc[i] = fmaf(G, dv, gacc[i]);
          }
          gd[(size_t)r * dp + col] = s;
        }
#pragma unroll
        for (int i = 0; i < kMaxLq; ++i) gq[(size_t)i * dp + col] += gacc[i];
      }
      __syncthreads();
      for (int r = warp; r < kWindow; r += kThreads / 32) {  // through the normalisation, into the chunk-row gradients
        float* out = growptr[r];
        if (!out) continue;
        float dot = 0.f;
        for (int c = lane; c < D; c += 32) dot = fmaf(ds[(size_t)r * dp + c], gd[(size_t)r * dp + c], dot);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        const float inv_s = 1.f / sd[r], f = nd[r] > 0.f ? dot / nd[r] : 0.f;
        for (int c = lane; c < D; c += 32) out[c] += gd[(size_t)r * dp + c] * inv_s - ds[(size_t)r * dp + c] * f;
      }
    }
    __syncthreads();
    // ---- query gradient: normalisation backward of the accumulated d q^ plus the sat_emb_reduce1 path ----
    for (int r = warp; r < Lq; r += kThreads / 32) {
      float dot = 0.f;
      for (int c = lane; c < D; c += 32) dot = fmaf(qs[(size_t)r * dp + c], gq[(size_t)r * dp + c], dot);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      const float inv_s = 1.f / sq[r], f = nq[r] > 0.f ? dot / nq[r] : 0.f, a0 = da0[r];
      float* out = P.grad_q + (b * Lq + r) * (int64_t)D;
      for (int c = lane; c < D; c += 32) {
        float v = gq[(size_t)r * dp + c] * inv_s - qs[(size_t)r * dp + c] * f;
        if (P.saturation == 0) v = fmaf(a0, P.sat_red_w[c], v);
        out[c] = v;
      }
    }
    float* wsb = P.ws + b * P.ws_stride;
    if (t < K) wsb[t] = acc_w[t];
    if (t < kNSat + KB) {
      const int nsat = P.saturation == 0 ? kNSat : K;
      if (t < nsat) wsb[K + 15 + t] = acc_sat[P.saturation == 0 ? t : kNSat + t];
    }
    if (P.saturation == 0) {
      const int base = K + 15 + kNSat;
      for (int c = t; c < D; c += kThreads) {  // d sat_emb_reduce1.weight[c] = sum_i da0_i * q_raw[i][c]
        float s = 0.f;
        for (int i = 0; i < Lq; ++i) s = fmaf(da0[i] * sq[i], qs[(size_t)i * dp + c], s);
        wsb[base + c] = s;
      }
    }
  }
}

__global__ void tkl_reduce_batch(const float* __restrict__ ws, float* __restrict__ out, int64_t B, int stride) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= stride) return;
  float s = 0.f;
  for (int64_t b = 0; b < B; ++b) s += ws[b * stride + j];
  out[j] = s;
}

// ================================================================================================================
// Wide backward (mmb200_tkl_bwd_wide): shared memory independent of D, work split by 64-feature blocks.
//
// The <= 15 gathered windows of a document lie in three "hills" of <= 5 consecutive windows, so they cover at most
// 3 x 38 = 114 document positions: at most three runs of positions (fewer where hills overlap), <= 128 in all.  The
// backward works over that union: every (query row, position) pair has one cosine and one gradient G_ip = d loss / d c_ip
// summed over the gathered windows that contain p (a window gathered twice counts twice, as in autograd).  The
// normalisation backward needs only the cosines: q^_i . d(q^_i) = sum_p G_ip c_ip and d^_p . d(d^_p) = sum_i G_ip c_ip.
//   1. tkl_bwd_wide_dot_kernel, per (document, feature block): partial q_i . d_p, |q_i|^2, |d_p|^2, red_w . q_i.
//   2. tkl_bwd_wide_g_kernel<KB>, per document: sums the partials in block order, recomputes window sums, saturation
//      and dense exactly as tkl_bwd_kernel, and writes A_ip = G_ip / ((|q_i|+eps)(|d_p|+eps)), the projection
//      coefficients, d (red_w . q_i) and the document's parameter partials.
//   3. tkl_bwd_wide_grad_kernel, per (document, feature block): grad q_i = sum_p A_ip d_p - alpha_i q_i + da0_i red_w,
//      grad d_p = sum_i A_ip q_i - beta_p d_p, and the document's red_w partial sum_i da0_i q_i.
// Every output element has one writer and one summation order: no atomics, bit-reproducible.
constexpr int kUPos = 128;                    // union positions per document (<= 114 used)
constexpr int kFB = 64;                       // features per block
constexpr int kFBS = kFB + 1;                 // shared row stride of a feature block
constexpr int kHill = 2 * 4 + kWindow;        // 38 positions of five consecutive windows
// one document's record in the workspace, both for the partials of each feature block and for the g kernel's output:
// [kMaxLq][kUPos] products | [kMaxLq] | [kUPos] | [kMaxLq]
constexpr int kWideRec = kMaxLq * kUPos + kMaxLq + kUPos + kMaxLq;

__host__ __device__ inline int wide_blocks(int D) { return (D + kFB - 1) / kFB; }
__host__ __device__ inline int64_t wide_param_floats(int64_t B, int stride) { return (B * stride + 3) & ~int64_t(3); }

// The union of the gathered windows' positions of one document: runs [run_p0[j], run_p0[j] + run_n[j]) of document
// positions at union indices run_u0[j].., sorted by position.  Hill c holds the windows clamp(top[c] + {-2..2}), i.e.
// every window of [lo, hi] = clamp(top[c] -+ 2), positions [2 lo, 2 hi + 30).
struct TklUnion {
  int run_p0[3], run_u0[3], run_n[3], nruns, npos;
  __device__ int position(int u) const {  // document position of union index u < npos
    int p = run_p0[0] + u;
    if (nruns > 1 && u >= run_u0[1]) p = run_p0[1] + u - run_u0[1];
    if (nruns > 2 && u >= run_u0[2]) p = run_p0[2] + u - run_u0[2];
    return p;
  }
  __device__ int index(int p) const {  // union index of a covered position p
    int u = p - run_p0[0];
    if (nruns > 1 && p >= run_p0[1]) u = run_u0[1] + p - run_p0[1];
    if (nruns > 2 && p >= run_p0[2]) u = run_u0[2] + p - run_p0[2];
    return u;
  }
};

__device__ inline void tkl_sort2(int& a0, int& e0, int& a1, int& e1) {
  if (a0 > a1) { const int a = a0, e = e0; a0 = a1; e0 = e1; a1 = a; e1 = e; }
}

// (fixed indices only, so that the runs stay in registers)
__device__ inline TklUnion tkl_union(const int64_t* top_idx, int W) {
  int a[3], e[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int t = (int)top_idx[c];
    const int lo = min(max(t - 2, 0), W - 1), hi = min(max(t + 2, 0), W - 1);
    a[c] = 2 * lo; e[c] = 2 * hi + kWindow;
  }
  tkl_sort2(a[0], e[0], a[1], e[1]);
  tkl_sort2(a[1], e[1], a[2], e[2]);
  tkl_sort2(a[0], e[0], a[1], e[1]);
  int p0 = a[0], n0 = e[0] - a[0], p1 = 0, n1 = 0, p2 = 0, n2 = 0, nr = 1;
  if (a[1] <= p0 + n0) n0 = max(p0 + n0, e[1]) - p0;     // hill 2 overlaps or touches run 0
  else { p1 = a[1]; n1 = e[1] - a[1]; nr = 2; }
  if (nr == 1) {
    if (a[2] <= p0 + n0) n0 = max(p0 + n0, e[2]) - p0;
    else { p1 = a[2]; n1 = e[2] - a[2]; nr = 2; }
  } else {
    if (a[2] <= p1 + n1) n1 = max(p1 + n1, e[2]) - p1;
    else { p2 = a[2]; n2 = e[2] - a[2]; nr = 3; }
  }
  TklUnion U;
  U.run_p0[0] = p0; U.run_p0[1] = p1; U.run_p0[2] = p2;
  U.run_n[0] = n0; U.run_n[1] = n1; U.run_n[2] = n2;
  U.run_u0[0] = 0; U.run_u0[1] = n0; U.run_u0[2] = n0 + n1;
  U.nruns = nr; U.npos = n0 + n1 + n2;
  return U;
}

// chunk row of union position u of document b (-1: past the union, or a chunk slot the packing dropped)
__device__ inline int64_t tkl_union_row(const TklBwdParams& P, const TklUnion& U, int64_t b, int u) {
  if (u >= U.npos) return -1;
  const int p = U.position(u);
  const int pk = P.slot_to_packed[b * P.C + p / kChunk];
  return pk < 0 ? -1 : (int64_t)pk * kChunk + p % kChunk;
}

// Loads feature block fb of the query rows [kMaxLq][kFBS] and of the union's chunk rows [kUPos][kFBS] (zeros past Lq,
// past D and for positions without a row) and the union's row indices.
__device__ inline void tkl_wide_load(const TklBwdParams& P, int64_t b, int fb, float* qs, float* ds, int64_t* rows,
                                     TklUnion* Us) {
  const int t = threadIdx.x;
  if (t == 0) *Us = tkl_union(P.top_idx + b * 3, P.W);
  __syncthreads();
  const TklUnion U = *Us;
  if (t < kUPos) rows[t] = tkl_union_row(P, U, b, t);
  __syncthreads();
  const int f0 = fb * kFB;
  for (int e = t; e < kMaxLq * kFB; e += kThreads) {
    const int i = e / kFB, c = e % kFB;
    qs[i * kFBS + c] = (i < P.Lq && f0 + c < P.D) ? P.q[(b * P.Lq + i) * (int64_t)P.D + f0 + c] : 0.f;
  }
  for (int e = t; e < kUPos * kFB; e += kThreads) {
    const int u = e / kFB, c = e % kFB;
    const int64_t row = rows[u];
    ds[u * kFBS + c] = (row >= 0 && f0 + c < P.D) ? P.chunks[row * P.D + f0 + c] : 0.f;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) tkl_bwd_wide_dot_kernel(TklBwdParams P, float* part) {
  __shared__ float qs[kMaxLq * kFBS], ds[kUPos * kFBS];
  __shared__ int64_t rows[kUPos];
  __shared__ TklUnion Us;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, NB = wide_blocks(P.D);
  for (int64_t item = blockIdx.x; item < P.B * NB; item += gridDim.x) {
    const int64_t b = item / NB;
    const int fb = (int)(item % NB);
    __syncthreads();
    tkl_wide_load(P, b, fb, qs, ds, rows, &Us);
    float* out = part + item * kWideRec;
    // products: warp w holds query rows 5w .. 5w+4, lane the positions lane + 32 j
    float acc[5][4];
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[r][j] = 0.f;
    for (int c = 0; c < kFB; ++c) {
      float dv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) dv[j] = ds[(lane + 32 * j) * kFBS + c];
#pragma unroll
      for (int r = 0; r < 5; ++r) {
        const float qv = qs[(5 * warp + r) * kFBS + c];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[r][j] = fmaf(qv, dv[j], acc[r][j]);
      }
    }
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) out[(5 * warp + r) * kUPos + lane + 32 * j] = acc[r][j];
    // squared norms and red_w . q, one row per thread
    if (t < kMaxLq + kUPos) {
      const float* row = t < kMaxLq ? qs + t * kFBS : ds + (t - kMaxLq) * kFBS;
      float ss = 0.f;
      for (int c = 0; c < kFB; ++c) ss = fmaf(row[c], row[c], ss);
      out[kMaxLq * kUPos + t] = ss;
    } else if (t < 2 * kMaxLq + kUPos) {
      const int i = t - kMaxLq - kUPos, f0 = fb * kFB;
      float rd = 0.f;
      if (P.saturation == 0)
        for (int c = 0; c < kFB && f0 + c < P.D; ++c) rd = fmaf(qs[i * kFBS + c], P.sat_red_w[f0 + c], rd);
      out[kMaxLq * kUPos + kMaxLq + kUPos + i] = rd;
    }
  }
}

template <int KB>
__global__ void __launch_bounds__(kThreads) tkl_bwd_wide_g_kernel(TklBwdParams P, const float* part, float* gout) {
  extern __shared__ __align__(16) float sm[];
  constexpr int kCS = kUPos + 1;
  float* cs = sm;                              // [40][129] cosines of the union
  float* dS = cs + kMaxLq * kCS;               // [15][40][KB] d window sums per gathered slot
  float* Tm = dS + 15 * kMaxLq * KB;           // [15][40][KB]
  float* parts = Tm + 15 * kMaxLq * KB;        // [15][40][kNSat + KB]
  float* da0p = parts + 15 * kMaxLq * (kNSat + KB);  // [15][40]
  float* nq = da0p + 15 * kMaxLq;              // [40] |q|
  float* sq = nq + kMaxLq;                     // [40] |q| + eps
  float* red = sq + kMaxLq;                    // [40] red_w . q_raw
  float* qm_s = red + kMaxLq;                  // [40]
  float* nd = qm_s + kMaxLq;                   // [128]
  float* sd = nd + kUPos;                      // [128]
  float* dm_u = sd + kUPos;                    // [128] position mask (0: masked, no row, or past the union)
  float* mu_s = dm_u + kUPos;                  // [KB]
  float* a_s = mu_s + KB;
  float* is2_s = a_s + KB;
  float* w_s = is2_s + KB;
  float* km_s = w_s + KB;
  float* sp = km_s + KB;                       // [16]
  float* gwin = sp + 16;                       // [16] gradient per gathered slot (duplicates merged into the first)
  int* wu0 = reinterpret_cast<int*>(gwin + 16);  // [16] union index of each slot's window's first position
  TklUnion* Us = reinterpret_cast<TklUnion*>(wu0 + 16);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, K = P.K, Lq = P.Lq, NB = wide_blocks(P.D);

  if (t < KB) {
    const bool ok = t < K;
    const float sg = ok ? P.sigma[t] : 1.f;
    mu_s[t] = ok ? P.mu[t] : 0.f;
    a_s[t] = ok ? rbf_scale(sg) : 0.f;
    is2_s[t] = ok ? 1.f / (sg * sg) : 0.f;
    w_s[t] = ok ? P.dense_w[t] : 0.f;
    km_s[t] = (ok && P.saturation == 1) ? P.sat_params[t] : 1.f;
  }
  if (t < 16) sp[t] = (P.saturation == 0 && t < kNSat) ? P.sat_params[t] : 0.f;

  for (int64_t b = blockIdx.x; b < P.B; b += gridDim.x) {
    __syncthreads();
    const float g = P.grad_score[b];
    if (t == 0) *Us = tkl_union(P.top_idx + b * 3, P.W);
    if (t < 15) {  // slot s gathers window clamp(best[c] + off) (sigir20_tkl.py:274-278); a sentinel/zero window passes nothing
      const int c = t % 3, sel = t / 3;
      const int off = sel == 0 ? 0 : (sel == 1 ? -1 : (sel == 2 ? 1 : (sel == 3 ? -2 : 2)));
      int w = (int)P.top_idx[b * 3 + c] + off;
      w = w < 0 ? 0 : (w >= P.W ? P.W - 1 : w);
      const float v = P.orig_score[b * P.W + w];
      wu0[t] = 2 * w;
      gwin[t] = (v != 0.f) ? g * P.chunk_scoring[t] : 0.f;
      P.ws[b * P.ws_stride + K + t] = g * v;  // d chunk_scoring[s] = g * top15[s]
    }
    if (t < kMaxLq) qm_s[t] = (t < Lq && mask_at(P.q_mask, P.q_mask ? P.mask_dtype : 0, b * (int64_t)Lq + t)) ? 1.f : 0.f;
    __syncthreads();
    const TklUnion U = *Us;
    if (t == 0) {  // merge slots that point at the same window
      for (int a = 0; a < 15; ++a)
        for (int c = a + 1; c < 15; ++c)
          if (wu0[c] == wu0[a] && gwin[c] != 0.f) { gwin[a] += gwin[c]; gwin[c] = 0.f; }
    }
    if (t < kUPos) {
      const int64_t row = tkl_union_row(P, U, b, t);
      dm_u[t] = (row >= 0 && mask_at(P.chunk_mask, P.chunk_mask ? P.mask_dtype : 0, row)) ? 1.f : 0.f;
    }
    // ---- the partials of every feature block, summed in block order ----
    const float* pb = part + b * NB * (int64_t)kWideRec;
    for (int e = t; e < kWideRec - kMaxLq * kUPos; e += kThreads) {
      float s = 0.f;
      for (int fb = 0; fb < NB; ++fb) s += pb[fb * (int64_t)kWideRec + kMaxLq * kUPos + e];
      if (e < kMaxLq) { const float n = sqrtf(s); nq[e] = n; sq[e] = n + kTinyNorm; }
      else if (e < kMaxLq + kUPos) { const float n = sqrtf(s); nd[e - kMaxLq] = n; sd[e - kMaxLq] = n + kTinyNorm; }
      else red[e - kMaxLq - kUPos] = s;
    }
    __syncthreads();
    if (t < 15) wu0[t] = U.index(wu0[t]);
    for (int e = t; e < kMaxLq * kUPos; e += kThreads) {
      const int i = e / kUPos, u = e % kUPos;
      float s = 0.f;
      for (int fb = 0; fb < NB; ++fb) s += pb[fb * (int64_t)kWideRec + e];
      cs[i * kCS + u] = s / (sq[i] * sd[u]);
    }
    __syncthreads();
    // ---- window sums, saturation and their backward per (gathered slot, query row) ----
    for (int e = t; e < 15 * kMaxLq; e += kThreads) {
      const int s = e / kMaxLq, i = e % kMaxLq;
      float da0 = 0.f;
      const float gw = gwin[s];
      if (gw != 0.f) {
        float S[KB];
        const float len = tkl_window_sums<KB>(cs + i * kCS + wu0[s], dm_u + wu0[s], mu_s, a_s, K, S);
        tkl_window_sat_bwd<KB>(S, len, i < Lq && qm_s[i] != 0.f, red[i], gw, K, P.saturation, sp, w_s, km_s,
                               Tm + e * KB, dS + e * KB, parts + e * (kNSat + KB), da0);
      }
      da0p[e] = da0;
    }
    __syncthreads();
    float* wsb = P.ws + b * P.ws_stride;
    if (t < K) {  // d dense_w[k] = sum over slots of gw * sum_i T[i][k]
      float acc = 0.f;
      for (int s = 0; s < 15; ++s) {
        if (gwin[s] == 0.f) continue;
        float x = 0.f;
        for (int i = 0; i < Lq; ++i) x += Tm[(s * kMaxLq + i) * KB + t];
        acc += gwin[s] * x;
      }
      wsb[t] = acc;
    }
    if (t >= 32 && t < 32 + kNSat + KB) {  // parameter pieces summed over query rows, then slots, in a fixed order
      const int x = t - 32, nsat = P.saturation == 0 ? kNSat : K, j = P.saturation == 0 ? x : x - kNSat;
      if (j >= 0 && j < nsat) {
        float acc = 0.f;
        for (int s = 0; s < 15; ++s) {
          if (gwin[s] == 0.f) continue;
          float y = 0.f;
          for (int i = 0; i < Lq; ++i) y += parts[(s * kMaxLq + i) * (kNSat + KB) + x];
          acc += y;
        }
        wsb[K + 15 + j] = acc;
      }
    }
    __syncthreads();  // Tm has been read: it holds G from here on
    float* Gs = Tm;   // [40][128]
    float* go = gout + b * (int64_t)kWideRec;
    // ---- G over the union: the window-sum gradients of every window that holds the position, then the RBF kernels ----
    for (int e = t; e < kMaxLq * kUPos; e += kThreads) {
      const int i = e / kUPos, u = e % kUPos;
      float G = 0.f;
      if (dm_u[u] != 0.f) {
        float Dk[KB];
#pragma unroll
        for (int k = 0; k < KB; ++k) Dk[k] = 0.f;
        for (int s = 0; s < 15; ++s) {
          if (gwin[s] == 0.f || u < wu0[s] || u >= wu0[s] + kWindow) continue;
          const float* d = dS + (s * kMaxLq + i) * KB;
#pragma unroll
          for (int k = 0; k < KB; ++k) Dk[k] += d[k];
        }
        G = tkl_dcos<KB>(cs[i * kCS + u], Dk, mu_s, a_s, is2_s);
      }
      go[e] = G / (sq[i] * sd[u]);   // A_iu
      Gs[e] = G;
    }
    __syncthreads();
    // alpha_i = (sum_u G_iu c_iu) / (|q_i| (|q_i| + eps)); beta_u likewise over i; da0_i summed over the slots in order
    for (int i = warp; i < kMaxLq; i += kThreads / 32) {
      float r = 0.f;
      for (int u = lane; u < kUPos; u += 32) r = fmaf(Gs[i * kUPos + u], cs[i * kCS + u], r);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
      if (lane == 0) {
        go[kMaxLq * kUPos + i] = nq[i] > 0.f ? r / (nq[i] * sq[i]) : 0.f;
        float a = 0.f;
        for (int s = 0; s < 15; ++s) a += da0p[s * kMaxLq + i];
        go[kMaxLq * kUPos + kMaxLq + kUPos + i] = a;
      }
    }
    if (t < kUPos) {
      float r = 0.f;
      for (int i = 0; i < Lq; ++i) r = fmaf(Gs[i * kUPos + t], cs[i * kCS + t], r);
      go[kMaxLq * kUPos + kMaxLq + t] = nd[t] > 0.f ? r / (nd[t] * sd[t]) : 0.f;
    }
  }
}

__global__ void __launch_bounds__(kThreads) tkl_bwd_wide_grad_kernel(TklBwdParams P, const float* gout) {
  extern __shared__ __align__(16) float sm[];
  float* As = sm;                                   // [40][128] A
  float* coef = As + kMaxLq * kUPos;                // [40 + 128 + 40] alpha | beta | da0
  float* qs = coef + kMaxLq + kUPos + kMaxLq;       // [40][kFBS]
  float* ds = qs + kMaxLq * kFBS;                   // [128][kFBS]
  int64_t* rows = reinterpret_cast<int64_t*>(ds + kUPos * kFBS);  // [128] (16248 floats in: 8-byte aligned)
  TklUnion& Us = *reinterpret_cast<TklUnion*>(rows + kUPos);
  const int t = threadIdx.x, NB = wide_blocks(P.D), Lq = P.Lq, D = P.D;
  const int c = t % kFB, grp = t / kFB;  // 4 groups of 64 feature columns
  for (int64_t item = blockIdx.x; item < P.B * NB; item += gridDim.x) {
    const int64_t b = item / NB;
    const int fb = (int)(item % NB), f = fb * kFB + c;
    __syncthreads();
    const float* go = gout + b * (int64_t)kWideRec;
    for (int e = t; e < kMaxLq * kUPos; e += kThreads) As[e] = go[e];
    for (int e = t; e < kMaxLq + kUPos + kMaxLq; e += kThreads) coef[e] = go[kMaxLq * kUPos + e];
    tkl_wide_load(P, b, fb, qs, ds, rows, &Us);
    const int npos = Us.npos;
    // query rows 10 grp .. 10 grp + 9: sum_u A_iu d_u - alpha_i q_i (+ da0_i red_w)
    {
      float acc[10];
#pragma unroll
      for (int r = 0; r < 10; ++r) acc[r] = 0.f;
      for (int u = 0; u < npos; ++u) {
        const float dv = ds[u * kFBS + c];
#pragma unroll
        for (int r = 0; r < 10; ++r) acc[r] = fmaf(As[(10 * grp + r) * kUPos + u], dv, acc[r]);
      }
      const float rw = (P.saturation == 0 && f < D) ? P.sat_red_w[f] : 0.f;
#pragma unroll
      for (int r = 0; r < 10; ++r) {
        const int i = 10 * grp + r;
        if (i < Lq && f < D) {
          float v = acc[r] - coef[i] * qs[i * kFBS + c];
          if (P.saturation == 0) v = fmaf(coef[kMaxLq + kUPos + i], rw, v);
          P.grad_q[(b * Lq + i) * (int64_t)D + f] = v;
        }
      }
    }
    // union positions 32 grp .. 32 grp + 31: sum_i A_iu q_i - beta_u d_u
    if (32 * grp < npos) {
      float acc[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = 0.f;
      for (int i = 0; i < Lq; ++i) {
        const float qv = qs[i * kFBS + c];
        const float4* a4 = reinterpret_cast<const float4*>(As + i * kUPos + 32 * grp);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 a = a4[j];
          acc[4 * j] = fmaf(a.x, qv, acc[4 * j]); acc[4 * j + 1] = fmaf(a.y, qv, acc[4 * j + 1]);
          acc[4 * j + 2] = fmaf(a.z, qv, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(a.w, qv, acc[4 * j + 3]);
        }
      }
      if (f < D) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int u = 32 * grp + j;
          const int64_t row = rows[u];
          if (row >= 0) P.grad_chunks[row * D + f] = acc[j] - coef[kMaxLq + u] * ds[u * kFBS + c];
        }
      }
    }
    if (P.saturation == 0 && t < kFB && f < D) {  // d sat_emb_reduce1.weight[f] of this document = sum_i da0_i q_i[f]
      float s = 0.f;
      for (int i = 0; i < Lq; ++i) s = fmaf(coef[kMaxLq + kUPos + i], qs[i * kFBS + c], s);
      P.ws[b * P.ws_stride + P.K + 15 + kNSat + f] = s;
    }
  }
}

constexpr size_t kWideGradSmem = (size_t)(kMaxLq * kUPos + kMaxLq + kUPos + kMaxLq + (kMaxLq + kUPos) * kFBS) *
                                       sizeof(float) + kUPos * sizeof(int64_t) + sizeof(TklUnion);

size_t wide_g_smem_bytes(int KB) {
  const size_t floats = (size_t)kMaxLq * (kUPos + 1) + 2 * 15 * kMaxLq * KB + 15 * kMaxLq * (kNSat + KB) + 15 * kMaxLq +
                        4 * kMaxLq + 3 * kUPos + 5 * KB + 16 + 16 + 16;
  return floats * sizeof(float) + sizeof(TklUnion) + 16;
}

int64_t wide_workspace_floats(int64_t B, int D, int K, int saturation) {
  const int stride = K + 15 + (saturation == 0 ? kNSat + D : K);
  return wide_param_floats(B, stride) + B * (int64_t)(wide_blocks(D) + 1) * kWideRec;
}

// dynamic shared memory of tkl_bwd_kernel<KB> at embedding dim D: the carve-up at the top of the kernel
size_t bwd_smem_bytes(int D, int KB) {
  const size_t dp = padded_row_stride(D);
  const size_t floats = (size_t)(2 * kMaxLq + 2 * kRows) * dp + 2 * kMaxLq * 33 + 3 * (size_t)kMaxLq * KB +
                        (size_t)kMaxLq * (kNSat + KB) + 6 * kMaxLq + 3 * kRows + 5 * KB + 16 + KB + (kNSat + KB) + 16 + 16;
  return floats * sizeof(float) + 4 * kRows * sizeof(float) + 64;
}

// the largest embedding dim (a multiple of 4) whose plan fits in `limit` bytes: 356 with either KB under the H100's
// 227 KB opt-in limit
int bwd_max_dim(int KB, size_t limit) {
  int d = 0;
  while (bwd_smem_bytes(d + 4, KB) <= limit) d += 4;
  return d;
}

}  // namespace
}  // namespace mmb

extern "C" int mmb200_tkl_bwd(const float* q, const void* q_mask, const float* chunks, const void* chunk_mask,
                              const int32_t* slot_to_packed, const float* mu, const float* sigma, const float* dense_w,
                              const float* sat_red_w, const float* sat_params, const float* chunk_scoring,
                              const int64_t* top_idx, const float* orig_score, const float* grad_score, float* grad_q,
                              float* grad_chunks, float* grad_params, float* workspace, int64_t B, int64_t n_chunks,
                              int32_t Lq, int32_t D, int32_t C, int32_t K, int32_t saturation, int32_t mask_dtype,
                              void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(q && chunks && slot_to_packed && mu && sigma && dense_w && sat_params && chunk_scoring && top_idx &&
                  orig_score && grad_score && grad_q && grad_chunks && grad_params && workspace, "null pointer");
  // the bound on D comes from the shared-memory plan below (it depends on K and on the device)
  MMB_REQUIRE(Lq >= 1 && Lq <= kMaxLq && D > 0 && D % 4 == 0 && K >= 1 && K <= 16 && C >= 1,
              "shape outside the TKL backward envelope (1 <= Lq <= 40, D a multiple of 4, 1 <= K <= 16)");
  MMB_REQUIRE(saturation == 0 || saturation == 1, "saturation: 0 = embedding, 1 = log");
  MMB_REQUIRE(saturation == 1 || sat_red_w != nullptr, "embedding saturation needs sat_emb_reduce1 weights");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TklBwdParams P{};
  P.q = q; P.q_mask = q_mask; P.chunks = chunks; P.chunk_mask = chunk_mask; P.slot_to_packed = slot_to_packed;
  P.mu = mu; P.sigma = sigma; P.dense_w = dense_w; P.sat_red_w = sat_red_w; P.sat_params = sat_params;
  P.chunk_scoring = chunk_scoring; P.top_idx = top_idx; P.orig_score = orig_score; P.grad_score = grad_score;
  P.grad_q = grad_q; P.grad_chunks = grad_chunks; P.ws = workspace; P.B = B; P.Lq = Lq; P.D = D; P.C = C; P.K = K;
  P.W = (C * kChunk - kWindow) / 2 + 1; P.mask_dtype = mask_dtype; P.saturation = saturation;
  P.ws_stride = K + 15 + (saturation == 0 ? kNSat + D : K);
  const int KB = K <= 12 ? 12 : 16;
  const size_t need = bwd_smem_bytes(D, KB);
  if (need > (size_t)dev.max_smem_optin) {
    const size_t limit = (size_t)dev.max_smem_optin;
    set_error("TKL backward: D=" + std::to_string(D) + " with K=" + std::to_string(K) + " needs " + std::to_string(need) +
              " bytes of shared memory, the device allows " + std::to_string(limit) + " (D <= " +
              std::to_string(bwd_max_dim(KB, limit)) + " fits with K <= " + std::to_string(KB) + ")");
    return MMB200_ERR_UNSUPPORTED;
  }
  MMB_CHECK_CUDA(cudaMemsetAsync(grad_chunks, 0, (size_t)n_chunks * kChunk * D * sizeof(float), stream));
  if (B == 0) return MMB200_OK;
  const int grid = (int)std::min<int64_t>(B, (int64_t)dev.sm_count * 2);
  if (KB == 12) {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_bwd_kernel<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    tkl_bwd_kernel<12><<<grid, kThreads, need, stream>>>(P);
  } else {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_bwd_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    tkl_bwd_kernel<16><<<grid, kThreads, need, stream>>>(P);
  }
  MMB_CHECK_CUDA(cudaGetLastError());
  tkl_reduce_batch<<<(P.ws_stride + 127) / 128, 128, 0, stream>>>(workspace, grad_params, B, P.ws_stride);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

namespace mmb {
namespace {
constexpr size_t kSm90SmemOptin = 227 * 1024;  // sm_90a's opt-in shared memory per block
constexpr int kWideMaxD = 1024;
}  // namespace
}  // namespace mmb

extern "C" int32_t mmb200_tkl_bwd_route(int32_t Lq, int32_t D, int32_t K) {
  using namespace mmb;
  if (Lq < 1 || Lq > kMaxLq || K < 1 || K > 16 || D < 4 || D % 4 != 0) return 0;
  if (bwd_smem_bytes(D, K <= 12 ? 12 : 16) <= kSm90SmemOptin) return 1;
  return D <= kWideMaxD ? 2 : 0;
}

extern "C" int64_t mmb200_tkl_bwd_wide_workspace_floats(int64_t B, int32_t D, int32_t K, int32_t saturation) {
  return mmb::wide_workspace_floats(B, D, K, saturation);
}

extern "C" int mmb200_tkl_bwd_wide(const float* q, const void* q_mask, const float* chunks, const void* chunk_mask,
                                   const int32_t* slot_to_packed, const float* mu, const float* sigma,
                                   const float* dense_w, const float* sat_red_w, const float* sat_params,
                                   const float* chunk_scoring, const int64_t* top_idx, const float* orig_score,
                                   const float* grad_score, float* grad_q, float* grad_chunks, float* grad_params,
                                   float* workspace, int64_t B, int64_t n_chunks, int32_t Lq, int32_t D, int32_t C,
                                   int32_t K, int32_t saturation, int32_t mask_dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(q && chunks && slot_to_packed && mu && sigma && dense_w && sat_params && chunk_scoring && top_idx &&
                  orig_score && grad_score && grad_q && grad_chunks && grad_params && workspace, "null pointer");
  if (!(Lq >= 1 && Lq <= kMaxLq && D >= 4 && D <= kWideMaxD && D % 4 == 0 && K >= 1 && K <= 16 && C >= 1)) {
    set_error("TKL wide backward: Lq=" + std::to_string(Lq) + ", D=" + std::to_string(D) + ", K=" + std::to_string(K) +
              ", C=" + std::to_string(C) + " is outside its envelope (1 <= Lq <= 40, D a multiple of 4 with " +
              "4 <= D <= 1024, 1 <= K <= 16, C >= 1)");
    return MMB200_ERR_UNSUPPORTED;
  }
  MMB_REQUIRE(saturation == 0 || saturation == 1, "saturation: 0 = embedding, 1 = log");
  MMB_REQUIRE(saturation == 1 || sat_red_w != nullptr, "embedding saturation needs sat_emb_reduce1 weights");
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TklBwdParams P{};
  P.q = q; P.q_mask = q_mask; P.chunks = chunks; P.chunk_mask = chunk_mask; P.slot_to_packed = slot_to_packed;
  P.mu = mu; P.sigma = sigma; P.dense_w = dense_w; P.sat_red_w = sat_red_w; P.sat_params = sat_params;
  P.chunk_scoring = chunk_scoring; P.top_idx = top_idx; P.orig_score = orig_score; P.grad_score = grad_score;
  P.grad_q = grad_q; P.grad_chunks = grad_chunks; P.ws = workspace; P.B = B; P.Lq = Lq; P.D = D; P.C = C; P.K = K;
  P.W = (C * kChunk - kWindow) / 2 + 1; P.mask_dtype = mask_dtype; P.saturation = saturation;
  P.ws_stride = K + 15 + (saturation == 0 ? kNSat + D : K);
  const int KB = K <= 12 ? 12 : 16;
  const size_t g_smem = wide_g_smem_bytes(KB);
  MMB_REQUIRE(g_smem <= (size_t)dev.max_smem_optin && kWideGradSmem <= (size_t)dev.max_smem_optin,
              "TKL wide backward: the device's shared memory per block is too small");
  MMB_CHECK_CUDA(cudaMemsetAsync(grad_chunks, 0, (size_t)n_chunks * kChunk * D * sizeof(float), stream));
  if (B == 0) return MMB200_OK;
  float* part = workspace + wide_param_floats(B, P.ws_stride);
  float* gout = part + B * (int64_t)wide_blocks(D) * kWideRec;
  const int64_t items = B * wide_blocks(D);
  const int fgrid = (int)std::min<int64_t>(items, (int64_t)dev.sm_count * 8);
  tkl_bwd_wide_dot_kernel<<<fgrid, kThreads, 0, stream>>>(P, part);
  MMB_CHECK_CUDA(cudaGetLastError());
  const int ggrid = (int)std::min<int64_t>(B, (int64_t)dev.sm_count);
  if (KB == 12) {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_bwd_wide_g_kernel<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g_smem));
    tkl_bwd_wide_g_kernel<12><<<ggrid, kThreads, g_smem, stream>>>(P, part, gout);
  } else {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_bwd_wide_g_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g_smem));
    tkl_bwd_wide_g_kernel<16><<<ggrid, kThreads, g_smem, stream>>>(P, part, gout);
  }
  MMB_CHECK_CUDA(cudaGetLastError());
  MMB_CHECK_CUDA(cudaFuncSetAttribute(tkl_bwd_wide_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kWideGradSmem));
  tkl_bwd_wide_grad_kernel<<<fgrid, kThreads, kWideGradSmem, stream>>>(P, gout);
  MMB_CHECK_CUDA(cudaGetLastError());
  tkl_reduce_batch<<<(P.ws_stride + 127) / 128, 128, 0, stream>>>(workspace, grad_params, B, P.ws_stride);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}
