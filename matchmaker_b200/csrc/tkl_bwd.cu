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
#pragma unroll
        for (int k = 0; k < KB; ++k) S[k] = 0.f;
        float len = 0.f;
        for (int r = 0; r < kWindow; ++r) {
          if (dm_s[r] == 0.f) continue;
          const float c = cs[i * 33 + r];
          float any = 0.f;
#pragma unroll
          for (int k = 0; k < KB; ++k) {
            const float u = (c - mu_s[k]) * a_s[k];
            const float v = k < K ? ex2_approx(-u * u) : 0.f;
            S[k] += v; any += v;
          }
          len += any != 0.f ? 1.f : 0.f;
        }
        const float gate = (i < Lq && qm_s[i] != 0.f && len > 0.f) ? 1.f : 0.f;
        float* pp = parts + i * (kNSat + KB);
#pragma unroll
        for (int x = 0; x < kNSat + KB; ++x) pp[x] = 0.f;
        if (P.saturation == 0) {
          const float a0 = red[i], a1 = len;
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
            Tm[i * KB + k] = (k < K) ? (sat1 * Pw - sat3) * gate : 0.f;
            dsat1 += dT * Pw; dsat3 -= dT;
            const float dP = dT * sat1;
            dsat2 += dP * Pw * lnS;
            dS[i * KB + k] = (S[k] >= kClamp) ? dP * sat2 * Pw / Sc : 0.f;
          }
          const float dz2 = -dsat2 * sat2 * sat2;
          const float dy0 = dsat1 * sp[4] + dz2 * sp[7] + dsat3 * sp[10];
          const float dy1 = dsat1 * sp[5] + dz2 * sp[8] + dsat3 * sp[11];
          const float dn0 = dy0 * sp[0], dn1 = dy1 * sp[1];
          // LayerNorm over two values: n1 = -n0, so d a0 = rstd (dn0 - dn1) / 2 (1 - n0^2) with 1 - n0^2 = eps rstd^2.  The
          // last form keeps full precision when |a0 - a1| >> sqrt(eps), where 1 - n0 * n0 is fp32 rounding noise.
          da0[i] += rstd * (dn0 - dn1) * 0.5f * (1e-5f * rstd * rstd);  // the length input (index 1) is a count: no gradient
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
            Tm[i * KB + k] = (k < K) ? logf(fmaxf(x, kClamp)) * gate : 0.f;
            dS[i * KB + k] = on ? dT / S[k] : 0.f;
            pp[kNSat + k] = on ? dT / km_s[k] : 0.f;  // d kernel_mult[0][k]
          }
        }
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
        float G = 0.f;
        if (r < kWindow && dm_s[r] != 0.f) {
          const float c = cs[i * 33 + r];
#pragma unroll
          for (int k = 0; k < KB; ++k) {
            const float diff = c - mu_s[k], u = diff * a_s[k];
            G = fmaf(dS[i * KB + k] * ex2_approx(-u * u), -diff * is2_s[k], G);
          }
        }
        dc[i * 33 + r] = G;
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
