// Cosine match matrix + RBF kernel pooling (KNRM / TK), forward and backward, CUDA-core version.
//
//   c_ij = <q^_i, d^_j>,  S_ik = sum_j dm_j exp(-(c_ij-mu_k)^2 / (2 sigma_k^2)),
//   score = sum_k w_k sum_i qm_i * log_scale * log(max(alpha_k S_ik, 1e-10))
//
// Reference arithmetic: matchmaker/models/knrm.py:52-84, models/published/ecai20_tk.py:105-124, and
// what torch autograd derives from them (SURVEY.md appendix A).  The reference materialises the
// [B,Lq,Ld,K] activation tensor and streams it through ~12 eager kernels (and saves several copies for
// backward); here one kernel per direction keeps the cosine tile and the K activations on chip, and
// backward recomputes them from the saved S[B,Lq,K].
//
// This file is the fp32-exact FFMA implementation: one CTA per pair, the normalised query block
// (32 rows) resident in shared memory, document rows streamed in tiles.  It serves every shape and is the
// validated baseline for the tensor-core kernels: forward kernel_pool_ts.cu, backward kernel_pool_bwd_wg.cu (the
// training pair mmb200_kernel_pool_fwd_train / _bwd_saved below routes to them).
#include <algorithm>

#include <cstdlib>

#include "device_util.cuh"
#include "host_util.cuh"
#include "kernel_pool.cuh"
#include "masks.cuh"

namespace mmb {

constexpr int kKpThreads = 256;
constexpr int kKpQ = 32;            // query rows per block pass

// Load `nrows` rows (row r of the tile = global row row0 + r, valid while < L) of a [L, D] matrix,
// L2-normalise them (x / (|x| + 1e-13)) and store into smem with stride dp.  Rows past L become zeros.
// One warp per row.  Optionally returns |x| and |x|+eps per row (backward).
__device__ __forceinline__ void kp_load_rows(const float* __restrict__ src, int row0, int L, int D, int dp, int nrows,
                                             float* __restrict__ dst, float* norm_out, float* s_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int d4 = D >> 2;
  for (int r = warp; r < nrows; r += nwarps) {
    float* drow = dst + (size_t)r * dp;
    const int g = row0 + r;
    if (g < L) {
      const float4* srow = reinterpret_cast<const float4*>(src + (size_t)g * D);
      float ss = 0.f;
      for (int c = lane; c < d4; c += 32) {
        const float4 v = __ldg(srow + c);
        ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
        *reinterpret_cast<float4*>(drow + 4 * c) = v;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float n = sqrtf(ss);
      const float s = n + kTinyNorm;
      const float inv = 1.0f / s;
      __syncwarp();
      for (int c = lane; c < d4; c += 32) {
        float4 v = *reinterpret_cast<float4*>(drow + 4 * c);
        v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
        *reinterpret_cast<float4*>(drow + 4 * c) = v;
      }
      if (lane == 0) {
        if (norm_out) norm_out[r] = n;
        if (s_out) s_out[r] = s;
      }
    } else {
      for (int c = lane; c < d4; c += 32) *reinterpret_cast<float4*>(drow + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (lane == 0) {
        if (norm_out) norm_out[r] = 0.f;
        if (s_out) s_out[r] = 1.f;
      }
    }
  }
}

// cos tile [32 x 32*JR]: thread t owns i = (t%8) + 8r (r<4), j = (t/8) + 32r' (r'<JR).
template <int JR>
__device__ __forceinline__ void kp_cos_tile(const float* __restrict__ qs, const float* __restrict__ ds, int D, int dp,
                                            float* __restrict__ cs, int cstride) {
  const int ti = threadIdx.x & 7, tj = threadIdx.x >> 3;
  float acc[4][JR];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < JR; ++s) acc[r][s] = 0.f;
  const int d4 = D >> 2;
  for (int c = 0; c < d4; ++c) {
    float4 qv[4], dv[JR];
#pragma unroll
    for (int r = 0; r < 4; ++r) qv[r] = *reinterpret_cast<const float4*>(qs + (size_t)(ti + 8 * r) * dp + 4 * c);
#pragma unroll
    for (int s = 0; s < JR; ++s) dv[s] = *reinterpret_cast<const float4*>(ds + (size_t)(tj + 32 * s) * dp + 4 * c);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < JR; ++s) {
        acc[r][s] = fmaf(qv[r].x, dv[s].x, acc[r][s]);
        acc[r][s] = fmaf(qv[r].y, dv[s].y, acc[r][s]);
        acc[r][s] = fmaf(qv[r].z, dv[s].z, acc[r][s]);
        acc[r][s] = fmaf(qv[r].w, dv[s].w, acc[r][s]);
      }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < JR; ++s) cs[(ti + 8 * r) * cstride + tj + 32 * s] = acc[r][s];
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
// The body of both forward entry points below; STORE: store mode (KpParams::doc_offsets), pair b reads query pair_q[b]
// and its passage's rows from the store
template <int KB, int JR, bool STORE>
__device__ __forceinline__ void kp_fwd_simt_body(const KpParams& P) {
  constexpr int TJ = 32 * JR;
  extern __shared__ __align__(16) float sm[];
  const int D = P.D, dp = padded_row_stride(D), Lq = P.Lq, Ld = P.Ld, K = P.K;
  float* qs = sm;                                  // [32][dp]
  float* ds = qs + (size_t)kKpQ * dp;              // [TJ][dp]
  float* cs = ds + (size_t)TJ * dp;                // [32][TJ+1]
  float* mu_s = cs + kKpQ * (TJ + 1);              // [32]
  float* a_s = mu_s + 32;                          // [32] sqrt(log2e / (2 sigma^2))
  float* al_s = a_s + 32;                          // [32] alpha
  float* w_s = al_s + 32;                          // [32] weight
  float* qm_s = w_s + 32;                          // [32]
  float* dm_s = qm_s + 32;                         // [TJ]
  float* pk_s = dm_s + TJ;                         // [32] per-kernel totals over query blocks
  float* lsm = pk_s + 32;                          // [KB][32]
  float* spart = lsm + KB * 32;                    // [8][KB][32]
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;

  if (t < 32) {
    const bool ok = t < K;
    mu_s[t] = ok ? P.mu[t] : 0.f;
    a_s[t] = ok ? rbf_scale(P.sigma[t]) : 0.f;
    al_s[t] = ok ? (P.alpha ? P.alpha[t] : 1.f) : 1.f;
    w_s[t] = ok ? P.weight[t] : 0.f;
  }
  for (int64_t b = blockIdx.x; b < P.B; b += gridDim.x) {
    int64_t qz = b, drow0 = b * (int64_t)Ld;   // query of the pair, first document row (and gate entry)
    int len = Ld;                              // document rows of the pair
    if constexpr (STORE) {
      qz = P.pair_q[b];
      len = kp_store_rows(P, b, &drow0);
    }
    const float* qb = P.q + qz * (int64_t)Lq * D;
    const float* db = P.d + drow0 * D;
    __syncthreads();
    if (t < 32) pk_s[t] = 0.f;
    for (int i0 = 0; i0 < Lq; i0 += kKpQ) {
      __syncthreads();
      kp_load_rows(qb, i0, Lq, D, dp, kKpQ, qs, nullptr, nullptr);
      if (t < 32) qm_s[t] = (i0 + t < Lq && mask_at(P.q_mask, P.q_mask ? P.mask_dtype : 0, qz * Lq + i0 + t)) ? 1.f : 0.f;
      float acc[KB];
#pragma unroll
      for (int k = 0; k < KB; ++k) acc[k] = 0.f;
      for (int j0 = 0; j0 < len; j0 += TJ) {
        __syncthreads();  // previous tile fully consumed
        kp_load_rows(db, j0, len, D, dp, TJ, ds, nullptr, nullptr);
        if (t < TJ) {   // dm_s = mask x gate: the weight of document term j in every activation sum
          const bool live = j0 + t < len && mask_at(P.d_mask, P.d_mask ? P.mask_dtype : 0, drow0 + j0 + t);
          dm_s[t] = live ? (P.gate ? fmaxf(P.gate[drow0 + j0 + t], 0.f) : 1.f) : 0.f;
        }
        __syncthreads();
        kp_cos_tile<JR>(qs, ds, D, dp, cs, TJ + 1);
        __syncthreads();
        if (P.cosine) {
          for (int e = t; e < kKpQ * TJ; e += kKpThreads) {
            const int i = e / TJ, j = e % TJ;
            if (i0 + i < Lq && j0 + j < Ld)
              P.cosine[(b * Lq + i0 + i) * (int64_t)Ld + j0 + j] =
                  cs[i * (TJ + 1) + j] * qm_s[i] *
                  (mask_at(P.d_mask, P.d_mask ? P.mask_dtype : 0, b * (int64_t)Ld + j0 + j) ? 1.f : 0.f);
          }
        }
        {  // kernel activations: thread = (query row i, eighth of the tile's document rows)
          const int i = lane, jg = warp;
#pragma unroll 1
          for (int jj = 0; jj < TJ / 8; ++jj) {
            const int j = jg * (TJ / 8) + jj;
            const float gj = dm_s[j];
            if (gj != 0.f) {  // warp-uniform
              const float c = cs[i * (TJ + 1) + j];
#pragma unroll
              for (int k = 0; k < KB; ++k) {
                const float u = (c - mu_s[k]) * a_s[k];
                acc[k] = fmaf(gj, ex2_approx(-u * u), acc[k]);
              }
            }
          }
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < KB; ++k) spart[(warp * KB + k) * 32 + lane] = acc[k];
      __syncthreads();
      for (int e = t; e < KB * 32; e += kKpThreads) {
        const int k = e >> 5, i = e & 31;
        float S = 0.f;
#pragma unroll
        for (int g = 0; g < 8; ++g) S += spart[(g * KB + k) * 32 + i];
        float L = 0.f;
        if (k < K && i0 + i < Lq) {
          if (P.per_kernel_query) P.per_kernel_query[(b * Lq + i0 + i) * (int64_t)K + k] = S;
          if (qm_s[i] != 0.f) L = P.log_scale * logf(fmaxf(S * al_s[k], P.clamp_min));
        }
        lsm[k * 32 + i] = L;
      }
      __syncthreads();
      for (int k = warp; k < KB; k += kKpThreads / 32) {
        float v = lsm[k * 32 + lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) pk_s[k] += v;
      }
    }
    __syncthreads();
    if (t < K && P.per_kernel) P.per_kernel[b * K + t] = pk_s[t];
    if (t == 0) {
      float s = 0.f;
      for (int k = 0; k < K; ++k) s = fmaf(pk_s[k], w_s[k], s);
      P.score[b] = STORE && len == 0 ? -INFINITY : s + P.bias;   // store mode: a pair without rows scores -inf
    }
  }
}

template <int KB, int JR>
__global__ void __launch_bounds__(kKpThreads) kernel_pool_fwd_simt(KpParams P) {
  kp_fwd_simt_body<KB, JR, false>(P);
}

// store mode (mmb200_kernel_pool_store_fwd); one CTA per SM: at the padded kernel's register choice (128) KB = 24 spills
template <int KB, int JR>
__global__ void __launch_bounds__(kKpThreads, 1) kernel_pool_fwd_simt_store(KpParams P) {
  kp_fwd_simt_body<KB, JR, true>(P);
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
template <int KB, int NC>
__global__ void __launch_bounds__(kKpThreads) kernel_pool_bwd_simt(KpParams P) {
  constexpr int TJ = 32;
  extern __shared__ __align__(16) float sm[];
  const int D = P.D, dp = padded_row_stride(D), Lq = P.Lq, Ld = P.Ld, K = P.K;
  float* qs = sm;                          // [32][dp] q^
  float* ds = qs + (size_t)32 * dp;        // [32][dp] d^
  float* gs = ds + (size_t)32 * dp;        // [32][dp] dd^ tile, later dq^
  float* cs = gs + (size_t)32 * dp;        // [32][33] cos
  float* Gs = cs + 32 * 33;                // [32 j][32 i]
  float* coef = Gs + 32 * 32;              // [32 i][KB]
  float* mu_s = coef + 32 * KB;            // [32]
  float* a_s = mu_s + 32;
  float* is2_s = a_s + 32;                 // 1 / sigma^2
  float* al_s = is2_s + 32;
  float* w_s = al_s + 32;
  float* qm_s = w_s + 32;
  float* dm_s = qm_s + 32;
  float* nq_s = dm_s + 32;                 // |q_i|
  float* sq_s = nq_s + 32;                 // |q_i| + eps
  float* nd_s = sq_s + 32;
  float* sd_s = nd_s + 32;
  float* pk_s = sd_s + 32;                 // [32] P_k over query blocks
  float* ga_s = pk_s + 32;                 // [32] d alpha over query blocks
  float* red = ga_s + 32;                  // [KB][32] scratch
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;

  if (t < 32) {
    const bool ok = t < K;
    const float sg = ok ? P.sigma[t] : 1.f;
    mu_s[t] = ok ? P.mu[t] : 0.f;
    a_s[t] = ok ? rbf_scale(sg) : 0.f;
    is2_s[t] = ok ? 1.0f / (sg * sg) : 0.f;
    al_s[t] = ok ? (P.alpha ? P.alpha[t] : 1.f) : 1.f;
    w_s[t] = ok ? P.weight[t] : 0.f;
  }
  for (int64_t b = blockIdx.x; b < P.B; b += gridDim.x) {
    const float* qb = P.q + b * (int64_t)Lq * D;
    const float* db = P.d + b * (int64_t)Ld * D;
    const float g = P.grad_score[b];
    __syncthreads();
    if (t < 32) { pk_s[t] = 0.f; ga_s[t] = 0.f; }
    for (int i0 = 0; i0 < Lq; i0 += 32) {
      __syncthreads();
      kp_load_rows(qb, i0, Lq, D, dp, 32, qs, nq_s, sq_s);
      if (t < 32) qm_s[t] = (i0 + t < Lq && mask_at(P.q_mask, P.q_mask ? P.mask_dtype : 0, b * (int64_t)Lq + i0 + t)) ? 1.f : 0.f;
      __syncthreads();
      // dS_ik (coef), and the per-pair pieces of d weight / d alpha
      for (int e = t; e < KB * 32; e += kKpThreads) {
        const int k = e >> 5, i = e & 31;
        float cf = 0.f, Lv = 0.f, da = 0.f;
        if (k < K && i0 + i < Lq && qm_s[i] != 0.f) {
          const float S = P.S[(b * Lq + i0 + i) * (int64_t)K + k];
          const float aS = S * al_s[k];
          Lv = P.log_scale * logf(fmaxf(aS, P.clamp_min));
          if (aS >= P.clamp_min) {  // torch.clamp passes the gradient at equality
            cf = g * w_s[k] * P.log_scale / S;
            da = g * w_s[k] * P.log_scale / al_s[k];
          }
        }
        coef[i * KB + k] = cf;
        red[k * 32 + i] = Lv;
        Gs[k * 32 + i] = da;  // Gs is free here; reused as scratch [KB<=32][32]
      }
      __syncthreads();
      for (int k = warp; k < KB; k += kKpThreads / 32) {
        float v = red[k * 32 + lane], u = Gs[k * 32 + lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          v += __shfl_xor_sync(0xffffffffu, v, o);
          u += __shfl_xor_sync(0xffffffffu, u, o);
        }
        if (lane == 0) { pk_s[k] += v; ga_s[k] += u; }
      }
      float accq[NC][32];
#pragma unroll
      for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) accq[c][i] = 0.f;

      for (int j0 = 0; j0 < Ld; j0 += TJ) {
        __syncthreads();
        kp_load_rows(db, j0, Ld, D, dp, TJ, ds, nd_s, sd_s);
        if (t < TJ) dm_s[t] = (j0 + t < Ld && mask_at(P.d_mask, P.d_mask ? P.mask_dtype : 0, b * (int64_t)Ld + j0 + t)) ? 1.f : 0.f;
        __syncthreads();
        kp_cos_tile<1>(qs, ds, D, dp, cs, 33);
        __syncthreads();
        {  // G_ij = dm_j g_j sum_k dS_ik K_ijk (-(c-mu_k)/sigma_k^2);  d gate_j = dm_j sum_i sum_k dS_ik K_ijk
          const int i = lane;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = warp + 8 * jj;
            float G = 0.f, H = 0.f;
            if (dm_s[j] != 0.f) {   // warp-uniform
              const float c = cs[i * 33 + j];
#pragma unroll
              for (int k = 0; k < KB; ++k) {
                const float diff = c - mu_s[k];
                const float u = diff * a_s[k];
                const float ck = coef[i * KB + k] * ex2_approx(-u * u);
                G = fmaf(ck, -diff * is2_s[k], G);
                H += ck;
              }
              if (P.gate) G *= fmaxf(P.gate[b * (int64_t)Ld + j0 + j], 0.f);
            }
            Gs[j * 32 + i] = G;
            if (P.grad_gate && j0 + j < Ld) {   // warp-uniform
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) H += __shfl_xor_sync(0xffffffffu, H, o);
              if (lane == 0) {
                // relu'(gate) = 0 for gate < 0 (the forward clamps a negative gate to 0)
                const float live = (P.gate && P.gate[b * (int64_t)Ld + j0 + j] < 0.f) ? 0.f : 1.f;
                float* gg = P.grad_gate + b * (int64_t)Ld + j0 + j;
                *gg = (i0 == 0) ? H * live : *gg + H * live;
              }
            }
          }
        }
        __syncthreads();
        // dd^_j[k] = sum_i G_ij q^_i[k];  dq^_i[k] += sum_j G_ij d^_j[k];  thread owns columns k = t + 256 c
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int k = t + kKpThreads * c;
          if (k < D) {
            float qcol[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) qcol[i] = qs[(size_t)i * dp + k];
#pragma unroll 2
            for (int j = 0; j < TJ; ++j) {
              const float dv = ds[(size_t)j * dp + k];
              float s = 0.f;
#pragma unroll
              for (int i4 = 0; i4 < 8; ++i4) {
                const float4 G4 = *reinterpret_cast<const float4*>(Gs + j * 32 + 4 * i4);
                s = fmaf(G4.x, qcol[4 * i4 + 0], s); accq[c][4 * i4 + 0] = fmaf(G4.x, dv, accq[c][4 * i4 + 0]);
                s = fmaf(G4.y, qcol[4 * i4 + 1], s); accq[c][4 * i4 + 1] = fmaf(G4.y, dv, accq[c][4 * i4 + 1]);
                s = fmaf(G4.z, qcol[4 * i4 + 2], s); accq[c][4 * i4 + 2] = fmaf(G4.z, dv, accq[c][4 * i4 + 2]);
                s = fmaf(G4.w, qcol[4 * i4 + 3], s); accq[c][4 * i4 + 3] = fmaf(G4.w, dv, accq[c][4 * i4 + 3]);
              }
              gs[(size_t)j * dp + k] = s;
            }
          }
        }
        __syncthreads();
        // through the normalisation: dd = dd^/s - d^ (d^ . dd^)/n   (second term 0 when n == 0)
        for (int r = warp; r < TJ; r += kKpThreads / 32) {
          const int j = j0 + r;
          if (j < Ld) {
            float dot = 0.f;
            for (int k = lane; k < D; k += 32) dot = fmaf(ds[(size_t)r * dp + k], gs[(size_t)r * dp + k], dot);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            const float inv_s = 1.0f / sd_s[r];
            const float f = nd_s[r] > 0.f ? dot / nd_s[r] : 0.f;
            float* out = P.grad_d + (b * Ld + j) * (int64_t)D;
            for (int k = lane; k < D; k += 32) {
              const float v = gs[(size_t)r * dp + k] * inv_s - ds[(size_t)r * dp + k] * f;
              out[k] = (i0 == 0) ? v : out[k] + v;
            }
          }
        }
      }
      __syncthreads();
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int k = t + kKpThreads * c;
        if (k < D) {
#pragma unroll
          for (int i = 0; i < 32; ++i) gs[(size_t)i * dp + k] = accq[c][i];
        }
      }
      __syncthreads();
      for (int r = warp; r < 32; r += kKpThreads / 32) {
        const int i = i0 + r;
        if (i < Lq) {
          float dot = 0.f;
          for (int k = lane; k < D; k += 32) dot = fmaf(qs[(size_t)r * dp + k], gs[(size_t)r * dp + k], dot);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
          const float inv_s = 1.0f / sq_s[r];
          const float f = nq_s[r] > 0.f ? dot / nq_s[r] : 0.f;
          float* out = P.grad_q + (b * Lq + i) * (int64_t)D;
          for (int k = lane; k < D; k += 32) out[k] = gs[(size_t)r * dp + k] * inv_s - qs[(size_t)r * dp + k] * f;
        }
      }
    }
    __syncthreads();
    if (t < K) {
      P.ws_weight[b * K + t] = g * pk_s[t];
      P.ws_alpha[b * K + t] = ga_s[t];
    }
  }
}

// grad_weight[k] = sum_b ws_weight[b,k]; grad_alpha likewise.  One block per kernel k, fixed summation order ->
// deterministic.  (One block for everything walked the batch with 128 dependent loads per thread: 40 us at B = 1024,
// a fifth of the tensor-core backward.)
__global__ void __launch_bounds__(256) kp_reduce_batch(const float* __restrict__ ws_w, const float* __restrict__ ws_a, float* gw,
                                                        float* ga, int64_t B, int K) {
  __shared__ float part[2][8];
  const int k = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  float sw[4] = {0.f, 0.f, 0.f, 0.f}, sa[4] = {0.f, 0.f, 0.f, 0.f};
  int64_t b = t;
  for (; b + 768 < B; b += 1024) {   // four independent loads in flight per thread
#pragma unroll
    for (int u = 0; u < 4; ++u) { sw[u] += ws_w[(b + 256 * u) * K + k]; sa[u] += ws_a[(b + 256 * u) * K + k]; }
  }
  for (; b < B; b += 256) { sw[0] += ws_w[b * K + k]; sa[0] += ws_a[b * K + k]; }
  float vw = (sw[0] + sw[1]) + (sw[2] + sw[3]), va = (sa[0] + sa[1]) + (sa[2] + sa[3]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vw += __shfl_xor_sync(0xffffffffu, vw, o);
    va += __shfl_xor_sync(0xffffffffu, va, o);
  }
  if (lane == 0) { part[0][warp] = vw; part[1][warp] = va; }
  __syncthreads();
  if (t == 0) {
    float a = 0.f, c = 0.f;
    for (int x = 0; x < 8; ++x) { a += part[0][x]; c += part[1][x]; }
    if (gw) gw[k] = a;
    if (ga) ga[k] = c;
  }
}

// ---------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------

// An empty batch (B == 0) is valid: its per-pair tensors are empty, so their pointers may be null (torch hands out a null
// data pointer for an empty tensor).
static int kp_validate(const KpParams& P) {
  MMB_REQUIRE(P.mu && P.sigma && P.weight, "null pointer");
  MMB_REQUIRE(P.B == 0 || (P.q && P.d), "null pointer");
  MMB_REQUIRE(P.B >= 0 && P.Lq > 0 && P.Ld > 0 && P.D > 0, "bad shape");
  MMB_REQUIRE(P.D % 4 == 0, "embedding dim must be a multiple of 4 floats (16-byte rows)");
  MMB_REQUIRE(P.K >= 1 && P.K <= 32, "1 <= K <= 32 kernels supported");
  MMB_REQUIRE(((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d)) & 15) == 0, "q/d must be 16-byte aligned");
  if (P.q_mask || P.d_mask) MMB_REQUIRE(mask_dtype_size(P.mask_dtype) != 0, "unknown mask dtype");
  return MMB200_OK;
}

template <int KB, int JR, bool STORE = false>
static int launch_fwd(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream) {
  const int dp = padded_row_stride(P.D), TJ = 32 * JR;
  const size_t need = ((size_t)(kKpQ + TJ) * dp + kKpQ * (TJ + 1) + 32 * 6 + TJ + (size_t)9 * KB * 32) * sizeof(float);
  if (need > (size_t)dev.max_smem_optin) {
    set_error("kernel_pool forward: embedding dim too large for the shared-memory tiles");
    return MMB200_ERR_UNSUPPORTED;
  }
  const int grid = (int)std::min<int64_t>(P.B, (int64_t)dev.sm_count * 4);
  if constexpr (STORE) {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_fwd_simt_store<KB, JR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    kernel_pool_fwd_simt_store<KB, JR><<<grid, kKpThreads, need, stream>>>(P);
  } else {
    MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_fwd_simt<KB, JR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
    kernel_pool_fwd_simt<KB, JR><<<grid, kKpThreads, need, stream>>>(P);
  }
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

template <int KB, int NC>
static int launch_bwd(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream) {
  const int dp = padded_row_stride(P.D);
  const size_t need = ((size_t)3 * 32 * dp + 32 * 33 + 32 * 32 + 32 * KB + 32 * 13 + (size_t)KB * 32) * sizeof(float);
  if (need > (size_t)dev.max_smem_optin) {
    set_error("kernel_pool backward: embedding dim too large for the shared-memory tiles");
    return MMB200_ERR_UNSUPPORTED;
  }
  MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_bwd_simt<KB, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need));
  const int grid = (int)std::min<int64_t>(P.B, (int64_t)dev.sm_count * 4);
  kernel_pool_bwd_simt<KB, NC><<<grid, kKpThreads, need, stream>>>(P);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

// the envelope of the tensor-core training pair (forward that saves its cosines + backward that consumes them): D <= 320
// on kernel_pool_bwd_wg.cu, 512 < D <= 1024 in whole 64-feature blocks (BERT widths) on kernel_pool_wide.cu
static bool kp_train_tc_shape_ok(int Lq, int Ld, int D, int K) {
  return (Lq >= 1 && Lq <= 32 && Ld >= 1 && K >= 1 && K <= 32 && D >= 4 && D % 4 == 0 && D <= 320) ||
         kp_wide_shape_ok(Lq, Ld, D, K);
}

// first float of the wide backward's part of the workspace, after ws_weight / ws_alpha (16-byte aligned)
static int64_t kp_wide_ws_off(int64_t B, int K) { return (2 * B * K + 3) / 4 * 4; }

static int kp_fwd_impl(const float* q, const float* d, const void* q_mask, const void* d_mask, const float* doc_gate,
                       const float* mu, const float* sigma, const float* alpha, const float* weight, float* score,
                       float* per_kernel, float* per_kernel_query, float* cosine, float* saved, int64_t B, int32_t Lq,
                       int32_t Ld, int32_t D, int32_t K, float log_scale, float clamp_min, float score_bias,
                       int32_t mask_dtype, int32_t impl, void* stream_) {
  MMB_REQUIRE(clamp_min > 0.f, "clamp_min must be positive");
  KpParams P{};
  P.saved = saved;
  P.gate = doc_gate; P.clamp_min = clamp_min; P.bias = score_bias;
  P.q = q; P.d = d; P.q_mask = q_mask; P.d_mask = d_mask; P.mu = mu; P.sigma = sigma; P.alpha = alpha; P.weight = weight;
  P.B = B; P.Lq = Lq; P.Ld = Ld; P.D = D; P.K = K; P.mask_dtype = mask_dtype; P.log_scale = log_scale;
  P.score = score; P.per_kernel = per_kernel; P.per_kernel_query = per_kernel_query; P.cosine = cosine;
  if (int rc = kp_validate(P)) return rc;
  MMB_REQUIRE(score != nullptr || B == 0, "score must be non-null");
  if (B == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (impl != MMB200_IMPL_SIMT) {
    bool handled = false;
    int rc = kernel_pool_fwd_ts(P, dev, stream, &handled);
    if (handled) return rc;
    if (impl == MMB200_IMPL_TCGEN05) {
      if (rc == MMB200_OK) { set_error("kernel_pool: shape not supported by the tensor-core kernel"); rc = MMB200_ERR_UNSUPPORTED; }
      return rc;
    }
  }
  const bool wide = Ld > 48;
  if (K <= 12) return wide ? launch_fwd<12, 2>(P, dev, stream) : launch_fwd<12, 1>(P, dev, stream);
  if (K <= 24) return wide ? launch_fwd<24, 2>(P, dev, stream) : launch_fwd<24, 1>(P, dev, stream);
  return wide ? launch_fwd<32, 2>(P, dev, stream) : launch_fwd<32, 1>(P, dev, stream);
}

// store mode: the routing of kp_fwd_impl (tensor-core kernel when it takes the shape, else the FFMA kernel with the tile
// width the padded [n_docs, max_doc_len, D] layout would get), so scores are bit-identical to that layout
static int kp_store_fwd_impl(KpParams& P, int32_t impl, cudaStream_t stream) {
  MMB_REQUIRE(P.clamp_min > 0.f, "clamp_min must be positive");
  if (int rc = kp_validate(P)) return rc;
  MMB_REQUIRE(P.B == 0 || (P.doc_offsets && P.pair_q && P.pair_d && P.score), "null pointer");
  MMB_REQUIRE(P.n_q >= 1 && P.n_rows >= 1, "the store needs at least one row and one query");
  MMB_REQUIRE(P.n_rows < (1ll << 31) - 1024, "at most 2^31 - 1024 store rows per device (TMA row coordinates are int32)");
  if (P.B == 0) return MMB200_OK;
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  if (impl != MMB200_IMPL_SIMT) {
    bool handled = false;
    int rc = kernel_pool_fwd_ts(P, dev, stream, &handled);
    if (handled) return rc;
    if (impl == MMB200_IMPL_TCGEN05) {
      if (rc == MMB200_OK) { set_error("kernel_pool_store: shape not supported by the tensor-core kernel"); rc = MMB200_ERR_UNSUPPORTED; }
      return rc;
    }
  }
  const bool wide = P.Ld > 48;
  if (P.K <= 12) return wide ? launch_fwd<12, 2, true>(P, dev, stream) : launch_fwd<12, 1, true>(P, dev, stream);
  if (P.K <= 24) return wide ? launch_fwd<24, 2, true>(P, dev, stream) : launch_fwd<24, 1, true>(P, dev, stream);
  return wide ? launch_fwd<32, 2, true>(P, dev, stream) : launch_fwd<32, 1, true>(P, dev, stream);
}

static int kp_bwd_impl(const float* q, const float* d, const void* q_mask, const void* d_mask, const float* doc_gate,
                       const float* mu, const float* sigma, const float* alpha, const float* weight,
                       const float* per_kernel_query, const float* saved, const float* grad_score, float* grad_q,
                       float* grad_d, float* grad_gate, float* grad_alpha, float* grad_weight, float* workspace,
                       int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K, float log_scale, float clamp_min,
                       int32_t mask_dtype, bool from_saved, void* stream_) {
  MMB_REQUIRE(clamp_min > 0.f, "clamp_min must be positive");
  KpParams P{};
  P.saved = const_cast<float*>(saved);
  // the tensor core drops the low 13 mantissa bits of the raw fp32 tiles: relative shrink 2^-10 u / m with u uniform in
  // [0, 1) and the mantissa m log-uniform in [1, 2) -> mean 2^-11 / ln 2 * (1 - 1/2) = 0.72 * 2^-11
  P.tf32_comp = 1.0f + 0.72f / 2048.0f;
#ifdef MMB200_ENABLE_PROF
  if (const char* e = getenv("MMB200_KPB_COMP")) P.tf32_comp = (float)atof(e);
#endif
  P.gate = doc_gate; P.clamp_min = clamp_min; P.grad_gate = grad_gate;
  P.q = q; P.d = d; P.q_mask = q_mask; P.d_mask = d_mask; P.mu = mu; P.sigma = sigma; P.alpha = alpha; P.weight = weight;
  P.B = B; P.Lq = Lq; P.Ld = Ld; P.D = D; P.K = K; P.mask_dtype = mask_dtype; P.log_scale = log_scale;
  P.S = per_kernel_query; P.grad_score = grad_score; P.grad_q = grad_q; P.grad_d = grad_d;
  if (int rc = kp_validate(P)) return rc;
  MMB_REQUIRE(B == 0 || (per_kernel_query && grad_score && grad_q && grad_d && workspace), "null pointer");
  const bool wide = from_saved && kp_wide_shape_ok(Lq, Ld, D, K);   // BERT widths, from the saved state (null when B = 0)
  MMB_REQUIRE(D <= 512 || wide, "kernel_pool backward supports embedding dim <= 512");
  P.ws_weight = workspace;
  P.ws_alpha = workspace + B * K;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (B == 0) {   // the weight and alpha gradients are sums over no pairs
    if (grad_weight) MMB_CHECK_CUDA(cudaMemsetAsync(grad_weight, 0, (size_t)K * sizeof(float), stream));
    if (grad_alpha) MMB_CHECK_CUDA(cudaMemsetAsync(grad_alpha, 0, (size_t)K * sizeof(float), stream));
    return MMB200_OK;
  }
  DeviceInfo dev;
  if (int rc = require_sm90(&dev)) return rc;
  int rc;
  if (wide) {
    if ((rc = kernel_pool_bwd_wide(P, workspace + kp_wide_ws_off(B, K), dev, stream))) return rc;
    kp_reduce_batch<<<K, 256, 0, stream>>>(P.ws_weight, P.ws_alpha, grad_weight, grad_alpha, B, K);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  }
  if (saved) {
    bool handled = false;
    rc = kernel_pool_bwd_tc(P, dev, stream, &handled);
    if (!handled) {
      if (rc == MMB200_OK) { set_error("kernel_pool_bwd_saved: arguments outside the tensor-core backward's envelope"); rc = MMB200_ERR_UNSUPPORTED; }
      return rc;
    }
    if (rc) return rc;
    kp_reduce_batch<<<K, 256, 0, stream>>>(P.ws_weight, P.ws_alpha, grad_weight, grad_alpha, B, K);
    MMB_CHECK_CUDA(cudaGetLastError());
    return MMB200_OK;
  }
  if (D <= 256) {
    if (K <= 12) rc = launch_bwd<12, 1>(P, dev, stream);
    else if (K <= 24) rc = launch_bwd<24, 1>(P, dev, stream);
    else rc = launch_bwd<32, 1>(P, dev, stream);
  } else {
    if (K <= 12) rc = launch_bwd<12, 2>(P, dev, stream);
    else if (K <= 24) rc = launch_bwd<24, 2>(P, dev, stream);
    else rc = launch_bwd<32, 2>(P, dev, stream);
  }
  if (rc) return rc;
  kp_reduce_batch<<<K, 256, 0, stream>>>(P.ws_weight, P.ws_alpha, grad_weight, grad_alpha, B, K);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

}  // namespace mmb

extern "C" int mmb200_kernel_pool_fwd(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                      const float* mu, const float* sigma, const float* alpha, const float* weight,
                                      float* score, float* per_kernel, float* per_kernel_query, float* cosine,
                                      int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K, float log_scale,
                                      int32_t mask_dtype, int32_t impl, void* stream_) {
  return mmb200_kernel_pool_fwd_ex(q, d, q_mask, d_mask, nullptr, mu, sigma, alpha, weight, score, per_kernel,
                                   per_kernel_query, cosine, B, Lq, Ld, D, K, log_scale, 1e-10f, 0.f, mask_dtype, impl, stream_);
}

extern "C" int mmb200_kernel_pool_fwd_ex(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                         const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                         const float* weight, float* score, float* per_kernel, float* per_kernel_query,
                                         float* cosine, int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K,
                                         float log_scale, float clamp_min, float score_bias, int32_t mask_dtype,
                                         int32_t impl, void* stream_) {
  return mmb::kp_fwd_impl(q, d, q_mask, d_mask, doc_gate, mu, sigma, alpha, weight, score, per_kernel, per_kernel_query,
                          cosine, nullptr, B, Lq, Ld, D, K, log_scale, clamp_min, score_bias, mask_dtype, impl, stream_);
}

extern "C" int mmb200_kernel_pool_store_fwd(const float* q, const void* q_mask, const float* store,
                                            const int64_t* doc_offsets, const float* gate, const int32_t* pair_q,
                                            const int32_t* pair_d, const float* mu, const float* sigma,
                                            const float* alpha, const float* weight, float* score, int64_t n_q,
                                            int64_t n_rows, int64_t n_pairs, int32_t Lq, int32_t max_doc_len,
                                            int32_t D, int32_t K, float log_scale, float clamp_min, float score_bias,
                                            int32_t mask_dtype, int32_t impl, void* stream) {
  mmb::KpParams P{};
  P.q = q; P.d = store; P.q_mask = q_mask; P.gate = gate; P.mu = mu; P.sigma = sigma; P.alpha = alpha; P.weight = weight;
  P.B = n_pairs; P.Lq = Lq; P.Ld = max_doc_len; P.D = D; P.K = K; P.mask_dtype = mask_dtype; P.log_scale = log_scale;
  P.clamp_min = clamp_min; P.bias = score_bias; P.score = score;
  P.doc_offsets = doc_offsets; P.pair_q = pair_q; P.pair_d = pair_d; P.n_q = n_q; P.n_rows = n_rows;
  return mmb::kp_store_fwd_impl(P, impl, static_cast<cudaStream_t>(stream));
}

extern "C" int32_t mmb200_kernel_pool_train_tc_supported(int32_t Lq, int32_t Ld, int32_t D, int32_t K) {
  return mmb::kp_train_tc_shape_ok(Lq, Ld, D, K) ? 1 : 0;
}

extern "C" int64_t mmb200_kernel_pool_saved_floats(int64_t B, int32_t Ld) { return mmb::kp_saved_floats(B, Ld); }

extern "C" int64_t mmb200_kernel_pool_bwd_saved_workspace_floats(int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K) {
  if (!mmb::kp_wide_shape_ok(Lq, Ld, D, K)) return 2 * B * K;
  return mmb::kp_wide_ws_off(B, K) + mmb::kp_wide_ws_floats(B, Ld);
}

extern "C" int mmb200_kernel_pool_fwd_train(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                            const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                            const float* weight,
                                            float* score, float* per_kernel, float* per_kernel_query, float* saved,
                                            int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K, float log_scale,
                                            float clamp_min, float score_bias, int32_t mask_dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE((saved != nullptr && per_kernel_query != nullptr) || B == 0, "saved and per_kernel_query must be non-null");
  if (!kp_train_tc_shape_ok(Lq, Ld, D, K)) {
    set_error("kernel_pool_fwd_train: shape outside the tensor-core training envelope (Lq <= 32, K <= 32; D % 4 == 0 and D <= 320, or D % 64 == 0 and 512 < D <= 1024)");
    return MMB200_ERR_UNSUPPORTED;
  }
  return kp_fwd_impl(q, d, q_mask, d_mask, doc_gate, mu, sigma, alpha, weight, score, per_kernel, per_kernel_query, nullptr,
                     saved, B, Lq, Ld, D, K, log_scale, clamp_min, score_bias, mask_dtype, MMB200_IMPL_TCGEN05, stream_);
}

extern "C" int mmb200_kernel_pool_bwd_saved(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                            const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                            const float* weight, const float* per_kernel_query, const float* saved,
                                            const float* grad_score, float* grad_q, float* grad_d, float* grad_gate,
                                            float* grad_alpha, float* grad_weight,
                                            float* workspace, int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K,
                                            float log_scale, float clamp_min, int32_t mask_dtype, void* stream_) {
  using namespace mmb;
  MMB_REQUIRE(saved != nullptr || B == 0, "saved must be non-null");
  if (!kp_train_tc_shape_ok(Lq, Ld, D, K)) {
    set_error("kernel_pool_bwd_saved: shape outside the tensor-core training envelope (Lq <= 32, K <= 32; D % 4 == 0 and D <= 320, or D % 64 == 0 and 512 < D <= 1024)");
    return MMB200_ERR_UNSUPPORTED;
  }
  return kp_bwd_impl(q, d, q_mask, d_mask, doc_gate, mu, sigma, alpha, weight, per_kernel_query, saved, grad_score, grad_q,
                     grad_d, grad_gate, grad_alpha, grad_weight, workspace, B, Lq, Ld, D, K, log_scale, clamp_min, mask_dtype,
                     true, stream_);
}

extern "C" int mmb200_kernel_pool_bwd(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                      const float* mu, const float* sigma, const float* alpha, const float* weight,
                                      const float* per_kernel_query, const float* grad_score, float* grad_q,
                                      float* grad_d, float* grad_alpha, float* grad_weight, float* workspace,
                                      int64_t B, int32_t Lq, int32_t Ld, int32_t D, int32_t K, float log_scale,
                                      int32_t mask_dtype, void* stream_) {
  return mmb200_kernel_pool_bwd_ex(q, d, q_mask, d_mask, nullptr, mu, sigma, alpha, weight, per_kernel_query, grad_score,
                                   grad_q, grad_d, nullptr, grad_alpha, grad_weight, workspace, B, Lq, Ld, D, K, log_scale,
                                   1e-10f, mask_dtype, stream_);
}

extern "C" int mmb200_kernel_pool_bwd_ex(const float* q, const float* d, const void* q_mask, const void* d_mask,
                                         const float* doc_gate, const float* mu, const float* sigma, const float* alpha,
                                         const float* weight, const float* per_kernel_query, const float* grad_score,
                                         float* grad_q, float* grad_d, float* grad_gate, float* grad_alpha,
                                         float* grad_weight, float* workspace, int64_t B, int32_t Lq, int32_t Ld,
                                         int32_t D, int32_t K, float log_scale, float clamp_min, int32_t mask_dtype,
                                         void* stream_) {
  return mmb::kp_bwd_impl(q, d, q_mask, d_mask, doc_gate, mu, sigma, alpha, weight, per_kernel_query, nullptr, grad_score,
                          grad_q, grad_d, grad_gate, grad_alpha, grad_weight, workspace, B, Lq, Ld, D, K, log_scale, clamp_min,
                          mask_dtype, false, stream_);
}
