// Cosine + RBF kernel pooling BACKWARD (KNRM / TK training step) on the tensor cores.
//
// Reference arithmetic: autograd through matchmaker/modules/cosine... -> models/knrm.py:52-84 /
// models/published/ecai20_tk.py:105-124 (restated in oracle/interaction_oracle.py, kernel_pool_backward).
//
// With c_ij the cosine, S_ik the pooled activations the forward saved and coef_ik = g w_k s / S_ik (0 for masked query
// terms and below the clamp):
//
//     G_ij  = dm_j * sum_k coef_ik K_ijk (mu_k - c_ij) / sigma_k^2                  (d loss / d c_ij)
//     dd^_j = sum_i G_ij q_i / (|q_i| + eps)          dq^_i = sum_j G_ij d_j / (|d_j| + eps)
//     dd_j  = dd^_j / (|d_j| + eps) - d_j (d^_j . dd^_j) / (|d_j| (|d_j| + eps)),  d^_j . dd^_j = sum_i G_ij c_ij
//     dq_i  likewise with q^_i . dq^_i = sum_j G_ij c_ij (per-warp partial sums, added in a fixed order).
//
// The cosines are not recomputed: the training forward (kernel_pool_ts_kernel<.., SAVE>) leaves them document-row-major
// together with the inverse norms (KpParams::saved).
//
// Both contractions run as wgmma kind tf32 with the FEATURES on M, so that both B operands are K-major (tf32 wgmma reads
// no MN-major operand) and are the G matrices the kernel writes itself; the embeddings are the A operand, gathered from
// shared memory into registers (the raw fp32 bits: the tensor core truncates them to tf32):
//
//   GEMM 1  dd^T[64 features x 64 doc rows]  = Q^T[64 features x 32 query rows]   * G1^T   (G1 [doc row][query row] = G / (|q| + eps))
//   GEMM 2  dq^T[64 features x 32 query rows] += D^T[64 features x 64 doc rows]    * G2     (G2^T [query row][doc row] = G / (|d| + eps))
//
// Per CTA (persistent over a contiguous range of pairs, 384 threads = 3 warpgroups), per pair: the query tile and the
// coefficient table, then per tile of 64 document rows: the document tile (all threads), G / G1 / G2 and the row terms
// (warps 0-7, thread = (document row, 8 query rows)), then the two GEMMs per 64-feature block (warpgroup w takes blocks
// w, w + 3), the document gradient written straight from the GEMM 1 accumulator; the query gradient at the end of the pair
// from the GEMM 2 accumulators, which stay in registers across the tiles.
//
// Operand precision: G is rounded to tf32 (cvt.rna); the raw embeddings are truncated by the tensor core (low 13 mantissa
// bits dropped, mean relative shrink 0.72 * 2^-11), which KpParams::tf32_comp undoes on average.
#include <algorithm>

#include "device_util.cuh"
#include "host_util.cuh"
#include "kernel_pool.cuh"
#include "masks.cuh"
#include "ptx.cuh"

namespace mmb {

namespace {

constexpr int kThreads = 384;
constexpr int kTile = 64;                 // document rows per tile (wgmma N of GEMM 1, K of GEMM 2)
constexpr int kMaxD = 320;
constexpr int kMaxFb = 2;                 // 64-feature blocks per warpgroup (D <= 320: 5 blocks over 3 warpgroups)
constexpr int kG1Bytes = kTile * 128;     // G1 [64 doc rows][32 query rows] fp32, K-major SWIZZLE_128B
constexpr int kG2Bytes = 2 * 32 * 128;    // G2^T [2 k-blocks][32 query rows][32 doc rows], K-major SWIZZLE_128B

__host__ __device__ inline int pitch_of(int D) { return (D + 63) / 64 * 64 + 8; }   // floats per row: 8 mod 32, conflict-free A gathers

template <int KBP>
struct BwShared {
  alignas(16) float T[KBP][32];      // [kernel][query row]: coef_ik / sigma_k^2
  float rsq[32];                     // 1 / (|q_i| + eps) of the pair
  float rsd[kTile];                  // 1 / (|d_j| + eps) of the tile's rows
  float pr[kTile];                   // (d^_j . dd^_j) / |d_j| times 1 / (|d_j| + eps); 0 for a zero row
  float ci[8][32];                   // [G warp][query row]: sum_j G_ij c_ij of the pair
  float mu[32], a[32], is2[32], sig2[32], alpha[32], w[32];
};

template <int KB, bool GATE>
__global__ void __launch_bounds__(kThreads, 1)
kernel_pool_bwd_tc_kernel(KpParams P) {
  constexpr int KBP = (KB + 3) & ~3;
  using Shared = BwShared<KBP>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int DP = pitch_of(P.D);
  uint8_t* g1 = smem;                                                  // SWIZZLE_128B operands first (1024-B aligned)
  uint8_t* g2 = g1 + kG1Bytes;
  float* qs = reinterpret_cast<float*>(g2 + kG2Bytes);                 // [32][DP] query rows (zero past Lq / D)
  float* ds = qs + 32 * DP;                                            // [64][DP] document tile (zero past Ld / D)
  Shared* S = reinterpret_cast<Shared*>(ds + kTile * DP);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles = (P.Ld + kTile - 1) / kTile;
  const int nfb = (P.D + 63) / 64;
  const int D4 = P.D >> 2, DP4 = DP >> 2;
  int64_t p_begin, p_end;
  cta_share(P.B, &p_begin, &p_end);

  if (tid < 32) {
    const bool ok = tid < P.K;
    const float sg = ok ? P.sigma[tid] : 1.f;
    S->mu[tid] = ok ? P.mu[tid] : 0.f;
    S->a[tid] = ok ? rbf_scale(sg) : 0.f;
    S->is2[tid] = ok ? 1.0f / (sg * sg) : 0.f;
    S->sig2[tid] = ok ? sg * sg : 0.f;
    S->alpha[tid] = ok ? (P.alpha ? P.alpha[tid] : 1.f) : 1.f;
    S->w[tid] = ok ? P.weight[tid] : 0.f;
  }
  // GEMM roles: warpgroup wg, feature blocks wg and wg + 3; thread rows (features) fr, fr + 8 of a block
  const int wg = warp >> 2, wq = warp & 3, tq = lane & 3;
  const int fr = 16 * wq + (lane >> 2);
  // G roles (warps 0-7): document row gj of the tile, query rows gi .. gi + 7
  const int gj = tid >> 2, gi = (tid & 3) * 8;
  const int dmt = P.d_mask ? P.mask_dtype : MMB200_MASK_NONE;
  const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
  __syncthreads();

  for (int64_t p = p_begin; p < p_end; ++p) {
    // ---- query tile, coefficient table, d weight / d alpha ----
    for (int e = tid; e < 32 * DP4; e += kThreads) {
      const int i = e / DP4, c4 = e - i * DP4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < P.Lq && c4 < D4) v = *reinterpret_cast<const float4*>(P.q + (p * P.Lq + i) * (int64_t)P.D + 4 * c4);
      reinterpret_cast<float4*>(qs)[e] = v;
    }
    if (warp == 0) {
      const float g = P.grad_score[p];
      const bool qlive = lane < P.Lq && mask_at(P.q_mask, qmt, p * (int64_t)P.Lq + lane);
      float Sr[KBP];   // the row's pooled activations, loaded back to back
#pragma unroll
      for (int k = 0; k < KBP; ++k) Sr[k] = (k < P.K && qlive) ? P.S[(p * P.Lq + lane) * (int64_t)P.K + k] : 1.f;
#pragma unroll
      for (int k = 0; k < KBP; ++k) {
        float cf = 0.f, Lv = 0.f, da = 0.f;
        if (k < P.K && qlive) {
          const float Sv = Sr[k];
          const float aS = Sv * S->alpha[k];
          Lv = P.log_scale * logf(fmaxf(aS, P.clamp_min));
          if (aS >= P.clamp_min) {   // torch.clamp passes the gradient at equality
            cf = g * S->w[k] * P.log_scale / Sv;
            da = g * S->w[k] * P.log_scale / S->alpha[k];
          }
        }
        S->T[k][lane] = cf * S->is2[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          Lv += __shfl_xor_sync(0xffffffffu, Lv, o);
          da += __shfl_xor_sync(0xffffffffu, da, o);
        }
        if (lane == 0 && k < P.K) {
          P.ws_weight[p * P.K + k] = g * Lv;
          P.ws_alpha[p * P.K + k] = da;
        }
      }
      S->rsq[lane] = P.saved[kp_saved_rsq_off(P.B, p, P.Ld) + lane];
    }
    float dq[kMaxFb][16];
#pragma unroll
    for (int b = 0; b < kMaxFb; ++b)
#pragma unroll
      for (int j = 0; j < 16; ++j) dq[b][j] = 0.f;
    float ci_acc[8];   // lanes 0..3 of each G warp: sum over the warp's rows of G_ij c_ij, query rows gi .. gi + 7
#pragma unroll
    for (int y = 0; y < 8; ++y) ci_acc[y] = 0.f;

    for (int t = 0; t < tiles; ++t) {
      const int t0 = t * kTile;
      __syncthreads();   // the previous tile's operands are no longer read; the query tile and the table are written
      for (int e = tid; e < kTile * DP4; e += kThreads) {
        const int j = e / DP4, c4 = e - j * DP4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t0 + j < P.Ld && c4 < D4) v = *reinterpret_cast<const float4*>(P.d + (p * P.Ld + t0 + j) * (int64_t)P.D + 4 * c4);
        reinterpret_cast<float4*>(ds)[e] = v;
      }
      if (warp < 8) {
        // ---- G, the GEMM operands G1 / G2^T, the row terms ----
        const int j = t0 + gj;
        const bool inb = j < P.Ld;
        bool valid = false;
        float rsd = 0.f;
        if (inb) {
          valid = mask_at(P.d_mask, dmt, p * (int64_t)P.Ld + j);
          rsd = P.saved[kp_saved_rsd_off(P.B, p, P.Ld) + j];
        }
        float c[8], G[8];
#pragma unroll
        for (int y = 0; y < 8; ++y) { c[y] = 0.f; G[y] = 0.f; }
        if (valid && gi < P.Lq) {
          const float4* crow = reinterpret_cast<const float4*>(P.saved + kp_saved_cos_off(p, P.Ld) + (int64_t)j * 32 + gi);
          const float4 v0 = crow[0], v1 = crow[1];
          c[0] = v0.x; c[1] = v0.y; c[2] = v0.z; c[3] = v0.w; c[4] = v1.x; c[5] = v1.y; c[6] = v1.z; c[7] = v1.w;
        }
        float H = 0.f;   // GATE: sum_i sum_k coef_ik K_ijk = d loss / d gate_j (this thread's 8 query rows)
        if (__any_sync(0xffffffffu, valid && gi < P.Lq)) {
#pragma unroll 3
          for (int k = 0; k < KB; ++k) {
            const float mu_k = S->mu[k], a_k = S->a[k];
            const float sig2_k = GATE ? S->sig2[k] : 0.f;
            const float4 T0 = *reinterpret_cast<const float4*>(&S->T[k][gi]), T1 = *reinterpret_cast<const float4*>(&S->T[k][gi + 4]);
            const float Tv[8] = {T0.x, T0.y, T0.z, T0.w, T1.x, T1.y, T1.z, T1.w};
#pragma unroll
            for (int y = 0; y < 8; ++y) {
              const float diff = mu_k - c[y];
              const float u = diff * a_k;
              const float te = Tv[y] * ex2_approx(-u * u);
              G[y] = fmaf(te, diff, G[y]);
              if constexpr (GATE) H = fmaf(te, sig2_k, H);
            }
          }
        }
        float gate_j = 1.f, gv = 0.f;
        if constexpr (GATE) {
          gv = valid ? P.gate[p * (int64_t)P.Ld + j] : 0.f;
          gate_j = fmaxf(gv, 0.f);   // the forward counts a negative gate as 0: relu'(gate) = 0 there
        }
        float cpr = 0.f, gc[8];
#pragma unroll
        for (int y = 0; y < 8; ++y) {
          G[y] = valid ? G[y] * gate_j : 0.f;
          gc[y] = G[y] * c[y];
          cpr += gc[y];
        }
        cpr += __shfl_xor_sync(0xffffffffu, cpr, 1);
        cpr += __shfl_xor_sync(0xffffffffu, cpr, 2);
        // G1 [doc row][query row]: G_ij / (|q_i| + eps), two 16-byte chunks of the row
        {
          uint32_t g1v[8];
#pragma unroll
          for (int y = 0; y < 8; ++y) g1v[y] = f32_to_tf32_rna(G[y] * S->rsq[gi + y]);
#pragma unroll
          for (int h = 0; h < 2; ++h)
            *reinterpret_cast<uint4*>(g1 + gj * 128 + ((((gi >> 2) + h) ^ (gj & 7)) << 4)) =
                make_uint4(g1v[4 * h], g1v[4 * h + 1], g1v[4 * h + 2], g1v[4 * h + 3]);
        }
        // G2^T [query row][doc row]: G_ij / (|d_j| + eps), k-block gj / 32
        {
          uint8_t* g2b = g2 + (gj >> 5) * (32 * 128);
          const int jj = gj & 31;
#pragma unroll
          for (int y = 0; y < 8; ++y) {
            const int i = gi + y;
            *reinterpret_cast<uint32_t*>(g2b + i * 128 + (((jj >> 2) ^ (i & 7)) << 4) + ((jj & 3) << 2)) = f32_to_tf32_rna(G[y] * rsd);
          }
        }
        if constexpr (GATE) {
          H += __shfl_xor_sync(0xffffffffu, H, 1);
          H += __shfl_xor_sync(0xffffffffu, H, 2);
          if (tq == 0 && inb && P.grad_gate) P.grad_gate[p * (int64_t)P.Ld + j] = (valid && gv >= 0.f) ? H : 0.f;
        }
        if (tq == 0) {
          S->rsd[gj] = rsd;
          S->pr[gj] = rsd * cpr * (rsd < 1e12f ? rsd : 0.f);   // 0 for a zero row
        }
        // q^_i . dq^_i = sum_j G_ij c_ij: over the warp's 8 rows (lanes with the same lane % 4 hold the same query rows)
#pragma unroll
        for (int y = 0; y < 8; ++y) {
          float v = gc[y];
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          v += __shfl_xor_sync(0xffffffffu, v, 8);
          v += __shfl_xor_sync(0xffffffffu, v, 16);
          ci_acc[y] += v;
        }
      }
      fence_proxy_async_smem();   // G1 / G2^T are read by the tensor core (async proxy)
      __syncthreads();
      // ---- the two GEMMs per 64-feature block ----
#pragma unroll
      for (int b = 0; b < kMaxFb; ++b) {
        const int fb = wg + 3 * b;
        if (fb >= nfb) break;   // warpgroup-uniform
        const int f0 = 64 * fb + fr, f1 = f0 + 8;
        // GEMM 1: A = Q^T (features x query rows), K = 32 query rows
        float dd[32];
#pragma unroll
        for (int x = 0; x < 32; ++x) dd[x] = 0.f;
        {
          uint32_t a[4][4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int i0 = 8 * k + tq, i1 = i0 + 4;
            a[k][0] = __float_as_uint(qs[i0 * DP + f0]);
            a[k][1] = __float_as_uint(qs[i0 * DP + f1]);
            a[k][2] = __float_as_uint(qs[i1 * DP + f0]);
            a[k][3] = __float_as_uint(qs[i1 * DP + f1]);
          }
          const uint64_t bd = make_wgmma_sw128_desc(smem_u32(g1));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n64k8_tf32_rs(dd, a[k], bd + (uint64_t)(2 * k), 1u);
          wgmma_commit();
        }
        wgmma_wait<0>();
        wgmma_fence_regs(dd);
        // document gradient: dd_j = dd^_j / (|d_j| + eps) (tf32-compensated) - d_j * pr_j
#pragma unroll
        for (int x = 0; x < 8; ++x)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int jl = 8 * x + 2 * tq + h, j = t0 + jl;
            if (j < P.Ld) {
              const float s1 = S->rsd[jl] * P.tf32_comp, s2 = S->pr[jl];
              float* gd = P.grad_d + (p * P.Ld + j) * (int64_t)P.D;
              if (f0 < P.D) gd[f0] = fmaf(s1, dd[4 * x + h], -ds[jl * DP + f0] * s2);
              if (f1 < P.D) gd[f1] = fmaf(s1, dd[4 * x + 2 + h], -ds[jl * DP + f1] * s2);
            }
          }
        // GEMM 2: A = D^T (features x document rows), K = 64 document rows
        {
          uint32_t a[8][4];
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int j0 = 8 * k + tq, j1 = j0 + 4;
            a[k][0] = __float_as_uint(ds[j0 * DP + f0]);
            a[k][1] = __float_as_uint(ds[j0 * DP + f1]);
            a[k][2] = __float_as_uint(ds[j1 * DP + f0]);
            a[k][3] = __float_as_uint(ds[j1 * DP + f1]);
          }
          const uint64_t bq = make_wgmma_sw128_desc(smem_u32(g2));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 8; ++k)
            wgmma_m64n32k8_tf32_rs(dq[b], a[k], bq + (uint64_t)((k >> 2) * (32 * 128 / 16) + 2 * (k & 3)), 1u);
          wgmma_commit();
        }
        wgmma_wait<0>();
        wgmma_fence_regs(dq[b]);
      }
    }
    // ---- query gradient: dq_i = dq^_i / (|q_i| + eps) (tf32-compensated) - q_i (q^_i . dq^_i) / (|q_i| (|q_i| + eps)) ----
    if (warp < 8 && lane < 4) {
#pragma unroll
      for (int y = 0; y < 8; ++y) S->ci[warp][gi + y] = ci_acc[y];
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < kMaxFb; ++b) {
      const int fb = wg + 3 * b;
      if (fb >= nfb) break;
      const int f0 = 64 * fb + fr, f1 = f0 + 8;
#pragma unroll
      for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = 8 * x + 2 * tq + h;
          if (i < P.Lq) {
            float cq = 0.f;
#pragma unroll
            for (int w8 = 0; w8 < 8; ++w8) cq += S->ci[w8][i];   // fixed order: deterministic
            const float rsq = S->rsq[i];
            const float s1 = rsq * P.tf32_comp, s2 = rsq * cq * (rsq < 1e12f ? rsq : 0.f);
            float* gq = P.grad_q + (p * P.Lq + i) * (int64_t)P.D;
            if (f0 < P.D) gq[f0] = fmaf(s1, dq[b][4 * x + h], -qs[i * DP + f0] * s2);
            if (f1 < P.D) gq[f1] = fmaf(s1, dq[b][4 * x + 2 + h], -qs[i * DP + f1] * s2);
          }
        }
    }
    __syncthreads();   // the next pair rewrites the query tile, the table and the partial sums
  }
}

template <int KB, bool GATE>
int launch(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream) {
  constexpr int KBP = (KB + 3) & ~3;
  const size_t smem = 1024 + kG1Bytes + kG2Bytes + (size_t)(32 + kTile) * pitch_of(P.D) * sizeof(float) + sizeof(BwShared<KBP>);
  if (smem > (size_t)dev.max_smem_optin) {
    set_error("kernel_pool tensor-core backward: shared-memory plan does not fit");
    return MMB200_ERR_UNSUPPORTED;
  }
  MMB_CHECK_CUDA(cudaFuncSetAttribute(kernel_pool_bwd_tc_kernel<KB, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::min<int64_t>(dev.sm_count, P.B);
  kernel_pool_bwd_tc_kernel<KB, GATE><<<grid, kThreads, smem, stream>>>(P);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

}  // namespace

int kernel_pool_bwd_tc(const KpParams& P, const DeviceInfo& dev, cudaStream_t stream, bool* handled) {
  *handled = false;
  if (P.saved == nullptr || P.Lq > 32 || P.K > 32 || P.D % 4 != 0 || P.D > kMaxD || (P.grad_gate != nullptr && P.gate == nullptr))
    return MMB200_OK;
  if (((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d) | reinterpret_cast<uintptr_t>(P.saved)) & 15) != 0)
    return MMB200_OK;
  *handled = true;
  if (P.B == 0) return MMB200_OK;
  if (P.gate) {   // TK-Sparse: gated activations, d loss / d gate
    if (P.K == 11) return launch<11, true>(P, dev, stream);
    if (P.K == 21) return launch<21, true>(P, dev, stream);
    if (P.K <= 12) return launch<12, true>(P, dev, stream);
    if (P.K <= 24) return launch<24, true>(P, dev, stream);
    return launch<32, true>(P, dev, stream);
  }
  if (P.K == 11) return launch<11, false>(P, dev, stream);
  if (P.K == 21) return launch<21, false>(P, dev, stream);
  if (P.K <= 12) return launch<12, false>(P, dev, stream);
  if (P.K <= 24) return launch<24, false>(P, dev, stream);
  return launch<32, false>(P, dev, stream);
}

}  // namespace mmb
