// Cosine + RBF kernel pooling BACKWARD at BERT widths (512 < D <= 1024, D % 64 == 0; Lq <= 32, K <= 32) on the tensor
// cores, from the state the training forward saved (kernel_pool_ts_kernel<.., SAVE>: cosines, inverse norms).
//
// Same arithmetic as kernel_pool_bwd_wg.cu (see there for G, the normalisation backward and the tf32 treatment), split
// in two kernels so that one pair at D = 768 spreads over several SMs:
//
//   kp_wide_g_kernel<KB, GATE>   one CTA per pair, nothing that depends on the features: G_ij from the saved cosines and
//                                per_kernel_query, the per-pair d weight / d alpha terms (for kp_reduce_batch), d gate, and
//                                the projection terms r_q[i] = sum_j G_ij c_ij, r_d[j] = sum_i G_ij c_ij (no full-D dot
//                                product: they come from the cosines).  Writes the GEMM operands G1 = G diag(1/(|q|+eps)),
//                                G2^T = (diag(1/(|d|+eps)) G)^T as tf32 and the normalisation terms to the workspace.
//   kp_wide_grad_kernel          one CTA (one warpgroup) per (pair, 64-feature block):
//                                  dd^T[64 features x 64 doc rows]   = Q^T[64 x 32 query rows] * G1^T   per document tile
//                                  dq^T[64 features x 32 query rows] += D^T[64 x 64 doc rows]  * G2     over the tiles
//                                with the normalisation backward in the epilogue.
//
// Every output element has one owner and one summation order (no atomics): two runs give the same bits.  Neither
// launch allocates or synchronises, so the training step can be captured in a CUDA graph.
#include <algorithm>

#include "device_util.cuh"
#include "host_util.cuh"
#include "kernel_pool.cuh"
#include "masks.cuh"
#include "ptx.cuh"

namespace mmb {

namespace {

constexpr int kTile = 64;            // document rows per tile (wgmma N of GEMM 1, K of GEMM 2)
constexpr int kGThreads = 256;       // G pass: thread = (document row of the tile, 8 query rows)
constexpr int kFThreads = 128;       // gradient GEMMs: one warpgroup, 64 features
constexpr int kFP = 64 + 8;          // floats per staged row: 8 mod 32, conflict-free A gathers
constexpr int kG1Bytes = kTile * 128;     // G1 [64 doc rows][32 query rows] fp32, K-major SWIZZLE_128B
constexpr int kG2Bytes = 2 * 32 * 128;    // G2^T [2 k-blocks][32 query rows][32 doc rows], K-major SWIZZLE_128B

template <int KBP>
struct GShared {
  alignas(16) float T[KBP][32];      // [kernel][query row]: coef_ik / sigma_k^2
  float rsq[32];
  float ci[8][32];                   // [warp][query row]: sum_j G_ij c_ij of the pair
  float mu[32], a[32], sig2[32], alpha[32], w[32], is2[32];
};

template <int KB, bool GATE>
__global__ void __launch_bounds__(kGThreads)
kp_wide_g_kernel(KpParams P, KpWideWs W) {
  constexpr int KBP = (KB + 3) & ~3;
  __shared__ GShared<KBP> S;
  const int64_t p = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, tq = lane & 3;
  const int gj = tid >> 2, gi = (tid & 3) * 8;
  const int dmt = P.d_mask ? P.mask_dtype : MMB200_MASK_NONE;
  const int qmt = P.q_mask ? P.mask_dtype : MMB200_MASK_NONE;
  const int Ldp = W.Ldp;
  uint32_t* g1 = W.g1 + p * (int64_t)Ldp * 32;     // [Ldp][32]
  uint32_t* g2 = W.g2t + p * (int64_t)Ldp * 32;    // [32][Ldp]
  float* prd = W.prd + p * (int64_t)Ldp;
  if (tid < 32) {
    const bool ok = tid < P.K;
    const float sg = ok ? P.sigma[tid] : 1.f;
    S.mu[tid] = ok ? P.mu[tid] : 0.f;
    S.a[tid] = ok ? rbf_scale(sg) : 0.f;
    S.is2[tid] = ok ? 1.0f / (sg * sg) : 0.f;
    S.sig2[tid] = ok ? sg * sg : 0.f;
    S.alpha[tid] = ok ? (P.alpha ? P.alpha[tid] : 1.f) : 1.f;
    S.w[tid] = ok ? P.weight[tid] : 0.f;
  }
  __syncthreads();
  // ---- coefficient table, d weight / d alpha (as kernel_pool_bwd_tc_kernel) ----
  if (warp == 0) {
    const float g = P.grad_score[p];
    const bool qlive = lane < P.Lq && mask_at(P.q_mask, qmt, p * (int64_t)P.Lq + lane);
    float Sr[KBP];
#pragma unroll
    for (int k = 0; k < KBP; ++k) Sr[k] = (k < P.K && qlive) ? P.S[(p * P.Lq + lane) * (int64_t)P.K + k] : 1.f;
#pragma unroll
    for (int k = 0; k < KBP; ++k) {
      float cf = 0.f, Lv = 0.f, da = 0.f;
      if (k < P.K && qlive) {
        const float Sv = Sr[k];
        const float aS = Sv * S.alpha[k];
        Lv = P.log_scale * logf(fmaxf(aS, P.clamp_min));
        if (aS >= P.clamp_min) {   // torch.clamp passes the gradient at equality
          cf = g * S.w[k] * P.log_scale / Sv;
          da = g * S.w[k] * P.log_scale / S.alpha[k];
        }
      }
      S.T[k][lane] = cf * S.is2[k];
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
    S.rsq[lane] = P.saved[kp_saved_rsq_off(P.B, p, P.Ld) + lane];
  }
  __syncthreads();
  float rsq8[8];
#pragma unroll
  for (int y = 0; y < 8; ++y) rsq8[y] = S.rsq[gi + y];
  float ci_acc[8];
#pragma unroll
  for (int y = 0; y < 8; ++y) ci_acc[y] = 0.f;

  for (int t0 = 0; t0 < Ldp; t0 += kTile) {
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
        const float mu_k = S.mu[k], a_k = S.a[k];
        const float sig2_k = GATE ? S.sig2[k] : 0.f;
        const float4 T0 = *reinterpret_cast<const float4*>(&S.T[k][gi]), T1 = *reinterpret_cast<const float4*>(&S.T[k][gi + 4]);
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
    // G1 row j: G_ij / (|q_i| + eps); G2^T column j: G_ij / (|d_j| + eps).  Rows Ld .. Ldp are written as zeros.
    {
      uint32_t v[8];
#pragma unroll
      for (int y = 0; y < 8; ++y) v[y] = f32_to_tf32_rna(G[y] * rsq8[y]);
      uint4* dst = reinterpret_cast<uint4*>(g1 + (int64_t)j * 32 + gi);
      dst[0] = make_uint4(v[0], v[1], v[2], v[3]);
      dst[1] = make_uint4(v[4], v[5], v[6], v[7]);
#pragma unroll
      for (int y = 0; y < 8; ++y) g2[(int64_t)(gi + y) * Ldp + j] = f32_to_tf32_rna(G[y] * rsd);
    }
    if constexpr (GATE) {
      H += __shfl_xor_sync(0xffffffffu, H, 1);
      H += __shfl_xor_sync(0xffffffffu, H, 2);
      if (tq == 0 && inb && P.grad_gate) P.grad_gate[p * (int64_t)P.Ld + j] = (valid && gv >= 0.f) ? H : 0.f;
    }
    // (d^_j . dd^_j) / |d_j| times 1 / (|d_j| + eps); 0 for a zero row
    if (tq == 0) prd[j] = rsd * cpr * (rsd < 1e12f ? rsd : 0.f);
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
  if (lane < 4) {
#pragma unroll
    for (int y = 0; y < 8; ++y) S.ci[warp][gi + y] = ci_acc[y];
  }
  __syncthreads();
  if (tid < 32) {
    float cq = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) cq += S.ci[w8][tid];   // fixed order: deterministic
    const float rsq = S.rsq[tid];
    W.prq[p * 32 + tid] = rsq * cq * (rsq < 1e12f ? rsq : 0.f);
  }
}

struct FShared {
  float rsd[kTile];   // 1 / (|d_j| + eps) of the tile's rows
  float prd[kTile];
  float rsq[32];
  float prq[32];
};

__global__ void __launch_bounds__(kFThreads)
kp_wide_grad_kernel(KpParams P, KpWideWs W) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* g1s = smem;                                          // SWIZZLE_128B operands first (1024-B aligned)
  uint8_t* g2s = g1s + kG1Bytes;
  float* qs = reinterpret_cast<float*>(g2s + kG2Bytes);         // [32][kFP] query rows of the block (zero past Lq)
  float* ds = qs + 32 * kFP;                                    // [64][kFP] document tile (zero past Ld)
  FShared* S = reinterpret_cast<FShared*>(ds + kTile * kFP);

  const int nfb = P.D >> 6;
  const int64_t p = blockIdx.x / nfb;
  const int f_base = (blockIdx.x - (int)(p * nfb)) * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, tq = lane & 3;
  const int fr = 16 * warp + (lane >> 2);
  const int Ldp = W.Ldp;
  const uint32_t* g1 = W.g1 + p * (int64_t)Ldp * 32;
  const uint32_t* g2 = W.g2t + p * (int64_t)Ldp * 32;

  for (int e = tid; e < 32 * 16; e += kFThreads) {
    const int i = e >> 4, c4 = e & 15;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < P.Lq) v = *reinterpret_cast<const float4*>(P.q + (p * P.Lq + i) * (int64_t)P.D + f_base + 4 * c4);
    *reinterpret_cast<float4*>(qs + i * kFP + 4 * c4) = v;
  }
  if (tid < 32) {
    S->rsq[tid] = P.saved[kp_saved_rsq_off(P.B, p, P.Ld) + tid];
    S->prq[tid] = W.prq[p * 32 + tid];
  }
  float dq[16];
#pragma unroll
  for (int x = 0; x < 16; ++x) dq[x] = 0.f;

  for (int t0 = 0; t0 < Ldp; t0 += kTile) {
    __syncthreads();   // the previous tile's operands are no longer read
    for (int e = tid; e < kTile * 16; e += kFThreads) {
      const int j = e >> 4, c4 = e & 15;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t0 + j < P.Ld) v = *reinterpret_cast<const float4*>(P.d + (p * P.Ld + t0 + j) * (int64_t)P.D + f_base + 4 * c4);
      *reinterpret_cast<float4*>(ds + j * kFP + 4 * c4) = v;
    }
    for (int e = tid; e < kTile * 8; e += kFThreads) {   // G1 [doc row][query row], 16-byte chunk c of row r
      const int r = e >> 3, c = e & 7;
      const uint4 v = *reinterpret_cast<const uint4*>(g1 + (int64_t)(t0 + r) * 32 + 4 * c);
      *reinterpret_cast<uint4*>(g1s + r * 128 + ((c ^ (r & 7)) << 4)) = v;
    }
    for (int e = tid; e < 32 * 16; e += kFThreads) {     // G2^T [query row][doc row]: k-block c / 8, chunk c % 8
      const int i = e >> 4, c = e & 15;
      const uint4 v = *reinterpret_cast<const uint4*>(g2 + (int64_t)i * Ldp + t0 + 4 * c);
      *reinterpret_cast<uint4*>(g2s + (c >> 3) * (32 * 128) + i * 128 + (((c & 7) ^ (i & 7)) << 4)) = v;
    }
    if (tid < kTile) {
      const int j = t0 + tid;
      S->rsd[tid] = j < P.Ld ? P.saved[kp_saved_rsd_off(P.B, p, P.Ld) + j] : 0.f;
      S->prd[tid] = W.prd[p * (int64_t)Ldp + j];
    }
    fence_proxy_async_smem();   // G1 / G2^T are read by the tensor core (async proxy)
    __syncthreads();
    const int f0 = fr, f1 = fr + 8;
    // A operands: Q^T (features x query rows) for GEMM 1, D^T (features x document rows) for GEMM 2, both gathered before
    // the fence that orders them before the wgmma
    uint32_t aq[4][4], ad[8][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i0 = 8 * k + tq, i1 = i0 + 4;
      aq[k][0] = __float_as_uint(qs[i0 * kFP + f0]);
      aq[k][1] = __float_as_uint(qs[i0 * kFP + f1]);
      aq[k][2] = __float_as_uint(qs[i1 * kFP + f0]);
      aq[k][3] = __float_as_uint(qs[i1 * kFP + f1]);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int j0 = 8 * k + tq, j1 = j0 + 4;
      ad[k][0] = __float_as_uint(ds[j0 * kFP + f0]);
      ad[k][1] = __float_as_uint(ds[j0 * kFP + f1]);
      ad[k][2] = __float_as_uint(ds[j1 * kFP + f0]);
      ad[k][3] = __float_as_uint(ds[j1 * kFP + f1]);
    }
    float dd[32];
#pragma unroll
    for (int x = 0; x < 32; ++x) dd[x] = 0.f;
    wgmma_fence();
    {   // GEMM 1: dd^T = Q^T G1^T, K = 32 query rows
      const uint64_t bd = make_wgmma_sw128_desc(smem_u32(g1s));
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64k8_tf32_rs(dd, aq[k], bd + (uint64_t)(2 * k), 1u);
      wgmma_commit();
    }
    {   // GEMM 2: dq^T += D^T G2, K = 64 document rows; in flight during GEMM 1's epilogue
      const uint64_t bq = make_wgmma_sw128_desc(smem_u32(g2s));
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_m64n32k8_tf32_rs(dq, ad[k], bq + (uint64_t)((k >> 2) * (32 * 128 / 16) + 2 * (k & 3)), 1u);
      wgmma_commit();
    }
    wgmma_wait<1>();
    wgmma_fence_regs(dd);
    // document gradient: dd_j = dd^_j / (|d_j| + eps) (tf32-compensated) - d_j * pr_j
#pragma unroll
    for (int x = 0; x < 8; ++x)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int jl = 8 * x + 2 * tq + h, j = t0 + jl;
        if (j < P.Ld) {
          const float s1 = S->rsd[jl] * P.tf32_comp, s2 = S->prd[jl];
          float* gd = P.grad_d + (p * P.Ld + j) * (int64_t)P.D + f_base;
          gd[f0] = fmaf(s1, dd[4 * x + h], -ds[jl * kFP + f0] * s2);
          gd[f1] = fmaf(s1, dd[4 * x + 2 + h], -ds[jl * kFP + f1] * s2);
        }
      }
    wgmma_wait<0>();
    wgmma_fence_regs(dq);
  }
  // query gradient: dq_i = dq^_i / (|q_i| + eps) (tf32-compensated) - q_i (q^_i . dq^_i) / (|q_i| (|q_i| + eps))
  const int f0 = fr, f1 = fr + 8;
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = 8 * x + 2 * tq + h;
      if (i < P.Lq) {
        const float s1 = S->rsq[i] * P.tf32_comp, s2 = S->prq[i];
        float* gq = P.grad_q + (p * P.Lq + i) * (int64_t)P.D + f_base;
        gq[f0] = fmaf(s1, dq[4 * x + h], -qs[i * kFP + f0] * s2);
        gq[f1] = fmaf(s1, dq[4 * x + 2 + h], -qs[i * kFP + f1] * s2);
      }
    }
}

template <int KB, bool GATE>
int launch_g(const KpParams& P, const KpWideWs& W, cudaStream_t stream) {
  kp_wide_g_kernel<KB, GATE><<<(unsigned)P.B, kGThreads, 0, stream>>>(P, W);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

template <bool GATE>
int launch_g_for(const KpParams& P, const KpWideWs& W, cudaStream_t stream) {
  if (P.K == 11) return launch_g<11, GATE>(P, W, stream);
  if (P.K == 21) return launch_g<21, GATE>(P, W, stream);
  if (P.K <= 12) return launch_g<12, GATE>(P, W, stream);
  if (P.K <= 24) return launch_g<24, GATE>(P, W, stream);
  return launch_g<32, GATE>(P, W, stream);
}

constexpr size_t kFSmem = 1024 + kG1Bytes + kG2Bytes + (size_t)(32 + kTile) * kFP * sizeof(float) + sizeof(FShared);

}  // namespace

bool kp_wide_shape_ok(int Lq, int Ld, int D, int K) {
  return Lq >= 1 && Lq <= 32 && Ld >= 1 && K >= 1 && K <= 32 && D > 512 && D <= 1024 && D % 64 == 0;
}

int64_t kp_wide_ws_floats(int64_t B, int Ld) {
  const int64_t Ldp = (Ld + kTile - 1) / kTile * kTile;
  return B * (65 * Ldp + 32);
}

int kernel_pool_bwd_wide(const KpParams& P, float* ws, const DeviceInfo& dev, cudaStream_t stream) {
  if (P.grad_gate != nullptr && P.gate == nullptr) {
    set_error("kernel_pool_bwd_saved: grad_gate needs doc_gate");
    return MMB200_ERR_INVALID;
  }
  if (((reinterpret_cast<uintptr_t>(P.q) | reinterpret_cast<uintptr_t>(P.d) | reinterpret_cast<uintptr_t>(P.saved) |
        reinterpret_cast<uintptr_t>(ws)) & 15) != 0) {
    set_error("kernel_pool_bwd_saved: q, d, saved and the workspace must be 16-byte aligned");
    return MMB200_ERR_INVALID;
  }
  if (kFSmem > (size_t)dev.max_smem_optin) {
    set_error("kernel_pool wide backward: shared-memory plan does not fit");
    return MMB200_ERR_UNSUPPORTED;
  }
  KpWideWs W;
  W.Ldp = (P.Ld + kTile - 1) / kTile * kTile;
  W.g1 = reinterpret_cast<uint32_t*>(ws);
  W.g2t = W.g1 + P.B * (int64_t)W.Ldp * 32;
  W.prd = reinterpret_cast<float*>(W.g2t + P.B * (int64_t)W.Ldp * 32);
  W.prq = W.prd + P.B * (int64_t)W.Ldp;
  int rc = P.gate ? launch_g_for<true>(P, W, stream) : launch_g_for<false>(P, W, stream);
  if (rc) return rc;
  MMB_CHECK_CUDA(cudaFuncSetAttribute(kp_wide_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFSmem));
  const int64_t grid = P.B * (P.D / 64);
  kp_wide_grad_kernel<<<(unsigned)grid, kFThreads, kFSmem, stream>>>(P, W);
  MMB_CHECK_CUDA(cudaGetLastError());
  return MMB200_OK;
}

}  // namespace mmb
