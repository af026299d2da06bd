// lseg_b200 — fused multi-head self-attention for sm_90a (the kernel the engine runs).
//
// softmax( (Q K^T) * dh^-0.5 [+ causal mask] ) V for head_dim 64, reading the packed QKV rows
// produced by the QKV GEMM ([B, N, 3*D] fp16; q | k | v thirds, head h at columns h*64) and
// writing [B*N, D] fp16. Restates timm Attention (SURVEY.md Appendix A.1; corroborated in-tree at
// modules/models/lseg_vit.py:26-39) and CLIP's causal nn.MultiheadAttention (Appendix A.2) without
// ever materialising the [B, heads, N, N] score tensor.
//
// One CTA = one 128-row query tile of one (image, head); 2 CTAs co-reside per SM. 9 warps:
//   warps 0..7  two consumer warpgroups, 64 query rows each, online softmax in registers:
//                 S_j = Q K_j^T   wgmma m64n64k16, both operands from smem (K-major)
//                 P_j = exp2(S_j * scale * log2 e - m)  in the accumulator fragment, repacked in place as fp16 A operand
//                 O  += P_j V_j   wgmma m64n64k16, A = P from registers, B = V from smem (MN-major)
//               a thread holds 2 query rows x 16 keys of S and 2 rows x 16 columns of O; row max / sum are reduced
//               over the 4 threads that share a row.
//   warp 8      TMA producer: Q once (128 x 64 box), K and V 64-key tiles through separate 4-deep rings; a K slot is
//               released once both warpgroups' S MMAs have read it, a V slot after their PV MMAs.
// Keys beyond the sequence are zero-filled by TMA and masked to -inf; query rows beyond it compute on zero rows and
// are not stored.
#pragma once
#include "common.cuh"

namespace lseg {

constexpr int kMhsaThreads = 288;
constexpr int kMhsaTile = 128;   // query rows per CTA
constexpr int kMhsaKT = 64;      // keys per tile
constexpr int kMhsaDh = 64;
constexpr int kMhsaStages = 4;
constexpr int kMhsaQBytes = kMhsaTile * kMhsaDh * 2;  // 16 KB
constexpr int kMhsaKvBytes = kMhsaKT * kMhsaDh * 2;   // 8 KB
// Q | K ring | V ring | mbarriers, plus the slack that aligns the base to the 1024 B swizzle atom
constexpr int kMhsaSmemBytes = kMhsaQBytes + 2 * kMhsaStages * kMhsaKvBytes + 256 + 1024;

struct MhsaParams {
  CUtensorMap tma_qkv;  // 3-D {3*D, N, B} fp16, box {64, 128, 1} (Q tiles)
  CUtensorMap tma_t64;  // same tensor, box {64, 64, 1} (K / V tiles)
  __half* out;          // [B*N, D]
  int n_tokens;
  int heads;
  int D;
  int causal;
  float scale_log2e;    // dh^-0.5 * log2(e)
  unsigned long long* trace;  // debug timeline buffer (TRACE instantiation only), else nullptr
};

struct MhsaDesc {
  const __half* qkv;  // [B, N, 3*D]
  __half* out;        // [B*N, D]
  int B, N, heads;    // D = heads * 64
  int causal;
};

// POLY: how many of every 8 exponentials run on the FMA pipe (exp2_poly<3>, relative error 7.5e-5 — below the fp16
// rounding of P) instead of the MUFU pipe. TRACE: debug instantiation that stamps clock64() at the hand-off points of
// 16 sampled CTAs into p.trace ([16 CTAs][10 warps][256] of (clock << 8 | tag)).
template <int POLY, bool TRACE = false>
__global__ void __launch_bounds__(kMhsaThreads, 2) mhsa_kernel(const __grid_constant__ MhsaParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = sQ + kMhsaQBytes;
  uint8_t* sV = sK + kMhsaStages * kMhsaKvBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kMhsaStages * kMhsaKvBytes);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;                    // [kMhsaStages]
  uint64_t* k_empty = k_full + kMhsaStages;
  uint64_t* v_full = k_empty + kMhsaStages;
  uint64_t* v_empty = v_full + kMhsaStages;

  const int warp = warp_idx_sync();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y / p.heads;
  const int h = blockIdx.y % p.heads;
  const int q0 = blockIdx.x * kMhsaTile;
  int trace_n = 0;
  unsigned long long* trace_w = nullptr;
  if (TRACE) {
    const int cta_lin = blockIdx.y * gridDim.x + blockIdx.x;
    const int slot = (cta_lin % 128 == 0) ? cta_lin / 128 : ((cta_lin % 128 == 7) ? 8 + cta_lin / 128 : -1);
    if (slot >= 0 && slot < 16 && lane == 0) trace_w = p.trace + (slot * 10 + warp) * 256;
  }
  auto TR = [&](int tag) {
    if (TRACE && trace_w && trace_n < 254) trace_w[trace_n++] = (static_cast<unsigned long long>(clock64()) << 8) | tag;
  };

  const int kv_end = p.causal ? min(p.n_tokens, q0 + kMhsaTile) : p.n_tokens;
  const int nkt = (kv_end + kMhsaKT - 1) / kMhsaKT;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&p.tma_qkv);
    tma_prefetch_desc(&p.tma_t64);
    mbar_init(q_full, 1);
    for (int i = 0; i < kMhsaStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);  // one arrival per consumer warp
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    mbar_fence_init();
  }
  griddep_launch_dependents();
  __syncthreads();
  griddep_wait();  // the QKV GEMM must have completed before the first TMA load / output store
  TR(0);

  if (warp == 8) {
    // ===================== TMA producer (converged warp, elected issuing lane) =====================
    const bool leader = elect_one_sync();
    if (leader) {
      mbar_expect_tx(q_full, kMhsaQBytes);
      tma_load_3d(sQ, &p.tma_qkv, q_full, h * kMhsaDh, q0, b);
    }
    __syncwarp();
    for (int j = 0; j < nkt; ++j) {
      const int slot = j % kMhsaStages;
      const uint32_t par = ((j / kMhsaStages) & 1) ^ 1;
      mbar_wait(&k_empty[slot], par, 11);
      if (leader) {
        mbar_expect_tx(&k_full[slot], kMhsaKvBytes);
        tma_load_3d(sK + slot * kMhsaKvBytes, &p.tma_t64, &k_full[slot], p.D + h * kMhsaDh, j * kMhsaKT, b);
      }
      __syncwarp();
      mbar_wait(&v_empty[slot], par, 12);
      if (leader) {
        mbar_expect_tx(&v_full[slot], kMhsaKvBytes);
        tma_load_3d(sV + slot * kMhsaKvBytes, &p.tma_t64, &v_full[slot], 2 * p.D + h * kMhsaDh, j * kMhsaKT, b);
      }
      __syncwarp();
      TR(20);
    }
  } else {
    // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) =====================
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows r0 and r0 + 8
    const int qa = q0 + r0, qb = qa + 8;
    const int cq = 2 * (lane & 3);                            // first of this thread's two columns per 8-column block
    const float c = p.scale_log2e;
    const int lim_a = p.causal ? qa : 0x7fffffff, lim_b = p.causal ? qb : 0x7fffffff;
    const uint32_t q_base = smem_u32(sQ) + wg * (64 * 128);
    float m_a = -INFINITY, m_b = -INFINITY;  // running row maxima (already scaled by c)
    float l_a = 0.f, l_b = 0.f;              // this thread's partial row sums
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0, 13);
    for (int j = 0; j < nkt; ++j) {
      const int slot = j % kMhsaStages;
      const uint32_t par = (j / kMhsaStages) & 1;
      const int kv0 = j * kMhsaKT;
      float s[32];
      mbar_wait(&k_full[slot], par, 19);
      __syncwarp();
      TR(1);
      {
        const uint32_t k_base = smem_u32(sK + slot * kMhsaKvBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kMhsaDh / 16; ++k)
          wgmma_m64n64k16_ss(s, wgmma_desc_sw128(q_base + k * 32, 1024, 16), wgmma_desc_sw128(k_base + k * 32, 1024, 16),
                             k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(s);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[slot]);
      // mask (key tail of the sequence, causal upper triangle) and row maxima
      const bool need_mask = (kv0 + kMhsaKT > kv_end) || (p.causal && kv0 + kMhsaKT - 1 > q0);
      float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (need_mask) {
          const int kv = kv0 + 8 * (i >> 2) + cq + (i & 1);
          const int lim = (i & 2) ? lim_b : lim_a;
          if (!(kv < kv_end && kv <= lim)) s[i] = -INFINITY;
        }
        if (i & 2) mx_b = fmaxf(mx_b, s[i]); else mx_a = fmaxf(mx_a, s[i]);
      }
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
      const float mn_a = fmaxf(m_a, mx_a * c), mn_b = fmaxf(m_b, mx_b * c);
      const float mu_a = (mn_a == -INFINITY) ? 0.f : mn_a, mu_b = (mn_b == -INFINITY) ? 0.f : mn_b;
      const float f_a = (m_a == -INFINITY) ? 0.f : ex2_approx(m_a - mu_a);
      const float f_b = (m_b == -INFINITY) ? 0.f : ex2_approx(m_b - mu_b);
      m_a = mn_a;
      m_b = mn_b;
      float sum_a = 0.f, sum_b = 0.f;
      uint32_t pa[16];  // P as fp16 pairs, in the A-fragment order of the PV MMA
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const float mu = (i & 2) ? mu_b : mu_a;
        const float x0 = fmaf(s[i], c, -mu), x1 = fmaf(s[i + 1], c, -mu);
        const float p0 = ((i & 7) < POLY) ? exp2_poly<3>(fmaxf(x0, -126.f)) : ex2_approx(x0);
        const float p1 = (((i + 1) & 7) < POLY) ? exp2_poly<3>(fmaxf(x1, -126.f)) : ex2_approx(x1);
        const float q0v = (s[i] == -INFINITY) ? 0.f : p0, q1v = (s[i + 1] == -INFINITY) ? 0.f : p1;
        if (i & 2) sum_b += q0v + q1v; else sum_a += q0v + q1v;
        __half2 hp = __floats2half2_rn(q0v, q1v);
        pa[i >> 1] = *reinterpret_cast<uint32_t*>(&hp);
      }
      l_a = l_a * f_a + sum_a;
      l_b = l_b * f_b + sum_b;
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= (i & 2) ? f_b : f_a;
      mbar_wait(&v_full[slot], par, 20);
      __syncwarp();
      {
        const uint32_t v_base = smem_u32(sV + slot * kMhsaKvBytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kMhsaKT / 16; ++kk) {
          const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
          wgmma_m64n64k16_rs_bmn(o, a, wgmma_desc_sw128(v_base + kk * 2048, 1024, 8192), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(o);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[slot]);
      TR(5);
    }
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float inv_a = 1.0f / l_a, inv_b = 1.0f / l_b;
    __half* out_a = p.out + (static_cast<long long>(b) * p.n_tokens + qa) * p.D + h * kMhsaDh + cq;
    __half* out_b = out_a + 8ll * p.D;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      if (qa < p.n_tokens)
        *reinterpret_cast<__half2*>(out_a + 8 * jj) = __floats2half2_rn(o[4 * jj] * inv_a, o[4 * jj + 1] * inv_a);
      if (qb < p.n_tokens)
        *reinterpret_cast<__half2*>(out_b + 8 * jj) = __floats2half2_rn(o[4 * jj + 2] * inv_b, o[4 * jj + 3] * inv_b);
    }
  }
  TR(8);
}

}  // namespace lseg
