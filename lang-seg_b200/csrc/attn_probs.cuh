// lseg_b200 — attention probabilities of a ViT block for sm_90a: P = softmax(Q K^T * dh^-0.5) written out as fp32
// [B, heads, N, N], contiguous. This is the tensor the reference's attention hook records (get_attention,
// modules/models/lseg_vit.py:22-42: softmax((q @ k^T) * scale) of blocks[h].attn), read from the same packed QKV rows
// the fused attention kernel (mhsa.cuh) reads: [B, N, 3*D] fp16, q | k | v thirds, head h at columns h*64. Non-causal,
// head_dim 64. V is never read.
//
// One CTA = one 128-row query tile of one (image, head), 9 warps (as mhsa_kernel):
//   warps 0..7  two consumer warpgroups of 64 query rows each. Both passes compute S_j = Q K_j^T with wgmma
//               m64n64k16, both operands from shared memory (K-major); a thread holds 2 rows x 16 keys of S_j.
//               Pass 1 keeps the running row max m (scaled by scale * log2 e) and this thread's partial row sum
//               l = sum exp2(S * c - m), rescaled whenever m grows. The partial sums are then reduced over the 4 threads
//               of a row and inverted once.
//               Pass 2 recomputes S_j (the same MMAs on the same tiles: the same bits) and forms
//               p = exp2(fmaf(S, c, -m)) * (1 / l) with the FINAL m and l, stages the warp's 16 x 64 fp32 tile in
//               shared memory and stores it row by row: two 128-byte warp-contiguous runs per row.
//   warp 8      TMA producer: Q once (128 x 64 box), then the K tiles of the sequence twice (pass 1, pass 2) through one
//               4-deep ring of 64-key tiles; a slot is released once both warpgroups' S MMAs have read it.
// Keys beyond the sequence are zero-filled by TMA and masked to -inf in pass 1; query rows and key columns beyond it
// are never stored. The output row pitch is 4N bytes, which is not 16-byte aligned for most N (N = 901: 3604 B), so
// the stores are 4-byte scalar stores, coalesced across the warp; every offset is 64-bit (B*heads*N^2 passes 2^31
// elements at B = 32, 736^2).
#pragma once
#include "common.cuh"
#include "mhsa.cuh"

namespace lseg {

constexpr int kAttnPThreads = 288;
constexpr int kAttnPStages = 4;
constexpr int kAttnPStagePitch = 64 + 8;  // floats per staged row: the padding makes the fragment writes conflict-free
constexpr int kAttnPStageBytes = 8 * 16 * kAttnPStagePitch * 4;  // 8 consumer warps x 16 rows
// Q | K ring | staging | mbarriers, plus the slack that aligns the base to the 1024 B swizzle atom
constexpr int kAttnPSmemBytes = kMhsaQBytes + kAttnPStages * kMhsaKvBytes + kAttnPStageBytes + 128 + 1024;

struct AttnProbsParams {
  CUtensorMap tma_qkv;  // 3-D {3*D, N, B} fp16, box {64, 128, 1} (Q tiles)
  CUtensorMap tma_t64;  // same tensor, box {64, 64, 1} (K tiles)
  float* out;           // [B, heads, N, N]
  int n_tokens;
  int heads;
  int D;
  float scale_log2e;    // dh^-0.5 * log2(e)
};

__global__ void __launch_bounds__(kAttnPThreads, 2) attn_probs_kernel(const __grid_constant__ AttnProbsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sQ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = sQ + kMhsaQBytes;
  float* sStage = reinterpret_cast<float*>(sK + kAttnPStages * kMhsaKvBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sStage) + kAttnPStageBytes);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;  // [kAttnPStages]
  uint64_t* k_empty = k_full + kAttnPStages;

  const int warp = warp_idx_sync();
  const int lane = threadIdx.x & 31;
  const int bh = blockIdx.y;  // image * heads + head: the [B, heads] plane of the output
  const int b = bh / p.heads;
  const int h = bh % p.heads;
  const int q0 = blockIdx.x * kMhsaTile;
  const int N = p.n_tokens;
  const int nkt = (N + kMhsaKT - 1) / kMhsaKT;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&p.tma_qkv);
    tma_prefetch_desc(&p.tma_t64);
    mbar_init(q_full, 1);
    for (int i = 0; i < kAttnPStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);  // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  griddep_launch_dependents();
  __syncthreads();
  griddep_wait();  // the kernel that wrote qkv must have completed before the first TMA load

  if (warp == 8) {
    // ===================== TMA producer (converged warp, elected issuing lane) =====================
    const bool leader = elect_one_sync();
    if (leader) {
      mbar_expect_tx(q_full, kMhsaQBytes);
      tma_load_3d(sQ, &p.tma_qkv, q_full, h * kMhsaDh, q0, b);
    }
    __syncwarp();
    for (int j = 0; j < 2 * nkt; ++j) {  // the key tiles of pass 1, then again those of pass 2
      const int slot = j % kAttnPStages;
      const uint32_t par = ((j / kAttnPStages) & 1) ^ 1;
      const int kt = (j < nkt) ? j : j - nkt;
      mbar_wait(&k_empty[slot], par, 11);
      if (leader) {
        mbar_expect_tx(&k_full[slot], kMhsaKvBytes);
        tma_load_3d(sK + slot * kMhsaKvBytes, &p.tma_t64, &k_full[slot], p.D + h * kMhsaDh, kt * kMhsaKT, b);
      }
      __syncwarp();
    }
  } else {
    // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) =====================
    const int wg = warp >> 2;
    const int wr = (warp & 3) * 16;      // first of this warp's 16 rows within the warpgroup's 64; the thread holds
                                         // rows wr + lane / 4 and wr + lane / 4 + 8
    const int cq = 2 * (lane & 3);       // first of this thread's two columns per 8-column block
    const float c = p.scale_log2e;
    const uint32_t q_base = smem_u32(sQ) + wg * (64 * 128);
    float* stage = sStage + warp * (16 * kAttnPStagePitch);  // this warp's 16 x 64 tile
    float m_a = -INFINITY, m_b = -INFINITY;  // running row maxima (already scaled by c)
    float l_a = 0.f, l_b = 0.f;              // this thread's partial row sums
    mbar_wait(q_full, 0, 13);

    // S_j = Q K_j^T for ring position j into s; releases the K slot once the MMAs have read it.
    auto scores = [&](int j, float (&s)[32]) {
      const int slot = j % kAttnPStages;
      mbar_wait(&k_full[slot], (j / kAttnPStages) & 1, 19);
      __syncwarp();
      const uint32_t k_base = smem_u32(sK + slot * kMhsaKvBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kMhsaDh / 16; ++k)
        wgmma_m64n64k16_ss(s, wgmma_desc_sw128(q_base + k * 32, 1024, 16), wgmma_desc_sw128(k_base + k * 32, 1024, 16),
                           k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence(s);
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[slot]);
    };

    // ---- pass 1: row max and row sum ----
    for (int j = 0; j < nkt; ++j) {
      const int kv0 = j * kMhsaKT;
      float s[32];
      scores(j, s);
      const bool need_mask = kv0 + kMhsaKT > N;
      float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (need_mask && kv0 + 8 * (i >> 2) + cq + (i & 1) >= N) s[i] = -INFINITY;
        if (i & 2) mx_b = fmaxf(mx_b, s[i]); else mx_a = fmaxf(mx_a, s[i]);
      }
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
      mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
      mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
      // every tile holds at least one key < N, so the maxima are finite from the first tile on
      const float mn_a = fmaxf(m_a, mx_a * c), mn_b = fmaxf(m_b, mx_b * c);
      const float f_a = (m_a == -INFINITY) ? 0.f : ex2_approx(m_a - mn_a);
      const float f_b = (m_b == -INFINITY) ? 0.f : ex2_approx(m_b - mn_b);
      m_a = mn_a;
      m_b = mn_b;
      float sum_a = 0.f, sum_b = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float e = (s[i] == -INFINITY) ? 0.f : ex2_approx(fmaf(s[i], c, -((i & 2) ? mn_b : mn_a)));
        if (i & 2) sum_b += e; else sum_a += e;
      }
      l_a = l_a * f_a + sum_a;
      l_b = l_b * f_b + sum_b;
    }
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
    l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
    l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
    const float inv_a = 1.0f / l_a, inv_b = 1.0f / l_b;

    // ---- pass 2: probabilities with the final m and l, staged per warp and stored row by row ----
    const int row0 = q0 + wg * 64 + wr;  // query index of the warp's first staged row
    const int rows = min(16, N - row0);  // rows of the warp's tile that lie in the sequence (<= 0: none)
    float* out_plane = p.out + static_cast<long long>(bh) * N * N;
    for (int j = 0; j < nkt; ++j) {
      const int kv0 = j * kMhsaKT;
      float s[32];
      scores(nkt + j, s);
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const bool rb = (i & 2) != 0;
        const float mu = rb ? m_b : m_a, inv = rb ? inv_b : inv_a;
        float2 v;
        v.x = ex2_approx(fmaf(s[i], c, -mu)) * inv;
        v.y = ex2_approx(fmaf(s[i + 1], c, -mu)) * inv;
        *reinterpret_cast<float2*>(stage + ((lane >> 2) + (rb ? 8 : 0)) * kAttnPStagePitch + 8 * (i >> 2) + cq) = v;
      }
      __syncwarp();
      const int cols = min(kMhsaKT, N - kv0);
      float* dst = out_plane + static_cast<long long>(row0) * N + kv0;
      for (int r = 0; r < rows; ++r, dst += N) {
        const float* src = stage + r * kAttnPStagePitch;
        if (lane < cols) dst[lane] = src[lane];
        if (lane + 32 < cols) dst[lane + 32] = src[lane + 32];
      }
      __syncwarp();  // the tile is read before the next one is staged
    }
  }
}

}  // namespace lseg
