// lseg_b200 — rounding-faithful causal attention for the CLIP text tower.
//
// CLIP's ResidualAttentionBlock calls nn.MultiheadAttention on fp16 tensors (SURVEY.md Appendix A.2; the tower is
// fp16 because clip.load(device='cuda') converts it, modules/models/lseg_vit.py:224). torch's
// multi_head_attention_forward rounds to fp16 after EVERY step:
//     q = q * head_dim^-0.5                  (fp16; exact, a power of two)
//     attn = bmm(q, k^T) + mask              (fp32 accumulate, fp16 result)
//     attn = softmax(attn, -1)               (fp32 arithmetic inside, NORMALISED result rounded to fp16)
//     out  = bmm(attn, v)                    (fp32 accumulate, fp16 result)
// which oracle/lseg_oracle.py:185-196 restates. The flash-style tensor-core kernel (mhsa.cuh) keeps S in fp32 and
// rounds the UN-normalised P, i.e. it has different rounding points; the text tower runs once per label set on K*77
// tokens, so this kernel trades speed for those exact rounding points: plain CUDA cores, one CTA per (label, head),
// one warp per query row, fp32 dot products in a fixed order. L <= 77 keys, head_dim 64.
#pragma once
#include "common.cuh"

namespace lseg {

constexpr int kTaMaxL = 80;     // context length 77, padded
constexpr int kTaDh = 64;
constexpr int kTaStride = 66;   // halves per smem row: 132 B rows -> lane j reads bank (j + d/2) % 32, conflict-free
constexpr int kTaWarps = 8;

__global__ void __launch_bounds__(kTaWarps * 32) text_attn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out,
                                                                  int L, int heads) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ __align__(16) __half sq[kTaMaxL * kTaStride];
  __shared__ __align__(16) __half sk[kTaMaxL * kTaStride];
  __shared__ __align__(16) __half sv[kTaMaxL * kTaStride];
  __shared__ float sp[kTaWarps][kTaMaxL];  // the current row's probabilities (fp16 values held as fp32)
  const int h = blockIdx.x, label = blockIdx.y;
  const int D = heads * kTaDh;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* base = qkv + static_cast<long long>(label) * L * 3 * D + h * kTaDh;
  const __half eighth = __float2half_rn(0.125f);
  // rows of q | k | v for this (label, head): 64 halves = 128 B contiguous each
  for (int idx = threadIdx.x; idx < L * 32; idx += blockDim.x) {
    const int row = idx >> 5, c = idx & 31;  // half2 column
    const __half* src = base + static_cast<long long>(row) * 3 * D + 2 * c;
    __half2 q2 = *reinterpret_cast<const __half2*>(src);
    q2 = __hmul2(q2, __half2half2(eighth));  // q * dh^-0.5 in fp16
    *reinterpret_cast<__half2*>(&sq[row * kTaStride + 2 * c]) = q2;
    *reinterpret_cast<__half2*>(&sk[row * kTaStride + 2 * c]) = *reinterpret_cast<const __half2*>(src + D);
    *reinterpret_cast<__half2*>(&sv[row * kTaStride + 2 * c]) = *reinterpret_cast<const __half2*>(src + 2 * D);
  }
  __syncthreads();
  for (int i = warp; i < L; i += kTaWarps) {
    // ---- scores of row i against keys j <= i (the additive -inf mask removes the rest exactly) ----
    float s[3];
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      const int j = lane + 32 * t;
      s[t] = -INFINITY;
      if (j <= i) {
        float acc = 0.f;
        const __half2* qr = reinterpret_cast<const __half2*>(&sq[i * kTaStride]);
        const __half2* kr = reinterpret_cast<const __half2*>(&sk[j * kTaStride]);
#pragma unroll 8
        for (int d = 0; d < kTaDh / 2; ++d) {
          const float2 a = __half22float2(qr[d]), b = __half22float2(kr[d]);
          acc = fmaf(a.x, b.x, acc);
          acc = fmaf(a.y, b.y, acc);
        }
        s[t] = __half2float(__float2half_rn(acc));  // bmm result is an fp16 tensor
      }
      mx = fmaxf(mx, s[t]);
    }
    mx = warp_max(mx);
    float e[3], sum = 0.f;
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      e[t] = (lane + 32 * t <= i) ? expf(s[t] - mx) : 0.f;
      sum += e[t];
    }
    sum = warp_sum(sum);
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      const int j = lane + 32 * t;
      if (j < kTaMaxL) sp[warp][j] = (j <= i) ? __half2float(__float2half_rn(e[t] / sum)) : 0.f;  // softmax output fp16
    }
    __syncwarp();
    // ---- out row = P V : lane owns output columns 2*lane, 2*lane+1 ----
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j <= i; ++j) {
      const float pj = sp[warp][j];
      const float2 v2 = __half22float2(*reinterpret_cast<const __half2*>(&sv[j * kTaStride + 2 * lane]));
      o0 = fmaf(pj, v2.x, o0);
      o1 = fmaf(pj, v2.y, o1);
    }
    __half* dst = out + (static_cast<long long>(label) * L + i) * D + h * kTaDh + 2 * lane;
    *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(o0, o1);
    __syncwarp();  // sp[warp] is rewritten by the next row
  }
}

static inline int launch_text_attn(const __half* qkv, __half* out, int K, int L, int heads, cudaStream_t s) {
  if (L > kTaMaxL || L <= 0) {
    set_error("text_attn: L=%d must be in 1..%d", L, kTaMaxL);
    return -1;
  }
  if (K <= 0 || K > 65535) {
    set_error("text_attn: K=%d must be in 1..65535", K);
    return -1;
  }
  if (heads <= 0 || heads > 65535) {
    set_error("text_attn: heads=%d must be in 1..65535", heads);
    return -1;
  }
  // __half2 loads and stores
  if (!qkv || (reinterpret_cast<uintptr_t>(qkv) & 3) != 0) {
    set_error("text_attn: qkv pointer %p is null or not 4-byte aligned", static_cast<const void*>(qkv));
    return -1;
  }
  if (!out || (reinterpret_cast<uintptr_t>(out) & 3) != 0) {
    set_error("text_attn: out pointer %p is null or not 4-byte aligned", static_cast<const void*>(out));
    return -1;
  }
  launch_pdl(text_attn_kernel, dim3(heads, K), dim3(kTaWarps * 32), 0, s, qkv, out, L, heads);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace lseg
