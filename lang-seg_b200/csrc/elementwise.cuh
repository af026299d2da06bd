// lseg_b200 — HBM-bound helper kernels (vectorised / warp-shuffle) for the LSeg forward path.
// Each kernel cites the reference line it restates. Index math is kept OFF the per-element path: rows /
// planes / pixels come from blockIdx (2-D/3-D grids), so a thread's work is "load 16 B, convert, store
// 16 B" without the 64-bit div/mod chains of a flat grid-stride loop (those made the first version of
// the x2 logits upsample instruction-bound at 1.6 TB/s instead of HBM-bound).
#pragma once
#include "common.cuh"

namespace lseg {

#define LSEG_LAUNCH_CHECK()                   \
  do {                                        \
    LSEG_CHECK_CUDA(cudaGetLastError());      \
    return 0;                                 \
  } while (0)

// ------------------------------------------------------------------------------------------
// patchify: x fp32 NCHW [B,3,H,W] -> A fp16 [B*gh*gw, 3*P*P], column = c*P*P + py*P + px, which is
// the flattening of the patch-embed Conv2d(3,D,kP,sP) weight (modules/models/lseg_vit.py:179; P = 16 for
// vit_large_patch16_384, 32 for vit_base_patch32_384), so the conv becomes one GEMM with the weight used as stored.
// grid (ceil(gw*3*P*P/4 / 256), B*gh): one thread = 4 pixels of one patch row.
// ------------------------------------------------------------------------------------------
template <int P>
__global__ void patchify_kernel(const float* __restrict__ x, __half* __restrict__ a, int H, int W) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int kQuads = P / 4;           // float4 groups per patch row
  constexpr int kPerPatchCh = P * kQuads;  // threads per (patch, channel)
  const int gh = H / P, gw = W / P;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= gw * 3 * kPerPatchCh) return;
  const int b = blockIdx.y / gh, gy = blockIdx.y - b * gh;
  const int px4 = i % kQuads, py = (i / kQuads) % P;
  const int rest = i / kPerPatchCh;  // gx*3 + c
  const int gx = rest / 3, c = rest - gx * 3;
  const float4 v = *reinterpret_cast<const float4*>(
      x + ((static_cast<long long>(b) * 3 + c) * H + gy * P + py) * W + gx * P + px4 * 4);
  __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  uint2 o;
  o.x = *reinterpret_cast<uint32_t*>(&h0);
  o.y = *reinterpret_cast<uint32_t*>(&h1);
  __half* dst = a + (static_cast<long long>(blockIdx.y) * gw + gx) * (3 * P * P) + c * P * P + py * P + px4 * 4;
  *reinterpret_cast<uint2*>(dst) = o;
}
static inline int launch_patchify(const float* x, __half* a, int B, int H, int W, int P, cudaStream_t s) {
  if ((P != 16 && P != 32) || H % P != 0 || W % P != 0) {
    set_error("patchify: patch size %d (16 or 32) must divide H=%d and W=%d", P, H, W);
    return -1;
  }
  const int gw = W / P, gh = H / P;
  dim3 grid((gw * 3 * P * (P / 4) + 255) / 256, B * gh);
  if (P == 16)
    launch_pdl(patchify_kernel<16>, grid, dim3(256), 0, s, x, a, H, W);
  else
    launch_pdl(patchify_kernel<32>, grid, dim3(256), 0, s, x, a, H, W);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// pos-embed resize, bilinear align_corners=False (modules/models/lseg_vit.py:149-163); weight-only,
// computed once per token grid. pos [1+g0*g0, D] -> out [1+gh*gw, D]; row 0 (cls) copied.
// ------------------------------------------------------------------------------------------
__global__ void pos_resize_kernel(const float* __restrict__ pos, float* __restrict__ out, int g0, int gh, int gw,
                                  int D) {
  const int row = blockIdx.x;  // 0 .. gh*gw
  if (row == 0) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) out[d] = pos[d];
    return;
  }
  const int oy = (row - 1) / gw, ox = (row - 1) % gw;
  const float sy = static_cast<float>(g0) / gh, sx = static_cast<float>(g0) / gw;
  float fy = fmaxf((oy + 0.5f) * sy - 0.5f, 0.f), fx = fmaxf((ox + 0.5f) * sx - 0.5f, 0.f);
  const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
  const int y1 = y0 + ((y0 < g0 - 1) ? 1 : 0), x1 = x0 + ((x0 < g0 - 1) ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const float* p00 = pos + (1 + y0 * g0 + x0) * static_cast<long long>(D);
  const float* p01 = pos + (1 + y0 * g0 + x1) * static_cast<long long>(D);
  const float* p10 = pos + (1 + y1 * g0 + x0) * static_cast<long long>(D);
  const float* p11 = pos + (1 + y1 * g0 + x1) * static_cast<long long>(D);
  for (int d = threadIdx.x; d < D; d += blockDim.x)
    out[static_cast<long long>(row) * D + d] = hy * (hx * p00[d] + lx * p01[d]) + ly * (hx * p10[d] + lx * p11[d]);
}

// ------------------------------------------------------------------------------------------
// token assembly (modules/models/lseg_vit.py:188-193): x[b,0] = cls + pos[0];
// x[b,1+t] = patch[b*T+t] (bias already added by the GEMM) + pos[1+t].   fp32 [B, 1+T, D]
// one block per token row.
// ------------------------------------------------------------------------------------------
__global__ void assemble_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ pos, float* __restrict__ x, int T, int D) {
  griddep_launch_dependents();
  griddep_wait();
  const int row = blockIdx.x;
  const int b = row / (T + 1), t = row - b * (T + 1);
  const float* src = (t == 0) ? cls : patch + (static_cast<long long>(b) * T + (t - 1)) * D;
  const float* pe = pos + static_cast<long long>(t) * D;
  float* dst = x + static_cast<long long>(row) * D;
  for (int c = threadIdx.x; c < D / 4; c += blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(src)[c];
    const float4 q = reinterpret_cast<const float4*>(pe)[c];
    v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    reinterpret_cast<float4*>(dst)[c] = v;
  }
}
static inline int launch_assemble_tokens(const float* patch, const float* cls, const float* pos, float* x, int B, int T,
                                         int D, cudaStream_t s) {
  launch_pdl(assemble_tokens_kernel, dim3(B * (T + 1)), dim3(256), 0, s, patch, cls, pos, x, T, D);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// LayerNorm over the last dim, one warp per row, fp32 statistics (two-pass in registers), fp16 out.
// timm: eps 1e-6 on the fp32 residual stream; CLIP: eps 1e-5 on the fp16 stream computed in fp32
// (SURVEY.md Appendix A.1/A.2). C in {512, 1024} is a template constant (fully unrolled, no predicates).
// HBM-bound: 6 B per element. A lane owns chunks of 8 consecutive elements (32 B loads in, one 16 B store out per
// chunk); gamma / beta are staged in shared memory by the whole block while the row loads are in flight, so the
// normalisation does not wait for a second round trip after the statistics.
// ------------------------------------------------------------------------------------------
template <typename TIn, int C>
__global__ void __launch_bounds__(256) layernorm_kernel(const TIn* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, __half* __restrict__ y,
                                                        long long M, float eps) {
  constexpr int kChunks = C / 256;  // 8-element chunks per lane
  __shared__ __align__(16) float sg[C];
  __shared__ __align__(16) float sb[C];
  griddep_launch_dependents();
  for (int i = threadIdx.x; i < C / 4; i += blockDim.x) {  // weights: not produced by the previous kernel
    reinterpret_cast<float4*>(sg)[i] = __ldg(reinterpret_cast<const float4*>(gamma) + i);
    reinterpret_cast<float4*>(sb)[i] = __ldg(reinterpret_cast<const float4*>(beta) + i);
  }
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  float v[8 * kChunks];
  if (row < M) {
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {
      const int col = (i * 32 + lane) * 8;
      if constexpr (sizeof(TIn) == 4) {
        const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + row * C + col);
        const float4 q0 = p[0], q1 = p[1];
        v[8 * i] = q0.x; v[8 * i + 1] = q0.y; v[8 * i + 2] = q0.z; v[8 * i + 3] = q0.w;
        v[8 * i + 4] = q1.x; v[8 * i + 5] = q1.y; v[8 * i + 6] = q1.z; v[8 * i + 7] = q1.w;
      } else {
        const uint4 q = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(x) + row * C + col);
        const __half2* qh = reinterpret_cast<const __half2*>(&q);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __half22float2(qh[k]);
          v[8 * i + 2 * k] = f.x;
          v[8 * i + 2 * k + 1] = f.y;
        }
      }
    }
  }
  __syncthreads();  // gamma / beta staged (all threads reach this, also those of rows beyond M)
  if (row >= M) return;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8 * kChunks; ++i) s += v[i];
  const float mean = warp_sum(s) / C;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8 * kChunks; ++i) {
    const float d = v[i] - mean;
    ss += d * d;
  }
  const float rstd = rsqrtf(warp_sum(ss) / C + eps);
#pragma unroll
  for (int i = 0; i < kChunks; ++i) {
    const int col = (i * 32 + lane) * 8;
    const float4 g0 = *reinterpret_cast<const float4*>(sg + col), g1 = *reinterpret_cast<const float4*>(sg + col + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(sb + col), b1 = *reinterpret_cast<const float4*>(sb + col + 4);
    __half2 h[4];
    h[0] = __floats2half2_rn((v[8 * i] - mean) * rstd * g0.x + b0.x, (v[8 * i + 1] - mean) * rstd * g0.y + b0.y);
    h[1] = __floats2half2_rn((v[8 * i + 2] - mean) * rstd * g0.z + b0.z, (v[8 * i + 3] - mean) * rstd * g0.w + b0.w);
    h[2] = __floats2half2_rn((v[8 * i + 4] - mean) * rstd * g1.x + b1.x, (v[8 * i + 5] - mean) * rstd * g1.y + b1.y);
    h[3] = __floats2half2_rn((v[8 * i + 6] - mean) * rstd * g1.z + b1.z, (v[8 * i + 7] - mean) * rstd * g1.w + b1.w);
    *reinterpret_cast<uint4*>(y + row * C + col) = *reinterpret_cast<uint4*>(h);
  }
}

// ------------------------------------------------------------------------------------------
// readout split (modules/models/lseg_vit.py:79-90): tap fp32 [B, 1+T, D] ->
//   tok fp16 [B*T, D] (patch tokens) and cls fp16 [B, D].   one block per token row.
// ------------------------------------------------------------------------------------------
__global__ void readout_split_kernel(const float* __restrict__ tap, __half* __restrict__ tok,
                                     __half* __restrict__ cls, int T, int D) {
  griddep_launch_dependents();
  griddep_wait();
  const int row = blockIdx.x;
  const int b = row / (T + 1), t = row - b * (T + 1);
  const float* src = tap + static_cast<long long>(row) * D;
  __half* dst = (t == 0) ? cls + static_cast<long long>(b) * D : tok + (static_cast<long long>(b) * T + (t - 1)) * D;
  for (int c = threadIdx.x; c < D / 4; c += blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(src)[c];
    __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&h0);
    o.y = *reinterpret_cast<uint32_t*>(&h1);
    reinterpret_cast<uint2*>(dst)[c] = o;
  }
}
static inline int launch_readout_split(const float* tap, __half* tok, __half* cls, int B, int T, int D,
                                       cudaStream_t s) {
  launch_pdl(readout_split_kernel, dim3(B * (T + 1)), dim3(256), 0, s, tap, tok, cls, T, D);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// im2col for the one strided conv (act_postprocess4[4]: 3x3 s2 p1, modules/models/lseg_vit.py:516-522):
// NHWC fp16 [B,H,W,C] -> [B*Ho*Wo, 9*C], tap-major columns, zero halo. grid (Wo, Ho, B).
// ------------------------------------------------------------------------------------------
__global__ void im2col_3x3_s2_kernel(const __half* __restrict__ x, __half* __restrict__ a, int H, int W, int C) {
  griddep_launch_dependents();
  griddep_wait();
  const int ox = blockIdx.x, oy = blockIdx.y, b = blockIdx.z;
  const int Wo = gridDim.x, Ho = gridDim.y;
  const int c8 = C / 8;
  __half* dst = a + ((static_cast<long long>(b) * Ho + oy) * Wo + ox) * 9 * C;
  for (int tap = 0; tap < 9; ++tap) {
    const int iy = oy * 2 - 1 + tap / 3, ix = ox * 2 - 1 + tap % 3;
    const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
    const __half* src = x + ((static_cast<long long>(b) * H + iy) * W + ix) * C;
    for (int c = threadIdx.x; c < c8; c += blockDim.x) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (in) v = reinterpret_cast<const uint4*>(src)[c];
      reinterpret_cast<uint4*>(dst + static_cast<long long>(tap) * C)[c] = v;
    }
  }
}
static inline int launch_im2col_3x3_s2(const __half* x, __half* a, int B, int H, int W, int C, cudaStream_t s) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  launch_pdl(im2col_3x3_s2_kernel, dim3(Wo, Ho, B), dim3(128), 0, s, x, a, H, W, C);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// ResNet-101 trunk of the zero-shot model (lseg_net_zs.py:307-310; torchvision resnet101 split by
// _make_resnet_backbone, lseg_blocks_zs.py:109-119). Three glue kernels around the GEMMs:
//   stem_im2col   x fp32 NCHW [B,3,H,W] -> rows fp16 [B*(H/2)*(W/2), 192] of the 7x7 stride-2 pad-3 stem conv; column
//                 c*49 + ky*7 + kx (the flattening of conv1.weight [64,3,7,7]), columns 147..191 zero (K = 3 chunks of 64)
//   maxpool3x3s2  NHWC fp16 [B,Hi,Wi,C] -> [B,Hi/2,Wi/2,C], kernel 3 stride 2 pad 1 (padding never wins: -inf)
//   subsample2    NHWC fp16 [B,Hi,Wi,C] -> [B,Hi/2,Wi/2,C], pixel (2y, 2x): the A operand of a 1x1 stride-2 conv
// ------------------------------------------------------------------------------------------
constexpr int kStemK = 192;
__global__ void __launch_bounds__(192) stem_im2col_kernel(const float* __restrict__ x, __half* __restrict__ a, int H, int W) {
  griddep_launch_dependents();
  griddep_wait();
  const int Ho = H / 2, Wo = W / 2;
  const long long pix = blockIdx.x;  // b*Ho*Wo + oy*Wo + ox
  const int ox = static_cast<int>(pix % Wo);
  const int oy = static_cast<int>((pix / Wo) % Ho);
  const int b = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
  const int t = threadIdx.x;
  float v = 0.f;
  if (t < 147) {
    const int c = t / 49, r = t - c * 49;
    const int ky = r / 7, kx = r - ky * 7;
    const int iy = 2 * oy - 3 + ky, ix = 2 * ox - 3 + kx;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[((static_cast<long long>(b) * 3 + c) * H + iy) * W + ix];
  }
  a[pix * kStemK + t] = __float2half_rn(v);
}
static inline int launch_stem_im2col(const float* x, __half* a, int B, int H, int W, cudaStream_t s) {
  if (H % 2 || W % 2) {
    set_error("stem_im2col: H=%d, W=%d must be even", H, W);
    return -1;
  }
  launch_pdl(stem_im2col_kernel, dim3(static_cast<unsigned>(static_cast<long long>(B) * (H / 2) * (W / 2))), dim3(192), 0, s,
             x, a, H, W);
  LSEG_LAUNCH_CHECK();
}

__global__ void __launch_bounds__(256) maxpool3x3s2_nhwc_kernel(const __half* __restrict__ x, __half* __restrict__ y, int Hi,
                                                                int Wi, int C) {
  griddep_launch_dependents();
  griddep_wait();
  const int Ho = Hi / 2, Wo = Wi / 2, c8 = C / 8;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long total = static_cast<long long>(gridDim.y) * Ho * Wo * c8;
  (void)total;
  const int b = blockIdx.y;
  if (i >= static_cast<long long>(Ho) * Wo * c8) return;
  const int c = static_cast<int>(i % c8);
  const int ox = static_cast<int>((i / c8) % Wo);
  const int oy = static_cast<int>(i / (static_cast<long long>(c8) * Wo));
  __half2 m[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) m[k] = __float2half2_rn(-INFINITY);
  for (int dy = 0; dy < 3; ++dy) {
    const int iy = 2 * oy - 1 + dy;
    if (iy < 0 || iy >= Hi) continue;
    for (int dx = 0; dx < 3; ++dx) {
      const int ix = 2 * ox - 1 + dx;
      if (ix < 0 || ix >= Wi) continue;
      const uint4 q = reinterpret_cast<const uint4*>(x + ((static_cast<long long>(b) * Hi + iy) * Wi + ix) * C)[c];
      const __half2* qh = reinterpret_cast<const __half2*>(&q);
#pragma unroll
      for (int k = 0; k < 4; ++k) m[k] = __hmax2(m[k], qh[k]);
    }
  }
  reinterpret_cast<uint4*>(y + ((static_cast<long long>(b) * Ho + oy) * Wo + ox) * C)[c] = *reinterpret_cast<uint4*>(m);
}
static inline int launch_maxpool3x3s2_nhwc(const __half* x, __half* y, int B, int Hi, int Wi, int C, cudaStream_t s) {
  if (C % 8 || Hi % 2 || Wi % 2) {
    set_error("maxpool3x3s2: C %% 8 == 0 and even H, W (C=%d H=%d W=%d)", C, Hi, Wi);
    return -1;
  }
  const long long n = static_cast<long long>(Hi / 2) * (Wi / 2) * (C / 8);
  launch_pdl(maxpool3x3s2_nhwc_kernel, dim3(static_cast<unsigned>((n + 255) / 256), B), dim3(256), 0, s, x, y, Hi, Wi, C);
  LSEG_LAUNCH_CHECK();
}

__global__ void __launch_bounds__(256) subsample2_nhwc_kernel(const __half* __restrict__ x, __half* __restrict__ y, int Hi, int Wi,
                                                              int C) {
  griddep_launch_dependents();
  griddep_wait();
  const int Ho = Hi / 2, Wo = Wi / 2, c8 = C / 8;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= static_cast<long long>(Ho) * Wo * c8) return;
  const int c = static_cast<int>(i % c8);
  const int ox = static_cast<int>((i / c8) % Wo);
  const int oy = static_cast<int>(i / (static_cast<long long>(c8) * Wo));
  reinterpret_cast<uint4*>(y + ((static_cast<long long>(b) * Ho + oy) * Wo + ox) * C)[c] =
      reinterpret_cast<const uint4*>(x + ((static_cast<long long>(b) * Hi + 2 * oy) * Wi + 2 * ox) * C)[c];
}
static inline int launch_subsample2_nhwc(const __half* x, __half* y, int B, int Hi, int Wi, int C, cudaStream_t s) {
  if (C % 8 || Hi % 2 || Wi % 2) {
    set_error("subsample2: C %% 8 == 0 and even H, W (C=%d H=%d W=%d)", C, Hi, Wi);
    return -1;
  }
  const long long n = static_cast<long long>(Hi / 2) * (Wi / 2) * (C / 8);
  launch_pdl(subsample2_nhwc_kernel, dim3(static_cast<unsigned>((n + 255) / 256), B), dim3(256), 0, s, x, y, Hi, Wi, C);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// bilinear x2, align_corners=True, NHWC fp16 -> NHWC fp16 (fusion blocks, lseg_blocks.py:352-354).
// src = dst * (in-1)/(out-1), computed like ATen (float scale, float product).
// grid (ceil(Wo/32), Ho, B), 256 threads: a warp produces 4 consecutive output pixels (32 channel groups of 8 per
// pixel) with all 16 source loads in flight before the first use — one pixel per warp (4 loads, then a store) was
// bound by the load round trip (1.6 TB/s of output at 240x240x256).
// ------------------------------------------------------------------------------------------
__global__ void upsample2x_nhwc_kernel(const __half* __restrict__ x, __half* __restrict__ y, int H, int W, int C) {
  griddep_launch_dependents();
  griddep_wait();
  const int Ho = 2 * H, Wo = 2 * W, c8 = C / 8;
  const int oy = blockIdx.y, b = blockIdx.z;
  const int ox0 = blockIdx.x * 32 + (threadIdx.x >> 5) * 4;
  if (ox0 >= Wo) return;
  const float sh = (Ho > 1) ? static_cast<float>(H - 1) / (Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? static_cast<float>(W - 1) / (Wo - 1) : 0.f;
  const float fy = sh * oy;
  const int y0 = static_cast<int>(fy);
  const int y1 = min(y0 + 1, H - 1);
  const float ly = fy - y0, hy = 1.f - ly;
  const __half* base = x + static_cast<long long>(b) * H * W * C;
  const __half* row0 = base + static_cast<long long>(y0) * W * C;
  const __half* row1 = base + static_cast<long long>(y1) * W * C;
  __half* dst = y + ((static_cast<long long>(b) * Ho + oy) * Wo + ox0) * C;
  for (int c = threadIdx.x & 31; c < c8; c += 32) {
    uint4 q00[4], q01[4], q10[4], q11[4];
    float lx[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ox = min(ox0 + k, Wo - 1);  // clamped duplicates are computed but not stored
      const float fx = sw * ox;
      const int x0 = static_cast<int>(fx);
      const int x1 = min(x0 + 1, W - 1);
      lx[k] = fx - x0;
      q00[k] = reinterpret_cast<const uint4*>(row0 + static_cast<long long>(x0) * C)[c];
      q01[k] = reinterpret_cast<const uint4*>(row0 + static_cast<long long>(x1) * C)[c];
      q10[k] = reinterpret_cast<const uint4*>(row1 + static_cast<long long>(x0) * C)[c];
      q11[k] = reinterpret_cast<const uint4*>(row1 + static_cast<long long>(x1) * C)[c];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (ox0 + k >= Wo) break;
      const float hx = 1.f - lx[k];
      const __half2* a00 = reinterpret_cast<const __half2*>(&q00[k]);
      const __half2* a01 = reinterpret_cast<const __half2*>(&q01[k]);
      const __half2* a10 = reinterpret_cast<const __half2*>(&q10[k]);
      const __half2* a11 = reinterpret_cast<const __half2*>(&q11[k]);
      uint4 o;
      __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f00 = __half22float2(a00[j]), f01 = __half22float2(a01[j]);
        const float2 f10 = __half22float2(a10[j]), f11 = __half22float2(a11[j]);
        oh[j] = __floats2half2_rn(hy * (hx * f00.x + lx[k] * f01.x) + ly * (hx * f10.x + lx[k] * f11.x),
                                  hy * (hx * f00.y + lx[k] * f01.y) + ly * (hx * f10.y + lx[k] * f11.y));
      }
      reinterpret_cast<uint4*>(dst + static_cast<long long>(k) * C)[c] = o;
    }
  }
}
static inline int launch_upsample2x_nhwc(const __half* x, __half* y, int B, int H, int W, int C, cudaStream_t s) {
  launch_pdl(upsample2x_nhwc_kernel, dim3((2 * W + 31) / 32, 2 * H, B), dim3(256), 0, s, x, y, H, W, C);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// bilinear x2, align_corners=True, NHWC fp32 -> NHWC fp32 | fp16, C = 256: the fusion blocks' upsample applied AFTER
// out_conv (lseg_blocks.py:352-356 runs interpolate, then the 1x1 out_conv; both are linear per pixel and the
// interpolation weights sum to one, so conv-then-interpolate is the same map with a quarter of the conv's pixels, and —
// with the conv result kept in fp32 — one fp16 rounding less than interpolating an fp16 tensor first).
// A warp owns 4 consecutive output pixels of one output row (lane = 4 channels, two passes of 128): the <= 4 source
// pixels x 2 rows they touch are loaded once (8 x 16 B per lane in flight), each output picks its pair by a
// warp-uniform offset. `add` (nullable, fp32, output shape) is summed into the result: the engine passes the next
// fusion block's other input so that its residual conv needs one skip operand instead of two.
// grid (ceil(Wo/32), Ho, B), 256 threads.
// ------------------------------------------------------------------------------------------
// (256, 3): 80 registers with a 16-24 B spill measured FASTER than spill-free at 2 blocks / SM (121 vs 144 us at level 1)
template <typename TOut>
__global__ void __launch_bounds__(256, 3) upsample2x_nhwc256_f32_kernel(const float* __restrict__ x, TOut* __restrict__ y,
                                                                        const float* __restrict__ add, int H, int W) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int C = 256;
  const int Ho = 2 * H, Wo = 2 * W;
  const int oy = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31;
  const int ox0 = blockIdx.x * 32 + (threadIdx.x >> 5) * 4;
  if (ox0 >= Wo) return;
  const float sh = (Ho > 1) ? static_cast<float>(H - 1) / (Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? static_cast<float>(W - 1) / (Wo - 1) : 0.f;
  const float fy = __fmul_rn(sh, oy);  // rounded product, as torch forms the source index (no FMA into ly)
  const int y0 = static_cast<int>(fy);
  const int y1 = min(y0 + 1, H - 1);
  const float ly = fy - y0, hy = 1.f - ly;
  const int xs = static_cast<int>(sw * ox0);  // first source column; the 4 outputs use columns xs .. xs+3
  const float* base = x + static_cast<long long>(b) * H * W * C;
  const long long opix = (static_cast<long long>(b) * Ho + oy) * Wo + ox0;
  TOut* dst = y + opix * C;
#pragma unroll
  for (int p = 0; p < 2; ++p) {  // two passes of 128 channels: a lane holds 4 channels, loads are 512 B per warp
    const int ch = p * 128 + lane * 4;
    const float* row0 = base + static_cast<long long>(y0) * W * C + ch;
    const float* row1 = base + static_cast<long long>(y1) * W * C + ch;
    float4 q0[4], q1[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long off = static_cast<long long>(min(xs + j, W - 1)) * C;
      q0[j] = *reinterpret_cast<const float4*>(row0 + off);
      q1[j] = *reinterpret_cast<const float4*>(row1 + off);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (ox0 + k >= Wo) break;  // warp-uniform
      const float fx = __fmul_rn(sw, ox0 + k);
      const int x0 = static_cast<int>(fx);
      const float lx = fx - x0, hx = 1.f - lx;
      const int d = x0 - xs;  // 0..2, warp-uniform
      float4 a0 = q0[0], a1 = q0[1], b0 = q1[0], b1 = q1[1];
      if (d == 1) { a0 = q0[1]; a1 = q0[2]; b0 = q1[1]; b1 = q1[2]; }
      if (d == 2) { a0 = q0[2]; a1 = q0[3]; b0 = q1[2]; b1 = q1[3]; }
      float4 o;
      o.x = hy * (hx * a0.x + lx * a1.x) + ly * (hx * b0.x + lx * b1.x);
      o.y = hy * (hx * a0.y + lx * a1.y) + ly * (hx * b0.y + lx * b1.y);
      o.z = hy * (hx * a0.z + lx * a1.z) + ly * (hx * b0.z + lx * b1.z);
      o.w = hy * (hx * a0.w + lx * a1.w) + ly * (hx * b0.w + lx * b1.w);
      if (add) {  // the next block's skip term folded in here: xs[0] + xs[1] of lseg_blocks.py:345-347 (uniform branch)
        const float4 r = *reinterpret_cast<const float4*>(add + (opix + k) * C + ch);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      if constexpr (sizeof(TOut) == 4) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(dst) + static_cast<long long>(k) * C + ch) = o;
      } else {
        __half2 h[2] = {__floats2half2_rn(o.x, o.y), __floats2half2_rn(o.z, o.w)};
        *reinterpret_cast<uint2*>(reinterpret_cast<__half*>(dst) + static_cast<long long>(k) * C + ch) =
            *reinterpret_cast<uint2*>(h);
      }
    }
  }
}
// The same with an fp16 source (the engine's choice: the low-res out_conv result leaves its GEMM through the fp16
// TMA-store epilogue, 3x faster than the register-direct fp32 one at K = 256): a lane holds 8 channels, one pass.
template <typename TOut>
__global__ void __launch_bounds__(256, 3) upsample2x_nhwc256_f16_kernel(const __half* __restrict__ x, TOut* __restrict__ y,
                                                                        const float* __restrict__ add, int H, int W) {
  griddep_launch_dependents();
  griddep_wait();
  constexpr int C = 256;
  const int Ho = 2 * H, Wo = 2 * W;
  const int oy = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31;
  const int ox0 = blockIdx.x * 32 + (threadIdx.x >> 5) * 4;
  if (ox0 >= Wo) return;
  const float sh = (Ho > 1) ? static_cast<float>(H - 1) / (Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? static_cast<float>(W - 1) / (Wo - 1) : 0.f;
  const float fy = __fmul_rn(sh, oy);  // rounded product, as torch forms the source index (no FMA into ly)
  const int y0 = static_cast<int>(fy);
  const int y1 = min(y0 + 1, H - 1);
  const float ly = fy - y0, hy = 1.f - ly;
  const int xs = static_cast<int>(sw * ox0);
  const int ch = lane * 8;
  const __half* base = x + static_cast<long long>(b) * H * W * C + ch;
  const __half* row0 = base + static_cast<long long>(y0) * W * C;
  const __half* row1 = base + static_cast<long long>(y1) * W * C;
  const long long opix = (static_cast<long long>(b) * Ho + oy) * Wo + ox0;
  uint4 q0[4], q1[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long off = static_cast<long long>(min(xs + j, W - 1)) * C;
    q0[j] = *reinterpret_cast<const uint4*>(row0 + off);
    q1[j] = *reinterpret_cast<const uint4*>(row1 + off);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (ox0 + k >= Wo) break;  // warp-uniform
    const float fx = __fmul_rn(sw, ox0 + k);
    const int x0 = static_cast<int>(fx);
    const float lx = fx - x0, hx = 1.f - lx;
    const int d = x0 - xs;  // 0..2, warp-uniform
    uint4 a0 = q0[0], a1 = q0[1], b0 = q1[0], b1 = q1[1];
    if (d == 1) { a0 = q0[1]; a1 = q0[2]; b0 = q1[1]; b1 = q1[2]; }
    if (d == 2) { a0 = q0[2]; a1 = q0[3]; b0 = q1[2]; b1 = q1[3]; }
    const __half2* pa0 = reinterpret_cast<const __half2*>(&a0);
    const __half2* pa1 = reinterpret_cast<const __half2*>(&a1);
    const __half2* pb0 = reinterpret_cast<const __half2*>(&b0);
    const __half2* pb1 = reinterpret_cast<const __half2*>(&b1);
    float o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f00 = __half22float2(pa0[j]), f01 = __half22float2(pa1[j]);
      const float2 f10 = __half22float2(pb0[j]), f11 = __half22float2(pb1[j]);
      o[2 * j] = hy * (hx * f00.x + lx * f01.x) + ly * (hx * f10.x + lx * f11.x);
      o[2 * j + 1] = hy * (hx * f00.y + lx * f01.y) + ly * (hx * f10.y + lx * f11.y);
    }
    if (add) {
      const float4* rp = reinterpret_cast<const float4*>(add + (opix + k) * C + ch);
      const float4 r0 = rp[0], r1 = rp[1];
      o[0] += r0.x; o[1] += r0.y; o[2] += r0.z; o[3] += r0.w;
      o[4] += r1.x; o[5] += r1.y; o[6] += r1.z; o[7] += r1.w;
    }
    if constexpr (sizeof(TOut) == 4) {
      float* d32 = reinterpret_cast<float*>(y) + (opix + k) * C + ch;
      *reinterpret_cast<float4*>(d32) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(d32 + 4) = make_float4(o[4], o[5], o[6], o[7]);
    } else {
      __half2 h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(o[2 * j], o[2 * j + 1]);
      *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(y) + (opix + k) * C + ch) = *reinterpret_cast<uint4*>(h);
    }
  }
}
template <typename TOut>
static inline int launch_upsample2x_nhwc256_f16(const __half* x, TOut* y, const float* add, int B, int H, int W,
                                                cudaStream_t s) {
  launch_pdl(upsample2x_nhwc256_f16_kernel<TOut>, dim3((2 * W + 31) / 32, 2 * H, B), dim3(256), 0, s, x, y, add, H, W);
  LSEG_LAUNCH_CHECK();
}
template <typename TOut>
static inline int launch_upsample2x_nhwc256_f32(const float* x, TOut* y, const float* add, int B, int H, int W,
                                                cudaStream_t s) {
  launch_pdl(upsample2x_nhwc256_f32_kernel<TOut>, dim3((2 * W + 31) / 32, 2 * H, B), dim3(256), 0, s, x, y, add, H, W);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// pixel-feature normalisation (modules/models/lseg_net.py:191,194): row / ||row||_2 in fp32, cast to
// fp16, then multiply by logit_scale in fp16 (the reference's `logit_scale * image_features.half()`
// rounds the product to fp16 before the matmul). One warp per row of C=512.
// ------------------------------------------------------------------------------------------
__global__ void l2norm_scale_kernel(const float* __restrict__ x, __half* __restrict__ y, long long M, int C,
                                    float logit_scale) {
  const int lane = threadIdx.x & 31;
  const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int nv = C / 128;
  float v[16];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i < nv) {
      const float4 q = *reinterpret_cast<const float4*>(x + row * C + (i * 32 + lane) * 4);
      v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
      ss += q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    }
  }
  const float nrm = sqrtf(warp_sum(ss));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (i < nv) {
      __half h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __half u = __float2half_rn(v[4 * i + j] / nrm);
        h[j] = __float2half_rn(logit_scale * __half2float(u));
      }
      *reinterpret_cast<uint2*>(y + row * C + (i * 32 + lane) * 4) = *reinterpret_cast<uint2*>(h);
    }
  }
}

// text-feature normalisation in fp16 (modules/models/lseg_net.py:192): norm rounded to fp16, then
// an fp16 division. One warp per row.
__global__ void l2norm_f16_kernel(const __half* __restrict__ x, __half* __restrict__ y, int M, int C) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  float ss = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float f = __half2float(x[static_cast<long long>(row) * C + c]);
    ss += f * f;
  }
  const float nrm = __half2float(__float2half_rn(sqrtf(warp_sum(ss))));
  for (int c = lane; c < C; c += 32)
    y[static_cast<long long>(row) * C + c] = __float2half_rn(__half2float(x[static_cast<long long>(row) * C + c]) / nrm);
}

// w0*a + w1*b with ONE fixed rounding sequence (product, then fused multiply-add): the logits upsample and the fused
// argmax below must produce bit-identical interpolated values, which FMA contraction left to the compiler would not
// guarantee across two kernels.
__device__ __forceinline__ float lerp2(float w0, float a, float w1, float b) { return __fmaf_rn(w0, a, __fmul_rn(w1, b)); }

// ------------------------------------------------------------------------------------------
// output head (modules/models/lseg_net.py:196,203): fp16 logits [planes,H,W] (values of the fp16
// matmul) -> .float() -> bilinear x2 align_corners=True -> fp32 [planes,2H,2W].
// HBM-write-bound (K*H*W*4 B per image). Separable: a WARP owns kUpRows consecutive output rows of one
// plane; per row it (1) blends the two source rows vertically into a private smem line (16 B loads,
// coalesced; stored split by column parity), (2) blends horizontally from that line — 2 LDS + 2 FMA per output — and streams float4
// stores (512 B contiguous per warp instruction). The horizontal taps/weights live in registers and are
// reused for all of the warp's rows. grid (ceil(Ho / (8 warps * kUpRows)), planes), W % 8 == 0, W <= 512.
// ------------------------------------------------------------------------------------------
static int g_upsample_split = getenv("LSEG_UPSAMPLE_SPLIT") ? atoi(getenv("LSEG_UPSAMPLE_SPLIT")) : 0;
constexpr int kUpRows = 4;      // output rows per warp
constexpr int kUpMaxW = 512;    // widest source row (smem line)
// 8 consecutive source values as fp32 (TIn = __half: one 16-byte load; float: two)
__device__ __forceinline__ void load8_f32(const __half* p, float (&o)[8]) {
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const __half2* ah = reinterpret_cast<const __half2*>(&a);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = __half22float2(ah[k]);
    o[2 * k] = f.x;
    o[2 * k + 1] = f.y;
  }
}
__device__ __forceinline__ void load8_f32(const float* p, float (&o)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}
// TIn = __half: the fp16 matmul result (arch_option 0); float: the output of the arch_option 1/2 head blocks
// SPLIT: smem line stored split by column parity (A/B switch lseg_debug_upsample_layout / LSEG_UPSAMPLE_SPLIT)
template <bool STREAM, typename TIn = __half, bool SPLIT = false>  // STREAM: st.global.cs stores (LSEG_UPSAMPLE_CS=1)
__global__ void upsample2x_nchw_kernel(const TIn* __restrict__ x, float* __restrict__ y, int H, int W) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ __align__(16) float line[8][kUpMaxW];
  const int Ho = 2 * H, Wo = 2 * W, w4 = Wo / 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long pl = blockIdx.y;
  const float sh = (Ho > 1) ? static_cast<float>(H - 1) / (Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? static_cast<float>(W - 1) / (Wo - 1) : 0.f;
  const TIn* plane = x + pl * H * W;
  float* oplane = y + pl * Ho * Wo;
  float* v = line[warp];
  const int oy0 = (blockIdx.x * 8 + warp) * kUpRows;
  for (int rr = 0; rr < kUpRows; ++rr) {
    const int oy = oy0 + rr;
    if (oy >= Ho) break;  // warp-uniform
    const float fy = sh * oy;
    const int y0 = static_cast<int>(fy);
    const int y1 = min(y0 + 1, H - 1);
    const float ly = fy - y0, hy = 1.f - ly;
    const TIn* r0 = plane + y0 * W;
    const TIn* r1 = plane + y1 * W;
    __syncwarp();
    for (int c = lane; c < W / 8; c += 32) {
      float fa[8], fb[8], o[8];
      load8_f32(r0 + 8 * c, fa);
      load8_f32(r1 + 8 * c, fb);
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] = lerp2(hy, fa[k], ly, fb[k]);
      // de-interleaved line: even source columns in v[0..), odd ones in v[kUpMaxW/2..). The horizontal pass of a
      // lane reads columns ~2*xq + const, i.e. a stride of two words across the warp: interleaved that is a 2-way bank
      // conflict on every LDS (the kernel is LSU-bound), split by parity it is one conflict-free wavefront
      if (SPLIT) {
        reinterpret_cast<float4*>(v)[c] = make_float4(o[0], o[2], o[4], o[6]);
        reinterpret_cast<float4*>(v + kUpMaxW / 2)[c] = make_float4(o[1], o[3], o[5], o[7]);
      } else {
        reinterpret_cast<float4*>(v)[2 * c] = make_float4(o[0], o[1], o[2], o[3]);
        reinterpret_cast<float4*>(v)[2 * c + 1] = make_float4(o[4], o[5], o[6], o[7]);
      }
    }
    __syncwarp();
    float* orow = oplane + static_cast<long long>(oy) * Wo;
    // horizontal taps are recomputed per output (4 flops) instead of cached: caching them cost 64
    // registers per thread and capped the SM at one resident block
#pragma unroll 1
    for (int xq = lane; xq < w4; xq += 32) {
      {
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float fx = sw * (xq * 4 + k);
          const int xi = static_cast<int>(fx);
          const float lxk = fx - xi;
          const int xa = min(xi, W - 1), xb = min(xa + 1, W - 1);
          if (SPLIT)
            o[k] = lerp2(1.f - lxk, v[(xa & 1) * (kUpMaxW / 2) + (xa >> 1)], lxk, v[(xb & 1) * (kUpMaxW / 2) + (xb >> 1)]);
          else
            o[k] = lerp2(1.f - lxk, v[xa], lxk, v[xb]);
        }
        if (STREAM)
          __stcs(reinterpret_cast<float4*>(orow + xq * 4), make_float4(o[0], o[1], o[2], o[3]));
        else
          *reinterpret_cast<float4*>(orow + xq * 4) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}
template <typename TIn>
static inline int launch_upsample2x_nchw(const TIn* x, float* y, long long planes, int H, int W, cudaStream_t s) {
  if (W % 8 != 0 || W > kUpMaxW || planes > 65535) {
    set_error("upsample2x_nchw: needs W %% 8 == 0, W <= %d, planes <= 65535 (W=%d planes=%lld)", kUpMaxW, W, planes);
    return -1;
  }
  const int rows_per_block = 8 * kUpRows;
  static const bool stream_stores = getenv("LSEG_UPSAMPLE_CS") != nullptr;
  const dim3 grid((2 * H + rows_per_block - 1) / rows_per_block, static_cast<unsigned>(planes));
  if (stream_stores)
    launch_pdl(upsample2x_nchw_kernel<true, TIn, false>, grid, dim3(256), 0, s, x, y, H, W);
  else if (g_upsample_split)
    launch_pdl(upsample2x_nchw_kernel<false, TIn, true>, grid, dim3(256), 0, s, x, y, H, W);
  else
    launch_pdl(upsample2x_nchw_kernel<false, TIn, false>, grid, dim3(256), 0, s, x, y, H, W);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// "Background" variant of the logits upsample for the multi-GPU gather (lang-seg_b200/parallel.py::LogitsGather): the
// gathering rank expands every shard's fp16 low-res logits to fp32 on a side stream while its NEXT step's trunk runs.
// The trunk's GEMM / attention CTAs own all of an SM's shared memory and all but ~4 K of its registers, so a kernel
// that is to run BESIDE them (instead of serialising with them, which is what upsample2x_nchw_kernel does) must use no
// shared memory and <= 32 registers x 128 threads: source values are read straight from global memory (the fp16 source
// is 1/8 of the bytes and L1/L2-resident), 8 scalar loads + one streaming 16 B store per 4 outputs. It does not need
// HBM peak: 8.85 GB (N = 8) within one 8.4 ms step is 1.05 TB/s. Same lerp2 sequence as upsample2x_nchw_kernel ->
// bit-identical values. grid (ceil(Ho / kBgRows), planes), 128 threads: a block walks kBgRows output rows, a thread
// owns 4 consecutive output columns per 512-column pass.
// ------------------------------------------------------------------------------------------
constexpr int kBgRows = 16;
__global__ void __launch_bounds__(128, 16) upsample2x_nchw_bg_kernel(const __half* __restrict__ x, float* __restrict__ y,
                                                                     int H, int W) {
  const int Ho = 2 * H, Wo = 2 * W;
  const float sh = (Ho > 1) ? static_cast<float>(H - 1) / (Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? static_cast<float>(W - 1) / (Wo - 1) : 0.f;
  const long long pl = blockIdx.y;
  const __half* plane = x + pl * H * W;
  float* oplane = y + pl * Ho * Wo;
  const int oy_end = min(Ho, static_cast<int>(blockIdx.x + 1) * kBgRows);
  for (int oy = blockIdx.x * kBgRows; oy < oy_end; ++oy) {
    const float fy = sh * oy;
    const int y0 = static_cast<int>(fy);
    const int y1 = min(y0 + 1, H - 1);
    const float ly = fy - y0, hy = 1.f - ly;
    const __half* r0 = plane + y0 * W;
    const __half* r1 = plane + y1 * W;
    for (int ox = threadIdx.x * 4; ox < Wo; ox += 512) {
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float fx = sw * (ox + k);
        const int xi = static_cast<int>(fx);
        const float lxk = fx - xi;
        const int xa = min(xi, W - 1), xb = min(xa + 1, W - 1);
        const float va = lerp2(hy, __half2float(__ldg(r0 + xa)), ly, __half2float(__ldg(r1 + xa)));
        const float vb = lerp2(hy, __half2float(__ldg(r0 + xb)), ly, __half2float(__ldg(r1 + xb)));
        o[k] = lerp2(1.f - lxk, va, lxk, vb);
      }
      __stcs(reinterpret_cast<float4*>(oplane + static_cast<long long>(oy) * Wo + ox), make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}
static inline int launch_upsample2x_nchw_bg(const __half* x, float* y, long long planes, int H, int W, cudaStream_t s) {
  if (W % 2 != 0 || planes > 65535 || planes <= 0) {
    set_error("upsample2x_nchw_bg: needs W %% 2 == 0, 0 < planes <= 65535 (W=%d planes=%lld)", W, planes);
    return -1;
  }
  const dim3 grid((2 * H + kBgRows - 1) / kBgRows, static_cast<unsigned>(planes));
  upsample2x_nchw_bg_kernel<<<grid, 128, 0, s>>>(x, y, H, W);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// Fused scratch.output_conv + class argmax (SURVEY.md §8(f) next row 2): the callers of LSeg.forward only ever take
// torch.max(logits, 1)[1] (lseg_app.py:357-360, test_lseg.py:397, test_lseg_zs.py:301). This kernel interpolates the
// fp16 low-resolution logits [B, K, H, W] exactly like upsample2x_nchw_kernel (same lerp2 sequence, so the values are
// bit-identical to the fp32 logits forward() returns) and keeps only the first maximal class per output pixel:
// 8 B per pixel leave the GPU instead of 4*K.
// One warp = one output row of one image, all K classes in turn: the two source rows of class k are interpolated
// vertically into a (double-buffered) smem line, then every lane updates the running (max, argmax) of its
// lane + 32 j outputs, j < kArgJ. Output columns beyond 32*kArgJ are handled in further passes.
// ------------------------------------------------------------------------------------------
constexpr int kArgJ = 16;  // outputs per lane per pass (Wo <= 512 in one pass)
template <typename TIn>
__global__ void __launch_bounds__(256) upsample2x_argmax_kernel(const TIn* __restrict__ lr, long long* __restrict__ mask,
                                                                int K, int H, int W) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ __align__(16) float line[8][2][kUpMaxW];
  const int Ho = 2 * H, Wo = 2 * W;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int oy = blockIdx.x * 8 + warp;
  if (oy >= Ho) return;  // warp-uniform
  const float sh = (Ho > 1) ? static_cast<float>(H - 1) / (Ho - 1) : 0.f;
  const float sw = (Wo > 1) ? static_cast<float>(W - 1) / (Wo - 1) : 0.f;
  const float fy = sh * oy;
  const int y0 = static_cast<int>(fy);
  const int y1 = min(y0 + 1, H - 1);
  const float ly = fy - y0, hy = 1.f - ly;
  const long long plane_sz = static_cast<long long>(H) * W;
  const TIn* img = lr + static_cast<long long>(b) * K * plane_sz;
  long long* orow = mask + (static_cast<long long>(b) * Ho + oy) * Wo;
  for (int ox0 = 0; ox0 < Wo; ox0 += 32 * kArgJ) {
    int xa[kArgJ], xb[kArgJ];
    float lx[kArgJ], best[kArgJ];
    int arg[kArgJ];
#pragma unroll
    for (int j = 0; j < kArgJ; ++j) {
      const int ox = min(ox0 + lane + 32 * j, Wo - 1);
      const float fx = sw * ox;
      const int xi = static_cast<int>(fx);
      lx[j] = fx - xi;
      xa[j] = min(xi, W - 1);
      xb[j] = min(xa[j] + 1, W - 1);
      best[j] = -INFINITY;
      arg[j] = 0;
    }
    for (int k = 0; k < K; ++k) {
      const TIn* r0 = img + k * plane_sz + static_cast<long long>(y0) * W;
      const TIn* r1 = img + k * plane_sz + static_cast<long long>(y1) * W;
      float* v = line[warp][k & 1];
      for (int c = lane; c < W / 8; c += 32) {
        float fa[8], fb[8], o[8];
        load8_f32(r0 + 8 * c, fa);
        load8_f32(r1 + 8 * c, fb);
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] = lerp2(hy, fa[q], ly, fb[q]);
        reinterpret_cast<float4*>(v)[2 * c] = make_float4(o[0], o[1], o[2], o[3]);
        reinterpret_cast<float4*>(v)[2 * c + 1] = make_float4(o[4], o[5], o[6], o[7]);
      }
      __syncwarp();  // line k visible; line k-1 (other buffer) is free again after this point for iteration k+1
#pragma unroll
      for (int j = 0; j < kArgJ; ++j) {
        const float val = lerp2(1.f - lx[j], v[xa[j]], lx[j], v[xb[j]]);
        if (val > best[j]) {  // strict: the first maximal class wins, like torch.max on the logits
          best[j] = val;
          arg[j] = k;
        }
      }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < kArgJ; ++j) {
      const int ox = ox0 + lane + 32 * j;
      if (ox < Wo) orow[ox] = arg[j];
    }
  }
}
template <typename TIn>
static inline int launch_upsample2x_argmax(const TIn* lr, long long* mask, int B, int K, int H, int W, cudaStream_t s) {
  if (W % 8 != 0 || W > kUpMaxW || B > 65535 || K <= 0) {
    set_error("upsample2x_argmax: needs W %% 8 == 0, W <= %d, B <= 65535, K > 0 (W=%d B=%d K=%d)", kUpMaxW, W, B, K);
    return -1;
  }
  launch_pdl(upsample2x_argmax_kernel<TIn>, dim3((2 * H + 7) / 8, B), dim3(256), 0, s, lr, mask, K, H, W);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// arch_option 1 / 2 head blocks (modules/models/lseg_net.py:29-79, applied at :198-201 to the fp32 view of the
// low-resolution logits [B,K,h,w]): ONE 3x3 convolution kernel (Conv2d(1,1,3,padding=1), weight [1,1,3,3] + bias)
// shared by every class plane (`depthwise_conv` reshapes the classes into the batch), optionally plus the per-pixel
// maximum over the classes (`bottleneck_block`: x.max(dim=1) skip), optionally an activation. fp32 arithmetic.
// ------------------------------------------------------------------------------------------
enum HeadAct { HEAD_ACT_NONE = 0, HEAD_ACT_RELU = 1, HEAD_ACT_LRELU = 2, HEAD_ACT_TANH = 3 };
struct HeadBlockW {
  float w[9];
  float bias;
};
__device__ __forceinline__ float ld_f32(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ float ld_f32(const float* p) { return *p; }

// cmax[b, y, x] = max_k x[b, k, y, x]; grid (ceil(h*w/256), B)
template <typename TIn>
__global__ void channel_max_kernel(const TIn* __restrict__ x, float* __restrict__ cmax, int K, int P) {
  griddep_launch_dependents();
  griddep_wait();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= P) return;
  const TIn* src = x + static_cast<long long>(blockIdx.y) * K * P + pix;
  float m = -INFINITY;
  for (int k = 0; k < K; ++k) m = fmaxf(m, ld_f32(src + static_cast<long long>(k) * P));
  cmax[static_cast<long long>(blockIdx.y) * P + pix] = m;
}

// y[plane, i, j] = act( bias + sum_{a,b} w[a][b] x[plane, i+a-1, j+b-1] (+ cmax[b, i, j]) ), zero padding.
// grid (ceil(w/32), ceil(h/8), B*K), block (32, 8)
template <typename TIn>
__global__ void head_block_kernel(const TIn* __restrict__ x, const float* __restrict__ cmax, float* __restrict__ y, int K,
                                  int h, int w, HeadBlockW hw, int act) {
  griddep_launch_dependents();
  griddep_wait();
  const int j = blockIdx.x * 32 + threadIdx.x, i = blockIdx.y * 8 + threadIdx.y;
  if (i >= h || j >= w) return;
  const long long plane = blockIdx.z;
  const TIn* src = x + plane * h * w;
  float acc = 0.f;  // torch accumulates the taps first and adds the bias last
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int ii = i + a - 1;
    if (ii < 0 || ii >= h) continue;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const int jj = j + b - 1;
      if (jj < 0 || jj >= w) continue;
      acc = fmaf(hw.w[a * 3 + b], ld_f32(src + static_cast<long long>(ii) * w + jj), acc);
    }
  }
  acc += hw.bias;
  if (cmax) acc += cmax[(plane / K) * static_cast<long long>(h) * w + static_cast<long long>(i) * w + j];
  if (act == HEAD_ACT_RELU) acc = fmaxf(acc, 0.f);
  else if (act == HEAD_ACT_LRELU) acc = acc > 0.f ? acc : 0.01f * acc;
  else if (act == HEAD_ACT_TANH) acc = tanhf(acc);
  y[plane * h * w + static_cast<long long>(i) * w + j] = acc;
}

// one application of scratch.head_block; mode 1 = bottleneck_block (channel-max skip), 2 = depthwise_block
template <typename TIn>
static inline int launch_head_block(const TIn* x, float* cmax_ws, float* y, int B, int K, int h, int w, const HeadBlockW& hw,
                                    int mode, int act, cudaStream_t s) {
  const int P = h * w;
  if (static_cast<long long>(B) * K > 65535) {
    set_error("head_block: B*K = %lld planes exceed 65535", static_cast<long long>(B) * K);
    return -1;
  }
  if (mode == 1) {
    launch_pdl(channel_max_kernel<TIn>, dim3((P + 255) / 256, B), dim3(256), 0, s, x, cmax_ws, K, P);
    LSEG_CHECK_CUDA(cudaGetLastError());
  }
  launch_pdl(head_block_kernel<TIn>, dim3((w + 31) / 32, (h + 7) / 8, B * K), dim3(32, 8), 0, s, x,
             static_cast<const float*>(mode == 1 ? cmax_ws : nullptr), y, K, h, w, hw, act);
  LSEG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// CLIP text tower glue (SURVEY.md Appendix A.2)
// ------------------------------------------------------------------------------------------
// x = token_embedding(text).half() + positional_embedding.half()   (fp16 add). one block per token.
__global__ void text_embed_kernel(const long long* __restrict__ tokens, const float* __restrict__ tok_emb,
                                  const float* __restrict__ pos_emb, __half* __restrict__ x, int L, int Wd) {
  const int row = blockIdx.x;
  const int t = row % L;
  const long long id = tokens[row];
  const float* e = tok_emb + id * Wd;
  const float* pe = pos_emb + static_cast<long long>(t) * Wd;
  for (int d = threadIdx.x; d < Wd; d += blockDim.x)
    x[static_cast<long long>(row) * Wd + d] = __hadd(__float2half_rn(e[d]), __float2half_rn(pe[d]));
}
// rows at the EOT position: text.argmax(-1) (first maximal id), gathered after ln_final.
__global__ void text_eot_gather_kernel(const long long* __restrict__ tokens, const __half* __restrict__ x,
                                       __half* __restrict__ out, int K, int L, int Wd) {
  const int k = blockIdx.x;
  if (k >= K) return;
  __shared__ int s_pos;
  if (threadIdx.x == 0) {
    long long best = tokens[static_cast<long long>(k) * L];
    int bp = 0;
    for (int t = 1; t < L; ++t) {
      const long long v = tokens[static_cast<long long>(k) * L + t];
      if (v > best) { best = v; bp = t; }
    }
    s_pos = bp;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < Wd; d += blockDim.x)
    out[static_cast<long long>(k) * Wd + d] = x[(static_cast<long long>(k) * L + s_pos) * Wd + d];
}

}  // namespace lseg
