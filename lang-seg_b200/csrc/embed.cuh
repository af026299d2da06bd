// lseg_b200 — export of the pixel embedding as the reference's normalised image_features (lseg_net.py:185-191).
//
// The engine keeps the embedding as fp16 rows emb [B*P, C] (head1's output, un-normalised) plus fp32 partial squared
// norms [B*P, C/32] of head1's fp32 accumulators; the pixel x text GEMM applies 1/||row|| in its epilogue. This kernel
// writes image_features = emb * rsqrt(sum of the partials) as fp32 NCHW [B, C, h, w] (h*w = P), the partials summed in
// index order exactly as that epilogue sums them.
//
// Memory-bound: per pixel 2C + C/8 bytes read and 4C written (3136 B at C = 512). A CTA owns 32 consecutive pixels of
// one image and walks the channels in chunks of 64: 16-byte loads along the channel rows (8 threads per 128-byte row
// segment), a transpose through shared memory, and 16-byte stores along the pixel rows of each output channel plane
// (8 threads per 128-byte segment).
#pragma once

namespace lseg {

constexpr int kEmbPx = 32;     // pixels per CTA
constexpr int kEmbCh = 64;     // channels per chunk
constexpr int kEmbThreads = 256;
constexpr int kEmbMaxParts = 24;  // C <= 768

__global__ void __launch_bounds__(kEmbThreads) embed_features_kernel(const __half* __restrict__ emb,
                                                                     const float* __restrict__ sumsq,
                                                                     float* __restrict__ out, int C, long long P) {
  // odd row stride: the transposed reads (4 channels x 8 pixel quads per warp) hit 32 distinct banks
  __shared__ float tile[kEmbPx][kEmbCh + 1];
  __shared__ float part[kEmbPx * kEmbMaxParts];
  __shared__ float scale[kEmbPx];
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const long long p0 = static_cast<long long>(blockIdx.x) * kEmbPx;
  const int npx = static_cast<int>(P - p0 < kEmbPx ? P - p0 : kEmbPx);
  const int parts = C >> 5;
  const long long row0 = static_cast<long long>(b) * P + p0;  // first embedding row of this CTA

  // partial squared norms of the CTA's pixels: contiguous in memory, loaded coalesced
  for (int i = tid; i < npx * parts; i += kEmbThreads) part[i] = sumsq[row0 * parts + i];
  __syncthreads();
  if (tid < kEmbPx) {
    float ss = 0.f;
    for (int i = 0; i < parts; ++i) ss += (tid < npx) ? part[tid * parts + i] : 1.f;
    scale[tid] = rsqrtf(ss);
  }
  __syncthreads();

  const int lpx = tid >> 3, lch = (tid & 7) * 8;   // load: pixel, first of 8 channels
  const int sq = (tid & 7) * 4, sch = tid >> 3;    // store: first of 4 pixels, channel (and +32)
  const bool full = npx == kEmbPx;
  for (int c0 = 0; c0 < C; c0 += kEmbCh) {
    if (lpx < npx) {
      const uint4 v = *reinterpret_cast<const uint4*>(emb + (row0 + lpx) * C + c0 + lch);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
      const float s = scale[lpx];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        tile[lpx][lch + 2 * j] = f.x * s;
        tile[lpx][lch + 2 * j + 1] = f.y * s;
      }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int ch = sch + 32 * r;
      float* dst = out + (static_cast<long long>(b) * C + c0 + ch) * P + p0 + sq;
      if (full) {
        *reinterpret_cast<float4*>(dst) = make_float4(tile[sq][ch], tile[sq + 1][ch], tile[sq + 2][ch], tile[sq + 3][ch]);
      } else {
        for (int q = 0; q < 4; ++q)
          if (sq + q < npx) dst[q] = tile[sq + q][ch];
      }
    }
    __syncthreads();
  }
}

// emb fp16 [B, P, C] (16-byte aligned), sumsq fp32 [B, P, C/32], out fp32 [B, C, P] (16-byte aligned, P % 4 == 0 for
// the vector stores; any P otherwise works through the scalar tail).
static inline int launch_embed_features(const __half* emb, const float* sumsq, float* out, int B, long long P, int C,
                                        cudaStream_t s) {
  if (C % kEmbCh != 0 || C / 32 > kEmbMaxParts) return set_error("embedding_features: C=%d (512 or 768)", C), -1;
  if (P % 4 != 0) return set_error("embedding_features: h*w=%lld must be a multiple of 4", P), -1;
  const long long blocks = (P + kEmbPx - 1) / kEmbPx;
  if (blocks > 0x7fffffffLL || B > 65535) return set_error("embedding_features: B=%d, h*w=%lld too large", B, P), -1;
  embed_features_kernel<<<dim3(static_cast<unsigned>(blocks), B), kEmbThreads, 0, s>>>(emb, sumsq, out, C, P);
  LSEG_LAUNCH_CHECK();
}

}  // namespace lseg
