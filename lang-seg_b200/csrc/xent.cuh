// lseg_b200 — validation cross-entropy on the device: CrossEntropyLoss(ignore_index) with mean reduction, which is what
// PyTorch-Encoding's SegmentationLosses reduces to for LSeg (se_loss = aux = False, no class weight).
//
// Per pixel of image b with target t and fp32 logits v_0 .. v_{K-1}:
//     t == ignore_index  : skipped (neither summed nor counted)
//     t outside [0, K)   : loss = NaN, counted; the first such pixel is recorded (tag kXentTag) for lseg_read_watchdog
//     otherwise          : loss = (m + log(s)) - v_t, counted
// where m and s are an online log-sum-exp over the classes in index order (xent_lse_step): m = max_k v_k and
// s = sum_k exp(v_k - m), rescaled each time m grows. A NaN logit makes s, hence the loss, NaN.
//
// Reduction without floating-point atomics, so the same call gives the same bits every time: each block sums its pixels'
// losses and counts in fp64 in a fixed order (per thread in pixel order, then a fixed shuffle tree, then the warps in
// index order) into its own slot of a caller workspace, and a one-block kernel adds the slots in index order to the
// caller's accumulator double[2] = {sum of losses, counted pixels}. The accumulator is added to and never cleared.
#pragma once
#include "common.cuh"

namespace lseg {

constexpr int kXentTag = 79;  // lseg_read_watchdog tag of a loss target outside [0, K) that is not ignore_index
// [0] = kXentTag (0 = no error), [1] = image, [2] = pixel index within the image (y * W + x, clamped to int), [3] = the
// target value (clamped to int). Read and cleared by lseg_read_watchdog; kept apart from g_watchdog, whose record makes
// pending barrier waits give up, and from g_segstats_error, so neither hides the other.
__device__ int g_xent_error[4];

struct XentArgs {
  const long long* target;  // int64 [B, H, W]
  long long ignore_index;
  double* partials;         // 2 doubles per block of the loss kernel (xent_partials_fused / xent_partials_scores)
  double* acc;              // double[2] = {sum of losses, counted pixels}, added to
};

static inline long long xent_partials_fused(int B, int H) { return 2ll * B * ((H + 7) / 8); }
static inline long long xent_partials_scores(int B, long long P) { return 2ll * B * ((P + 1023) / 1024); }

// One class of the online log-sum-exp. m is the running maximum BEFORE v (the caller raises it to v when v > m); s the
// running sum relative to m. Start: m = -inf, s = 0. An equal value adds exactly 1 (also when both are infinite, where
// exp(v - m) would be NaN), so leading -inf logits do not poison s.
__device__ __forceinline__ void xent_lse_step(float v, float m, float& s) {
  s = v > m ? fmaf(s, expf(m - v), 1.f) : s + (v == m ? 1.f : expf(v - m));
}

// Class index of a target: t in [0, K), -1 for ignore_index, -2 for anything else (recorded).
__device__ __forceinline__ int xent_class(long long t, const XentArgs& a, int K, int b, long long pix) {
  if (t == a.ignore_index) return -1;
  if (t >= 0 && t < K) return static_cast<int>(t);
  if (atomicCAS(&g_xent_error[0], 0, kXentTag) == 0) {
    g_xent_error[1] = b;
    g_xent_error[2] = static_cast<int>(pix < INT_MAX ? pix : INT_MAX);
    g_xent_error[3] = static_cast<int>(t < INT_MIN ? INT_MIN : (t > INT_MAX ? INT_MAX : t));
  }
  return -2;
}

// Adds one pixel's loss to a thread's running (sum, count); tk as xent_class returns it.
__device__ __forceinline__ void xent_add_pixel(int tk, float m, float s, float vt, double& sum, int& count) {
  if (tk == -1) return;
  const float l = tk == -2 ? __int_as_float(0x7fffffff) : (m + logf(s)) - vt;
  sum += static_cast<double>(l);
  ++count;
}

// Block reduction in a fixed order into partials[2 * slot .. 2 * slot + 1]. Every thread of the block calls it; `red` is
// 16 bytes per warp of shared memory that the block no longer needs once all its threads arrive here.
__device__ __forceinline__ void xent_block_store(double sum, double c, double* red, double* partials, long long slot) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  const int warp = threadIdx.x >> 5;
  __syncthreads();  // red may alias shared memory other warps were still reading
  if ((threadIdx.x & 31) == 0) {
    red[2 * warp] = sum;
    red[2 * warp + 1] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ts = 0.0, tc = 0.0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {
      ts += red[2 * w];
      tc += red[2 * w + 1];
    }
    partials[2 * slot] = ts;
    partials[2 * slot + 1] = tc;
  }
}

// acc[0..1] += the sum of the n partial pairs, in index order per thread and then in a fixed tree: one block of 256.
__global__ void __launch_bounds__(256) xent_finish_kernel(const double* __restrict__ partials, long long n,
                                                          double* __restrict__ acc) {
  __shared__ double red[8 * 2];
  double s = 0.0, c = 0.0;
  for (long long i = threadIdx.x; i < n; i += 256) {
    s += partials[2 * i];
    c += partials[2 * i + 1];
  }
  __shared__ double total[2];
  xent_block_store(s, c, red, total, 0);
  if (threadIdx.x == 0) {
    acc[0] += total[0];
    acc[1] += total[1];
  }
}

// Standalone loss on fp32 scores [B, K, P]: grid (ceil(P / 1024), B), 256 threads, one thread per pixel with the K planes
// read in turn (coalesced across the warp, as seg_stats_scores_kernel reads them). Ignored pixels read no scores.
__global__ void __launch_bounds__(256) xent_scores_kernel(const float* __restrict__ scores, int K, long long P, XentArgs a) {
  __shared__ double red[8 * 2];
  const int b = blockIdx.y;
  const float* img = scores + static_cast<long long>(b) * K * P;
  const long long* tgt = a.target + static_cast<long long>(b) * P;
  double sum = 0.0;
  int count = 0;
  const long long base = static_cast<long long>(blockIdx.x) * 1024 + threadIdx.x;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    const long long pix = base + 256 * i;
    if (pix >= P) break;
    const int tk = xent_class(__ldg(tgt + pix), a, K, b, pix);
    if (tk == -1) continue;
    float m = -INFINITY, s = 0.f, vt = 0.f;
    if (tk >= 0) {
      const float* p = img + pix;
#pragma unroll 4
      for (int k = 0; k < K; ++k) {
        const float v = __ldg(p + static_cast<long long>(k) * P);
        xent_lse_step(v, m, s);
        m = v > m ? v : m;
      }
      vt = __ldg(p + static_cast<long long>(tk) * P);
    }
    xent_add_pixel(tk, m, s, vt, sum, count);
  }
  xent_block_store(sum, static_cast<double>(count), red, a.partials,
                   static_cast<long long>(b) * gridDim.x + blockIdx.x);
}

// Argument rules shared by every loss entry point; `need` = doubles of partials the launch writes.
static inline int xent_check(const char* fn, const XentArgs& a, long long partials_len, long long need) {
  if (!a.target) return set_error("%s: null loss target pointer", fn), -1;
  if (!a.acc) return set_error("%s: null loss accumulator pointer", fn), -1;
  if (!a.partials) return set_error("%s: null partials pointer", fn), -1;
  if (reinterpret_cast<uintptr_t>(a.target) % 8 != 0) return set_error("%s: loss target must be 8-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(a.acc) % 8 != 0) return set_error("%s: loss accumulator must be 8-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(a.partials) % 8 != 0) return set_error("%s: partials must be 8-byte aligned", fn), -1;
  if (partials_len < need)
    return set_error("%s: partials_len=%lld doubles, this call needs %lld", fn, partials_len, need), -1;
  return 0;
}

static inline int launch_xent_finish(const XentArgs& a, long long n, cudaStream_t s) {
  xent_finish_kernel<<<1, 256, 0, s>>>(a.partials, n, a.acc);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static inline int launch_xent_scores(const float* scores, int B, int K, int H, int W, const XentArgs& a,
                                     long long partials_len, cudaStream_t s) {
  const char* fn = "lseg_xent_scores";
  if (!scores) return set_error("%s: null scores pointer", fn), -1;
  if (reinterpret_cast<uintptr_t>(scores) % 4 != 0) return set_error("%s: scores must be 4-byte aligned", fn), -1;
  if (B <= 0 || B > 65535) return set_error("%s: B=%d must be in [1, 65535]", fn, B), -1;
  if (K <= 0) return set_error("%s: K=%d must be positive", fn, K), -1;
  if (H <= 0 || W <= 0) return set_error("%s: H=%d, W=%d must be positive", fn, H, W), -1;
  const long long P = static_cast<long long>(H) * W;
  if (xent_check(fn, a, partials_len, xent_partials_scores(B, P))) return -1;
  const long long blocks = (P + 1023) / 1024;
  xent_scores_kernel<<<dim3(static_cast<unsigned>(blocks), B), 256, 0, s>>>(scores, K, P, a);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return launch_xent_finish(a, blocks * B, s);
}

}  // namespace lseg
