// lseg_b200 — segmentation metric counters (pixAcc, mIoU, FB-IoU) accumulated on the device.
//
// The evaluation callers of LSeg.forward score its output with PyTorch-Encoding's SegmentationMetric (test_lseg.py:314-395:
// torch.max + numpy histograms on the host) or with the few-shot Evaluator.classify_prediction / AverageMeter
// (test_lseg_zs.py:290-316: per-image torch.histc, float32 counters). Both reduce to one per-pixel rule over integer
// counters, kept here in int64 rows of 3*nclass + 2 entries:
//     [ inter(nclass) | pred(nclass) | label(nclass) | correct | labeled ]
// For a pixel of image b with predicted class p and target t, row g = group[b] (row 0 without a group table):
//     t < 0           : ignored, no counter changes
//     otherwise       : labeled += 1
//       p == t        : correct += 1; inter[t] += 1 if t < nclass
//       0 <= p < nclass: pred[p] += 1
//       t < nclass    : label[t] += 1
// union = pred + label - inter is formed when the counters are read. The kernels ADD to the rows and never clear them.
// Each block holds one image (so one row): it counts into an int32 shared-memory histogram and flushes the non-zero bins
// with 64-bit global atomics, once per block. Above kSegSmemMaxClass classes the bins go straight to global memory.
#pragma once
#include "common.cuh"

namespace lseg {

constexpr int kSegStatsTag = 78;  // lseg_read_watchdog tag of a group id outside [0, G)
// Largest nclass whose block histogram (3*nclass + 2 int32 bins) fits the 16 KiB that upsample2x_argmax_kernel's static
// 32 KiB line buffer leaves below the 48 KiB a block may use without opting in: 4 * (3 * 1364 + 2) = 16376 bytes.
constexpr int kSegSmemMaxClass = 1364;
constexpr int kSegMaxClass = 1 << 24;   // keeps every bin index and row offset in int range
constexpr int kSegPixPerThread = 4;     // standalone kernels: a block of 256 threads covers 1024 pixels of one image
// [0] = kSegStatsTag (0 = no error), [1] = image, [2] = its group id, [3] = G. Read and cleared by lseg_read_watchdog.
// Kept apart from g_watchdog: a set g_watchdog makes pending barrier waits give up, which a bad group id must not do.
__device__ int g_segstats_error[4];

struct SegStatsArgs {
  const long long* target;  // int64 [B, H, W]
  const int* group;         // int32 [B], or nullptr: every image counts into row 0
  long long* stats;         // int64 [G, 3*nclass + 2], 8-byte aligned
  int nclass, G;
};

// Row of image b, or -1 when group[b] is outside [0, G): the image is skipped and the first such image is recorded.
__device__ __forceinline__ int seg_group_row(const SegStatsArgs& a, int b, bool report) {
  const int g = a.group ? a.group[b] : 0;
  if (g >= 0 && g < a.G) return g;
  if (report && atomicCAS(&g_segstats_error[0], 0, kSegStatsTag) == 0) {
    g_segstats_error[1] = b;
    g_segstats_error[2] = g;
    g_segstats_error[3] = a.G;
  }
  return -1;
}

__device__ __forceinline__ void seg_bin(int* hist, unsigned long long* grow, int i) {
  if (hist) atomicAdd(hist + i, 1);
  else atomicAdd(grow + i, 1ull);
}

// One pixel. correct / labeled are kept in registers by the caller: every pixel would otherwise hit the same two bins.
__device__ __forceinline__ void seg_count_pixel(long long p, long long t, int nclass, int* hist, unsigned long long* grow,
                                                int& labeled, int& correct) {
  if (t < 0) return;
  ++labeled;
  const bool hit = p == t;
  correct += hit;
  if (t < nclass) {
    seg_bin(hist, grow, 2 * nclass + static_cast<int>(t));
    if (hit) seg_bin(hist, grow, static_cast<int>(t));
  }
  if (p >= 0 && p < nclass) seg_bin(hist, grow, nclass + static_cast<int>(p));
}

// Zeroes the block histogram (nullptr: global mode, nothing to do). Every thread of the block calls it.
__device__ __forceinline__ void seg_block_begin(int* hist, int nclass) {
  if (!hist) return;
  for (int i = threadIdx.x; i < 3 * nclass + 2; i += blockDim.x) hist[i] = 0;
  __syncthreads();
}

// Adds the threads' correct / labeled counts and flushes the block histogram into the row. Every thread of the block calls
// it (hist and grow are block-uniform).
__device__ __forceinline__ void seg_block_finish(int* hist, unsigned long long* grow, int nclass, int labeled, int correct) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    labeled += __shfl_xor_sync(0xffffffffu, labeled, o);
    correct += __shfl_xor_sync(0xffffffffu, correct, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (hist) {
      atomicAdd(hist + 3 * nclass, correct);
      atomicAdd(hist + 3 * nclass + 1, labeled);
    } else {
      if (correct) atomicAdd(grow + 3 * nclass, static_cast<unsigned long long>(correct));
      if (labeled) atomicAdd(grow + 3 * nclass + 1, static_cast<unsigned long long>(labeled));
    }
  }
  if (!hist) return;
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * nclass + 2; i += blockDim.x) {
    const int v = hist[i];
    if (v) atomicAdd(grow + i, static_cast<unsigned long long>(v));
  }
}

// Prediction = first maximal class of fp32 scores [B, K, P] (strict '>': torch.max(scores, 1)[1] on NaN-free input; a NaN
// score never wins, and a pixel whose scores are all NaN or -inf is class 0). grid (ceil(P / 1024), B), 256 threads: one
// thread per pixel, the K planes read in turn, so every load is coalesced across the warp. Ignored pixels (t < 0) read no
// scores.
__global__ void __launch_bounds__(256) seg_stats_scores_kernel(const float* __restrict__ scores, int K, long long P,
                                                               SegStatsArgs a) {
  extern __shared__ int seg_hist[];
  const int b = blockIdx.y;
  const int g = seg_group_row(a, b, blockIdx.x == 0 && threadIdx.x == 0);
  if (g < 0) return;  // block-uniform
  int* hist = a.nclass <= kSegSmemMaxClass ? seg_hist : nullptr;
  unsigned long long* grow = reinterpret_cast<unsigned long long*>(a.stats + static_cast<long long>(g) * (3 * a.nclass + 2));
  seg_block_begin(hist, a.nclass);
  const float* img = scores + static_cast<long long>(b) * K * P;
  const long long* tgt = a.target + static_cast<long long>(b) * P;
  int labeled = 0, correct = 0;
  const long long base = static_cast<long long>(blockIdx.x) * (256 * kSegPixPerThread) + threadIdx.x;
#pragma unroll 1
  for (int i = 0; i < kSegPixPerThread; ++i) {
    const long long pix = base + 256 * i;
    if (pix >= P) break;
    const long long t = __ldg(tgt + pix);
    if (t < 0) continue;
    float best = -INFINITY;
    int arg = 0;
    const float* s = img + pix;
#pragma unroll 8
    for (int k = 0; k < K; ++k) {
      const float v = __ldg(s + static_cast<long long>(k) * P);
      if (v > best) {
        best = v;
        arg = k;
      }
    }
    seg_count_pixel(arg, t, a.nclass, hist, grow, labeled, correct);
  }
  seg_block_finish(hist, grow, a.nclass, labeled, correct);
}

// Prediction = an int64 mask [B, P]. grid (ceil(P / 1024), B), 256 threads.
__global__ void __launch_bounds__(256) seg_stats_mask_kernel(const long long* __restrict__ pred, long long P, SegStatsArgs a) {
  extern __shared__ int seg_hist[];
  const int b = blockIdx.y;
  const int g = seg_group_row(a, b, blockIdx.x == 0 && threadIdx.x == 0);
  if (g < 0) return;  // block-uniform
  int* hist = a.nclass <= kSegSmemMaxClass ? seg_hist : nullptr;
  unsigned long long* grow = reinterpret_cast<unsigned long long*>(a.stats + static_cast<long long>(g) * (3 * a.nclass + 2));
  seg_block_begin(hist, a.nclass);
  const long long* pm = pred + static_cast<long long>(b) * P;
  const long long* tgt = a.target + static_cast<long long>(b) * P;
  int labeled = 0, correct = 0;
  const long long base = static_cast<long long>(blockIdx.x) * (256 * kSegPixPerThread) + threadIdx.x;
#pragma unroll
  for (int i = 0; i < kSegPixPerThread; ++i) {
    const long long pix = base + 256 * i;
    if (pix < P) seg_count_pixel(__ldg(pm + pix), __ldg(tgt + pix), a.nclass, hist, grow, labeled, correct);
  }
  seg_block_finish(hist, grow, a.nclass, labeled, correct);
}

static inline size_t seg_smem_bytes(int nclass) {
  return nclass <= kSegSmemMaxClass ? sizeof(int) * (3 * static_cast<size_t>(nclass) + 2) : 0;
}

// Argument checks shared by every entry point that accumulates counters; `pred` is the scores / mask / input image.
static inline int seg_stats_check(const char* fn, const void* pred, const SegStatsArgs& a, int B, int H, int W) {
  if (!pred) return set_error("%s: null prediction / input pointer", fn), -1;
  if (!a.target) return set_error("%s: null target pointer", fn), -1;
  if (!a.stats) return set_error("%s: null stats pointer", fn), -1;
  if (reinterpret_cast<uintptr_t>(a.stats) % 8 != 0) return set_error("%s: stats must be 8-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(a.target) % 8 != 0) return set_error("%s: target must be 8-byte aligned", fn), -1;
  if (a.group && reinterpret_cast<uintptr_t>(a.group) % 4 != 0) return set_error("%s: group must be 4-byte aligned", fn), -1;
  if (a.nclass <= 0 || a.nclass > kSegMaxClass)
    return set_error("%s: nclass=%d must be in [1, %d]", fn, a.nclass, kSegMaxClass), -1;
  if (a.G <= 0) return set_error("%s: G=%d rows must be positive", fn, a.G), -1;
  if (static_cast<long long>(a.G) * (3ll * a.nclass + 2) > (1ll << 40))
    return set_error("%s: G=%d x nclass=%d counters are too many", fn, a.G, a.nclass), -1;
  if (B <= 0 || B > 65535) return set_error("%s: B=%d must be in [1, 65535]", fn, B), -1;
  if (H <= 0 || W <= 0) return set_error("%s: H=%d, W=%d must be positive", fn, H, W), -1;
  return 0;
}

static inline int launch_seg_stats_scores(const float* scores, int B, int K, int H, int W, const SegStatsArgs& a,
                                          cudaStream_t s) {
  if (seg_stats_check("seg_stats_scores", scores, a, B, H, W)) return -1;
  if (K <= 0) return set_error("seg_stats_scores: K=%d must be positive", K), -1;
  const long long P = static_cast<long long>(H) * W;
  const long long blocks = (P + 256 * kSegPixPerThread - 1) / (256 * kSegPixPerThread);
  seg_stats_scores_kernel<<<dim3(static_cast<unsigned>(blocks), B), 256, seg_smem_bytes(a.nclass), s>>>(scores, K, P, a);
  LSEG_LAUNCH_CHECK();
}

static inline int launch_seg_stats_mask(const long long* pred, int B, int H, int W, const SegStatsArgs& a, cudaStream_t s) {
  if (seg_stats_check("seg_stats_mask", pred, a, B, H, W)) return -1;
  if (reinterpret_cast<uintptr_t>(pred) % 8 != 0) return set_error("seg_stats_mask: pred must be 8-byte aligned"), -1;
  const long long P = static_cast<long long>(H) * W;
  const long long blocks = (P + 256 * kSegPixPerThread - 1) / (256 * kSegPixPerThread);
  seg_stats_mask_kernel<<<dim3(static_cast<unsigned>(blocks), B), 256, seg_smem_bytes(a.nclass), s>>>(pred, P, a);
  LSEG_LAUNCH_CHECK();
}

}  // namespace lseg
