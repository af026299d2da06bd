// lseg_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   C[M,N] = epilogue( A[M,K] * W[N,K]^T )       fp16 operands, fp32 accumulate in registers
//
// One kernel family covers every dense contraction of the LSeg forward path (SURVEY.md §2b k1,k4,k6-k8,
// k10-k17,k19): linear layers, 1x1 convs, kernel==stride transposed convs (depth-to-space store),
// and 3x3 stride-1 convs as implicit GEMM (the A tile of tap (dy,dx) is a shifted 4-D TMA box of
// the NHWC activation; TMA zero-fills the padding halo).
//
// Roles (one CTA per SM, persistent over a static round-robin list of 128 x 128 tiles):
//   warpgroup 0   TMA producer (warp 0, one elected lane): fills the A/B smem ring (128B-swizzled, K-major)
//   warpgroups 1-2  consumers: each issues wgmma m64n128k16 for 64 of the tile's 128 rows (accumulator in registers),
//                 then stages its fp32 accumulators in shared memory, and the 8 consumer warps run the epilogue with
//                 thread <-> output row (warp = 32 rows x 64 columns): scale/bias/act/residual -> global.
// The producer runs up to kStages k-chunks ahead, so the next tile's operands stream in during the epilogue.
//
// Epilogue modes:
//   EPI_DIRECT   stores straight from registers, thread <-> accumulator row.
//   EPI_TMA_F16  fp16 row-major outputs: each epilogue warp packs 32 rows x 64 columns into a private
//                128B-swizzled smem tile and one elected lane issues a bulk tensor store.
//   EPI_TMA_ADD  in-place fp32 residual stream (x += A W^T + b): the warp stages 32 x 32 fp32 results and
//                issues a bulk tensor REDUCE-ADD, so the residual is never read by the SM at all.
// Per-column constants (bias, folded-BN scale) live in registers per tile and are distributed by shuffle.
#pragma once
#include "common.cuh"

namespace lseg {

constexpr int kGemmBM = 128;
constexpr int kGemmBN = 128;
constexpr int kGemmBK = 64;
constexpr int kConvTH = 8;   // conv M tile = 8 x 16 output pixels
constexpr int kConvTW = 16;

enum GemmAct { ACT_NONE = 0, ACT_GELU = 1, ACT_QUICKGELU = 2, ACT_RELU = 3 };
enum GemmStore { STORE_ROWMAJOR = 0, STORE_D2S = 1, STORE_NCHW_T = 2 };
enum GemmEpiMode { EPI_DIRECT = 0, EPI_TMA_F16 = 1, EPI_TMA_ADD = 2 };

struct GemmEpi {
  const float* bias;       // [N] (or [groups, N] when bias_group_rows > 0); nullable
  int bias_group_rows;     // rows sharing one bias row (per-image broadcast bias, readout k10)
  const float* scale;      // [N] per-column scale applied before bias (folded BatchNorm); nullable
  int act;                 // GemmAct
  const float* res_f32;    // fp32 residual, same row-major layout as the output; nullable
  const float* res2_f32;   // second fp32 residual (fusion-block skip add); nullable
  const __half* res_f16;   // fp16 residual (CLIP text tower: fp16 residual stream); nullable
  float* out_f32;          // nullable
  __half* out_f16;         // nullable
  __half* out_f16_relu;    // nullable: relu(result) copy in fp16 (input of the next RCU conv)
  long long ldc;           // row stride in elements (row-major store + residual)
  int store;               // GemmStore
  int d2s_s, d2s_cout, d2s_h, d2s_w;  // depth-to-space: input grid h x w, upscale s, cout channels
  int nchw_p, nchw_k;      // STORE_NCHW_T: pixels per image, channel count (n < nchw_k stored)
  int nchw_group;          // STORE_NCHW_T, > 0: the N columns are per-image blocks of `nchw_group` columns; a row of image
                           // b stores only columns [b*group, b*group + nchw_k) as channels 0..nchw_k-1 (zero-shot path)
  const float* row_sumsq;  // STORE_NCHW_T only, nullable: [rows, row_sumsq_parts] partial squared norms;
  int row_sumsq_parts;     //   result *= row_scale * rsqrt(sum of the row's parts)
  float row_scale;
  float* out_row_sumsq;    // nullable: [rows, ceil(N/32)] partial sums of result^2 (fp32, pre-rounding)
  int relu_after_res;      // EPI_DIRECT, row-major: ReLU applied AFTER the fp32 residual add, to every output
                           // (torchvision Bottleneck: relu(bn3(conv3) + identity)); a compile-time kernel variant
};

struct GemmParams {
  CUtensorMap tma_a;  // plain: 2-D {K, M}; conv: 4-D {C, W, H, B}
  CUtensorMap tma_b;  // 2-D {Ktot, N}, Ktot = taps * C, tap-major
  CUtensorMap tma_c;  // output map of the TMA epilogues. EPI_TMA_F16: fp16, plain 2-D {N, M} box {64, 32} /
                      // conv 4-D {N, W, H, B} box {64, 16, 2, 1}. EPI_TMA_ADD: fp32 2-D {N, M} box {32, 32}.
                      // The map clips the M / H / W / N tails, so partial tiles need no masking.
  int M, N;
  int k_iters;   // total K chunks of 64 (taps * C/64)
  int k_chunks;  // chunks per tap (C/64); == k_iters for plain
  int conv;      // 0 plain, 1 implicit-GEMM conv
  int H, W, kw, pad;
  int tiles_h, tiles_w;
  int num_m_tiles, num_n_tiles;
  int split_k;   // EPI_TMA_ADD only: balance (tile, k-chunk) units over the CTAs instead of whole tiles
  int split_fixed;       // EPI_DIRECT, >= 2: every tile's K loop is cut into this many equal segments, each a work unit of
  long long split_rows;  //   its own; segment s stores its RAW fp32 partial at row (s * split_rows + row) of out_f32 and
                         //   splitk_reduce_kernel sums the segments in index order (deterministic) and applies the epilogue
  unsigned long long* trace;  // debug timeline ([2 CTAs][20 warps][512] of clock64 << 8 | tag), normally nullptr
  int probe;  // measurement only (results are garbage when non-zero):
              //   1 = skip epilogue work, 2 = skip TMA loads, 4 = skip MMA issue
  GemmEpi e;
};

// Debug timeline of one warp (lseg_debug_gemm_trace): stamps are dropped when w == nullptr (always, unless enabled).
// The stamp itself is an out-of-line call so that the untraced kernel pays one predicated branch per site, not a
// predicated copy of the stamp code.
__device__ __noinline__ int gemm_trace_stamp(unsigned long long* w, int n, int tag) {
  if (n < 510) w[n++] = (static_cast<unsigned long long>(clock64()) << 8) | static_cast<unsigned>(tag);
  return n;
}
struct GemmTrace {
  unsigned long long* w = nullptr;
  int n = 0;
  __device__ __forceinline__ void operator()(int tag) {
    if (w) n = gemm_trace_stamp(w, n, tag);
  }
};

// ------------------------------------------------------------------------------------------
// Epilogue math of one 32-column chunk of one output row: f = act(v * scale + bias), plus the optional
// partial squared row norm. v = the row's fp32 accumulators for columns [n0, n0+32).
// ------------------------------------------------------------------------------------------
// Per-column constants of the (up to) 128 columns a warp handles in one tile, held in registers: lane l keeps
// columns 4l..4l+3 (zeros beyond N), fetched with ONE coalesced 16-byte load per lane before the accumulator is
// even awaited; chunk c then takes them by shuffle instead of issuing dependent global loads per 32-column chunk.
struct GemmColConst {
  float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 scale = make_float4(0.f, 0.f, 0.f, 0.f);
  bool on = false;  // warp-uniform: false -> per-chunk global loads (row-dependent bias)
};
__device__ __forceinline__ GemmColConst gemm_col_const(const GemmEpi& e, int N, int n_base, int ncols, int lane) {
  GemmColConst cc;
  cc.on = (e.bias_group_rows == 0) && ((N & 3) == 0);
  if (cc.on) {
    const int col = n_base + 4 * lane;
    const bool in = (4 * lane < ncols) && (col < N);
    if (e.bias && in) cc.bias = __ldg(reinterpret_cast<const float4*>(e.bias + col));
    if (e.scale && in) cc.scale = __ldg(reinterpret_cast<const float4*>(e.scale + col));
  }
  return cc;
}

__device__ __forceinline__ void gemm_epilogue_math(const GemmEpi& e, int N, const uint32_t (&v)[32], long long grow,
                                                   int n0, long long bias_off, bool row_valid, float (&f)[32],
                                                   const GemmColConst& cc, int chunk, bool use_bias = true) {
  const int nvalid = min(32, N - n0);
#pragma unroll
  for (int i = 0; i < 32; ++i) f[i] = __uint_as_float(v[i]);
  if (cc.on) {
    if (e.scale) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int src = chunk * 8 + j;
        f[4 * j] *= __shfl_sync(0xffffffffu, cc.scale.x, src);
        f[4 * j + 1] *= __shfl_sync(0xffffffffu, cc.scale.y, src);
        f[4 * j + 2] *= __shfl_sync(0xffffffffu, cc.scale.z, src);
        f[4 * j + 3] *= __shfl_sync(0xffffffffu, cc.scale.w, src);
      }
    }
    if (e.bias && use_bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int src = chunk * 8 + j;
        f[4 * j] += __shfl_sync(0xffffffffu, cc.bias.x, src);
        f[4 * j + 1] += __shfl_sync(0xffffffffu, cc.bias.y, src);
        f[4 * j + 2] += __shfl_sync(0xffffffffu, cc.bias.z, src);
        f[4 * j + 3] += __shfl_sync(0xffffffffu, cc.bias.w, src);
      }
    }
  } else if (nvalid == 32) {  // uniform-address 16 B loads: one broadcast transaction each
    if (e.scale) {
      const float4* sp = reinterpret_cast<const float4*>(e.scale + n0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 s = __ldg(sp + j);
        f[4 * j] *= s.x; f[4 * j + 1] *= s.y; f[4 * j + 2] *= s.z; f[4 * j + 3] *= s.w;
      }
    }
    if (e.bias) {
      const float4* bp = reinterpret_cast<const float4*>(e.bias + bias_off + n0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 b = __ldg(bp + j);
        f[4 * j] += b.x; f[4 * j + 1] += b.y; f[4 * j + 2] += b.z; f[4 * j + 3] += b.w;
      }
    }
  } else {
    if (e.scale) {
#pragma unroll
      for (int i = 0; i < 32; ++i) f[i] *= (i < nvalid) ? __ldg(e.scale + n0 + i) : 0.f;
    }
    if (e.bias) {
      const float* bp = e.bias + bias_off + n0;
#pragma unroll
      for (int i = 0; i < 32; ++i) f[i] += (i < nvalid) ? __ldg(bp + i) : 0.f;
    }
  }
  if (e.act == ACT_GELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) f[i] = gelu_erf(f[i]);
  } else if (e.act == ACT_QUICKGELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) f[i] = quick_gelu(f[i]);
  } else if (e.act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < 32; ++i) f[i] = fmaxf(f[i], 0.f);
  }
  if (e.out_row_sumsq && row_valid) {  // per-(row, 32-column chunk) partial, summed in fixed order by the
    float ss = 0.f;                    // consumer: deterministic (no atomics), batch-8 == batch-1 bit for bit
#pragma unroll
    for (int i = 0; i < 32; ++i) ss = fmaf((i < nvalid) ? f[i] : 0.f, f[i], ss);
    e.out_row_sumsq[grow * ((N + 31) >> 5) + (n0 >> 5)] = ss;
  }
}

// EPI_DIRECT store part, straight from registers (thread <-> row). GROUPED: STORE_NCHW_T with per-image column blocks
// (zero-shot path) — a compile-time variant: as a runtime case it costs the common kernel 4 registers and 128
// instructions (the one-label-set instantiation is instruction-for-instruction the round-1 kernel again).
// RELU_RES: GemmEpi::relu_after_res (ResNet bottleneck output), row-major full chunks and tails alike.
template <bool GROUPED = false, bool RELU_RES = false>
__device__ __forceinline__ void gemm_epilogue_store(const GemmEpi& e, int N, float (&f)[32], const float4 (&res)[8],
                                                    bool has_res, long long grow, int n0) {
  const int nvalid = min(32, N - n0);
  if (e.store == STORE_ROWMAJOR) {
    const long long off = grow * e.ldc + n0;
    if (nvalid == 32) {
      if (e.res_f32) {
        if (has_res) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            f[4 * i + 0] += res[i].x; f[4 * i + 1] += res[i].y; f[4 * i + 2] += res[i].z; f[4 * i + 3] += res[i].w;
          }
        } else {
          const float4* rp = reinterpret_cast<const float4*>(e.res_f32 + off);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 q = rp[i];
            f[4 * i + 0] += q.x; f[4 * i + 1] += q.y; f[4 * i + 2] += q.z; f[4 * i + 3] += q.w;
          }
        }
      }
      if (e.res2_f32) {
        const float4* rp = reinterpret_cast<const float4*>(e.res2_f32 + off);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 q = rp[i];
          f[4 * i + 0] += q.x; f[4 * i + 1] += q.y; f[4 * i + 2] += q.z; f[4 * i + 3] += q.w;
        }
      }
      if constexpr (RELU_RES) {
#pragma unroll
        for (int i = 0; i < 32; ++i) f[i] = fmaxf(f[i], 0.f);
      }
      if (e.out_f32) {
        float4* op = reinterpret_cast<float4*>(e.out_f32 + off);
#pragma unroll
        for (int i = 0; i < 8; ++i) op[i] = make_float4(f[4 * i], f[4 * i + 1], f[4 * i + 2], f[4 * i + 3]);
      }
      if (e.out_f16) {
        __half2 h[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        if (e.res_f16) {  // fp16 residual stream: round the branch output first, then add in fp16
          const uint4* rp = reinterpret_cast<const uint4*>(e.res_f16 + off);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint4 q = rp[i];
            const __half2* qh = reinterpret_cast<const __half2*>(&q);
#pragma unroll
            for (int j = 0; j < 4; ++j) h[4 * i + j] = __hadd2(qh[j], h[4 * i + j]);
          }
        }
        uint4* op = reinterpret_cast<uint4*>(e.out_f16 + off);
#pragma unroll
        for (int i = 0; i < 4; ++i) op[i] = *reinterpret_cast<uint4*>(&h[4 * i]);
      }
      if (e.out_f16_relu) {
        __half2 h[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) h[i] = __floats2half2_rn(fmaxf(f[2 * i], 0.f), fmaxf(f[2 * i + 1], 0.f));
        uint4* op = reinterpret_cast<uint4*>(e.out_f16_relu + off);
#pragma unroll
        for (int i = 0; i < 4; ++i) op[i] = *reinterpret_cast<uint4*>(&h[4 * i]);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        if (i < nvalid) {
          float x = f[i];
          if (e.res_f32) x += e.res_f32[off + i];
          if (e.res2_f32) x += e.res2_f32[off + i];
          if constexpr (RELU_RES) x = fmaxf(x, 0.f);
          if (e.out_f32) e.out_f32[off + i] = x;
          if (e.out_f16) {
            __half hx = __float2half_rn(x);
            if (e.res_f16) hx = __hadd(e.res_f16[off + i], hx);
            e.out_f16[off + i] = hx;
          }
          if (e.out_f16_relu) e.out_f16_relu[off + i] = __float2half_rn(fmaxf(x, 0.f));
        }
      }
    }
  } else if (e.store == STORE_D2S) {
    // column n = (i*s + j)*cout + co ; row grow = (b*h + y)*w + x  ->  NHWC [B, h*s, w*s, cout]
    const int ij = n0 / e.d2s_cout;
    const int co0 = n0 - ij * e.d2s_cout;
    const int di = ij / e.d2s_s, dj = ij - di * e.d2s_s;
    const int hw = e.d2s_h * e.d2s_w;
    const int b = static_cast<int>(grow / hw);
    const int yx = static_cast<int>(grow - static_cast<long long>(b) * hw);
    const int y = yx / e.d2s_w, x = yx - y * e.d2s_w;
    const long long orow =
        (static_cast<long long>(b) * (e.d2s_h * e.d2s_s) + (y * e.d2s_s + di)) * (e.d2s_w * e.d2s_s) +
        (x * e.d2s_s + dj);
    __half2 h[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    uint4* op = reinterpret_cast<uint4*>(e.out_f16 + orow * e.d2s_cout + co0);
#pragma unroll
    for (int i = 0; i < 4; ++i) op[i] = *reinterpret_cast<uint4*>(&h[4 * i]);
  } else {  // STORE_NCHW_T : out[(b*K + n)*P + p], fp16 (lanes = consecutive pixels -> coalesced)
    const int b = static_cast<int>(grow / e.nchw_p);
    const int pix = static_cast<int>(grow - static_cast<long long>(b) * e.nchw_p);
    if constexpr (!GROUPED) {  // one label set for all images: the chunk's columns are channels n0 .. n0+31
      __half* op = e.out_f16 + (static_cast<long long>(b) * e.nchw_k + n0) * e.nchw_p + pix;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (n0 + i < e.nchw_k) op[static_cast<long long>(i) * e.nchw_p] = __float2half_rn(f[i]);
    } else {
      // per-image column blocks: a row of image b keeps columns [b*group, b*group + nchw_k) as channels 0 .. nchw_k-1:
      // "store element i of the chunk iff lo <= i < hi" on a pointer shifted by the block start
      const int c_lo = b * e.nchw_group;
      const int lo = max(0, c_lo - n0);
      const int hi = min(min(32, c_lo + e.nchw_k - n0), N - n0);
      __half* op = e.out_f16 + (static_cast<long long>(b) * e.nchw_k + (n0 - c_lo)) * e.nchw_p + pix;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (i >= lo && i < hi) op[static_cast<long long>(i) * e.nchw_p] = __float2half_rn(f[i]);
    }
  }
}

// tile-local row -> global row (pixel) index + validity
__device__ __forceinline__ bool gemm_row_map(const GemmParams& p, int m_tile, int r, long long& grow) {
  if (p.conv) {
    const int per_img = p.tiles_h * p.tiles_w;
    const int b = m_tile / per_img;
    const int t = m_tile % per_img;
    const int h = (t / p.tiles_w) * kConvTH + r / kConvTW;
    const int w = (t % p.tiles_w) * kConvTW + r % kConvTW;
    grow = (static_cast<long long>(b) * p.H + h) * p.W + w;
    return (m_tile < p.num_m_tiles) && (h < p.H) && (w < p.W);
  }
  grow = static_cast<long long>(m_tile) * kGemmBM + r;
  return (m_tile < p.num_m_tiles) && (grow < p.M);
}

constexpr int kEpiStageBytes = 2 * 4096;  // per epilogue warp: two 32-row x 128 B swizzled tiles (TMA epilogues)

// 32 consecutive fp32 accumulators of one row of the staged tile (16-byte aligned)
__device__ __forceinline__ void gemm_acc_ld32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 q = reinterpret_cast<const float4*>(src)[i];
    v[4 * i] = __float_as_uint(q.x);
    v[4 * i + 1] = __float_as_uint(q.y);
    v[4 * i + 2] = __float_as_uint(q.z);
    v[4 * i + 3] = __float_as_uint(q.w);
  }
}

// Epilogue of one 128 x (ncols) accumulator slab for one warp (r = quarter*32 + lane = this thread's row); acc_row is
// this thread's row of the fp32 accumulator tile staged in shared memory, at the warp's first column.
// SINGLE_BUF: one 4 KB staging tile per warp instead of two (leaves the shared memory to the accumulator tile and the
// operand ring; the warp then waits for its previous bulk store to finish reading before it refills the buffer).
template <int EPI, bool SINGLE_BUF = false, bool GROUPED = false, bool RELU_RES = false, typename WaitFn>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmParams& p, const float* acc_row, int n_base, int ncols,
                                                   int m_tile, int r, WaitFn wait_accumulator, uint8_t* stage_buf,
                                                   int& store_groups, GemmTrace& tr, bool first_k = true,
                                                   int split_seg = 0) {
  const GemmEpi& e = p.e;
  long long grow;
  const bool valid = gemm_row_map(p, m_tile, r, grow);
  // split_fixed: this segment's plane of the partial-sum workspace (split_rows is 0 otherwise)
  if constexpr (EPI == EPI_DIRECT) grow += split_seg * p.split_rows;
  if constexpr (EPI == EPI_DIRECT) {
    // The fp32 residual of chunk c+1 is requested before chunk c is processed, and that of chunk 0 before the
    // accumulator is even ready, so the residual read latency overlaps the main loop / the previous chunk.
    const bool pre = valid && e.res_f32 && (e.store == STORE_ROWMAJOR);
    const long long bias_off =
        (e.bias_group_rows > 0 && valid) ? (grow / e.bias_group_rows) * static_cast<long long>(p.N) : 0;
    float4 rnext[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) rnext[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pre && n_base + 32 <= p.N) {
      const float4* rp = reinterpret_cast<const float4*>(e.res_f32 + grow * e.ldc + n_base);
#pragma unroll
      for (int j = 0; j < 8; ++j) rnext[j] = rp[j];
    }
    const GemmColConst cc = gemm_col_const(e, p.N, n_base, ncols, r & 31);
    float row_mul = 1.f;
    if (e.row_sumsq && valid) {  // deferred pixel normalisation: logit_scale / ||feature row||, once per tile
      float ss = 0.f;
      const float* sp = e.row_sumsq + grow * e.row_sumsq_parts;
      for (int i = 0; i < e.row_sumsq_parts; ++i) ss += __ldg(sp + i);
      row_mul = e.row_scale * rsqrtf(ss);
    }
    wait_accumulator();
    if (p.probe & 1) return;
#pragma unroll 1
    for (int c = 0; c < ncols / 32; ++c) {
      const int n0 = n_base + c * 32;
      if (n0 >= p.N) break;  // warp-uniform
      float4 rcur[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) rcur[j] = rnext[j];
      const bool has_res = pre && (n0 + 32 <= p.N);
      if (pre && (c + 1) * 32 < ncols && n0 + 64 <= p.N) {
        const float4* rp = reinterpret_cast<const float4*>(e.res_f32 + grow * e.ldc + n0 + 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) rnext[j] = rp[j];
      }
      uint32_t v[32];
      __syncwarp();
      gemm_acc_ld32(acc_row + c * 32, v);
      float f[32];
      gemm_epilogue_math(e, p.N, v, grow, n0, bias_off, valid, f, cc, c);  // all lanes: it shuffles
      if (valid) {
        if (e.row_sumsq) {
#pragma unroll
          for (int i = 0; i < 32; ++i) f[i] *= row_mul;
        }
        gemm_epilogue_store<GROUPED, RELU_RES>(e, p.N, f, rcur, has_res, grow, n0);
      }
    }
  } else {
    // ---------------- TMA epilogues: results leave through a per-warp swizzled smem tile ----------------
    const int lane = r & 31, quarter = r >> 5;
    const long long grow_c = valid ? grow : 0;  // keep per-row lookups in range; the tensor map clips the rest
    const long long bias_off = (e.bias_group_rows > 0) ? (grow_c / e.bias_group_rows) * static_cast<long long>(p.N) : 0;
    int crd_w = 0, crd_h = 0, crd_b = 0;
    if (p.conv) {
      const int per_img = p.tiles_h * p.tiles_w;
      crd_b = m_tile / per_img;
      const int t = m_tile % per_img;
      crd_h = (t / p.tiles_w) * kConvTH + quarter * 2;
      crd_w = (t % p.tiles_w) * kConvTW;
    }
    const GemmColConst cc = gemm_col_const(e, p.N, n_base, ncols, lane);
    const bool leader = elect_one_sync();  // issues (and owns the bulk groups of) this warp's TMA stores
    wait_accumulator();
    tr(1);
    if (p.probe & 1) return;
    int groups = store_groups;
#pragma unroll 1
    for (int c = 0; c < ncols / 32; ++c) {
      const int n0 = n_base + c * 32;
      if (n0 >= p.N) break;  // warp-uniform
      uint32_t v[32];
      __syncwarp();
      gemm_acc_ld32(acc_row + c * 32, v);
      tr(2);
      float f[32];
      gemm_epilogue_math(e, p.N, v, grow_c, n0, bias_off, valid, f, cc, c, first_k);
      tr(3);
      uint8_t* buf = SINGLE_BUF ? stage_buf : stage_buf + (groups & 1) * 4096;
      const bool first_of_group = (EPI == EPI_TMA_ADD) || ((c & 1) == 0);
      if (first_of_group && groups >= (SINGLE_BUF ? 1 : 2)) {  // the bulk op that last used this buffer must be done READING it
        if (leader) {
          if (SINGLE_BUF)
            tma_store_wait_read<0>();
          else
            tma_store_wait_read<1>();
        }
        __syncwarp();
      }
      tr(4);
      if constexpr (EPI == EPI_TMA_F16) {
        // 32 rows x 64 fp16 columns per group: this chunk fills 16-byte slots (c&1)*4 .. +3 of the row
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          __half2 h[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[8 * t + 2 * i], f[8 * t + 2 * i + 1]);
          const int slot = ((c & 1) * 4 + t) ^ (lane & 7);
          *reinterpret_cast<uint4*>(buf + lane * 128 + slot * 16) = *reinterpret_cast<uint4*>(h);
        }
      } else {
        // 32 rows x 32 fp32 columns per group
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int slot = t ^ (lane & 7);
          *reinterpret_cast<float4*>(buf + lane * 128 + slot * 16) =
              make_float4(f[4 * t], f[4 * t + 1], f[4 * t + 2], f[4 * t + 3]);
        }
      }
      tr(5);
      const bool last_of_group =
          (EPI == EPI_TMA_ADD) || ((c & 1) == 1) || (c + 1 == ncols / 32) || (n0 + 32 >= p.N);
      if (last_of_group) {
        fence_proxy_async_smem();
        __syncwarp();
        const int col0 = n_base + (c & ~1) * 32;
        const int row0 = m_tile * kGemmBM + quarter * 32;
        if (leader) {
          if constexpr (EPI == EPI_TMA_F16) {
            if (p.conv)
              tma_store_4d(&p.tma_c, buf, col0, crd_w, crd_h, crd_b);
            else
              tma_store_2d(&p.tma_c, buf, col0, row0);
          } else {
            tma_reduce_add_2d(&p.tma_c, buf, n0, row0);
          }
          tma_store_commit();
        }
        ++groups;
        tr(6);
      }
    }
    store_groups = groups;
  }
}

// ==========================================================================================
// The kernel: persistent CTAs over 128 x 128 output tiles (warp roles in the header comment).
//   full barrier  : per stage, armed by the producer with the stage's byte count; the TMA loads credit it
//   empty barrier : per stage, one arrival per consumer warp once its warpgroup's MMAs have read the stage
// ==========================================================================================
template <int EPI>
struct GemmCfg {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;  // 16 KB
  static constexpr int kBBytes = kGemmBN * kGemmBK * 2;  // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiWarps = 8;                     // the two consumer warpgroups
  static constexpr int kThreads = 128 + 32 * kEpiWarps;   // + the producer warpgroup
  static constexpr int kEpiBufBytes = 4096;               // one 32-row x 128 B TMA-store staging tile per warp
  static constexpr int kStageOutBytes = (EPI == EPI_DIRECT) ? 0 : kEpiWarps * kEpiBufBytes;
  static constexpr int kAccStride = kGemmBN + 4;          // fp32 row stride of the staged accumulators (bank spread)
  static constexpr int kAccBytes = kGemmBM * kAccStride * 4;
  // operand ring | per-warp TMA-store staging (1024 B aligned) | accumulator tile | mbarriers: <= 227 KB
  static constexpr int kStages = (EPI == EPI_DIRECT) ? 4 : 3;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStageOutBytes + kAccBytes + 1024 + 256;
};

__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// FIXED_SPLIT: the deterministic split-K schedule (GemmParams::split_fixed) is its own instantiation, so its index
// arithmetic stays out of the other kernels.
template <int EPI, bool FIXED_SPLIT = false, bool GROUPED = false, bool RELU_RES = false>
__global__ void __launch_bounds__(GemmCfg<EPI>::kThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  static_assert(!RELU_RES || (EPI == EPI_DIRECT && !FIXED_SPLIT && !GROUPED), "relu-after-residual: plain register-direct");
  static_assert(!FIXED_SPLIT || EPI == EPI_DIRECT, "split-K partials leave through the register-direct epilogue");
  static_assert(!GROUPED || (EPI == EPI_DIRECT && !FIXED_SPLIT), "per-image column blocks: NCHW-T store, register-direct");
  using Cfg = GemmCfg<EPI>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_out = smem + Cfg::kStages * Cfg::kStageBytes;
  float* acc_tile = reinterpret_cast<float*>(stage_out + Cfg::kStageOutBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_tile) + Cfg::kAccBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;

  const int warp = warp_idx_sync();  // provably warp-uniform: role branches and their operands stay on the uniform datapath
  const int lane = threadIdx.x & 31;
  const int cta = blockIdx.x;
  const int num_ctas = gridDim.x;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tma_a);
    tma_prefetch_desc(&p.tma_b);
    if (EPI != EPI_DIRECT) tma_prefetch_desc(&p.tma_c);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], Cfg::kEpiWarps);
    }
    mbar_fence_init();
  }
  griddep_launch_dependents();
  __syncthreads();
  griddep_wait();  // everything above overlapped the previous kernel's tail; operands / outputs are touched below

  const int num_tiles = p.num_m_tiles * p.num_n_tiles;

  // Work schedule of this CTA. Default: whole tiles cta, cta + G, ... . split_k (in-place residual GEMMs only, whose
  // epilogue is a reduce-add and therefore composes over partial sums): the (tile, k-chunk) units are dealt out evenly,
  // so a CTA handles a contiguous range that may start / end inside a tile. The bias is added by the k = 0 segment.
  struct Sched {
    int tile_next, tile_step, num_tiles, k_iters;
    long long unit, unit_end;
    bool split;
    int fixed, seg;
    __device__ bool next(int& tile, int& k0, int& k1) {
      if constexpr (FIXED_SPLIT) {  // units = (tile, segment), dealt round-robin; 32-bit arithmetic (seg < 16)
        if (tile_next >= num_tiles * fixed) return false;
        tile = tile_next / fixed;
        seg = tile_next - tile * fixed;
        tile_next += tile_step;
        k0 = seg * k_iters / fixed;
        k1 = (seg + 1) * k_iters / fixed;
        return true;
      }
      if (!split) {
        if (tile_next >= num_tiles) return false;
        tile = tile_next;
        tile_next += tile_step;
        k0 = 0;
        k1 = k_iters;
        return true;
      }
      if (unit >= unit_end) return false;
      tile = static_cast<int>(unit / k_iters);
      k0 = static_cast<int>(unit - static_cast<long long>(tile) * k_iters);
      const long long left = unit_end - unit;
      k1 = (k_iters - k0 < left) ? k_iters : k0 + static_cast<int>(left);
      unit += k1 - k0;
      return true;
    }
  };
  auto make_sched = [&]() {
    Sched sc;
    sc.tile_next = cta;
    sc.tile_step = num_ctas;
    sc.num_tiles = num_tiles;
    sc.k_iters = p.k_iters;
    sc.split = (EPI == EPI_TMA_ADD) && p.split_k;
    sc.fixed = FIXED_SPLIT ? p.split_fixed : 0;
    sc.seg = 0;
    const long long units = static_cast<long long>(num_tiles) * p.k_iters;
    // boundaries on multiples of 4 k-chunks: no sliver segments whose epilogue would cost more than their MMAs
    sc.unit = ((units * cta / num_ctas) + 3) & ~3ll;
    sc.unit_end = (cta + 1 == num_ctas) ? units : (((units * (cta + 1) / num_ctas) + 3) & ~3ll);
    if (sc.unit_end > units) sc.unit_end = units;
    return sc;
  };

  if (warp == 0) {
    // ===================== TMA producer (converged warp, elected issuing lane) =====================
    const bool leader = elect_one_sync();
    int stage = 0;
    uint32_t phase = 0;
    Sched sc = make_sched();
    int tile, k_begin, k_end;
    while (sc.next(tile, k_begin, k_end)) {
      const int m_tile = tile % p.num_m_tiles;
      const int n0 = (tile / p.num_m_tiles) * kGemmBN;
      int cb = 0, ch0 = 0, cw0 = 0;
      if (p.conv) {
        const int per_img = p.tiles_h * p.tiles_w;
        cb = m_tile / per_img;
        const int t = m_tile % per_img;
        ch0 = (t / p.tiles_w) * kConvTH;
        cw0 = (t % p.tiles_w) * kConvTW;
      }
      for (int kit = k_begin; kit < k_end; ++kit) {
        mbar_wait(&empty_bar[stage], phase ^ 1, 21);
        uint8_t* sa = smem + stage * Cfg::kStageBytes;
        uint8_t* sb = sa + Cfg::kABytes;
        if (p.probe & 2) {
          if (leader) mbar_arrive(&full_bar[stage]);
          __syncwarp();
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
          continue;
        }
        int c0 = kit * kGemmBK, c1 = m_tile * kGemmBM, c2 = 0;
        if (p.conv) {
          const int tap = kit / p.k_chunks;
          const int c = kit - tap * p.k_chunks;
          const int dy = tap / p.kw, dx = tap - dy * p.kw;
          c0 = c * kGemmBK;
          c1 = cw0 + dx - p.pad;
          c2 = ch0 + dy - p.pad;
        }
        if (leader) {
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (p.conv)
            tma_load_4d(sa, &p.tma_a, &full_bar[stage], c0, c1, c2, cb);
          else
            tma_load_2d(sa, &p.tma_a, &full_bar[stage], c0, c1);
          tma_load_2d(sb, &p.tma_b, &full_bar[stage], kit * kGemmBK, n0);
        }
        __syncwarp();
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: MMA main loop, then the epilogue =====================
    const int wg = (warp - 4) >> 2;  // rows [64 wg, 64 wg + 64) of the tile in the main loop
    const int wl = warp & 3;         // warp within its warpgroup: accumulator rows 16 wl .. 16 wl + 15
    const int ew = warp - 4;
    const int quarter = ew & 3;      // epilogue: rows [32 quarter, +32), columns [64 half, +64)
    const int half = ew >> 2;
    const int r = quarter * 32 + lane;
    const int col0 = half * 64;
    const float* acc_row = acc_tile + r * Cfg::kAccStride + col0;
    uint8_t* stage_buf = stage_out + ew * Cfg::kEpiBufBytes;
    int store_groups = 0;
    int stage = 0;
    uint32_t phase = 0;
    GemmTrace tr;
    if (p.trace && lane == 0 && (cta == 0 || cta == num_ctas / 2)) tr.w = p.trace + ((cta == 0 ? 0 : 1) * 20 + warp) * 512;
    tr(0);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    Sched sc = make_sched();
    int tile, k_begin, k_end;
    while (sc.next(tile, k_begin, k_end)) {
      const int m_tile = tile % p.num_m_tiles;
      const int n_tile = tile / p.num_m_tiles;
      int prev = -1;
      for (int kit = k_begin; kit < k_end; ++kit) {
        mbar_wait(&full_bar[stage], phase, 23);
        __syncwarp();
        const uint32_t a_base = smem_u32(smem + stage * Cfg::kStageBytes) + wg * (64 * 128);
        const uint32_t b_base = smem_u32(smem + stage * Cfg::kStageBytes + Cfg::kABytes);
        if (!(p.probe & 4)) {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kGemmBK / 16; ++k)
            wgmma_m64n128k16_ss(acc, wgmma_desc_sw128(a_base + k * 32, 1024, 16),
                                wgmma_desc_sw128(b_base + k * 32, 1024, 16), (kit != k_begin) || (k != 0));
          wgmma_commit();
        }
        wgmma_wait<1>();  // the previous chunk's MMAs have read their stage: hand it back to the producer
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      tr(12);
      // stage the accumulators (fragment rows 64 wg + 16 wl + lane/4 (+8), columns 8 j + 2 (lane % 4) (+1)) once the
      // previous tile's epilogue has read the tile
      consumer_bar_sync();
      {
        float* d0 = acc_tile + (wg * 64 + wl * 16 + (lane >> 2)) * Cfg::kAccStride + 2 * (lane & 3);
        float* d1 = d0 + 8 * Cfg::kAccStride;
#pragma unroll
        for (int j = 0; j < kGemmBN / 8; ++j) {
          *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(d1 + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      // the next tile's first MMA ignores the accumulator (scale-d = 0): dead values, not 64 registers held across the
      // epilogue
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      consumer_bar_sync();
      gemm_epilogue_tile<EPI, true, GROUPED, RELU_RES>(p, acc_row, n_tile * kGemmBN + col0, 64, m_tile, r, []() {},
                                                       stage_buf, store_groups, tr, k_begin == 0,
                                                       FIXED_SPLIT ? sc.seg : 0);
      tr(7);
    }
    if (EPI != EPI_DIRECT && elect_one_sync()) tma_store_wait_all();  // outstanding bulk ops read this CTA's smem
  }
}

// ------------------------------------------------------------------------------------------
// Deterministic split-K, second half: out = epilogue(sum_s partial[s]) for the GEMMs whose tile count leaves most of
// the CTAs idle (3x3 convs on the 15x15 decoder level, K up to 9216).
// ws fp32 [S][M][N] (N == ldc of the partials); one thread = 4 consecutive columns of one row, segments summed in index
// order. Epilogue = the row-major subset of gemm_epilogue_math / gemm_epilogue_store: scale, bias (per column), act, two
// fp32 residuals, fp32 / fp16 / relu-fp16 outputs with the FINAL row stride e.ldc.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, int S, long long M, int N,
                                                            GemmEpi e) {
  griddep_launch_dependents();
  griddep_wait();
  const int n4 = N >> 2;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= M * n4) return;
  const long long row = i / n4;
  const int col = static_cast<int>(i - row * n4) * 4;
  const long long plane = M * static_cast<long long>(N);
  const float* src = ws + row * N + col;
  float4 a = *reinterpret_cast<const float4*>(src);
  for (int s = 1; s < S; ++s) {
    const float4 q = *reinterpret_cast<const float4*>(src + s * plane);
    a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
  }
  if (e.scale) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(e.scale + col));
    a.x *= q.x; a.y *= q.y; a.z *= q.z; a.w *= q.w;
  }
  if (e.bias) {
    const float4 q = __ldg(reinterpret_cast<const float4*>(e.bias + col));
    a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
  }
  if (e.act == ACT_GELU) {
    a.x = gelu_erf(a.x); a.y = gelu_erf(a.y); a.z = gelu_erf(a.z); a.w = gelu_erf(a.w);
  } else if (e.act == ACT_QUICKGELU) {
    a.x = quick_gelu(a.x); a.y = quick_gelu(a.y); a.z = quick_gelu(a.z); a.w = quick_gelu(a.w);
  } else if (e.act == ACT_RELU) {
    a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
  }
  const long long off = row * e.ldc + col;
  if (e.res_f32) {
    const float4 q = *reinterpret_cast<const float4*>(e.res_f32 + off);
    a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
  }
  if (e.res2_f32) {
    const float4 q = *reinterpret_cast<const float4*>(e.res2_f32 + off);
    a.x += q.x; a.y += q.y; a.z += q.z; a.w += q.w;
  }
  if (e.relu_after_res) {
    a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
  }
  if (e.out_f32) *reinterpret_cast<float4*>(e.out_f32 + off) = a;
  if (e.out_f16) {
    __half2 h[2] = {__floats2half2_rn(a.x, a.y), __floats2half2_rn(a.z, a.w)};
    *reinterpret_cast<uint2*>(e.out_f16 + off) = *reinterpret_cast<uint2*>(h);
  }
  if (e.out_f16_relu) {
    __half2 h[2] = {__floats2half2_rn(fmaxf(a.x, 0.f), fmaxf(a.y, 0.f)), __floats2half2_rn(fmaxf(a.z, 0.f), fmaxf(a.w, 0.f))};
    *reinterpret_cast<uint2*>(e.out_f16_relu + off) = *reinterpret_cast<uint2*>(h);
  }
}

// ------------------------------------------------------------------------------------------
// Host-side description of one GEMM
// ------------------------------------------------------------------------------------------
struct GemmDesc {
  // A operand
  const __half* a;      // plain: [a_rows >= M, lda] ; conv: NHWC [B, H, W, C]
  long long lda;        // plain only (elements)
  int a_rows;           // plain only: allocated rows (tensor-map extent)
  // B operand (weights) [N, Ktot] row-major fp16, rows padded to a multiple of 128
  const __half* w;
  int w_rows;           // allocated rows of w (>= N)
  int M, N, K;          // plain: K ; conv: K = C (per tap)
  int conv, B, H, W, kh, kw, pad;
  GemmEpi e;
};

}  // namespace lseg
