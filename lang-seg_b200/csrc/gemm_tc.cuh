// lseg_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   C[M,N] = epilogue( A[M,K] * W[N,K]^T )       fp16 operands, fp32 accumulate in registers
//
// One kernel family covers every dense contraction of the LSeg forward path (SURVEY.md §2b k1,k4,k6-k8,
// k10-k17,k19): linear layers, 1x1 convs, kernel==stride transposed convs (depth-to-space store),
// and 3x3 stride-1 convs as implicit GEMM (the A tile of tap (dy,dx) is a shifted 4-D TMA box of
// the NHWC activation; TMA zero-fills the padding halo).
//
// Roles (one CTA per SM, persistent over a static round-robin list of 128 x 128 tiles), "ping-pong" schedule:
//   warpgroup 0   TMA producer (warp 0, one elected lane; 24 registers): fills the A/B smem ring (128B-swizzled,
//                 K-major) in list order
//   warpgroups 1-2  consumers (240 registers): the list's entries alternate between them. A warpgroup computes its whole
//                 tile (two wgmma m64n128k16 per k16 step, 2 x 64 fp32 accumulators per thread), then runs its epilogue:
//                 the TMA epilogues straight from each warp's accumulator fragment (gemm_epilogue_frag); the register-
//                 direct one, and the fp16 TMA store of GEMMs with row sums, stage the tile in the warpgroup's own
//                 shared-memory area one 64-column half at a time and map thread <-> output row (warp = 32 rows x 64
//                 columns per half): scale/bias/act/residual -> global.
// The MMA turn passes from one warpgroup to the other in list order (named barriers), so one warpgroup's epilogue
// runs while the other's MMAs keep the tensor cores busy; the tensor pipe idles only where an epilogue takes longer
// than a main loop, or where a CTA owns a single tile. The accumulation order of every output element (the same
// k16 chunks through the same m64n128k16 instruction) does not depend on which warpgroup computes the tile.
// Grids with more work units than SMs and an even n-tile count run as 2-CTA clusters that share the A tile (CLUSTER,
// see the kernel); lseg_b200.cu (gemm_plan_grid) has the rule and the numbers behind it.
// Measured (B=8, 480x480, H100 80GB HBM3 SXM at a 700 W power limit, tools/gemm_shapes.py, as planned): ViT linears
// 530-600 TFLOP/s (QKV, fc1) and 350-490 (proj, fc2); 3x3 decoder convs 320-480 at 60^2 / 120^2; head1 (staged row-sum
// form) 290-300.
//
// Epilogue modes:
//   EPI_DIRECT   stores straight from registers, thread <-> accumulator row.
//   EPI_TMA_F16  fp16 row-major outputs: each warp converts its own fragment rows (16 per m64 half) and packs 16 rows x
//                64 columns into a private 128B-swizzled smem box; one elected lane issues a bulk tensor store.
//   EPI_TMA_ADD  in-place fp32 residual stream (x += A W^T + b): the warp packs 16 x 32 fp32 results the same way and
//                issues a bulk tensor REDUCE-ADD, so the residual is never read by the SM at all.
//   The TMA epilogues need no accumulator staging area and no warpgroup barrier, so their operand ring has 6 stages
//   (register-direct: 5). Exception: EPI_TMA_F16 plans with row sums (head1's out_row_sumsq, summed per row in column
//   order) run the staged form EPI_TMA_F16_STAGED (4 stages, gemm_tma_f16_staged), where a thread holds whole rows.
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
// EPI_TMA_F16_STAGED is no plan's mode but a kernel form: the EPI_TMA_F16 plans with row sums (out_row_sumsq) run the
// fp16 TMA store through the staged accumulators (gemm_tma_f16_staged).
enum GemmEpiMode { EPI_DIRECT = 0, EPI_TMA_F16 = 1, EPI_TMA_ADD = 2, EPI_TMA_F16_STAGED = 3 };

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
  CUtensorMap tma_c;  // output map of the TMA epilogues, one box = one warp's 16 fragment rows. EPI_TMA_F16: fp16, plain
                      // 2-D {N, M} box {64, 16} / conv 4-D {N, W, H, B} box {64, 16, 1, 1}. EPI_TMA_ADD: fp32 2-D {N, M}
                      // box {32, 16}.
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
  unsigned long long* trace;  // debug timeline ([2 CTAs][20 warps][512] of clock64 << 8 | tag; rows 4-11 = consumer
                              // warps, layout in lseg_debug_gemm_trace), normally nullptr
  int probe;  // measurement only (results are garbage when non-zero):
              //   1 = skip epilogue work, 2 = skip TMA loads, 4 = skip MMA issue
  GemmEpi e;
};

// Ragged pixel x text product (gemm_tc_kernel RAGGED): B images, each with its own label set. Image b's P pixel rows
// (rows b*P .. b*P + P - 1 of A, P a multiple of 128, so no tile straddles two images) meet only text rows
// text_row[b] .. text_row[b] + k[b] - 1 of the one packed text operand (tma_b), and its k[b] columns are stored as planes
// koff[b] .. koff[b] + k[b] - 1 of a packed fp16 [sum k, h, w] output (STORE_NCHW_T, nchw_p = P). The work list is
// image-major, m-fastest within an image: image b owns tiles tile0[b] .. tile0[b+1] - 1, m_tiles(P) * ceil(k[b] / 128).
// The table travels in the kernel's __grid_constant__ parameters (no host synchronisation, no device copy), so the
// image count is capped (kRaggedMaxImages).
struct GemmRaggedTable {
  int n;         // images
  int m_tiles;   // 128-row tiles per image (P / 128)
  int tile0[kRaggedMaxImages + 1];
  int k[kRaggedMaxImages];
  int text_row[kRaggedMaxImages];
  int koff[kRaggedMaxImages];
};
struct GemmRaggedParams : GemmParams {
  GemmRaggedTable rt;
};
template <bool RAGGED> struct GemmParamsOf { using type = GemmParams; };
template <> struct GemmParamsOf<true> { using type = GemmRaggedParams; };

// Work-list entry -> (m_tile, n_tile) and the first B row of the tile. Plain lists are m-fastest over
// num_m_tiles x num_n_tiles (CLUSTER: over pair units, the CTA of rank r takes n-tile 2 j + r); ragged lists are decoded
// through the table (img = the image, whose label count / first output plane the epilogue needs).
struct GemmTileCoord {
  int m_tile, n_tile, b_row, img;
};
template <bool CLUSTER>
__device__ __forceinline__ GemmTileCoord gemm_tile_coord(const GemmParams& p, int tile, int rank) {
  GemmTileCoord c;
  c.m_tile = tile % p.num_m_tiles;
  c.n_tile = CLUSTER ? 2 * (tile / p.num_m_tiles) + rank : tile / p.num_m_tiles;
  c.b_row = c.n_tile * kGemmBN;
  c.img = 0;
  return c;
}
template <bool CLUSTER>
__device__ __forceinline__ GemmTileCoord gemm_tile_coord(const GemmRaggedParams& p, int tile, int) {
  GemmTileCoord c;
  int b = 0;
  while (b + 1 < p.rt.n && tile >= p.rt.tile0[b + 1]) ++b;
  const int local = tile - p.rt.tile0[b];
  c.m_tile = b * p.rt.m_tiles + local % p.rt.m_tiles;
  c.n_tile = local / p.rt.m_tiles;
  c.b_row = p.rt.text_row[b] + c.n_tile * kGemmBN;
  c.img = b;
  return c;
}
__device__ __forceinline__ int gemm_num_units(const GemmParams& p, bool cluster) {
  return p.num_m_tiles * (cluster ? p.num_n_tiles / 2 : p.num_n_tiles);
}
__device__ __forceinline__ int gemm_num_units(const GemmRaggedParams& p, bool) { return p.rt.tile0[p.rt.n]; }
// label count / first output plane of image img (ragged epilogue); 0 for plain lists
__device__ __forceinline__ int gemm_ragged_k(const GemmParams&, int) { return 0; }
__device__ __forceinline__ int gemm_ragged_k(const GemmRaggedParams& p, int img) { return p.rt.k[img]; }
__device__ __forceinline__ int gemm_ragged_koff(const GemmParams&, int) { return 0; }
__device__ __forceinline__ int gemm_ragged_koff(const GemmRaggedParams& p, int img) { return p.rt.koff[img]; }

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
// partial squared row norm. v = the row's fp32 accumulators for columns [n0, n0+32). use_bias = false: a stream-K
// segment that does not start at k = 0 (its partial sum is reduce-added to the one that carries the bias).
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
  } else if (nvalid == 32 && (N & 3) == 0) {  // uniform-address 16 B loads: one broadcast transaction each (a grouped
    if (e.scale) {                             // bias row starts at group * N: 16-byte aligned only when N % 4 == 0)
      const float4* sp = reinterpret_cast<const float4*>(e.scale + n0);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 s = __ldg(sp + j);
        f[4 * j] *= s.x; f[4 * j + 1] *= s.y; f[4 * j + 2] *= s.z; f[4 * j + 3] *= s.w;
      }
    }
    if (e.bias && use_bias) {
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
    if (e.bias && use_bias) {
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
// RAGGED: STORE_NCHW_T of one image of a ragged list — N is the image's label count and koff its first output plane.
template <bool GROUPED = false, bool RELU_RES = false, bool RAGGED = false>
__device__ __forceinline__ void gemm_epilogue_store(const GemmEpi& e, int N, float (&f)[32], const float4 (&res)[8],
                                                    bool has_res, long long grow, int n0, int koff = 0) {
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
    if constexpr (RAGGED) {  // the image's own label set: columns n0 .. n0+31 are planes koff + n0 .. of the packed output
      __half* op = e.out_f16 + (static_cast<long long>(koff) + n0) * e.nchw_p + pix;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (n0 + i < N) op[static_cast<long long>(i) * e.nchw_p] = __float2half_rn(f[i]);
    } else if constexpr (!GROUPED) {  // one label set for all images: the chunk's columns are channels n0 .. n0+31
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

// Staged accumulators: one warpgroup's 128 rows x 64 fp32 columns (a column half of its tile), rows of 256 B with no
// padding; the 16-byte chunk q of row r sits at chunk q ^ (r & 7), so the 8 rows a quarter-warp reads (thread <-> row)
// and the 4 rows a fragment store touches spread over the banks.
constexpr int kAccCols = kGemmBN / 2;
__device__ __forceinline__ int gemm_acc_chunk(int q, int r) { return q ^ (r & 7); }

// fp32 accumulators [32 c, 32 c + 32) of staged row r (acc_row = the row's start)
__device__ __forceinline__ void gemm_acc_ld32(const float* acc_row, int c, int r, uint32_t (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 q = reinterpret_cast<const float4*>(acc_row)[gemm_acc_chunk(8 * c + i, r)];
    v[4 * i] = __float_as_uint(q.x);
    v[4 * i + 1] = __float_as_uint(q.y);
    v[4 * i + 2] = __float_as_uint(q.z);
    v[4 * i + 3] = __float_as_uint(q.w);
  }
}

// Register-direct epilogue of one 128 x (ncols) accumulator slab for one warp (r = quarter*32 + lane = this thread's
// row); acc_row is this thread's row of the staged accumulators (gemm_acc_ld32), whose column 0 is output column n_base.
// RAGGED: the tile belongs to an image with rag_k labels whose first output plane is rag_koff (gemm_epilogue_store); its
// column count takes the place of p.N.
template <bool GROUPED = false, bool RELU_RES = false, bool RAGGED = false, typename WaitFn>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmParams& p, const float* acc_row, int n_base, int ncols,
                                                   int m_tile, int r, WaitFn wait_accumulator, int split_seg = 0,
                                                   int rag_k = 0, int rag_koff = 0) {
  const GemmEpi& e = p.e;
  long long grow;
  const bool valid = gemm_row_map(p, m_tile, r, grow);
  // split_fixed: this segment's plane of the partial-sum workspace (split_rows is 0 otherwise)
  grow += split_seg * p.split_rows;
  const int& N = RAGGED ? rag_k : p.N;  // plain lists: p.N itself (a parameter-space operand, as before)
  // The fp32 residual of chunk c+1 is requested before chunk c is processed, and that of chunk 0 before the
  // accumulator is even ready, so the residual read latency overlaps the main loop / the previous chunk.
  const bool pre = valid && e.res_f32 && (e.store == STORE_ROWMAJOR);
  const long long bias_off =
      (e.bias_group_rows > 0 && valid) ? (grow / e.bias_group_rows) * static_cast<long long>(N) : 0;
  float4 rnext[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) rnext[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (pre && n_base + 32 <= N) {
    const float4* rp = reinterpret_cast<const float4*>(e.res_f32 + grow * e.ldc + n_base);
#pragma unroll
    for (int j = 0; j < 8; ++j) rnext[j] = rp[j];
  }
  const GemmColConst cc = gemm_col_const(e, N, n_base, ncols, r & 31);
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
    if (n0 >= N) break;  // warp-uniform
    float4 rcur[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) rcur[j] = rnext[j];
    const bool has_res = pre && (n0 + 32 <= N);
    if (pre && (c + 1) * 32 < ncols && n0 + 64 <= N) {
      const float4* rp = reinterpret_cast<const float4*>(e.res_f32 + grow * e.ldc + n0 + 32);
#pragma unroll
      for (int j = 0; j < 8; ++j) rnext[j] = rp[j];
    }
    uint32_t v[32];
    __syncwarp();
    gemm_acc_ld32(acc_row, c, r, v);
    float f[32];
    gemm_epilogue_math(e, N, v, grow, n0, bias_off, valid, f, cc, c);  // all lanes: it shuffles
    if (valid) {
      if (e.row_sumsq) {
#pragma unroll
        for (int i = 0; i < 32; ++i) f[i] *= row_mul;
      }
      gemm_epilogue_store<GROUPED, RELU_RES, RAGGED>(e, N, f, rcur, has_res, grow, n0, rag_koff);
    }
  }
}

// fp16 TMA store of one 128 x (ncols) staged accumulator slab for one warp (thread <-> row r = quarter*32 + lane, as in
// gemm_epilogue_tile), for the EPI_TMA_F16 plans with row sums: gemm_epilogue_math sums each row's 32-column chunks in
// column order from the thread's own row. The warp packs 32 rows x 64 columns into its 4 KB 128B-swizzled staging tile
// (waiting until its previous bulk store has read it) and the elected lane issues the store: tensor-map box {64, 32},
// or {64, 16, 2, 1} for a conv.
__device__ __forceinline__ void gemm_tma_f16_staged(const GemmParams& p, const float* acc_row, int n_base, int ncols,
                                                    int m_tile, int r, uint8_t* stage_buf, int& store_groups,
                                                    bool leader, GemmTrace& tr) {
  const GemmEpi& e = p.e;
  long long grow;
  const bool valid = gemm_row_map(p, m_tile, r, grow);
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
  tr(1);
  if (p.probe & 1) return;
  int groups = store_groups;
#pragma unroll 1
  for (int c = 0; c < ncols / 32; ++c) {
    const int n0 = n_base + c * 32;
    if (n0 >= p.N) break;  // warp-uniform
    uint32_t v[32];
    __syncwarp();
    gemm_acc_ld32(acc_row, c, r, v);
    tr(2);
    float f[32];
    gemm_epilogue_math(e, p.N, v, grow_c, n0, bias_off, valid, f, cc, c);
    tr(3);
    if ((c & 1) == 0 && groups >= 1) {  // the previous bulk store must be done READING the staging tile
      if (leader) tma_store_wait_read<0>();
      __syncwarp();
    }
    tr(4);
    // 32 rows x 64 fp16 columns per group: this chunk fills 16-byte slots (c&1)*4 .. +3 of the row
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      __half2 h[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[8 * t + 2 * i], f[8 * t + 2 * i + 1]);
      const int slot = ((c & 1) * 4 + t) ^ (lane & 7);
      *reinterpret_cast<uint4*>(stage_buf + lane * 128 + slot * 16) = *reinterpret_cast<uint4*>(h);
    }
    tr(5);
    if ((c & 1) == 1 || c + 1 == ncols / 32 || n0 + 32 >= p.N) {
      fence_proxy_async_smem();
      __syncwarp();
      const int col0 = n_base + (c & ~1) * 32;
      if (leader) {
        if (p.conv)
          tma_store_4d(&p.tma_c, stage_buf, col0, crd_w, crd_h, crd_b);
        else
          tma_store_2d(&p.tma_c, stage_buf, col0, m_tile * kGemmBM + quarter * 32);
        tma_store_commit();
      }
      ++groups;
      tr(6);
    }
  }
  store_groups = groups;
}

// TMA epilogues, straight from one warp's wgmma fragments. acc0 / acc1 hold tile rows 64 h + 16 wl + lane / 4 (acc[4 j],
// acc[4 j + 1]) and + 8 (acc[4 j + 2], acc[4 j + 3]) of m64 half h = 0 / 1, columns 8 j + 2 (lane % 4) and + 1 (j = 0 .. 15;
// column 0 = output column n_base). Row slot s = 2 h + t is the thread's row 64 h + 16 wl + lane / 4 + 8 t.
// Each element gets gemm_epilogue_math's arithmetic in its order (scale, bias unless a stream-K segment starts past k = 0,
// activation) with the same column constants (zero beyond N), so the results are those of the register-direct path.
// The warp's 16 rows of a half leave in tensor-map boxes of 16 rows x 128 B: 64 fp16 columns (EPI_TMA_F16; a conv box is
// one pixel row of the 8 x 16 tile), or 32 fp32 columns reduce-added into the residual stream (EPI_TMA_ADD). A box is
// written into one of the warp's two 128B-swizzled staging buffers (bufs, 2 x 2 KB, 1024 B aligned), and the elected lane
// issues the bulk op; before a buffer is refilled, the bulk op that last read it must be done reading. The tensor map
// clips the M / H / W / N tails.

// scale, bias and activation of one m64 half (row slots 2 h, 2 h + 1). sv / bv: the non-grouped column constants, lane l
// holding columns 2 l, 2 l + 1 (index 0) and 64 + 2 l, + 1 (index 1) of the tile; column group j takes them from lane
// 4 (j % 8) + lane % 4 by shuffle. A per-image bias depends on the row: each row slot loads its 16 pairs at once. Multiply
// and add stay separate roundings (__fmul_rn / __fadd_rn), as in gemm_epilogue_math.
__device__ __forceinline__ void gemm_frag_math(const GemmParams& p, float (&acc)[64], int h, int m_tile, int n_base,
                                               int wl, int lane, const float2 (&sv)[2], const float2 (&bv)[2],
                                               bool use_bias) {
  const GemmEpi& e = p.e;
  const int N = p.N;
  const int q = lane & 3;
  if (e.scale) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int src = 4 * (j & 7) + q;
      const float sx = __shfl_sync(0xffffffffu, sv[j >> 3].x, src), sy = __shfl_sync(0xffffffffu, sv[j >> 3].y, src);
      acc[4 * j] = __fmul_rn(acc[4 * j], sx);
      acc[4 * j + 1] = __fmul_rn(acc[4 * j + 1], sy);
      acc[4 * j + 2] = __fmul_rn(acc[4 * j + 2], sx);
      acc[4 * j + 3] = __fmul_rn(acc[4 * j + 3], sy);
    }
  }
  if (use_bias && e.bias_group_rows == 0) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int src = 4 * (j & 7) + q;
      const float bx = __shfl_sync(0xffffffffu, bv[j >> 3].x, src), by = __shfl_sync(0xffffffffu, bv[j >> 3].y, src);
      acc[4 * j] = __fadd_rn(acc[4 * j], bx);
      acc[4 * j + 1] = __fadd_rn(acc[4 * j + 1], by);
      acc[4 * j + 2] = __fadd_rn(acc[4 * j + 2], bx);
      acc[4 * j + 3] = __fadd_rn(acc[4 * j + 3], by);
    }
  } else if (use_bias) {
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      long long grow;
      const bool valid = gemm_row_map(p, m_tile, 64 * h + 16 * wl + (lane >> 2) + 8 * t, grow);
      // keep per-row lookups in range; the tensor map clips the rest
      const long long boff = (valid ? grow / e.bias_group_rows : 0) * static_cast<long long>(N);
      float2 b[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = n_base + 8 * j + 2 * q;  // N % 8 == 0: col + 1 < N iff col < N
        const float2 v = __ldg(reinterpret_cast<const float2*>(e.bias + boff + (col < N ? col : 0)));
        b[j] = col < N ? v : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        acc[4 * j + 2 * t] = __fadd_rn(acc[4 * j + 2 * t], b[j].x);
        acc[4 * j + 2 * t + 1] = __fadd_rn(acc[4 * j + 2 * t + 1], b[j].y);
      }
    }
  }
  if (e.act == ACT_GELU) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = gelu_erf(acc[i]);
  } else if (e.act == ACT_QUICKGELU) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = quick_gelu(acc[i]);
  } else if (e.act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = fmaxf(acc[i], 0.f);
  }
}

// The stores of one m64 half h: one box per 64 fp16 / 32 fp32 columns.
template <int EPI>
__device__ __forceinline__ void gemm_frag_store(const GemmParams& p, const float (&acc)[64], int h, int m_tile,
                                                int n_base, int wl, int q, int rq, uint8_t* bufs, int& groups,
                                                bool leader, GemmTrace& tr) {
  constexpr int kBufBytes = 2048;
  constexpr int kBoxes = (EPI == EPI_TMA_F16) ? 2 : 4;
  constexpr int kBoxCols = kGemmBN / kBoxes;
  constexpr int kJ = kBoxCols / 8;  // fragment column groups per box
  const int row0 = 64 * h + 16 * wl;  // first tile row of the warp's 16
#pragma unroll
  for (int bx = 0; bx < kBoxes; ++bx) {
    const int col0 = n_base + bx * kBoxCols;
    if (col0 >= p.N) break;  // warp-uniform
    uint8_t* buf = bufs + (groups & 1) * kBufBytes;
    if (groups >= 2) {  // the bulk op that last used this buffer must be done READING it
      if (leader) tma_store_wait_read<1>();
      __syncwarp();
    }
    uint8_t* r_lo = buf + rq * 128;  // box rows rq and rq + 8 share the swizzle phase rq
    uint8_t* r_hi = r_lo + 8 * 128;
#pragma unroll
    for (int jj = 0; jj < kJ; ++jj) {
      const int j = bx * kJ + jj;
      if constexpr (EPI == EPI_TMA_F16) {  // columns 8 jj + 2 q, + 1: 16-byte chunk jj, bytes 4 q .. 4 q + 3
        const int off = ((jj ^ rq) << 4) + 4 * q;
        const __half2 lo = __floats2half2_rn(acc[4 * j], acc[4 * j + 1]);
        const __half2 hi = __floats2half2_rn(acc[4 * j + 2], acc[4 * j + 3]);
        *reinterpret_cast<__half2*>(r_lo + off) = lo;
        *reinterpret_cast<__half2*>(r_hi + off) = hi;
      } else {  // columns 8 jj + 2 q, + 1: 16-byte chunk 2 jj + q / 2, bytes 8 (q % 2) ..
        const int off = (((2 * jj + (q >> 1)) ^ rq) << 4) + 8 * (q & 1);
        *reinterpret_cast<float2*>(r_lo + off) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(r_hi + off) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (leader) {
      if constexpr (EPI == EPI_TMA_F16) {
        if (p.conv) {  // the warp's 16 rows are pixel row 4 h + wl of the 8 x 16 conv tile
          const int per_img = p.tiles_h * p.tiles_w;
          const int t = m_tile % per_img;
          tma_store_4d(&p.tma_c, buf, col0, (t % p.tiles_w) * kConvTW, (t / p.tiles_w) * kConvTH + row0 / kConvTW,
                       m_tile / per_img);
        } else {
          tma_store_2d(&p.tma_c, buf, col0, m_tile * kGemmBM + row0);
        }
      } else {
        tma_reduce_add_2d(&p.tma_c, buf, col0, m_tile * kGemmBM + row0);
      }
      tma_store_commit();
    }
    ++groups;
    tr(6);
  }
}

template <int EPI>
__device__ __forceinline__ void gemm_epilogue_frag(const GemmParams& p, float (&acc0)[64], float (&acc1)[64], int m_tile,
                                                   int n_base, int wl, int lane, uint8_t* bufs, int& groups, bool leader,
                                                   bool first_k, GemmTrace& tr) {
  const GemmEpi& e = p.e;
  const int N = p.N;
  const bool use_bias = e.bias && first_k;
  float2 sv[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)}, bv[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
#pragma unroll
  for (int k = 0; k < 2; ++k) {  // independent loads, issued together
    const int col = n_base + 64 * k + 2 * lane;
    if (e.scale && col < N) sv[k] = __ldg(reinterpret_cast<const float2*>(e.scale + col));
    if (use_bias && e.bias_group_rows == 0 && col < N) bv[k] = __ldg(reinterpret_cast<const float2*>(e.bias + col));
  }
  gemm_frag_math(p, acc0, 0, m_tile, n_base, wl, lane, sv, bv, use_bias);
  gemm_frag_math(p, acc1, 1, m_tile, n_base, wl, lane, sv, bv, use_bias);
  const int q = lane & 3, rq = lane >> 2;
  gemm_frag_store<EPI>(p, acc0, 0, m_tile, n_base, wl, q, rq, bufs, groups, leader, tr);
  gemm_frag_store<EPI>(p, acc1, 1, m_tile, n_base, wl, q, rq, bufs, groups, leader, tr);
}

// ==========================================================================================
// The kernel: persistent CTAs over 128 x 128 output tiles (warp roles in the header comment).
//   full barrier  : per stage, armed by the producer with the stage's byte count; the TMA loads credit it
//   empty barrier : per stage, one arrival per warp of the consumer warpgroup whose MMAs have read the stage
//   named barriers 1 / 2 : the MMA turn of consumer warpgroup 0 / 1 (ping-pong order, see the kernel)
//   named barriers 3 / 4 : consumer warpgroup 0 / 1 alone (its accumulator staging area, staged epilogues)
// ==========================================================================================
template <int EPI>
struct GemmCfg {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;  // 16 KB
  static constexpr int kBBytes = kGemmBN * kGemmBK * 2;  // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiWarps = 8;                     // the two consumer warpgroups
  static constexpr int kThreads = 128 + 32 * kEpiWarps;   // + the producer warpgroup
  // staged epilogues (register-direct, and the fp16 TMA store with row sums) go through the accumulator staging areas
  static constexpr bool kStaged = (EPI == EPI_DIRECT) || (EPI == EPI_TMA_F16_STAGED);
  // TMA epilogues: 4 KB of TMA-store staging per warp (two 16-row boxes, gemm_epilogue_frag; one 32-row tile,
  // gemm_tma_f16_staged)
  static constexpr int kStageOutBytes = (EPI == EPI_DIRECT) ? 0 : kEpiWarps * 4096;
  // staged epilogues: per consumer warpgroup, one staged column half of its tile
  static constexpr int kAccBytes = kGemmBM * kAccCols * 4;
  static constexpr int kAccAreaBytes = kStaged ? 2 * kAccBytes : 0;
  // operand ring | per-warp TMA-store staging (1024 B aligned) | 2 accumulator staging areas | mbarriers: <= 227 KB
  static constexpr int kStages = (EPI == EPI_DIRECT) ? 5 : (EPI == EPI_TMA_F16_STAGED) ? 4 : 6;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStageOutBytes + kAccAreaBytes + 1024 + 256;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory per CTA");
  // 128 x 24 + 256 x 240 <= 65536 (= 384 x 168 at launch): what the producer warpgroup gives back, the consumers take
  // (two 64 x 128 fp32 accumulators are 128 registers per consumer thread)
  static constexpr int kProducerRegs = 24;
  static constexpr int kConsumerRegs = 240;
};

// Fragment -> staging for column half H of the 64 tile rows whose staged row 0 is acc_half; acc holds them as wgmma lays
// them out (warp wl: rows 16 wl + lane/4 (+8), columns 8 j + 2 (lane % 4) (+1)). The staged registers are zeroed
// afterwards: the next tile's first MMA ignores the accumulator (scale-d = 0), so they are dead values instead of
// registers held across the epilogue.
template <int H>
__device__ __forceinline__ void gemm_stage_half(float* acc_half, float (&acc)[64], int wl, int lane) {
  const int r = wl * 16 + (lane >> 2);
  float* d0 = acc_half + r * kAccCols + 2 * (lane & 1);
  float* d1 = d0 + 8 * kAccCols;  // row r + 8: same swizzle as row r
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    const int j = 8 * H + jj;
    const int q = gemm_acc_chunk(2 * jj + ((lane & 3) >> 1), r);
    *reinterpret_cast<float2*>(d0 + 4 * q) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(d1 + 4 * q) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    acc[4 * j] = acc[4 * j + 1] = acc[4 * j + 2] = acc[4 * j + 3] = 0.f;
  }
}

// FIXED_SPLIT: the deterministic split-K schedule (GemmParams::split_fixed) is its own instantiation, so its index
// arithmetic stays out of the other kernels.
// CLUSTER: the grid is made of 2-CTA clusters, and both CTAs of a cluster walk the same work list of pair units
// (m_tile, n_pair) — (m_tile, n_pair, segment) under FIXED_SPLIT — in the m-fastest order of the unclustered list; the CTA
// of rank r computes n-tile 2 n_pair + r. The A tile is the same for both, so rank r loads only its rows 64 r .. 64 r + 63
// (the A tensor map's box is half a tile: {64, 64}, or {64, 16, 4, 1} = pixel rows 4 r .. 4 r + 3 of a conv tile) and
// multicasts them to the same ring offset in both CTAs; B stays per CTA. Each full barrier still expects the whole stage
// (16 KB of A, half from each rank, + 16 KB of B). Since either producer writes a stage of both CTAs, a stage is free only
// once the on-turn consumer warps of both CTAs have released it: every consumer warp arrives on the empty barrier of its
// own CTA and on the peer's (count 8). The two lists have the same k ranges, so the ring stage / parity sequence and the
// ping-pong turn order are the same in both CTAs. Every output element sums the same k16 chunks in the same order through
// the same instruction as without clusters: results are bit-identical. Needs an even n-tile count and no stream-K split.
// RAGGED: the parameters carry a per-image problem table (GemmRaggedTable) and the work list is decoded through it; the
// K loop and the epilogue arithmetic are the plain NCHW-T kernel's, so image b's logits are bit-identical to those of a
// one-image call with its own label set (an accumulator column does not depend on its neighbours). Unclustered.
template <int EPI, bool FIXED_SPLIT = false, bool GROUPED = false, bool RELU_RES = false, bool CLUSTER = false,
          bool RAGGED = false>
__global__ void __launch_bounds__(GemmCfg<EPI>::kThreads, 1)
    gemm_tc_kernel(const __grid_constant__ typename GemmParamsOf<RAGGED>::type p) {
  static_assert(!RELU_RES || (EPI == EPI_DIRECT && !FIXED_SPLIT && !GROUPED), "relu-after-residual: plain register-direct");
  static_assert(!RAGGED || (EPI == EPI_DIRECT && !FIXED_SPLIT && !GROUPED && !RELU_RES && !CLUSTER),
                "ragged pixel x text: NCHW-T store, register-direct, unclustered");
  static_assert(!FIXED_SPLIT || EPI == EPI_DIRECT, "split-K partials leave through the register-direct epilogue");
  static_assert(!GROUPED || (EPI == EPI_DIRECT && !FIXED_SPLIT), "per-image column blocks: NCHW-T store, register-direct");
  using Cfg = GemmCfg<EPI>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage_out = smem + Cfg::kStages * Cfg::kStageBytes;
  float* acc_stage = reinterpret_cast<float*>(stage_out + Cfg::kStageOutBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_stage) + Cfg::kAccAreaBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;

  const int warp = warp_idx_sync();  // provably warp-uniform: role branches and their operands stay on the uniform datapath
  const int lane = threadIdx.x & 31;
  // work list index and count: one list per CTA, or per cluster
  const int cta = CLUSTER ? static_cast<int>(cluster_id_x()) : static_cast<int>(blockIdx.x);
  const int num_ctas = CLUSTER ? static_cast<int>(num_clusters_x()) : static_cast<int>(gridDim.x);
  const int rank = CLUSTER ? static_cast<int>(cluster_ctarank()) : 0;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tma_a);
    tma_prefetch_desc(&p.tma_b);
    if (EPI != EPI_DIRECT) tma_prefetch_desc(&p.tma_c);
    for (int i = 0; i < Cfg::kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CLUSTER ? 8 : 4);
    }
    mbar_fence_init();
  }
  griddep_launch_dependents();
  if constexpr (CLUSTER)
    cluster_sync();  // the peer's barriers are initialised before its first multicast or remote arrival reaches them
  else
    __syncthreads();
  griddep_wait();  // everything above overlapped the previous kernel's tail; operands / outputs are touched below

  // CLUSTER: the list is over pair units (num_n_tiles is even); RAGGED: the table's tile count
  const int num_tiles = gemm_num_units(p, CLUSTER);

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
    sc.split = (EPI == EPI_TMA_ADD) && !CLUSTER && p.split_k;
    sc.fixed = FIXED_SPLIT ? p.split_fixed : 0;
    sc.seg = 0;
    const long long units = static_cast<long long>(num_tiles) * p.k_iters;
    // boundaries on multiples of 4 k-chunks: no sliver segments whose epilogue would cost more than their MMAs
    sc.unit = ((units * cta / num_ctas) + 3) & ~3ll;
    sc.unit_end = (cta + 1 == num_ctas) ? units : (((units * (cta + 1) / num_ctas) + 3) & ~3ll);
    if (sc.unit_end > units) sc.unit_end = units;
    return sc;
  };

  if (warp < 4) {
    // ===================== TMA producer warpgroup: warp 0 issues, warps 1-3 only hand their registers back =====================
    // (CLUSTER: warps 1-3 stay until the final cluster barrier instead of exiting)
    setmaxnreg_dec<Cfg::kProducerRegs>();
    if (!CLUSTER && warp != 0) return;
    const bool leader = elect_one_sync();  // converged warp, elected issuing lane
    int stage = 0;
    uint32_t phase = 0;
    Sched sc = make_sched();
    int tile, k_begin, k_end;
    while ((!CLUSTER || warp == 0) && sc.next(tile, k_begin, k_end)) {
      const GemmTileCoord tc = gemm_tile_coord<CLUSTER>(p, tile, rank);
      const int m_tile = tc.m_tile;
      const int n0 = tc.b_row;
      int cb = 0, ch0 = 0, cw0 = 0;
      if (p.conv) {
        const int per_img = p.tiles_h * p.tiles_w;
        cb = m_tile / per_img;
        const int t = m_tile % per_img;
        ch0 = (t / p.tiles_w) * kConvTH;
        cw0 = (t % p.tiles_w) * kConvTW;
      }
      for (int kit = k_begin; kit < k_end; ++kit) {
        // inlined wait: an out-of-line callee cannot be shared by warpgroups with different setmaxnreg budgets
        mbar_wait_inl(&empty_bar[stage], phase ^ 1, 21);
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
          if constexpr (CLUSTER) {  // this rank's half of the A tile, into both CTAs
            uint8_t* sa_half = sa + rank * (Cfg::kABytes / 2);
            if (p.conv)
              tma_load_4d_multicast(sa_half, &p.tma_a, &full_bar[stage], c0, c1, c2 + rank * (kConvTH / 2), cb, 0x3);
            else
              tma_load_2d_multicast(sa_half, &p.tma_a, &full_bar[stage], c0, c1 + rank * (kGemmBM / 2), 0x3);
          } else {
            if (p.conv)
              tma_load_4d(sa, &p.tma_a, &full_bar[stage], c0, c1, c2, cb);
            else
              tma_load_2d(sa, &p.tma_a, &full_bar[stage], c0, c1);
          }
          tma_load_2d(sb, &p.tma_b, &full_bar[stage], kit * kGemmBK, n0);
        }
        __syncwarp();
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumers: ping-pong over the CTA's work list =====================
    // Entry i of the list belongs to warpgroup i % 2, which runs the main loop of the whole 128 x 128 tile (two
    // m64n128k16 per k16 step: rows 0-63 and 64-127) and then its epilogue. The producer fills the ring in list order,
    // so the warpgroups take their MMA turns in list order: warpgroup w waits for its turn (barrier 1 + w) before its
    // first full-barrier wait (the parity of a ring stage names one fill only once the previous entry has consumed its
    // chunks) and hands the turn on as soon as its MMAs are issued. Its epilogue then runs during the other
    // warpgroup's main loop.
    setmaxnreg_inc<Cfg::kConsumerRegs>();
    const int wg = (warp - 4) >> 2;
    const int wl = warp & 3;       // warp within its warpgroup: main loop fragment rows 16 wl .. 16 wl + 15 of each
    const int r = wl * 32 + lane;  // 64-row half; epilogue tile row r (thread <-> row)
    float* acc_half = Cfg::kStaged ? acc_stage + wg * (Cfg::kAccBytes / 4) : nullptr;  // staged epilogues
    const float* acc_row = Cfg::kStaged ? acc_half + r * kAccCols : nullptr;
    uint8_t* stage_bufs = stage_out + (warp - 4) * (Cfg::kStageOutBytes / Cfg::kEpiWarps);  // TMA epilogues
    int store_groups = 0;
    // TMA epilogues: the lane that issues (and owns the bulk groups of) this warp's TMA stores
    const bool leader = (EPI != EPI_DIRECT) && elect_one_sync();
    int stage = 0;
    uint32_t phase = 0;
    GemmTrace tr;
    const int bid = blockIdx.x;  // traced: CTAs 0 and gridDim.x / 2 (clustered plans: both are rank 0 of their pair)
    if (p.trace && lane == 0 && (bid == 0 || bid == static_cast<int>(gridDim.x) / 2)) tr.w = p.trace + ((bid == 0 ? 0 : 1) * 20 + warp) * 512;
    tr(0);
    float acc0[64], acc1[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc0[i] = acc1[i] = 0.f;
    Sched sc = make_sched();
    int tile, k_begin, k_end;
    bool more = sc.next(tile, k_begin, k_end);
    for (int idx = 0; more; ++idx) {
      const GemmTileCoord tc = gemm_tile_coord<CLUSTER>(p, tile, rank);
      const int m_tile = tc.m_tile;
      const int n_tile = tc.n_tile;
      const int img = tc.img;
      const int kb = k_begin, ke = k_end;
      const int seg = FIXED_SPLIT ? sc.seg : 0;
      more = sc.next(tile, k_begin, k_end);  // entry idx + 1
      if ((idx & 1) != wg) {  // the other warpgroup's entry: step over its ring fills
        const int s = stage + (ke - kb);
        phase ^= (s / Cfg::kStages) & 1;
        stage = s % Cfg::kStages;
        continue;
      }
      if (idx > 0) bar_sync(1 + wg, 256);
      int prev = -1;
      for (int kit = kb; kit < ke; ++kit) {
        mbar_wait_inl(&full_bar[stage], phase, 23);
        __syncwarp();
        const uint32_t a_base = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint32_t b_base = a_base + Cfg::kABytes;
        if (!(p.probe & 4)) {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kGemmBK / 16; ++k) {
            const uint64_t db = wgmma_desc_sw128(b_base + k * 32, 1024, 16);
            const uint32_t accumulate = (kit != kb) || (k != 0);
            wgmma_m64n128k16_ss(acc0, wgmma_desc_sw128(a_base + k * 32, 1024, 16), db, accumulate);
            wgmma_m64n128k16_ss(acc1, wgmma_desc_sw128(a_base + 64 * 128 + k * 32, 1024, 16), db, accumulate);
          }
          wgmma_commit();
        }
        wgmma_wait<1>();  // the previous chunk's MMAs have read their stage (complete): hand it back to the producer(s)
        if (prev >= 0 && lane == 0) {
          mbar_arrive(&empty_bar[prev]);
          if constexpr (CLUSTER) mbar_arrive_cluster(&empty_bar[prev], rank ^ 1);
        }
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      if (more) bar_arrive(1 + (wg ^ 1), 256);  // entry idx + 1 is the other warpgroup's
      wgmma_wait<0>();
      wgmma_reg_fence(acc0);
      wgmma_reg_fence(acc1);
      if (prev >= 0 && lane == 0) {
        mbar_arrive(&empty_bar[prev]);
        if constexpr (CLUSTER) mbar_arrive_cluster(&empty_bar[prev], rank ^ 1);
      }
      tr(12);
      if constexpr (Cfg::kStaged) {
        // Epilogue, one column half at a time through this warpgroup's staging area. Barrier 3 + wg: no warp of the
        // warpgroup still reads the area (previous half or tile) when it is rewritten, and all of it is written before
        // any warp reads it.
        auto epilogue_half = [&](int n_base) {
          if constexpr (EPI == EPI_DIRECT)
            gemm_epilogue_tile<GROUPED, RELU_RES, RAGGED>(p, acc_row, n_base, kAccCols, m_tile, r, []() {}, seg,
                                                          gemm_ragged_k(p, img), gemm_ragged_koff(p, img));
          else
            gemm_tma_f16_staged(p, acc_row, n_base, kAccCols, m_tile, r, stage_bufs, store_groups, leader, tr);
        };
        bar_sync(3 + wg, 128);
        gemm_stage_half<0>(acc_half, acc0, wl, lane);
        gemm_stage_half<0>(acc_half + 64 * kAccCols, acc1, wl, lane);
        bar_sync(3 + wg, 128);
        epilogue_half(n_tile * kGemmBN);
        bar_sync(3 + wg, 128);
        gemm_stage_half<1>(acc_half, acc0, wl, lane);
        gemm_stage_half<1>(acc_half + 64 * kAccCols, acc1, wl, lane);
        bar_sync(3 + wg, 128);
        epilogue_half(n_tile * kGemmBN + kAccCols);
      } else if (!(p.probe & 1)) {
        gemm_epilogue_frag<EPI>(p, acc0, acc1, m_tile, n_tile * kGemmBN, wl, lane, stage_bufs, store_groups, leader, kb == 0,
                                tr);
      }
      tr(7);
    }
    if (EPI != EPI_DIRECT && leader) tma_store_wait_all();  // outstanding bulk ops read this CTA's smem
  }
  // CLUSTER: no CTA leaves while its peer may still arrive on its barriers (the peer's consumers release their last
  // stages on both CTAs)
  if constexpr (CLUSTER) cluster_sync();
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
