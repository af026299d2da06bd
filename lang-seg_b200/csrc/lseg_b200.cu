// lseg_b200 — single translation unit of liblseg_b200.so: host launchers, the C ABI declared in
// include/lseg_b200.h, and (engine.cuh) the whole-model forward. Compiled for sm_90a only.
#include "../../include/lseg_b200.h"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"
#include "elementwise.cuh"
#include "gemm_tc.cuh"
#include "mhsa.cuh"
#include "text_attn.cuh"
#include "p2p.cuh"
#include "evaluator.cuh"

namespace lseg {

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local char t_error[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_error, sizeof(t_error), fmt, ap);
  va_end(ap);
}
const char* get_error() { return t_error; }

// ------------------------------------------------------------------------------------------
// device / driver entry points
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;
static int g_num_sms = 0;        // SM count of the devices this process uses (all must agree: H100 SXM = 132)
static int g_deterministic = 1;  // 1 (default): fixed summation order; 0: split-K allowed (LSEG_SPLITK=1 / lseg_set_deterministic(0))
static int g_plan_epoch = 0;     // bumped when an option that is baked into cached plans changes
static unsigned long long* g_gemm_trace = nullptr;  // debug (lseg_debug_gemm_trace)
static int g_gemm_probe = 0;
static int g_mhsa_variant = 0;   // kernel the engine's ViT attention runs (lseg_mhsa_variant documents the numbering)
static std::mutex g_init_mutex;
static bool g_global_init = false;
constexpr int kMaxDevices = 64;
static int g_dev_status[kMaxDevices];  // 0 = not initialised, 1 = ready, -1 = unusable

// Process-wide part: driver entry point and environment switches.
static int init_global() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
    set_error("lseg_b200: cuTensorMapEncodeTiled not available from the driver");
    return -1;
  }
  g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  if (getenv("LSEG_SPLITK")) g_deterministic = 0;
  const char* pr = getenv("LSEG_GEMM_PROBE");  // measurement only, see GemmParams::probe
  g_gemm_probe = pr ? atoi(pr) : 0;
  const char* mv = getenv("LSEG_MHSA_VARIANT");
  if (mv) g_mhsa_variant = atoi(mv);
  return 0;
}

// Per-device part: architecture check and the function attributes (opt-in shared memory sizes are a property of
// (function, device); a process that drives several GPUs — DataParallel replicas, additional_utils/models.py:183-248 —
// must set them on each one).
static int init_device(int dev) {
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
    set_error("lseg_b200: cudaGetDeviceProperties failed");
    return -1;
  }
  if (prop.major != 9 || prop.minor != 0) {
    set_error("lseg_b200: device '%s' is sm_%d%d; this library contains sm_90a code only", prop.name, prop.major,
              prop.minor);
    return -1;
  }
  if (g_num_sms != 0 && g_num_sms != prop.multiProcessorCount) {
    set_error("lseg_b200: devices with different SM counts in one process (%d vs %d)", g_num_sms,
              prop.multiProcessorCount);
    return -1;
  }
  g_num_sms = prop.multiProcessorCount;
#define LSEG_SET_SMEM(KERNEL, EPI_) \
  cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<EPI_>::kSmemBytes)
  LSEG_SET_SMEM((gemm_tc_kernel<EPI_DIRECT>), EPI_DIRECT);
  LSEG_SET_SMEM((gemm_tc_kernel<EPI_TMA_F16>), EPI_TMA_F16);
  LSEG_SET_SMEM((gemm_tc_kernel<EPI_TMA_ADD>), EPI_TMA_ADD);
  LSEG_SET_SMEM((gemm_tc_kernel<EPI_DIRECT, true>), EPI_DIRECT);
  LSEG_SET_SMEM((gemm_tc_kernel<EPI_DIRECT, false, true>), EPI_DIRECT);
  LSEG_SET_SMEM((gemm_tc_kernel<EPI_DIRECT, false, false, true>), EPI_DIRECT);
#undef LSEG_SET_SMEM
  cudaFuncSetAttribute(mhsa_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(mhsa_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(mhsa_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(mhsa_kernel<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  if (cudaGetLastError() != cudaSuccess) {
    set_error("lseg_b200: cudaFuncSetAttribute failed on device %d", dev);
    return -1;
  }
  return 0;
}

// Makes the CURRENT device usable (idempotent, thread-safe). Every entry point calls it after cudaSetDevice.
static int ensure_init() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("lseg_b200: no CUDA device available (there is no CPU fallback)");
    return -1;
  }
  if (dev < 0 || dev >= kMaxDevices) {
    set_error("lseg_b200: device index %d out of range", dev);
    return -1;
  }
  if (g_dev_status[dev] == 1) return 0;
  std::lock_guard<std::mutex> lock(g_init_mutex);
  if (g_dev_status[dev] == 1) return 0;
  if (!g_global_init) {
    if (init_global()) return -1;
    g_global_init = true;
  }
  if (init_device(dev)) return -1;
  g_dev_status[dev] = 1;
  return 0;
}

static int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box);
int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box) {
  return make_tmap(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, rank, dims, strides_bytes, box);
}
static int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("tensor map base %p is not 16-byte aligned", base);
    return -1;
  }
  CUresult r = g_encode(out, dtype, rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with %d (rank %d dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)", (int)r, rank,
              (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
              (unsigned long long)(rank > 2 ? gdim[2] : 0), (unsigned long long)(rank > 3 ? gdim[3] : 0), bdim[0],
              rank > 1 ? bdim[1] : 0, rank > 2 ? bdim[2] : 0, rank > 3 ? bdim[3] : 0);
    return -1;
  }
  return 0;
}

int read_watchdog(int out[4], cudaStream_t stream) {
  LSEG_CHECK_CUDA(cudaStreamSynchronize(stream));
  LSEG_CHECK_CUDA(cudaMemcpyFromSymbol(out, g_watchdog, sizeof(int) * 4));
  int zero[4] = {0, 0, 0, 0};
  LSEG_CHECK_CUDA(cudaMemcpyToSymbol(g_watchdog, zero, sizeof(zero)));
  return 0;
}

// ------------------------------------------------------------------------------------------
// GEMM planning / launch
// ------------------------------------------------------------------------------------------
struct GemmPlan {
  GemmParams p;
  int grid;
  int epi;      // GemmEpiMode
  // deterministic split-K (gemm_tc.cuh splitk_reduce_kernel): p.split_fixed segments per tile write raw partials to a
  // workspace the CALLER provides (gemm_set_workspace) before gemm_run; final_epi is the epilogue the reduce applies
  size_t ws_bytes;
  GemmEpi final_epi;
};

// Split the K loop of the implicit-GEMM convs whose tile count leaves most CTAs idle (3x3 convs on the 15x15 decoder
// level, layer4_rn). The segment count is a function of the PER-IMAGE geometry only — it is sized
// for a batch of kSplitRefBatch images whatever the actual batch — so the summation order, and with it every bit of the
// result, is the same for batch 1 and batch 64 (the evaluator's batched and one-by-one runs must agree exactly).
constexpr int kSplitRefBatch = 8;
static int gemm_pick_split(const GemmDesc& d, const GemmParams& p, int n_tiles, int max_ctas) {
  static const int mode = getenv("LSEG_SPLITK_FIXED") ? atoi(getenv("LSEG_SPLITK_FIXED")) : -1;  // 0 off, >1 forced, -1 auto
  if (mode == 0 || !d.conv) return 0;
  const GemmEpi& e = d.e;
  const bool plain_epi = e.store == STORE_ROWMAJOR && e.bias_group_rows == 0 && !e.out_row_sumsq && !e.res_f16 &&
                         !e.row_sumsq && (d.N % 8 == 0) && (e.out_f32 || e.out_f16 || e.out_f16_relu);
  const bool inplace = e.res_f32 && e.res_f32 == e.out_f32;
  if (!plain_epi || inplace) return 0;
  const int ref_tiles = kSplitRefBatch * p.tiles_h * p.tiles_w * n_tiles;
  if (ref_tiles * 2 > max_ctas) return 0;
  int s = max_ctas / ref_tiles;
  if (mode > 1) s = mode;
  if (s > p.k_iters / 4) s = p.k_iters / 4;
  if (s > 16) s = 16;
  // two or three segments only pay where the unsplit GEMM would leave through the register-direct epilogue (fp32 /
  // residual / multi-output); a plain fp16 output keeps its TMA-store epilogue
  const bool tma_f16 = e.out_f16 && !e.out_f32 && !e.out_f16_relu && !e.res_f32 && !e.res2_f32;
  if (s < 4 && tma_f16 && mode <= 1) return 0;
  return s >= 2 ? s : 0;
}

static void gemm_set_workspace(GemmPlan* plan, float* ws) { plan->p.e.out_f32 = ws; }

static int gemm_plan(const GemmDesc& d, GemmPlan* plan) {
  if (ensure_init()) return -1;
  GemmParams& p = plan->p;
  memset(&p, 0, sizeof(p));
  if (d.K % kGemmBK != 0) {
    set_error("gemm: K=%d must be a multiple of %d", d.K, kGemmBK);
    return -1;
  }
  const int taps = d.conv ? d.kh * d.kw : 1;
  const long long ktot = static_cast<long long>(taps) * d.K;
  if (d.w_rows < kGemmBN && d.w_rows < d.N) {
    set_error("gemm: weight rows %d < N %d", d.w_rows, d.N);
    return -1;
  }
  p.M = d.M;
  p.N = d.N;
  p.k_chunks = d.K / kGemmBK;
  p.k_iters = p.k_chunks * taps;
  p.conv = d.conv;
  p.probe = g_gemm_probe;
  p.trace = g_gemm_trace;
  p.e = d.e;
  if (d.conv) {
    p.H = d.H;
    p.W = d.W;
    p.kw = d.kw;
    p.pad = d.pad;
    p.tiles_h = (d.H + kConvTH - 1) / kConvTH;
    p.tiles_w = (d.W + kConvTW - 1) / kConvTW;
    p.num_m_tiles = d.B * p.tiles_h * p.tiles_w;
    const uint64_t dims[4] = {(uint64_t)d.K, (uint64_t)d.W, (uint64_t)d.H, (uint64_t)d.B};
    const uint64_t str[3] = {(uint64_t)d.K * 2, (uint64_t)d.K * d.W * 2, (uint64_t)d.K * d.W * d.H * 2};
    const uint32_t box[4] = {kGemmBK, kConvTW, kConvTH, 1};
    if (make_tmap_f16(&p.tma_a, d.a, 4, dims, str, box)) return -1;
  } else {
    p.num_m_tiles = (d.M + kGemmBM - 1) / kGemmBM;
    const uint64_t dims[2] = {(uint64_t)d.K, (uint64_t)d.a_rows};
    const uint64_t str[1] = {(uint64_t)d.lda * 2};
    const uint32_t box[2] = {kGemmBK, kGemmBM};
    if (make_tmap_f16(&p.tma_a, d.a, 2, dims, str, box)) return -1;
  }
  p.num_n_tiles = (d.N + kGemmBN - 1) / kGemmBN;
  {
    const uint64_t dims[2] = {(uint64_t)ktot, (uint64_t)d.w_rows};
    const uint64_t str[1] = {(uint64_t)ktot * 2};
    const uint32_t box[2] = {kGemmBK, kGemmBN};
    if (make_tmap_f16(&p.tma_b, d.w, 2, dims, str, box)) return -1;
  }
  // TMA-store epilogue: plain fp16 row-major outputs (QKV, fc1, readout, 1x1 / 3x3 convs feeding the next conv,
  // head1, text in_proj / c_fc)
  plan->epi = EPI_DIRECT;
  plan->ws_bytes = 0;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  {
    const int split = gemm_pick_split(d, p, p.num_n_tiles, g_num_sms);
    if (split) {
      plan->final_epi = d.e;
      p.split_fixed = split;
      p.split_rows = d.M;
      p.e = GemmEpi{};
      memset(&p.e, 0, sizeof(p.e));
      p.e.store = STORE_ROWMAJOR;
      p.e.ldc = d.N;
      p.e.row_scale = 1.f;
      plan->ws_bytes = sizeof(float) * static_cast<size_t>(split) * d.M * d.N;
      const int units = tiles * split;
      plan->grid = units < g_num_sms ? units : g_num_sms;
      if (d.e.store == STORE_ROWMAJOR && (d.e.ldc % 8 != 0)) {
        set_error("gemm: ldc must be a multiple of 8");
        return -1;
      }
      return 0;
    }
  }
  {
    const GemmEpi& e = p.e;
    static const bool disabled = getenv("LSEG_GEMM_NO_TMA_STORE") != nullptr;
    const bool rowmajor = !disabled && e.store == STORE_ROWMAJOR && (d.N % 8 == 0) && d.N >= 64;
    if (e.relu_after_res && (e.store != STORE_ROWMAJOR || !e.res_f32 || e.res_f16 || e.out_row_sumsq)) {
      set_error("gemm: relu_after_res needs a row-major store and an fp32 residual");
      return -1;
    }
    if (rowmajor && e.out_f16 && !e.out_f32 && !e.out_f16_relu && !e.res_f16 && !e.res_f32 && !e.res2_f32 &&
        (e.ldc % 8 == 0)) {
      if (d.conv) {
        const uint64_t dims[4] = {(uint64_t)d.N, (uint64_t)d.W, (uint64_t)d.H, (uint64_t)d.B};
        const uint64_t str[3] = {(uint64_t)e.ldc * 2, (uint64_t)e.ldc * d.W * 2, (uint64_t)e.ldc * d.W * d.H * 2};
        const uint32_t box[4] = {64, kConvTW, 2, 1};
        if (make_tmap_f16(&p.tma_c, e.out_f16, 4, dims, str, box)) return -1;
      } else {
        const uint64_t dims[2] = {(uint64_t)d.N, (uint64_t)d.M};
        const uint64_t str[1] = {(uint64_t)e.ldc * 2};
        const uint32_t box[2] = {64, 32};
        if (make_tmap_f16(&p.tma_c, e.out_f16, 2, dims, str, box)) return -1;
      }
      plan->epi = EPI_TMA_F16;
    } else if (rowmajor && !d.conv && e.out_f32 && e.res_f32 == e.out_f32 && !e.res2_f32 && !e.res_f16 &&
               !e.out_f16 && !e.out_f16_relu && !e.out_row_sumsq && !e.relu_after_res && (e.ldc % 4 == 0)) {
      // in-place fp32 residual stream: x += A W^T + b through a bulk tensor reduce-add (x is never read)
      const uint64_t dims[2] = {(uint64_t)d.N, (uint64_t)d.M};
      const uint64_t str[1] = {(uint64_t)e.ldc * 4};
      const uint32_t box[2] = {32, 32};
      if (make_tmap(&p.tma_c, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, e.out_f32, 2, dims, str, box)) return -1;
      plan->epi = EPI_TMA_ADD;
      // stream-K style balancing when whole tiles would leave a ragged last wave
      static const int min_kit = getenv("LSEG_SPLITK_MIN_KITERS") ? atoi(getenv("LSEG_SPLITK_MIN_KITERS")) : 32;
      p.split_k =
          (!g_deterministic && tiles > g_num_sms && tiles % g_num_sms != 0 && p.k_iters >= min_kit) ? 1 : 0;
    }
  }
  plan->grid = tiles < g_num_sms ? tiles : g_num_sms;
  if (p.e.store == STORE_D2S && (p.e.d2s_cout % 32 != 0 || !p.e.out_f16)) {
    set_error("gemm: depth-to-space store needs cout %% 32 == 0 and an fp16 output");
    return -1;
  }
  if (p.e.store == STORE_ROWMAJOR && (p.e.ldc % 8 != 0)) {
    set_error("gemm: ldc must be a multiple of 8");
    return -1;
  }
  return 0;
}

static int gemm_run_kernel(const GemmPlan& plan, cudaStream_t stream);
static int gemm_run(const GemmPlan& plan, cudaStream_t stream) {
  if (plan.grid <= 0) return 0;
  if (plan.p.split_fixed > 1) {
    if (!plan.p.e.out_f32) {
      set_error("gemm: split-K plan without a workspace (gemm_set_workspace)");
      return -1;
    }
    if (gemm_run_kernel(plan, stream)) return -1;
    const long long quads = static_cast<long long>(plan.p.M) * (plan.p.N / 4);
    launch_pdl(splitk_reduce_kernel, dim3(static_cast<unsigned>((quads + 255) / 256)), dim3(256), 0, stream,
               static_cast<const float*>(plan.p.e.out_f32), plan.p.split_fixed, static_cast<long long>(plan.p.M), plan.p.N,
               plan.final_epi);
    LSEG_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  return gemm_run_kernel(plan, stream);
}
static int gemm_run_kernel(const GemmPlan& plan, cudaStream_t stream) {
#define LSEG_LAUNCH(KERNEL, EPI_) \
  launch_pdl(KERNEL, dim3(plan.grid), dim3(GemmCfg<EPI_>::kThreads), GemmCfg<EPI_>::kSmemBytes, stream, plan.p)
  if (plan.epi == EPI_TMA_F16) LSEG_LAUNCH(gemm_tc_kernel<EPI_TMA_F16>, EPI_TMA_F16);
  else if (plan.epi == EPI_TMA_ADD) LSEG_LAUNCH(gemm_tc_kernel<EPI_TMA_ADD>, EPI_TMA_ADD);
  else if (plan.p.split_fixed > 1) LSEG_LAUNCH((gemm_tc_kernel<EPI_DIRECT, true>), EPI_DIRECT);
  else if (plan.p.e.store == STORE_NCHW_T && plan.p.e.nchw_group > 0)
    LSEG_LAUNCH((gemm_tc_kernel<EPI_DIRECT, false, true>), EPI_DIRECT);
  else if (plan.p.e.relu_after_res) LSEG_LAUNCH((gemm_tc_kernel<EPI_DIRECT, false, false, true>), EPI_DIRECT);
  else LSEG_LAUNCH(gemm_tc_kernel<EPI_DIRECT>, EPI_DIRECT);
#undef LSEG_LAUNCH
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// MHSA planning / launch
// ------------------------------------------------------------------------------------------
struct MhsaPlan {
  MhsaParams p;
  dim3 grid;
};
static int mhsa_plan(const MhsaDesc& d, MhsaPlan* plan) {
  if (ensure_init()) return -1;
  MhsaParams& p = plan->p;
  memset(&p, 0, sizeof(p));
  const int D = d.heads * kMhsaDh;
  const uint64_t dims[3] = {(uint64_t)3 * D, (uint64_t)d.N, (uint64_t)d.B};
  const uint64_t str[2] = {(uint64_t)3 * D * 2, (uint64_t)3 * D * d.N * 2};
  const uint32_t box[3] = {kMhsaDh, kMhsaTile, 1};
  if (make_tmap_f16(&p.tma_qkv, d.qkv, 3, dims, str, box)) return -1;
  const uint32_t box64[3] = {kMhsaDh, kMhsaKT, 1};
  if (make_tmap_f16(&p.tma_t64, d.qkv, 3, dims, str, box64)) return -1;
  p.out = d.out;
  p.n_tokens = d.N;
  p.heads = d.heads;
  p.D = D;
  p.causal = d.causal;
  p.scale_log2e = 0.125f * 1.44269504088896340736f;
  plan->grid = dim3((d.N + kMhsaTile - 1) / kMhsaTile, d.B * d.heads, 1);
  return 0;
}
// variant (include/lseg_b200.h): the share of exponentials evaluated on the FMA pipe — 0, 1, 2, 5, 6: none; 3, 7: one
// of four score pairs; 4, 8: two of four.
static int mhsa_run_variant(const MhsaPlan& plan, int variant, cudaStream_t stream) {
  switch (variant) {
    case 0: case 1: case 2: case 5: case 6:
      launch_pdl(mhsa_kernel<0>, plan.grid, dim3(kMhsaThreads), kMhsaSmemBytes, stream, plan.p);
      break;
    case 3: case 7: launch_pdl(mhsa_kernel<1>, plan.grid, dim3(kMhsaThreads), kMhsaSmemBytes, stream, plan.p); break;
    case 4: case 8: launch_pdl(mhsa_kernel<2>, plan.grid, dim3(kMhsaThreads), kMhsaSmemBytes, stream, plan.p); break;
    default: set_error("mhsa: unknown kernel variant %d", variant); return -1;
  }
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}
static int mhsa_run(const MhsaPlan& plan, cudaStream_t stream) { return mhsa_run_variant(plan, g_mhsa_variant, stream); }

// ------------------------------------------------------------------------------------------
// elementwise launch helpers
// ------------------------------------------------------------------------------------------
static int run_layernorm(const void* x, int in_f16, const float* g, const float* b, __half* y, long long M, int C,
                         float eps, cudaStream_t s) {
  const int rows_per_block = 8;
  const int grid = static_cast<int>((M + rows_per_block - 1) / rows_per_block);
  const dim3 blk(rows_per_block * 32);
#define LSEG_LN_CASE(CC)                                                                                            \
  case CC:                                                                                                          \
    if (in_f16)                                                                                                     \
      launch_pdl(layernorm_kernel<__half, CC>, dim3(grid), blk, 0, s, static_cast<const __half*>(x), g, b, y, M, eps); \
    else                                                                                                            \
      launch_pdl(layernorm_kernel<float, CC>, dim3(grid), blk, 0, s, static_cast<const float*>(x), g, b, y, M, eps);   \
    break;
  switch (C) {
    LSEG_LN_CASE(512)
    LSEG_LN_CASE(768)
    LSEG_LN_CASE(1024)
    default:
      set_error("layernorm: C=%d (the path has 512 — CLIP text —, 768 — ViT-B — and 1024 — ViT-L)", C);
      return -1;
  }
#undef LSEG_LN_CASE
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace lseg

#include "engine.cuh"

// ==========================================================================================
// C ABI
// ==========================================================================================
using namespace lseg;

extern "C" {

const char* lseg_last_error(void) { return get_error(); }
int lseg_abi_version(void) { return LSEG_B200_ABI_VERSION; }

int lseg_read_watchdog(int out[4], void* stream) {
  if (ensure_init()) return -1;
  return read_watchdog(out, static_cast<cudaStream_t>(stream));
}

static void fill_epi(const lseg_gemm_args* a, GemmEpi* e) {
  memset(e, 0, sizeof(*e));
  e->bias = a->bias;
  e->bias_group_rows = a->bias_group_rows;
  e->scale = a->scale;
  e->act = a->act;
  e->res_f32 = a->res_f32;
  e->res2_f32 = a->res2_f32;
  e->res_f16 = static_cast<const __half*>(a->res_f16);
  e->out_f32 = a->out_f32;
  e->out_f16 = static_cast<__half*>(a->out_f16);
  e->out_f16_relu = static_cast<__half*>(a->out_f16_relu);
  e->ldc = a->ldc;
  e->store = a->store;
  e->d2s_s = a->d2s_s;
  e->d2s_cout = a->d2s_cout;
  e->d2s_h = a->d2s_h;
  e->d2s_w = a->d2s_w;
  e->nchw_p = a->nchw_p;
  e->nchw_k = a->nchw_k;
  e->nchw_group = a->nchw_group;
  e->row_sumsq = a->row_sumsq;
  e->row_sumsq_parts = a->row_sumsq_parts;
  e->row_scale = a->row_scale;
  e->out_row_sumsq = a->out_row_sumsq;
  e->relu_after_res = a->relu_after_res;
}

int lseg_gemm(const lseg_gemm_args* a, void* stream) {
  if (!a) {
    set_error("lseg_gemm: null args");
    return -1;
  }
  GemmDesc d;
  memset(&d, 0, sizeof(d));
  d.a = static_cast<const __half*>(a->a);
  d.lda = a->lda;
  d.a_rows = a->a_rows > 0 ? a->a_rows : a->M;
  d.w = static_cast<const __half*>(a->w);
  d.w_rows = a->w_rows > 0 ? a->w_rows : a->N;
  d.M = a->M;
  d.N = a->N;
  d.K = a->K;
  d.conv = a->conv;
  d.B = a->B;
  d.H = a->H;
  d.W = a->W;
  d.kh = d.kw = a->ksize;
  d.pad = a->pad;
  fill_epi(a, &d.e);
  GemmPlan plan;
  if (gemm_plan(d, &plan)) return -1;
  if (plan.ws_bytes) {  // stage-op call: a per-device scratch that only grows (the engine plans own theirs)
    static std::mutex mu;
    static float* scratch[64] = {nullptr};
    static size_t cap[64] = {0};
    int dev = 0;
    LSEG_CHECK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    if (dev < 0 || dev >= 64) {
      set_error("lseg_gemm: device index %d", dev);
      return -1;
    }
    if (cap[dev] < plan.ws_bytes) {
      LSEG_CHECK_CUDA(cudaDeviceSynchronize());
      if (scratch[dev]) cudaFree(scratch[dev]);
      scratch[dev] = nullptr;
      cap[dev] = 0;
      LSEG_CHECK_CUDA(cudaMalloc(&scratch[dev], plan.ws_bytes));
      cap[dev] = plan.ws_bytes;
    }
    gemm_set_workspace(&plan, scratch[dev]);
  }
  return gemm_run(plan, static_cast<cudaStream_t>(stream));
}

int lseg_mhsa(const void* qkv, void* out, int B, int N, int heads, int causal, void* stream) {
  MhsaDesc d;
  d.qkv = static_cast<const __half*>(qkv);
  d.out = static_cast<__half*>(out);
  d.B = B;
  d.N = N;
  d.heads = heads;
  d.causal = causal;
  MhsaPlan plan;
  if (mhsa_plan(d, &plan)) return -1;
  return mhsa_run(plan, static_cast<cudaStream_t>(stream));
}

int lseg_mhsa_variant(const void* qkv, void* out, int B, int N, int heads, int causal, int variant, void* stream) {
  MhsaDesc d;
  d.qkv = static_cast<const __half*>(qkv);
  d.out = static_cast<__half*>(out);
  d.B = B;
  d.N = N;
  d.heads = heads;
  d.causal = causal;
  MhsaPlan plan;
  if (mhsa_plan(d, &plan)) return -1;
  return mhsa_run_variant(plan, variant, static_cast<cudaStream_t>(stream));
}

int lseg_text_attn(const void* qkv, void* out, int K, int L, int heads, void* stream) {
  if (ensure_init()) return -1;
  return launch_text_attn(static_cast<const __half*>(qkv), static_cast<__half*>(out), K, L, heads,
                          static_cast<cudaStream_t>(stream));
}

// ---- multi-scale evaluator glue + preprocessing (SURVEY.md section 8(f) rows 1 and 3) ----
static_assert(sizeof(lseg_eval_window) == sizeof(EvalWindow), "lseg_eval_window layout");

int lseg_eval_make_crops(const float* img, float* crops, const lseg_eval_window* wins, int n_inputs, int h, int w, int crop,
                         const float* pad3_host, void* stream) {
  if (ensure_init()) return -1;
  if (!img || !crops || !wins || !pad3_host || n_inputs <= 0 || n_inputs > 65535 || crop <= 0) {
    set_error("lseg_eval_make_crops: bad argument");
    return -1;
  }
  eval_make_crops_kernel<<<dim3((crop + 31) / 32, (crop + 7) / 8, n_inputs), dim3(32, 8), 0,
                           static_cast<cudaStream_t>(stream)>>>(img, crops, reinterpret_cast<const EvalWindow*>(wins), h, w,
                                                                crop, pad3_host[0], pad3_host[1], pad3_host[2]);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_eval_canvas(const float* outs, float* canvas, const lseg_eval_window* wins, int n_win, int K, int crop, int height,
                     int width, int flip, int whole, void* stream) {
  if (ensure_init()) return -1;
  if (!outs || !canvas || !wins || n_win <= 0 || K <= 0 || K > 65535) {
    set_error("lseg_eval_canvas: bad argument");
    return -1;
  }
  eval_canvas_kernel<<<dim3((width + 31) / 32, (height + 7) / 8, K), dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      outs, canvas, reinterpret_cast<const EvalWindow*>(wins), n_win, K, crop, height, width, flip, whole);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_eval_resize_add(const float* canvas, float* scores, int K, int height, int width, int h, int w, void* stream) {
  if (ensure_init()) return -1;
  if (!canvas || !scores || K <= 0 || K > 65535) {
    set_error("lseg_eval_resize_add: bad argument");
    return -1;
  }
  eval_resize_add_kernel<<<dim3((w + 31) / 32, (h + 7) / 8, K), dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      canvas, scores, height, width, h, w);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_preprocess(const unsigned char* img_hwc, float* out, int h, int w, int Ho, int Wo, int Hp, int Wp,
                    const float* mean3_host, const float* std3_host, const float* pad3_host, void* stream) {
  if (ensure_init()) return -1;
  if (!img_hwc || !out || !mean3_host || !std3_host || !pad3_host || h <= 0 || w <= 0 || Ho <= 0 || Wo <= 0 || Hp < Ho ||
      Wp < Wo) {
    set_error("lseg_preprocess: bad argument");
    return -1;
  }
  preprocess_kernel<<<dim3((Wp + 31) / 32, (Hp + 7) / 8), dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      img_hwc, out, h, w, Ho, Wo, Hp, Wp, mean3_host[0], mean3_host[1], mean3_host[2], std3_host[0], std3_host[1],
      std3_host[2], pad3_host[0], pad3_host[1], pad3_host[2]);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---- peer memory (the logits gather, SURVEY.md section 8(e)) ----
int lseg_p2p_alloc(unsigned long long bytes, void** dptr, unsigned char* handle64) {
  if (ensure_init()) return -1;
  if (!dptr || !handle64 || bytes == 0) {
    set_error("lseg_p2p_alloc: bad argument");
    return -1;
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  void* p = nullptr;
  LSEG_CHECK_CUDA(cudaMalloc(&p, bytes));
  LSEG_CHECK_CUDA(cudaMemset(p, 0, bytes));
  LSEG_CHECK_CUDA(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  cudaError_t err = cudaIpcGetMemHandle(&h, p);
  if (err != cudaSuccess) {
    cudaFree(p);
    set_error("lseg_p2p_alloc: cudaIpcGetMemHandle failed: %s", cudaGetErrorString(err));
    return -1;
  }
  memcpy(handle64, &h, 64);
  *dptr = p;
  return 0;
}

int lseg_p2p_open(const unsigned char* handle64, void** dptr) {
  if (ensure_init()) return -1;
  if (!dptr || !handle64) {
    set_error("lseg_p2p_open: bad argument");
    return -1;
  }
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t err = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (err != cudaSuccess) {
    cudaGetLastError();
    set_error("lseg_p2p_open: cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(err));
    return -1;
  }
  *dptr = p;
  return 0;
}

int lseg_p2p_close(void* dptr) {
  if (!dptr) return 0;
  LSEG_CHECK_CUDA(cudaIpcCloseMemHandle(dptr));
  return 0;
}

int lseg_p2p_free(void* dptr) {
  if (!dptr) return 0;
  LSEG_CHECK_CUDA(cudaFree(dptr));
  return 0;
}

int lseg_p2p_copy(void* dst, const void* src, unsigned long long bytes, void* stream) {
  LSEG_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
  return 0;
}

int lseg_p2p_signal(unsigned long long* flag, unsigned long long value, void* stream) {
  if (ensure_init()) return -1;
  p2p_signal_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(flag, value);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_p2p_wait(const unsigned long long* flags, int n, int stride, unsigned long long value, unsigned int timeout_ms,
                  void* stream) {
  if (ensure_init()) return -1;
  if (n <= 0) return 0;
  p2p_wait_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(flags, n, stride, value,
                                                                  static_cast<unsigned long long>(timeout_ms) * 1000000ull);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_set_deterministic(int on) {
  if (ensure_init()) return -1;
  if ((on != 0) != (g_deterministic != 0)) ++g_plan_epoch;
  g_deterministic = on ? 1 : 0;
  return 0;
}

int lseg_debug_gemm_trace(unsigned long long* trace) {
  g_gemm_trace = trace;
  return 0;
}

int lseg_mhsa_trace(const void* qkv, void* out, int B, int N, int heads, int causal, unsigned long long* trace,
                    void* stream) {
  MhsaDesc d;
  d.qkv = static_cast<const __half*>(qkv);
  d.out = static_cast<__half*>(out);
  d.B = B;
  d.N = N;
  d.heads = heads;
  d.causal = causal;
  MhsaPlan plan;
  if (mhsa_plan(d, &plan)) return -1;
  plan.p.trace = trace;
  mhsa_kernel<0, true><<<plan.grid, kMhsaThreads, kMhsaSmemBytes, static_cast<cudaStream_t>(stream)>>>(plan.p);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_layernorm(const void* x, int in_f16, const float* gamma, const float* beta, void* y, long long M, int C,
                   float eps, void* stream) {
  if (ensure_init()) return -1;
  return run_layernorm(x, in_f16, gamma, beta, static_cast<__half*>(y), M, C, eps, static_cast<cudaStream_t>(stream));
}

int lseg_patchify(const float* x, void* a, int B, int H, int W, int patch, void* stream) {
  if (ensure_init()) return -1;
  return launch_patchify(x, static_cast<__half*>(a), B, H, W, patch, static_cast<cudaStream_t>(stream));
}

int lseg_pos_resize(const float* pos, float* out, int g0, int gh, int gw, int D, void* stream) {
  if (ensure_init()) return -1;
  pos_resize_kernel<<<1 + gh * gw, 256, 0, static_cast<cudaStream_t>(stream)>>>(pos, out, g0, gh, gw, D);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_assemble_tokens(const float* patch, const float* cls, const float* pos, float* x, int B, int T, int D,
                         void* stream) {
  if (ensure_init()) return -1;
  return launch_assemble_tokens(patch, cls, pos, x, B, T, D, static_cast<cudaStream_t>(stream));
}

int lseg_readout_split(const float* tap, void* tok, void* cls, int B, int T, int D, void* stream) {
  if (ensure_init()) return -1;
  return launch_readout_split(tap, static_cast<__half*>(tok), static_cast<__half*>(cls), B, T, D,
                              static_cast<cudaStream_t>(stream));
}

int lseg_im2col_3x3_s2(const void* x, void* a, int B, int H, int W, int C, void* stream) {
  if (ensure_init()) return -1;
  return launch_im2col_3x3_s2(static_cast<const __half*>(x), static_cast<__half*>(a), B, H, W, C,
                              static_cast<cudaStream_t>(stream));
}

int lseg_stem_im2col(const float* x, void* a, int B, int H, int W, void* stream) {
  if (ensure_init()) return -1;
  return launch_stem_im2col(x, static_cast<__half*>(a), B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_maxpool3x3s2_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  if (ensure_init()) return -1;
  return launch_maxpool3x3s2_nhwc(static_cast<const __half*>(x), static_cast<__half*>(y), B, H, W, C,
                                  static_cast<cudaStream_t>(stream));
}

int lseg_subsample2_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  if (ensure_init()) return -1;
  return launch_subsample2_nhwc(static_cast<const __half*>(x), static_cast<__half*>(y), B, H, W, C,
                                static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  if (ensure_init()) return -1;
  return launch_upsample2x_nhwc(static_cast<const __half*>(x), static_cast<__half*>(y), B, H, W, C,
                                static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_nhwc256(const void* x, int in_f16, void* y, int out_f16, const float* add, int B, int H, int W,
                            void* stream) {
  if (ensure_init()) return -1;
  if (add && out_f16) {
    set_error("upsample2x_nhwc256: the skip operand goes with an fp32 output");
    return -1;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (in_f16) {
    if (out_f16) return launch_upsample2x_nhwc256_f16<__half>(static_cast<const __half*>(x), static_cast<__half*>(y), nullptr, B, H, W, s);
    return launch_upsample2x_nhwc256_f16<float>(static_cast<const __half*>(x), static_cast<float*>(y), add, B, H, W, s);
  }
  if (out_f16) return launch_upsample2x_nhwc256_f32<__half>(static_cast<const float*>(x), static_cast<__half*>(y), nullptr, B, H, W, s);
  return launch_upsample2x_nhwc256_f32<float>(static_cast<const float*>(x), static_cast<float*>(y), add, B, H, W, s);
}

int lseg_l2norm_scale(const float* x, void* y, long long M, int C, float logit_scale, void* stream) {
  if (ensure_init()) return -1;
  if (C % 128 != 0 || C > 512) {
    set_error("l2norm_scale: C=%d must be a multiple of 128 and <= 512", C);
    return -1;
  }
  const int grid = static_cast<int>((M + 7) / 8);
  l2norm_scale_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, static_cast<__half*>(y), M, C,
                                                                           logit_scale);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_l2norm_f16(const void* x, void* y, int M, int C, void* stream) {
  if (ensure_init()) return -1;
  l2norm_f16_kernel<<<(M + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __half*>(x),
                                                                               static_cast<__half*>(y), M, C);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_upsample2x_nchw(const void* x, float* y, long long planes, int H, int W, void* stream) {
  if (ensure_init()) return -1;
  if ((2 * W) % 4 != 0) {
    set_error("upsample2x_nchw: output width must be a multiple of 4");
    return -1;
  }
  return launch_upsample2x_nchw(static_cast<const __half*>(x), y, planes, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_debug_upsample_layout(int split) {
  const int old = g_upsample_split;
  g_upsample_split = split ? 1 : 0;
  return old;
}

int lseg_upsample2x_nchw_bg(const void* x, float* y, long long planes, int H, int W, void* stream) {
  if (ensure_init()) return -1;
  return launch_upsample2x_nchw_bg(static_cast<const __half*>(x), y, planes, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_nchw_f32(const float* x, float* y, long long planes, int H, int W, void* stream) {
  if (ensure_init()) return -1;
  if ((2 * W) % 4 != 0) {
    set_error("upsample2x_nchw: output width must be a multiple of 4");
    return -1;
  }
  return launch_upsample2x_nchw(x, y, planes, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_head_block(const void* x, int in_f16, float* cmax_ws, float* y, int B, int K, int h, int w, const float* w9_host,
                    float bias, int mode, int act, void* stream) {
  if (ensure_init()) return -1;
  if (!x || !y || !w9_host || (mode != 1 && mode != 2) || (mode == 1 && !cmax_ws)) {
    set_error("lseg_head_block: bad argument");
    return -1;
  }
  HeadBlockW hw;
  for (int i = 0; i < 9; ++i) hw.w[i] = w9_host[i];
  hw.bias = bias;
  if (in_f16)
    return launch_head_block(static_cast<const __half*>(x), cmax_ws, y, B, K, h, w, hw, mode, act,
                             static_cast<cudaStream_t>(stream));
  return launch_head_block(static_cast<const float*>(x), cmax_ws, y, B, K, h, w, hw, mode, act,
                           static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_argmax(const void* lr, long long* mask, int B, int K, int H, int W, void* stream) {
  if (ensure_init()) return -1;
  return launch_upsample2x_argmax(static_cast<const __half*>(lr), mask, B, K, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_text_embed(const int64_t* tokens, const float* tok_emb, const float* pos_emb, void* x, int K, int L, int Wd,
                    void* stream) {
  if (ensure_init()) return -1;
  text_embed_kernel<<<K * L, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(tokens), tok_emb, pos_emb, static_cast<__half*>(x), L, Wd);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_text_eot_gather(const int64_t* tokens, const void* x, void* out, int K, int L, int Wd, void* stream) {
  if (ensure_init()) return -1;
  text_eot_gather_kernel<<<K, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(tokens), static_cast<const __half*>(x), static_cast<__half*>(out), K, L, Wd);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
