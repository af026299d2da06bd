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
#include "attn_probs.cuh"
#include "text_attn.cuh"
#include "p2p.cuh"
#include "evaluator.cuh"
#include "embed.cuh"

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
static int g_gemm_cluster_mode = 2;  // lseg_debug_set_gemm_cluster: 1 never, 2 the planner's rule, 3 wherever allowed
static int g_trace_block = -1;       // lseg_debug_set_trace_block: trunk block whose intermediates image plans snapshot
// Which gemm_tc_kernel instantiation runs a plan (numbering of lseg_debug_gemm_plan's out[4]).
enum GemmKernel { GK_DIRECT = 0, GK_TMA_F16 = 1, GK_TMA_ADD = 2, GK_FIXED_SPLIT = 3, GK_GROUPED_NCHW = 4, GK_RELU_RES = 5,
                  GK_RAGGED = 6, GK_COUNT = 7 };
static int g_gemm_active_pairs[GK_COUNT];  // per instantiation: 2-CTA clusters of it that fit on the device at once
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

// Opt-in shared memory of both forms of one gemm_tc_kernel instantiation, and how many 2-CTA clusters of the clustered
// form the device holds at once (not simply SMs / 2: a cluster's CTAs share one GPC, and a GPC may have an odd SM count).
template <int EPI, bool FIXED_SPLIT = false, bool GROUPED = false, bool RELU_RES = false>
static int gemm_init_kernel(int* active_pairs) {
  auto plain = gemm_tc_kernel<EPI, FIXED_SPLIT, GROUPED, RELU_RES, false>;
  auto paired = gemm_tc_kernel<EPI, FIXED_SPLIT, GROUPED, RELU_RES, true>;
  const int smem = GemmCfg<EPI>::kSmemBytes;
  if (cudaFuncSetAttribute(plain, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
      cudaFuncSetAttribute(paired, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return -1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2);
  cfg.blockDim = dim3(GemmCfg<EPI>::kThreads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  return cudaOccupancyMaxActiveClusters(active_pairs, paired, &cfg) == cudaSuccess ? 0 : -1;
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
  int pairs[GK_COUNT];
  int pairs_staged = 0;  // GK_TMA_F16 plans with row sums launch the staged form (gemm_run_kernel)
  if (gemm_init_kernel<EPI_DIRECT>(&pairs[GK_DIRECT]) || gemm_init_kernel<EPI_TMA_F16>(&pairs[GK_TMA_F16]) ||
      gemm_init_kernel<EPI_TMA_F16_STAGED>(&pairs_staged) || gemm_init_kernel<EPI_TMA_ADD>(&pairs[GK_TMA_ADD]) ||
      gemm_init_kernel<EPI_DIRECT, true>(&pairs[GK_FIXED_SPLIT]) ||
      gemm_init_kernel<EPI_DIRECT, false, true>(&pairs[GK_GROUPED_NCHW]) ||
      gemm_init_kernel<EPI_DIRECT, false, false, true>(&pairs[GK_RELU_RES]) ||
      cudaFuncSetAttribute(gemm_tc_kernel<EPI_DIRECT, false, false, false, false, true>,
                           cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<EPI_DIRECT>::kSmemBytes) != cudaSuccess) {
    set_error("lseg_b200: GEMM kernel attributes / cluster occupancy query failed on device %d", dev);
    return -1;
  }
  pairs[GK_RAGGED] = 0;  // the ragged kernel has no clustered form
  if (pairs_staged < pairs[GK_TMA_F16]) pairs[GK_TMA_F16] = pairs_staged;
  memcpy(g_gemm_active_pairs, pairs, sizeof(pairs));
  cudaFuncSetAttribute(mhsa_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(mhsa_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(mhsa_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(mhsa_kernel<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMhsaSmemBytes);
  cudaFuncSetAttribute(attn_probs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnPSmemBytes);
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

// A barrier timeout (g_watchdog) is reported first; a bad metric group id (g_segstats_error, tag kSegStatsTag) when no
// timeout is pending; a bad loss target (g_xent_error, tag kXentTag) when neither is. Only the reported record is
// cleared, so further calls return the others.
int read_watchdog(int out[4], cudaStream_t stream) {
  LSEG_CHECK_CUDA(cudaStreamSynchronize(stream));
  LSEG_CHECK_CUDA(cudaMemcpyFromSymbol(out, g_watchdog, sizeof(int) * 4));
  int zero[4] = {0, 0, 0, 0};
  if (out[0] != 0) {
    LSEG_CHECK_CUDA(cudaMemcpyToSymbol(g_watchdog, zero, sizeof(zero)));
    return 0;
  }
  LSEG_CHECK_CUDA(cudaMemcpyFromSymbol(out, g_segstats_error, sizeof(int) * 4));
  if (out[0] != 0) {
    LSEG_CHECK_CUDA(cudaMemcpyToSymbol(g_segstats_error, zero, sizeof(zero)));
    return 0;
  }
  LSEG_CHECK_CUDA(cudaMemcpyFromSymbol(out, g_xent_error, sizeof(int) * 4));
  if (out[0] != 0) LSEG_CHECK_CUDA(cudaMemcpyToSymbol(g_xent_error, zero, sizeof(zero)));
  return 0;
}

// ------------------------------------------------------------------------------------------
// GEMM planning / launch
// ------------------------------------------------------------------------------------------
struct GemmPlan {
  GemmParams p;
  int grid;     // CTAs
  int cluster;  // 1, or 2: CTA pairs that share the A tile (gemm_tc_kernel CLUSTER); grid is then even
  int epi;      // GemmEpiMode
  // deterministic split-K (gemm_tc.cuh splitk_reduce_kernel): p.split_fixed segments per tile write raw partials to a
  // workspace the CALLER provides (gemm_set_workspace) before gemm_run; final_epi is the epilogue the reduce applies
  size_t ws_bytes;
  GemmEpi final_epi;
  int ragged = 0;      // 1: pixel x text over the per-image problem table rt (gemm_plan_ragged); never clustered
  GemmRaggedTable rt;
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

static int gemm_kernel_of(const GemmPlan& plan);
// Last step of gemm_plan: cluster size, grid, and the A tensor map, whose box is what one CTA loads (a whole 128-row
// tile, or the half a CTA of a pair multicasts). Pairs need an even n-tile count (no dummy tiles) and whole tiles per work
// unit (stream-K ranges are per CTA). The units are tiles, or tiles x segments under the fixed split-K schedule.
// The planner pairs CTAs only when there are more work units than SMs. Measured with tools/gemm_shapes.py (B = 8, 480^2,
// H100 80GB HBM3 at 700 W, paired vs unclustered, two runs): with several units per CTA, pairs were faster on the ViT
// proj / fc1 / fc2 (+4 to +8 %), the 120^2 and 60^2 3x3 convs (+4 to +18 %), the 120^2 1x1 out_conv (+12 %), head1
// (+40 %; its 236 MB A operand exceeds L2, and a pair fetches each A tile once for two n-tiles) and pixel x text
// (+5 %); QKV was within 1 % (-0.6 / -1.0 %). Where every CTA owns at most one unit (the 30^2 convs: 128 tiles; the
// 15^2 split-K convs: 128 units) pairs only add their barrier round trips: layer_rn and RCU conv2 at 30^2 and 15^2 were
// 0.4 to 3.2 % slower in both runs, RCU conv1 +4 % to -11 %.
static int gemm_plan_grid(const GemmDesc& d, GemmPlan* plan) {
  GemmParams& p = plan->p;
  const int pairs = g_gemm_active_pairs[gemm_kernel_of(*plan)];
  const int units = plan->ragged ? plan->rt.tile0[plan->rt.n]
                                 : p.num_m_tiles * p.num_n_tiles * (p.split_fixed > 1 ? p.split_fixed : 1);
  const bool allowed = !plan->ragged && p.num_n_tiles % 2 == 0 && !p.split_k && pairs > 0;
  const bool wanted = g_gemm_cluster_mode == 3 || (g_gemm_cluster_mode == 2 && units > g_num_sms);
  plan->cluster = (allowed && wanted) ? 2 : 1;
  if (plan->cluster == 2)
    plan->grid = 2 * (units / 2 < pairs ? units / 2 : pairs);
  else
    plan->grid = units < g_num_sms ? units : g_num_sms;
  const int rows = kGemmBM / plan->cluster;
  if (d.conv) {
    const uint64_t dims[4] = {(uint64_t)d.K, (uint64_t)d.W, (uint64_t)d.H, (uint64_t)d.B};
    const uint64_t str[3] = {(uint64_t)d.K * 2, (uint64_t)d.K * d.W * 2, (uint64_t)d.K * d.W * d.H * 2};
    const uint32_t box[4] = {kGemmBK, kConvTW, (uint32_t)rows / kConvTW, 1};
    return make_tmap_f16(&p.tma_a, d.a, 4, dims, str, box);
  }
  const uint64_t dims[2] = {(uint64_t)d.K, (uint64_t)d.a_rows};
  const uint64_t str[1] = {(uint64_t)d.lda * 2};
  const uint32_t box[2] = {kGemmBK, (uint32_t)rows};
  return make_tmap_f16(&p.tma_a, d.a, 2, dims, str, box);
}

static int gemm_plan(const GemmDesc& d, GemmPlan* plan) {
  if (ensure_init()) return -1;
  GemmParams& p = plan->p;
  memset(&p, 0, sizeof(p));
  if (d.K % kGemmBK != 0) {
    set_error("gemm: K=%d must be a multiple of %d", d.K, kGemmBK);
    return -1;
  }
  {  // the epilogue reads and writes these operands with 16-byte vector accesses
    const struct { const void* ptr; const char* name; } ops[] = {
        {d.e.bias, "bias"}, {d.e.scale, "scale"}, {d.e.res_f32, "res_f32"}, {d.e.res2_f32, "res2_f32"},
        {d.e.res_f16, "res_f16"}, {d.e.out_f32, "out_f32"}, {d.e.out_f16, "out_f16"},
        {d.e.out_f16_relu, "out_f16_relu"}};
    for (const auto& op : ops) {
      if ((reinterpret_cast<uintptr_t>(op.ptr) & 15) != 0) {
        set_error("gemm: %s pointer %p is not 16-byte aligned", op.name, op.ptr);
        return -1;
      }
    }
  }
  if (d.e.relu_after_res && (d.e.store != STORE_ROWMAJOR || !d.e.res_f32 || d.e.res_f16 || d.e.out_row_sumsq)) {
    set_error("gemm: relu_after_res needs a row-major store and an fp32 residual");
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
  } else {
    p.num_m_tiles = (d.M + kGemmBM - 1) / kGemmBM;
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
      if (d.e.store == STORE_ROWMAJOR && (d.e.ldc % 8 != 0)) {
        set_error("gemm: ldc must be a multiple of 8");
        return -1;
      }
      return gemm_plan_grid(d, plan);
    }
  }
  {
    const GemmEpi& e = p.e;
    static const bool disabled = getenv("LSEG_GEMM_NO_TMA_STORE") != nullptr;
    const bool rowmajor = !disabled && e.store == STORE_ROWMAJOR && (d.N % 8 == 0) && d.N >= 64;
    if (rowmajor && e.out_f16 && !e.out_f32 && !e.out_f16_relu && !e.res_f16 && !e.res_f32 && !e.res2_f32 &&
        (e.ldc % 8 == 0)) {
      // a box is one warp's 16 fragment rows, or 32 staged rows for the row-sum form (gemm_run_kernel)
      const uint32_t rows = e.out_row_sumsq ? 32 : 16;
      if (d.conv) {
        const uint64_t dims[4] = {(uint64_t)d.N, (uint64_t)d.W, (uint64_t)d.H, (uint64_t)d.B};
        const uint64_t str[3] = {(uint64_t)e.ldc * 2, (uint64_t)e.ldc * d.W * 2, (uint64_t)e.ldc * d.W * d.H * 2};
        const uint32_t box[4] = {64, kConvTW, rows / kConvTW, 1};  // whole pixel rows of the 8 x 16 tile
        if (make_tmap_f16(&p.tma_c, e.out_f16, 4, dims, str, box)) return -1;
      } else {
        const uint64_t dims[2] = {(uint64_t)d.N, (uint64_t)d.M};
        const uint64_t str[1] = {(uint64_t)e.ldc * 2};
        const uint32_t box[2] = {64, rows};
        if (make_tmap_f16(&p.tma_c, e.out_f16, 2, dims, str, box)) return -1;
      }
      plan->epi = EPI_TMA_F16;
    } else if (rowmajor && !d.conv && e.out_f32 && e.res_f32 == e.out_f32 && !e.res2_f32 && !e.res_f16 &&
               !e.out_f16 && !e.out_f16_relu && !e.out_row_sumsq && !e.relu_after_res && (e.ldc % 4 == 0)) {
      // in-place fp32 residual stream: x += A W^T + b through a bulk tensor reduce-add (x is never read)
      const uint64_t dims[2] = {(uint64_t)d.N, (uint64_t)d.M};
      const uint64_t str[1] = {(uint64_t)e.ldc * 4};
      const uint32_t box[2] = {32, 16};
      if (make_tmap(&p.tma_c, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, e.out_f32, 2, dims, str, box)) return -1;
      plan->epi = EPI_TMA_ADD;
      // stream-K style balancing when whole tiles would leave a ragged last wave. Only without an activation: the
      // segments of a tile reduce-add their epilogue results, and act(p1 + p2 + b) != act(p1 + b) + act(p2).
      static const int min_kit = getenv("LSEG_SPLITK_MIN_KITERS") ? atoi(getenv("LSEG_SPLITK_MIN_KITERS")) : 32;
      p.split_k = (!g_deterministic && e.act == ACT_NONE && tiles > g_num_sms && tiles % g_num_sms != 0 &&
                   p.k_iters >= min_kit) ? 1 : 0;
    }
  }
  if (p.e.store == STORE_D2S && (p.e.d2s_cout % 32 != 0 || !p.e.out_f16)) {
    set_error("gemm: depth-to-space store needs cout %% 32 == 0 and an fp16 output");
    return -1;
  }
  if (p.e.store == STORE_ROWMAJOR && (p.e.ldc % 8 != 0)) {
    set_error("gemm: ldc must be a multiple of 8");
    return -1;
  }
  return gemm_plan_grid(d, plan);
}

// Ragged pixel x text plan (gemm_tc_kernel RAGGED, the table in gemm_tc.cuh): d describes the whole product — A = the
// B * P pixel rows (P = d.e.nchw_p, a multiple of 128), w = the packed text operand with d.w_rows readable rows, e = the
// NCHW-T epilogue whose out_f16 is the packed fp16 [sum k, P] output. Image b's label count k[b] and first text row
// text_row[b] are host arrays: the tile counts are needed here. Unclustered: the pair rule needs an even n-tile count,
// and the per-image counts are generally odd.
static int gemm_plan_ragged(GemmDesc d, int B, const int* k, const int* text_row, GemmPlan* plan) {
  const int P = d.e.nchw_p;
  if (B < 1 || B > kRaggedMaxImages) return set_error("gemm_ragged: B=%d images (1 .. %d)", B, kRaggedMaxImages), -1;
  if (P <= 0 || P % kGemmBM != 0 || static_cast<long long>(B) * P != d.M)
    return set_error("gemm_ragged: P=%d pixels per image must be a positive multiple of %d (M=%d)", P, kGemmBM, d.M), -1;
  GemmRaggedTable& rt = plan->rt;
  memset(&rt, 0, sizeof(rt));
  rt.n = B;
  rt.m_tiles = P / kGemmBM;
  long long koff = 0, tiles = 0;
  int kmax = 0;
  for (int b = 0; b < B; ++b) {
    if (k[b] < 1 || text_row[b] < 0 || static_cast<long long>(text_row[b]) + k[b] > d.w_rows)
      return set_error("gemm_ragged: image %d: k=%d labels at text_row=%d do not fit %d text rows", b, k[b], text_row[b],
                       d.w_rows), -1;
    rt.k[b] = k[b];
    rt.text_row[b] = text_row[b];
    rt.koff[b] = static_cast<int>(koff);
    rt.tile0[b] = static_cast<int>(tiles);
    koff += k[b];
    tiles += static_cast<long long>(rt.m_tiles) * ((k[b] + kGemmBN - 1) / kGemmBN);
    if (koff > 65535 || tiles > (1 << 30)) return set_error("gemm_ragged: sum of k = %lld exceeds 65535", koff), -1;
    kmax = k[b] > kmax ? k[b] : kmax;
  }
  rt.tile0[B] = static_cast<int>(tiles);
  d.N = kmax;
  d.e.store = STORE_NCHW_T;
  d.e.nchw_k = kmax;
  d.e.nchw_group = 0;
  plan->ragged = 1;
  return gemm_plan(d, plan);
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
static int gemm_kernel_of(const GemmPlan& plan) {
  if (plan.ragged) return GK_RAGGED;
  if (plan.epi == EPI_TMA_F16) return GK_TMA_F16;
  if (plan.epi == EPI_TMA_ADD) return GK_TMA_ADD;
  if (plan.p.split_fixed > 1) return GK_FIXED_SPLIT;
  if (plan.p.e.store == STORE_NCHW_T && plan.p.e.nchw_group > 0) return GK_GROUPED_NCHW;
  if (plan.p.e.relu_after_res) return GK_RELU_RES;
  return GK_DIRECT;
}
template <int EPI, bool FIXED_SPLIT = false, bool GROUPED = false, bool RELU_RES = false>
static void gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
  const dim3 grid(plan.grid), block(GemmCfg<EPI>::kThreads);
  if (plan.cluster == 2)
    launch_pdl_cluster(gemm_tc_kernel<EPI, FIXED_SPLIT, GROUPED, RELU_RES, true>, grid, block, GemmCfg<EPI>::kSmemBytes,
                       2, stream, plan.p);
  else
    launch_pdl(gemm_tc_kernel<EPI, FIXED_SPLIT, GROUPED, RELU_RES>, grid, block, GemmCfg<EPI>::kSmemBytes, stream, plan.p);
}
static int gemm_run_kernel(const GemmPlan& plan, cudaStream_t stream) {
  switch (gemm_kernel_of(plan)) {
    case GK_TMA_F16:
      // Row sums (head1's partial squared norms, out_row_sumsq) must be summed in column order per row. The staged form
      // has each thread hold whole rows, so that order costs nothing. Split across the fragment's lanes, the sums took
      // head1 (K = 256, its epilogue longer than its main loop) from 0.405 to 0.45 ms (H100 80GB HBM3, 700 W).
      if (plan.p.e.out_row_sumsq)
        gemm_launch<EPI_TMA_F16_STAGED>(plan, stream);
      else
        gemm_launch<EPI_TMA_F16>(plan, stream);
      break;
    case GK_TMA_ADD: gemm_launch<EPI_TMA_ADD>(plan, stream); break;
    case GK_FIXED_SPLIT: gemm_launch<EPI_DIRECT, true>(plan, stream); break;
    case GK_GROUPED_NCHW: gemm_launch<EPI_DIRECT, false, true>(plan, stream); break;
    case GK_RELU_RES: gemm_launch<EPI_DIRECT, false, false, true>(plan, stream); break;
    case GK_RAGGED: {
      GemmRaggedParams rp;
      static_cast<GemmParams&>(rp) = plan.p;
      rp.rt = plan.rt;
      launch_pdl(gemm_tc_kernel<EPI_DIRECT, false, false, false, false, true>, dim3(plan.grid),
                 dim3(GemmCfg<EPI_DIRECT>::kThreads), GemmCfg<EPI_DIRECT>::kSmemBytes, stream, rp);
      break;
    }
    default: gemm_launch<EPI_DIRECT>(plan, stream); break;
  }
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
  // the rules of include/lseg_b200.h, checked before a tensor map is encoded: one CTA row per (image, head) in
  // gridDim.y, TMA loads of qkv (16-byte base) and __half2 stores to out (4-byte base)
  {
    const struct { int v; const char* name; } dims[] = {{d.B, "B"}, {d.N, "N"}, {d.heads, "heads"}};
    for (const auto& x : dims) {
      if (x.v <= 0) {
        set_error("mhsa: %s=%d must be positive", x.name, x.v);
        return -1;
      }
    }
  }
  if (static_cast<long long>(d.B) * d.heads > 65535) {
    set_error("mhsa: B*heads = %lld exceeds 65535 (B=%d, heads=%d)", static_cast<long long>(d.B) * d.heads, d.B,
              d.heads);
    return -1;
  }
  if (!d.qkv || (reinterpret_cast<uintptr_t>(d.qkv) & 15) != 0) {
    set_error("mhsa: qkv pointer %p is null or not 16-byte aligned", static_cast<const void*>(d.qkv));
    return -1;
  }
  if (!d.out || (reinterpret_cast<uintptr_t>(d.out) & 3) != 0) {
    set_error("mhsa: out pointer %p is null or not 4-byte aligned", static_cast<const void*>(d.out));
    return -1;
  }
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
// attention probabilities (attn_probs.cuh): planning / launch
// ------------------------------------------------------------------------------------------
struct AttnProbsPlan {
  AttnProbsParams p;  // p.out is set per call (the engine's plans take it from CallCtx)
  dim3 grid;
};
// Tensor maps and grid for qkv of (B, N, heads), whose arguments have been checked: those of the fused attention kernel.
static int attn_probs_maps(const __half* qkv, int B, int N, int heads, AttnProbsPlan* plan) {
  MhsaDesc d;
  d.qkv = qkv;
  d.out = const_cast<__half*>(qkv);  // mhsa_plan wants an output; this one is never written
  d.B = B;
  d.N = N;
  d.heads = heads;
  d.causal = 0;
  MhsaPlan mp;
  if (mhsa_plan(d, &mp)) return -1;
  AttnProbsParams& p = plan->p;
  memset(&p, 0, sizeof(p));
  p.tma_qkv = mp.p.tma_qkv;
  p.tma_t64 = mp.p.tma_t64;
  p.n_tokens = N;
  p.heads = heads;
  p.D = mp.p.D;
  p.scale_log2e = mp.p.scale_log2e;
  plan->grid = mp.grid;
  return 0;
}
// The rules of lseg_attn_probs (include/lseg_b200.h), each rejected by name before a tensor map is encoded.
static int attn_probs_plan(const char* fn, const __half* qkv, float* out, int B, int N, int heads, AttnProbsPlan* plan) {
  if (B <= 0) return set_error("%s: B=%d must be positive", fn, B), -1;
  if (N <= 0) return set_error("%s: N=%d must be positive", fn, N), -1;
  if (heads <= 0) return set_error("%s: heads=%d must be positive", fn, heads), -1;
  if (static_cast<long long>(B) * heads > 65535)
    return set_error("%s: B*heads = %lld exceeds 65535 (B=%d, heads=%d)", fn, static_cast<long long>(B) * heads, B, heads),
           -1;
  if (!qkv) return set_error("%s: null qkv", fn), -1;
  if (reinterpret_cast<uintptr_t>(qkv) % 16) return set_error("%s: qkv must be 16-byte aligned", fn), -1;
  if (!out) return set_error("%s: null out", fn), -1;
  if (reinterpret_cast<uintptr_t>(out) % 4) return set_error("%s: out must be 4-byte aligned", fn), -1;
  if (attn_probs_maps(qkv, B, N, heads, plan)) return -1;
  plan->p.out = out;
  return 0;
}
static int attn_probs_run(const AttnProbsPlan& plan, cudaStream_t stream) {
  launch_pdl(attn_probs_kernel, plan.grid, dim3(kAttnPThreads), kAttnPSmemBytes, stream, plan.p);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

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

// Argument rules of the glue entries (include/lseg_b200.h): each is checked, and a violation reported by entry and
// argument name, before anything is launched. Alignments are the kernels' vector widths; grid-y/z limits are 65535.
constexpr long long kGridYZ = 65535, kGridX = 2147483647;
static int arg_ptr(const char* fn, const char* name, const void* p, int align) {
  if (!p) return set_error("%s: null %s", fn, name), -1;
  if (reinterpret_cast<uintptr_t>(p) % align) return set_error("%s: %s must be %d-byte aligned", fn, name, align), -1;
  return 0;
}
static int arg_pos(const char* fn, const char* name, long long v) {
  if (v <= 0) return set_error("%s: %s=%lld must be positive", fn, name, v), -1;
  return 0;
}
static int arg_max(const char* fn, const char* what, long long v, long long lim) {
  if (v > lim) return set_error("%s: %s = %lld exceeds %lld", fn, what, v, lim), -1;
  return 0;
}
static int arg_mult(const char* fn, const char* name, long long v, int m) {
  if (v % m) return set_error("%s: %s=%lld must be a multiple of %d", fn, name, v, m), -1;
  return 0;
}
// the smem-line upsamples (lseg_upsample2x_nchw*, lseg_upsample2x_argmax): W % 8 == 0, W <= kUpMaxW
static int arg_up_w(const char* fn, int W) {
  if (arg_mult(fn, "W", W, 8)) return -1;
  return arg_max(fn, "W", W, kUpMaxW);
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

static int gemm_desc_of(const lseg_gemm_args* a, GemmDesc& d) {
  if (!a) {
    set_error("lseg_gemm: null args");
    return -1;
  }
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
  return 0;
}

int lseg_gemm(const lseg_gemm_args* a, void* stream) {
  GemmDesc d;
  if (gemm_desc_of(a, d)) return -1;
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

int lseg_gemm_ragged(const void* a, const float* row_sumsq, int row_sumsq_parts, float row_scale, int B, int P, int C,
                     const void* text, int text_rows, const int* text_row, const int* k, void* out, void* stream) {
  const char* fn = "lseg_gemm_ragged";
  if (!a) return set_error("%s: null a", fn), -1;
  if (!out) return set_error("%s: null out", fn), -1;
  if (reinterpret_cast<uintptr_t>(a) % 16) return set_error("%s: a must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(out) % 16) return set_error("%s: out must be 16-byte aligned", fn), -1;
  if (P <= 0 || P % kGemmBM != 0) return set_error("%s: P=%d must be a positive multiple of %d", fn, P, kGemmBM), -1;
  if (C <= 0 || C % kGemmBK != 0) return set_error("%s: C=%d must be a positive multiple of %d", fn, C, kGemmBK), -1;
  if (row_sumsq && row_sumsq_parts < 1)
    return set_error("%s: row_sumsq_parts=%d must be positive with row_sumsq", fn, row_sumsq_parts), -1;
  long long sum_k = 0;
  if (check_ragged(fn, B, text, text_rows, text_row, k, &sum_k)) return -1;
  if (static_cast<long long>(B) * P > (1ll << 31) - 1) return set_error("%s: B*P = %lld rows", fn, (long long)B * P), -1;
  GemmDesc d;
  memset(&d, 0, sizeof(d));
  d.a = static_cast<const __half*>(a);
  d.lda = C;
  d.a_rows = B * P;
  d.w = static_cast<const __half*>(text);
  d.w_rows = text_rows;
  d.M = B * P;
  d.K = C;
  d.e = epi_none();
  d.e.out_f16 = static_cast<__half*>(out);
  d.e.nchw_p = P;
  d.e.row_sumsq = row_sumsq;
  d.e.row_sumsq_parts = row_sumsq ? row_sumsq_parts : 0;
  d.e.row_scale = row_scale;
  GemmPlan plan;
  if (gemm_plan_ragged(d, B, k, text_row, &plan)) return -1;
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

int lseg_attn_probs(const void* qkv, float* out, int B, int N, int heads, void* stream) {
  AttnProbsPlan plan;
  if (attn_probs_plan("lseg_attn_probs", static_cast<const __half*>(qkv), out, B, N, heads, &plan)) return -1;
  return attn_probs_run(plan, static_cast<cudaStream_t>(stream));
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
  const char* fn = "lseg_preprocess";
  if (arg_ptr(fn, "img_hwc", img_hwc, 1) || arg_ptr(fn, "out", out, 4) || arg_ptr(fn, "mean3", mean3_host, 4) ||
      arg_ptr(fn, "std3", std3_host, 4) || arg_ptr(fn, "pad3", pad3_host, 4) || arg_pos(fn, "h", h) ||
      arg_pos(fn, "w", w) || arg_pos(fn, "Ho", Ho) || arg_pos(fn, "Wo", Wo) ||
      arg_max(fn, "ceil(Hp/8)", (static_cast<long long>(Hp) + 7) / 8, kGridYZ))
    return -1;
  if (Hp < Ho) return set_error("%s: Hp=%d must be >= Ho=%d", fn, Hp, Ho), -1;
  if (Wp < Wo) return set_error("%s: Wp=%d must be >= Wo=%d", fn, Wp, Wo), -1;
  if (ensure_init()) return -1;
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

int lseg_debug_gemm_plan(const lseg_gemm_args* a, int out[5]) {
  GemmDesc d;
  if (gemm_desc_of(a, d)) return -1;
  GemmPlan plan;
  if (gemm_plan(d, &plan)) return -1;
  out[0] = plan.epi;
  out[1] = plan.grid;
  out[2] = plan.p.split_k;
  out[3] = plan.p.split_fixed;
  out[4] = gemm_kernel_of(plan);
  return 0;
}

int lseg_debug_gemm_cluster(const lseg_gemm_args* a, int out[2]) {
  GemmDesc d;
  if (gemm_desc_of(a, d)) return -1;
  GemmPlan plan;
  if (gemm_plan(d, &plan)) return -1;
  out[0] = plan.cluster;
  out[1] = plan.grid / plan.cluster;
  return 0;
}

int lseg_debug_set_gemm_cluster(int mode) {
  if (mode < 1 || mode > 3) {
    set_error("debug_set_gemm_cluster: mode must be 1, 2 or 3, got %d", mode);
    return -1;
  }
  if (ensure_init()) return -1;
  if (mode != g_gemm_cluster_mode) ++g_plan_epoch;
  g_gemm_cluster_mode = mode;
  return 0;
}

int lseg_debug_set_trace_block(int block) {
  if (block < -1) {
    set_error("debug_set_trace_block: block must be -1 (off) or a trunk block index, got %d", block);
    return -1;
  }
  if (block != g_trace_block) ++g_plan_epoch;
  g_trace_block = block;
  return 0;
}

int lseg_debug_gemm_trace(unsigned long long* trace) {
  g_gemm_trace = trace;
  return 0;
}

int lseg_mhsa_trace(const void* qkv, void* out, int B, int N, int heads, int causal, unsigned long long* trace,
                    void* stream) {
  if (!trace) {
    set_error("mhsa_trace: trace pointer is null");
    return -1;
  }
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
  const char* fn = "lseg_layernorm";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "gamma", gamma, 16) || arg_ptr(fn, "beta", beta, 16) ||
      arg_ptr(fn, "y", y, 16) || arg_pos(fn, "M", M) || arg_max(fn, "M / 8 blocks", (M + 7) / 8, kGridX))
    return -1;
  if (C != 512 && C != 768 && C != 1024) return set_error("%s: C=%d must be 512, 768 or 1024", fn, C), -1;
  if (ensure_init()) return -1;
  return run_layernorm(x, in_f16, gamma, beta, static_cast<__half*>(y), M, C, eps, static_cast<cudaStream_t>(stream));
}

int lseg_patchify(const float* x, void* a, int B, int H, int W, int patch, void* stream) {
  const char* fn = "lseg_patchify";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "a", a, 8) || arg_pos(fn, "B", B) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_pos(fn, "patch", patch) ||
      arg_max(fn, "B*(H/patch)", static_cast<long long>(B) * (H / patch), kGridYZ))
    return -1;
  if (patch != 16 && patch != 32) return set_error("%s: patch=%d must be 16 or 32", fn, patch), -1;
  if (arg_mult(fn, "H", H, patch) || arg_mult(fn, "W", W, patch)) return -1;
  if (ensure_init()) return -1;
  return launch_patchify(x, static_cast<__half*>(a), B, H, W, patch, static_cast<cudaStream_t>(stream));
}

int lseg_pos_resize(const float* pos, float* out, int g0, int gh, int gw, int D, void* stream) {
  const char* fn = "lseg_pos_resize";
  if (arg_ptr(fn, "pos", pos, 4) || arg_ptr(fn, "out", out, 4) || arg_pos(fn, "g0", g0) || arg_pos(fn, "gh", gh) ||
      arg_pos(fn, "gw", gw) || arg_pos(fn, "D", D) ||
      arg_max(fn, "1 + gh*gw", 1 + static_cast<long long>(gh) * gw, kGridX))
    return -1;
  if (ensure_init()) return -1;
  pos_resize_kernel<<<1 + gh * gw, 256, 0, static_cast<cudaStream_t>(stream)>>>(pos, out, g0, gh, gw, D);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_assemble_tokens(const float* patch, const float* cls, const float* pos, float* x, int B, int T, int D,
                         void* stream) {
  const char* fn = "lseg_assemble_tokens";
  if (arg_ptr(fn, "patch", patch, 16) || arg_ptr(fn, "cls", cls, 16) || arg_ptr(fn, "pos", pos, 16) ||
      arg_ptr(fn, "x", x, 16) || arg_pos(fn, "B", B) || arg_pos(fn, "T", T) || arg_pos(fn, "D", D) ||
      arg_mult(fn, "D", D, 4) || arg_max(fn, "B*(T+1)", static_cast<long long>(B) * (T + 1), kGridX))
    return -1;
  if (ensure_init()) return -1;
  return launch_assemble_tokens(patch, cls, pos, x, B, T, D, static_cast<cudaStream_t>(stream));
}

int lseg_readout_split(const float* tap, void* tok, void* cls, int B, int T, int D, void* stream) {
  const char* fn = "lseg_readout_split";
  if (arg_ptr(fn, "tap", tap, 16) || arg_ptr(fn, "tok", tok, 8) || arg_ptr(fn, "cls", cls, 8) || arg_pos(fn, "B", B) ||
      arg_pos(fn, "T", T) || arg_pos(fn, "D", D) || arg_mult(fn, "D", D, 4) ||
      arg_max(fn, "B*(T+1)", static_cast<long long>(B) * (T + 1), kGridX))
    return -1;
  if (ensure_init()) return -1;
  return launch_readout_split(tap, static_cast<__half*>(tok), static_cast<__half*>(cls), B, T, D,
                              static_cast<cudaStream_t>(stream));
}

int lseg_im2col_3x3_s2(const void* x, void* a, int B, int H, int W, int C, void* stream) {
  const char* fn = "lseg_im2col_3x3_s2";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "a", a, 16) || arg_pos(fn, "B", B) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_pos(fn, "C", C) || arg_mult(fn, "C", C, 8) || arg_max(fn, "B", B, kGridYZ) ||
      arg_max(fn, "Ho", (H - 1) / 2 + 1, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  return launch_im2col_3x3_s2(static_cast<const __half*>(x), static_cast<__half*>(a), B, H, W, C,
                              static_cast<cudaStream_t>(stream));
}

int lseg_stem_im2col(const float* x, void* a, int B, int H, int W, void* stream) {
  const char* fn = "lseg_stem_im2col";
  if (arg_ptr(fn, "x", x, 4) || arg_ptr(fn, "a", a, 2) || arg_pos(fn, "B", B) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_max(fn, "B*(H/2)*(W/2)", static_cast<long long>(B) * (H / 2) * (W / 2), kGridX) ||
      arg_mult(fn, "H", H, 2) || arg_mult(fn, "W", W, 2))
    return -1;
  if (ensure_init()) return -1;
  return launch_stem_im2col(x, static_cast<__half*>(a), B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_maxpool3x3s2_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  const char* fn = "lseg_maxpool3x3s2_nhwc";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 16) || arg_pos(fn, "B", B) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_pos(fn, "C", C) || arg_max(fn, "B", B, kGridYZ) || arg_mult(fn, "C", C, 8) ||
      arg_mult(fn, "H", H, 2) || arg_mult(fn, "W", W, 2))
    return -1;
  if (ensure_init()) return -1;
  return launch_maxpool3x3s2_nhwc(static_cast<const __half*>(x), static_cast<__half*>(y), B, H, W, C,
                                  static_cast<cudaStream_t>(stream));
}

int lseg_subsample2_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  const char* fn = "lseg_subsample2_nhwc";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 16) || arg_pos(fn, "B", B) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_pos(fn, "C", C) || arg_max(fn, "B", B, kGridYZ) || arg_mult(fn, "C", C, 8) ||
      arg_mult(fn, "H", H, 2) || arg_mult(fn, "W", W, 2))
    return -1;
  if (ensure_init()) return -1;
  return launch_subsample2_nhwc(static_cast<const __half*>(x), static_cast<__half*>(y), B, H, W, C,
                                static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream) {
  const char* fn = "lseg_upsample2x_nhwc";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 16) || arg_pos(fn, "B", B) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_pos(fn, "C", C) || arg_mult(fn, "C", C, 8) || arg_max(fn, "B", B, kGridYZ) ||
      arg_max(fn, "2H", 2LL * H, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  return launch_upsample2x_nhwc(static_cast<const __half*>(x), static_cast<__half*>(y), B, H, W, C,
                                static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_nhwc256(const void* x, int in_f16, void* y, int out_f16, const float* add, int B, int H, int W,
                            void* stream) {
  const char* fn = "lseg_upsample2x_nhwc256";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 16) || (add && arg_ptr(fn, "add", add, 16)) ||
      arg_pos(fn, "B", B) || arg_pos(fn, "H", H) || arg_pos(fn, "W", W) || arg_max(fn, "B", B, kGridYZ) ||
      arg_max(fn, "2H", 2LL * H, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  if (add && out_f16) return set_error("%s: add (the skip operand) needs an fp32 output (out_f16=0)", fn), -1;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (in_f16) {
    if (out_f16) return launch_upsample2x_nhwc256_f16<__half>(static_cast<const __half*>(x), static_cast<__half*>(y), nullptr, B, H, W, s);
    return launch_upsample2x_nhwc256_f16<float>(static_cast<const __half*>(x), static_cast<float*>(y), add, B, H, W, s);
  }
  if (out_f16) return launch_upsample2x_nhwc256_f32<__half>(static_cast<const float*>(x), static_cast<__half*>(y), nullptr, B, H, W, s);
  return launch_upsample2x_nhwc256_f32<float>(static_cast<const float*>(x), static_cast<float*>(y), add, B, H, W, s);
}

int lseg_l2norm_scale(const float* x, void* y, long long M, int C, float logit_scale, void* stream) {
  const char* fn = "lseg_l2norm_scale";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 8) || arg_pos(fn, "M", M) || arg_pos(fn, "C", C) ||
      arg_max(fn, "M / 8 blocks", (M + 7) / 8, kGridX) || arg_mult(fn, "C", C, 128) || arg_max(fn, "C", C, 512))
    return -1;
  if (ensure_init()) return -1;
  const int grid = static_cast<int>((M + 7) / 8);
  l2norm_scale_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, static_cast<__half*>(y), M, C,
                                                                           logit_scale);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_l2norm_f16(const void* x, void* y, int M, int C, void* stream) {
  const char* fn = "lseg_l2norm_f16";
  if (arg_ptr(fn, "x", x, 2) || arg_ptr(fn, "y", y, 2) || arg_pos(fn, "M", M) || arg_pos(fn, "C", C)) return -1;
  if (ensure_init()) return -1;
  l2norm_f16_kernel<<<(M + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __half*>(x),
                                                                               static_cast<__half*>(y), M, C);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_upsample2x_nchw(const void* x, float* y, long long planes, int H, int W, void* stream) {
  const char* fn = "lseg_upsample2x_nchw";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 16) || arg_pos(fn, "planes", planes) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_up_w(fn, W) || arg_max(fn, "planes", planes, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  return launch_upsample2x_nchw(static_cast<const __half*>(x), y, planes, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_debug_upsample_layout(int split) {
  const int old = g_upsample_split;
  g_upsample_split = split ? 1 : 0;
  return old;
}

int lseg_upsample2x_nchw_bg(const void* x, float* y, long long planes, int H, int W, void* stream) {
  const char* fn = "lseg_upsample2x_nchw_bg";
  if (arg_ptr(fn, "x", x, 2) || arg_ptr(fn, "y", y, 16) || arg_pos(fn, "planes", planes) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_mult(fn, "W", W, 2) || arg_max(fn, "planes", planes, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  return launch_upsample2x_nchw_bg(static_cast<const __half*>(x), y, planes, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_upsample2x_nchw_f32(const float* x, float* y, long long planes, int H, int W, void* stream) {
  const char* fn = "lseg_upsample2x_nchw_f32";
  if (arg_ptr(fn, "x", x, 16) || arg_ptr(fn, "y", y, 16) || arg_pos(fn, "planes", planes) || arg_pos(fn, "H", H) ||
      arg_pos(fn, "W", W) || arg_up_w(fn, W) || arg_max(fn, "planes", planes, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  return launch_upsample2x_nchw(x, y, planes, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_head_block(const void* x, int in_f16, float* cmax_ws, float* y, int B, int K, int h, int w, const float* w9_host,
                    float bias, int mode, int act, void* stream) {
  const char* fn = "lseg_head_block";
  if (arg_ptr(fn, "x", x, in_f16 ? 2 : 4) || arg_ptr(fn, "y", y, 4) || arg_ptr(fn, "w9", w9_host, 4)) return -1;
  if (mode != 1 && mode != 2) return set_error("%s: mode=%d must be 1 or 2", fn, mode), -1;
  if (act < HEAD_ACT_NONE || act > HEAD_ACT_TANH) return set_error("%s: act=%d must be 0..3", fn, act), -1;
  if ((mode == 1 && arg_ptr(fn, "cmax_ws", cmax_ws, 4)) || arg_pos(fn, "B", B) || arg_pos(fn, "K", K) ||
      arg_pos(fn, "h", h) || arg_pos(fn, "w", w) || arg_max(fn, "ceil(h/8)", (h + 7) / 8, kGridYZ) ||
      arg_max(fn, "B", B, kGridYZ) || arg_max(fn, "B*K", static_cast<long long>(B) * K, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
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
  const char* fn = "lseg_upsample2x_argmax";
  if (arg_ptr(fn, "lr", lr, 16) || arg_ptr(fn, "mask", mask, 8) || arg_pos(fn, "B", B) || arg_pos(fn, "K", K) ||
      arg_pos(fn, "H", H) || arg_pos(fn, "W", W) || arg_up_w(fn, W) || arg_max(fn, "B", B, kGridYZ))
    return -1;
  if (ensure_init()) return -1;
  return launch_upsample2x_argmax(static_cast<const __half*>(lr), mask, B, K, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_seg_stats_scores(const float* scores, const long long* target, const int* group, int B, int K, int H, int W,
                          int nclass, int G, long long* stats, void* stream) {
  if (ensure_init()) return -1;
  return launch_seg_stats_scores(scores, B, K, H, W, SegStatsArgs{target, group, stats, nclass, G},
                                 static_cast<cudaStream_t>(stream));
}

int lseg_seg_stats_mask(const long long* pred, const long long* target, const int* group, int B, int H, int W, int nclass,
                        int G, long long* stats, void* stream) {
  if (ensure_init()) return -1;
  return launch_seg_stats_mask(pred, B, H, W, SegStatsArgs{target, group, stats, nclass, G},
                               static_cast<cudaStream_t>(stream));
}

int lseg_xent_scores(const float* scores, const long long* target, long long ignore_index, int B, int K, int H, int W,
                     double* loss, double* partials, long long partials_len, void* stream) {
  if (ensure_init()) return -1;
  return launch_xent_scores(scores, B, K, H, W, XentArgs{target, ignore_index, partials, loss}, partials_len,
                            static_cast<cudaStream_t>(stream));
}

int lseg_text_embed(const int64_t* tokens, const float* tok_emb, const float* pos_emb, void* x, int K, int L, int Wd,
                    void* stream) {
  const char* fn = "lseg_text_embed";
  if (arg_ptr(fn, "tokens", tokens, 8) || arg_ptr(fn, "tok_emb", tok_emb, 4) || arg_ptr(fn, "pos_emb", pos_emb, 4) ||
      arg_ptr(fn, "x", x, 2) || arg_pos(fn, "K", K) || arg_pos(fn, "L", L) || arg_pos(fn, "Wd", Wd) ||
      arg_max(fn, "K*L", static_cast<long long>(K) * L, kGridX))
    return -1;
  if (ensure_init()) return -1;
  text_embed_kernel<<<K * L, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(tokens), tok_emb, pos_emb, static_cast<__half*>(x), L, Wd);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int lseg_text_eot_gather(const int64_t* tokens, const void* x, void* out, int K, int L, int Wd, void* stream) {
  const char* fn = "lseg_text_eot_gather";
  if (arg_ptr(fn, "tokens", tokens, 8) || arg_ptr(fn, "x", x, 2) || arg_ptr(fn, "out", out, 2) || arg_pos(fn, "K", K) ||
      arg_pos(fn, "L", L) || arg_pos(fn, "Wd", Wd))
    return -1;
  if (ensure_init()) return -1;
  text_eot_gather_kernel<<<K, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(tokens), static_cast<const __half*>(x), static_cast<__half*>(out), K, L, Wd);
  LSEG_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
