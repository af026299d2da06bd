// lseg_b200 — shared device helpers for the sm_90a kernels.
//
// Thin inline-PTX wrappers (mbarrier, TMA, wgmma), shared-memory matrix descriptors and the host-side
// tensor-map factory. Everything here is written for sm_90a (Hopper) only; there is no fallback path.
#pragma once
#include <cstdlib>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace lseg {

// ------------------------------------------------------------------------------------------
// Device-side watchdog: a barrier wait that exceeds kWatchdogCycles records (tag, block, role)
// in g_watchdog and makes every later wait in the grid fall through, so a protocol bug shows
// up as a reported error code instead of a hung GPU box.
// ------------------------------------------------------------------------------------------
constexpr long long kWatchdogCycles = 1ll << 31;  // ~1 s at 1.9 GHz
__device__ int g_watchdog[4];                     // [0]=tag (0 = ok), [1]=blockIdx.x, [2]=threadIdx.x, [3]=parity

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ----------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// suspend-time hint: the waiting thread sleeps in hardware until the phase completes or this many ns
// pass, instead of re-polling every ~100 cycles and stealing issue slots from the compute warps that
// share its SM sub-partition.
constexpr uint32_t kTryWaitHintNs = 20000;
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(kTryWaitHintNs)
      : "memory");
  return ok != 0;
}
// Non-blocking phase test (for a thread that multiplexes several barriers), and a try_wait whose hardware
// suspend is bounded by `ns` instead of kTryWaitHintNs.
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ bool mbar_try_wait_ns(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
__device__ __noinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity, int tag) {
  // try_wait suspends the thread in hardware for a bounded time, so this loop is not a hot spin.
  // The watchdog bookkeeping (a global-memory flag read, ~1 us) runs only every 256 failed polls so
  // that it never sits on the critical path of a healthy pipeline.
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++polls & 0xFFu) != 0) continue;
    if (*reinterpret_cast<volatile int*>(&g_watchdog[0]) != 0) return;
    if (clock64() - t0 > kWatchdogCycles) {
      if (atomicCAS(&g_watchdog[0], 0, tag) == 0) {
        g_watchdog[1] = blockIdx.x;
        g_watchdog[2] = threadIdx.x;
        g_watchdog[3] = static_cast<int>(parity);
      }
      return;
    }
  }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag) {
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity, tag);
}
// Fully inlined wait (hinted try_wait): for waits that sit between long-lived register state — the out-of-line
// mbar_wait_slow is a real call, and live registers around it are spilled per the ABI.
__device__ __forceinline__ void mbar_wait_inl(uint64_t* bar, uint32_t parity, int tag) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++polls & 0xFFu) != 0) continue;
    if (*reinterpret_cast<volatile int*>(&g_watchdog[0]) != 0) return;
    if (clock64() - t0 > kWatchdogCycles) {
      if (atomicCAS(&g_watchdog[0], 0, tag) == 0) {
        g_watchdog[1] = blockIdx.x;
        g_watchdog[2] = threadIdx.x;
        g_watchdog[3] = static_cast<int>(parity);
      }
      return;
    }
  }
}
// Latency-critical variant: try_wait WITHOUT a suspend-time hint (the hardware re-checks after its short
// default window instead of parking the thread), for waits that sit on a kernel's critical path.
__device__ __forceinline__ bool mbar_try_wait_spin(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity, int tag) {
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait_spin(bar, parity)) {
    if ((++polls & 0xFFFu) != 0) continue;
    if (*reinterpret_cast<volatile int*>(&g_watchdog[0]) != 0) return;
    if (clock64() - t0 > kWatchdogCycles) {
      if (atomicCAS(&g_watchdog[0], 0, tag) == 0) {
        g_watchdog[1] = blockIdx.x;
        g_watchdog[2] = threadIdx.x;
        g_watchdog[3] = static_cast<int>(parity);
      }
      return;
    }
  }
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------
// Every per-step kernel is launched with programmaticStreamSerializationAllowed: its CTAs may become resident and
// run their prologue (barrier init, tensor-map prefetch) while the previous kernel of the stream is
// still draining. griddep_wait() blocks until that previous grid has completed and its writes are visible; it
// must precede the first access to any global memory another kernel of the step reads or writes.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// One lane of a converged warp (elect.sync): the MMA / TMA warps run converged with warp-uniform values (which the
// compiler then keeps in uniform registers) and only predicate the bulk-copy instruction itself on this
// — a `if (lane == 0) { ... }` region makes every descriptor operand go through an ELECT + R2UR waterfall
// (~20 dependent instructions per issue).
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ int warp_idx_sync() { return __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0); }


// ---- proxies / fences --------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (TMA stores / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA ---------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::
          "r"(smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA stores: smem tile -> global through a tensor map (clips rows/columns outside the tensor).
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(m),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// global[tile] += smem tile, performed by the TMA unit at L2 (element type from the tensor map: fp32)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(m),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their smem source
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- wgmma (warpgroup MMA) -----------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle (layout type 1 at bits [62,64)); addresses / offsets are encoded
// >>4. Tiles are 1024 B aligned (the 8-row swizzle atom), so the base-offset field stays 0.
//   K-major operand (rows of 64 halves = 128 B, as TMA writes a {64, rows} box): SBO = 1024 B between 8-row groups,
//   LBO unused; the k-th 16-element K slice starts k * 32 B into the tile.
//   MN-major operand (128 B along MN per K index, i.e. a row-major [K, 64] tile): SBO = 1024 B between 8-k groups,
//   LBO = byte stride between 64-element MN chunks; the k-th 16-row K slice starts k * 2048 B into the tile.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// Ordering of the accumulator registers against the asynchronous MMAs of this warpgroup.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across an MMA that is still in flight.
template <int N>
__device__ __forceinline__ void wgmma_reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] (smem) * B[128 x 16]^T (smem), both K-major; fp16 in, fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 64] (+)= A[64 x 16] (smem) * B[64 x 16]^T (smem), both K-major; fp16 in, fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 64] (+)= A[64 x 16] (registers: fp16 pairs in the accumulator-fragment order) * B[16 x 64] (smem,
// MN-major: the 64 columns contiguous, as a row-major [K, N] tile); fp32 accumulate.
__device__ __forceinline__ void wgmma_m64n64k16_rs_bmn(float (&d)[32], const uint32_t (&a)[4], uint64_t db,
                                                       uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}

// ---- misc math ---------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx(float x);
// Exact-erf GELU, 0.5 x (1 + erf(x / sqrt 2)) (timm Mlp / ProjectReadout use nn.GELU()), with erf from
// 2^x on the FMA/ALU pipes (no MUFU): Cody-Waite split x = n + f, f in [-0.5, 0.5] via the 1.5*2^23 rounding trick,
// minimax polynomial for 2^f (tools/fit_exp2.py: relative error 7.5e-5 / 2.7e-6 / 2.3e-7 for degree 3 / 4 / 5),
// exponent added by integer arithmetic on the bit pattern: ~9 issue slots instead of one MUFU instruction. Used by
// the attention variants that move part of the softmax exponentials off the MUFU pipe (lseg_mhsa_variant 3/4/7/8).
// Requires -126 <= x <= 126 (the callers clamp).
template <int DEG>
__device__ __forceinline__ float exp2_poly(float x) {
  const float r = x + 12582912.f;  // 1.5 * 2^23: the low mantissa bits of r now hold round(x)
  const float f = x - (r - 12582912.f);
  float p;
  if (DEG == 3) {
    p = fmaf(f, 5.517166885e-02f, 2.426111221e-01f);
    p = fmaf(p, f, 6.932609855e-01f);
    p = fmaf(p, f, 9.999280736e-01f);
  } else if (DEG == 4) {
    p = fmaf(f, 9.570101897e-03f, 5.591786033e-02f);
    p = fmaf(p, f, 2.402474483e-01f);
    p = fmaf(p, f, 6.931218147e-01f);
    p = fmaf(p, f, 9.999992614e-01f);
  } else {
    p = fmaf(f, 1.327647190e-03f, 9.675541334e-03f);
    p = fmaf(p, f, 5.550713274e-02f);
    p = fmaf(p, f, 2.402211972e-01f);
    p = fmaf(p, f, 6.931469671e-01f);
    p = fmaf(p, f, 1.000000072e+00f);
  }
  return __int_as_float(__float_as_int(p) + (__float_as_int(r) << 23));
}

// Exact-erf GELU x * Phi(x) with Phi(x) = 1 / (1 + 2^(x * P(x^2))): P is a degree-4 minimax fit (tools/fit_gelu.py:
// reweighted least squares against scipy erfc on [-7, 7], coefficients carry the -log2(e)); |gelu error| <= 3.7e-6 over
// all x in fp32 arithmetic, i.e. below the fp16 rounding of the stored activation wherever that activation is
// not already in fp16's subnormal range. 10 issue slots (2 MUFU) instead of the 20 of the Abramowitz-Stegun
// 7.1.26 form used before (the fc1 epilogue is issue-bound). P(u) < 0 for all u >= 0, so the sigmoid saturates
// monotonically outside the fitted range.
__device__ __forceinline__ float gelu_erf(float x) {
  const float u = x * x;
  float p = fmaf(u, -3.228989445e-06f, 8.823814435e-05f);
  p = fmaf(p, u, 3.602744768e-04f);
  p = fmaf(p, u, -1.052266877e-01f);
  p = fmaf(p, u, -2.302045391e+00f);
  const float e = ex2_approx(x * p);
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}
// CLIP QuickGELU evaluated the way the fp16 reference does it: h = half(x); half(1.702*h);
// half(sigmoid(.)); half(h * .)  (x * torch.sigmoid(1.702 * x) on a HalfTensor).
__device__ __forceinline__ float quick_gelu(float x) {
  const float h = __half2float(__float2half_rn(x));
  const float t = __half2float(__float2half_rn(1.702f * h));
  const float s = __half2float(__float2half_rn(1.0f / (1.0f + __expf(-t))));
  return h * s;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
// Thread-local last-error string surfaced through lseg_last_error().
void set_error(const char* fmt, ...);
const char* get_error();

#define LSEG_CHECK_CUDA(expr)                                                                  \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::lseg::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)

// Kernel launch with the PDL attribute (see griddep_wait above); LSEG_NO_PDL=1 falls back to plain launches.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args&&... args) {
  static const bool no_pdl = getenv("LSEG_NO_PDL") != nullptr;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = no_pdl ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Encode a tiled fp16 tensor map (rank 2..4), 128-byte swizzle, zero OOB fill.
// dims/box are innermost-first, strides_bytes[i] is the byte stride of dim i+1.
int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);

int read_watchdog(int out[4], cudaStream_t stream);  // also clears it

}  // namespace lseg
