// lseg_b200 — whole-model orchestration: LSeg.forward (modules/models/lseg_net.py:160-205) and
// CLIP encode_text (SURVEY.md Appendix A.2) as a static list of kernel launches over a bump-allocated
// HBM workspace. Plans (TMA descriptors, grids) are built once per input shape and replayed; nothing
// here touches the host between launches, so a forward is ~290 back-to-back async launches on one stream.
//
// Data layout in HBM (all activations stay resident for the whole forward):
//   residual stream      fp32 [B*N, 1024]   (taps of blocks 5/11/17/23 are separate fp32 buffers)
//   GEMM operands        fp16 row-major, K contiguous (tokens) / NHWC (decoder feature maps)
//   decoder residuals    fp32 NHWC
//   low-res logits       fp16 [B, K, H/2, W/2]; final logits fp32 NCHW [B, K, H, W]
#pragma once
#include <functional>
#include <map>
#include <memory>
#include <tuple>

namespace lseg {

struct CallCtx {
  const float* x;
  const __half* text;
  int K;
  long long text_image_stride;
  float* out;            // fp32 logits [B,K,H,W], or nullptr when only the mask / the low-res logits are wanted
  long long* out_mask;   // optional int64 class mask [B,H,W] (fused upsample + argmax)
  __half* out_lr;        // optional target of the fp16 low-res logits [B,K,H/2,W/2] (the exact result of the reference's
                         // fp16 matmul, lseg_net.py:194-196) instead of the plan's own buffer; may be PEER memory — the
                         // pixel x text GEMM then stores straight into another GPU's gather buffer over NVLink
  const SegStatsArgs* seg = nullptr;  // optional metric counters, fused with the argmax output stage (out_mask optional)
  const XentArgs* xent = nullptr;     // optional cross-entropy, fused with the same stage (seg and out_mask optional)
  // ragged batch (lseg_forward_ragged / lseg_query_ragged): image b's rag_k[b] labels are rows rag_text_row[b] .. of
  // `text` (rag_text_rows readable rows); K is then the sum of rag_k, and the logits / low-res planes are packed by image
  const int* rag_k = nullptr;
  const int* rag_text_row = nullptr;
  int rag_text_rows = 0;
  // lseg_encode_image_attention: attn[k] receives the attention probabilities of block hooks[k], fp32 [B, heads, N, N]
  // (read only by the steps of a plan built with ImagePlan::attn)
  float* const* attn = nullptr;
};
using StepFn = std::function<int(const CallCtx&, cudaStream_t)>;
enum StepKind { KIND_EW = 0, KIND_GEMM = 1, KIND_MHSA = 2, KIND_LN = 3, KIND_MEMSET = 4 };
// One launch of the forward: the closure plus what bench.py's roofline needs (kernel class and
// the ALGORITHMIC flops of this launch, 2*M*N*K for GEMMs, 4*N^2*dh per head for attention).
struct Step {
  StepFn fn;
  int kind = KIND_EW;
  double flops = 0.0;
  Step() {}
  template <class F, class = typename std::enable_if<!std::is_same<typename std::decay<F>::type, Step>::value>::type>
  Step(F&& f, int kind_ = KIND_EW, double flops_ = 0.0) : fn(std::forward<F>(f)), kind(kind_), flops(flops_) {}
  int operator()(const CallCtx& c, cudaStream_t s) const { return fn(c, s); }
};

struct Arena {
  // Bump allocator over a few large cudaMalloc'd slabs: a plan makes ~60 allocations, which as individual
  // cudaMalloc / cudaFree calls cost a device-wide synchronisation each when a plan is rebuilt.
  static constexpr size_t kSlab = size_t(512) << 20;
  std::vector<void*> slabs;
  uint8_t* cur = nullptr;
  size_t left = 0;
  size_t total = 0;
  void* alloc(size_t bytes) {
    bytes = (bytes + 1023) & ~size_t(1023);  // 1024 B: swizzled TMA tiles / tensor-map bases stay aligned
    if (bytes > left) {
      const size_t want = bytes > kSlab ? bytes : kSlab;
      void* p = nullptr;
      if (cudaMalloc(&p, want) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
      }
      slabs.push_back(p);
      total += want;
      if (bytes > kSlab) return p;  // oversized request: its own slab, the current one keeps its remainder
      cur = static_cast<uint8_t*>(p);
      left = want;
    }
    void* r = cur;
    cur += bytes;
    left -= bytes;
    return r;
  }
  void release() {
    for (void* p : slabs) cudaFree(p);
    slabs.clear();
    cur = nullptr;
    left = 0;
    total = 0;
  }
};

struct ImagePlan {
  int B = 0, H = 0, W = 0;
  int epoch = 0;  // g_plan_epoch at build time (options baked into the GEMM plans)
  bool attn = false;  // records the hooked blocks' attention probabilities into CallCtx::attn (one step per hooked block)
  Arena arena;
  std::vector<Step> steps;  // the trunk up to (not including) head1
  std::map<std::string, const void*> debug;
  // head1 (lseg_net.py:185): path1 -> the pixel embedding. forward writes the plan's own featn / feat_sumsq;
  // lseg_encode_image writes a caller's buffers, with one GEMM plan (host-encoded tensor maps) per destination
  GemmDesc head1_desc;
  float* head1_ws = nullptr;  // split-K workspace of head1 (shared by its plans: calls on an engine are stream-ordered)
  std::map<std::pair<const void*, const void*>, GemmPlan> head1;
  __half* featn = nullptr;
  float* feat_sumsq = nullptr;
  unsigned long long last_use = 0;
  ~ImagePlan() { arena.release(); }
};

// Buffers of the label-dependent tail at one (B, H, W): independent of the trunk's activation arena, so a query on a
// stored embedding at a shape the engine never ran a forward at allocates only these.
struct TailWs {
  int B = 0, H = 0, W = 0;
  int epoch = 0;  // g_plan_epoch of the cached pixel x text plans
  __half* logits_lr = nullptr;  // fp16 [B,K,H/2,W/2], grows with K
  size_t logits_cap_k = 0;
  float* head_ws[2] = {nullptr, nullptr};  // arch_option 1/2: fp32 [B,K,h,w] ping-pong, grows with K
  float* head_cmax = nullptr;              // [B,h,w]
  size_t head_cap_k = 0;
  // pixel x text GEMM plans (host-encoded tensor maps) keyed by (text pointer, K, per-image stride, output pointer,
  // embedding pointers, and for a ragged batch its text row count and k / text_row vectors)
  struct CorrKey {
    const void* text;
    int K;
    long long stride;
    const void* out;
    const void* emb;
    const void* sumsq;
    std::vector<int> rag;
    bool operator<(const CorrKey& o) const {
      return std::tie(text, K, stride, out, emb, sumsq, rag) < std::tie(o.text, o.K, o.stride, o.out, o.emb, o.sumsq, o.rag);
    }
  };
  std::map<CorrKey, std::vector<std::pair<GemmPlan, double>>> corr;
  unsigned long long last_use = 0;
  ~TailWs() {
    if (logits_lr) cudaFree(logits_lr);
    for (float* p : head_ws)
      if (p) cudaFree(p);
    if (head_cmax) cudaFree(head_cmax);
  }
};

struct TextPlan {
  int K = 0;
  Arena arena;
  std::vector<std::function<int(const long long*, __half*, cudaStream_t)>> steps;
  ~TextPlan() { arena.release(); }
};

}  // namespace lseg

struct lseg_engine {
  lseg_weights w;
  int device = 0;
  // a few image plans, least-recently-used eviction: the multi-scale evaluator alternates between its full batch and
  // the last partial one, the zero-shot and the ADE nets share an engine, ...
  static constexpr int kMaxImagePlans = 3;
  std::vector<std::unique_ptr<lseg::ImagePlan>> plans;
  lseg::ImagePlan* img = nullptr;  // the plan of the last forward (debug buffers)
  static constexpr int kMaxTails = 3;
  std::vector<std::unique_ptr<lseg::TailWs>> tails;  // least-recently-used, like the image plans
  unsigned long long use_counter = 0;
  std::unique_ptr<lseg::TextPlan> txt;
  std::map<std::pair<int, int>, float*> pos_cache;
  int last_launches = 0;
};

namespace lseg {

#define LSEG_ALLOC(var, type, count)                                                        \
  type* var = static_cast<type*>(arena.alloc(sizeof(type) * static_cast<size_t>(count)));   \
  if (!var) {                                                                               \
    set_error("workspace allocation of %zu bytes failed", sizeof(type) * (size_t)(count));  \
    return -1;                                                                              \
  }

// Arena of the plan under construction: split-K GEMMs (gemm_plan -> ws_bytes) take their partial-sum workspace from it.
static thread_local Arena* t_plan_arena = nullptr;
static int plan_workspace(GemmPlan* plan) {
  if (!plan->ws_bytes) return 0;
  float* ws = t_plan_arena ? static_cast<float*>(t_plan_arena->alloc(plan->ws_bytes)) : nullptr;
  if (!ws) {
    set_error("split-K workspace allocation of %zu bytes failed", plan->ws_bytes);
    return -1;
  }
  gemm_set_workspace(plan, ws);
  return 0;
}

static GemmEpi epi_none() {
  GemmEpi e;
  memset(&e, 0, sizeof(e));
  return e;
}

// Build a plain GEMM step: A [M,K] (lda) x lin.w -> epilogue e.
static int add_gemm(std::vector<Step>& steps, const __half* a, long long lda, int a_rows, int M,
                    const lseg_linear_w& lin, const GemmEpi& e) {
  GemmDesc d;
  memset(&d, 0, sizeof(d));
  d.a = a;
  d.lda = lda;
  d.a_rows = a_rows;
  d.w = static_cast<const __half*>(lin.w);
  d.w_rows = lin.rows;
  d.M = M;
  d.N = lin.out;
  d.K = lin.in;
  d.e = e;
  GemmPlan plan;
  if (gemm_plan(d, &plan) || plan_workspace(&plan)) return -1;
  steps.emplace_back([plan](const CallCtx&, cudaStream_t s) { return gemm_run(plan, s); }, KIND_GEMM,
                     2.0 * M * lin.out * lin.in);
  return 0;
}

// 3x3 stride-1 pad-1 conv over NHWC fp16 [B,H,W,C] with tap-major weights [N, 9*C].
static int add_conv3x3(std::vector<Step>& steps, const __half* a, int B, int H, int W, int C,
                       const lseg_linear_w& lin, const GemmEpi& e) {
  GemmDesc d;
  memset(&d, 0, sizeof(d));
  d.a = a;
  d.w = static_cast<const __half*>(lin.w);
  d.w_rows = lin.rows;
  d.M = B * H * W;
  d.N = lin.out;
  d.K = C;
  d.conv = 1;
  d.B = B;
  d.H = H;
  d.W = W;
  d.kh = d.kw = 3;
  d.pad = 1;
  d.e = e;
  GemmPlan plan;
  if (gemm_plan(d, &plan) || plan_workspace(&plan)) return -1;
  steps.emplace_back([plan](const CallCtx&, cudaStream_t s) { return gemm_run(plan, s); }, KIND_GEMM,
                     2.0 * B * H * W * lin.out * 9.0 * C);
  return 0;
}

static int add_layernorm(std::vector<Step>& steps, const void* x, int in_f16, const float* g, const float* b,
                         __half* y, long long M, int C, float eps) {
  steps.emplace_back([=](const CallCtx&, cudaStream_t s) { return run_layernorm(x, in_f16, g, b, y, M, C, eps, s); },
                     KIND_LN, 0.0);
  return 0;
}

// ResidualConvUnit_custom (modules/models/lseg_blocks.py:265-288) on NHWC [B,h,w,256]:
//   in_relu = relu(x) fp16, x_f32 = x;   out = bn2(conv2(relu(bn1(conv1(in_relu))))) + x (+ skip)
static int add_rcu(std::vector<Step>& steps, const lseg_rcu_w& rw, const __half* in_relu, const float* x_f32,
                   const float* skip_f32, __half* tmp, int B, int h, int w, float* out_f32, __half* out_f16,
                   __half* out_f16_relu) {
  GemmEpi e1 = epi_none();
  e1.scale = rw.bn1_scale;
  e1.bias = rw.bn1_shift;
  e1.act = ACT_RELU;
  e1.out_f16 = tmp;
  e1.ldc = 256;
  if (add_conv3x3(steps, in_relu, B, h, w, 256, rw.conv1, e1)) return -1;
  GemmEpi e2 = epi_none();
  e2.scale = rw.bn2_scale;
  e2.bias = rw.bn2_shift;
  e2.res_f32 = x_f32;
  e2.res2_f32 = skip_f32;
  e2.out_f32 = out_f32;
  e2.out_f16 = out_f16;
  e2.out_f16_relu = out_f16_relu;
  e2.ldc = 256;
  return add_conv3x3(steps, tmp, B, h, w, 256, rw.conv2, e2);
}

// Block trace (lseg_debug_set_trace_block): a device-to-device copy of `bytes` at `src`, taken at this point of the
// plan, into a buffer of its own that the plan's debug map names `name`.
static int add_snapshot(ImagePlan* plan, const char* name, const void* src, size_t bytes) {
  void* dst = plan->arena.alloc(bytes);
  if (!dst) {
    set_error("workspace allocation of %zu bytes failed (trace buffer %s)", bytes, name);
    return -1;
  }
  plan->debug[name] = dst;
  plan->steps.emplace_back(
      [=](const CallCtx&, cudaStream_t s) {
        LSEG_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s));
        return 0;
      },
      KIND_MEMSET, 0.0);
  return 0;
}

static int get_pos_embed(lseg_engine* eng, int gh, int gw, cudaStream_t stream, const float** out) {
  auto key = std::make_pair(gh, gw);
  auto it = eng->pos_cache.find(key);
  if (it != eng->pos_cache.end()) {
    *out = it->second;
    return 0;
  }
  float* buf = nullptr;
  const int D = eng->w.vit_dim;
  LSEG_CHECK_CUDA(cudaMalloc(&buf, sizeof(float) * (1 + (size_t)gh * gw) * D));
  pos_resize_kernel<<<1 + gh * gw, 256, 0, stream>>>(eng->w.pos_embed, buf, eng->w.pos_grid, gh, gw, D);
  LSEG_CHECK_CUDA(cudaGetLastError());
  eng->pos_cache[key] = buf;
  *out = buf;
  return 0;
}

// ViT trunk + readout + reassemble: fills layer_in[k] (NHWC fp16 inputs of scratch.layerN_rn), their stored channel
// counts and sizes.
static int build_vit_trunk(lseg_engine* eng, ImagePlan* plan, int B, int H, int W, cudaStream_t stream,
                           __half* (&layer_in)[4], int (&c_post)[4], int (&lh)[4], int (&lw)[4]) {
  const lseg_weights& w = eng->w;
  Arena& arena = plan->arena;
  std::vector<Step>& steps = plan->steps;
  // backbone geometry (lseg_vit.py:442-522 _make_pretrained_clip_vitl16_384 / _vitb32_384): token width, depth, heads,
  // patch size and the per-level reassemble recipe come with the weights
  const int P = w.patch_size, D = w.vit_dim, heads = w.vit_heads;
  const int gh = H / P, gw = W / P, T = gh * gw, N = T + 1;
  const int patch_k = 3 * P * P;
  const long long M = static_cast<long long>(B) * N;
  const long long BT = static_cast<long long>(B) * T;

  const float* pos = nullptr;
  if (get_pos_embed(eng, gh, gw, stream, &pos)) return -1;

  // ---- ViT trunk (modules/models/lseg_vit.py:166-201) ----
  LSEG_ALLOC(patch_a, __half, BT * patch_k);
  LSEG_ALLOC(patch_out, float, BT * D);
  plan->debug["patch_out"] = patch_out;  // [B*T, D]
  LSEG_ALLOC(xbuf, float, M * D);
  LSEG_ALLOC(xn, __half, M * D);
  LSEG_ALLOC(qkv, __half, M * 3 * D);
  LSEG_ALLOC(attn, __half, M * D);
  LSEG_ALLOC(hbuf, __half, M * 4 * D);
  float* taps[4];
  for (int k = 0; k < 4; ++k) {
    LSEG_ALLOC(t, float, M * D);
    taps[k] = t;
    char name[8];
    snprintf(name, sizeof(name), "tap%d", k);
    plan->debug[name] = t;
  }

  steps.push_back([=](const CallCtx& c, cudaStream_t s) {
    return launch_patchify(c.x, patch_a, B, H, W, P, s);
  });
  {
    GemmEpi e = epi_none();
    e.bias = w.patch.b;
    e.out_f32 = patch_out;
    e.ldc = D;
    if (add_gemm(steps, patch_a, patch_k, (int)BT, (int)BT, w.patch, e)) return -1;
  }
  {
    const float* cls = w.cls_token;
    steps.push_back([=](const CallCtx&, cudaStream_t s) {
      return launch_assemble_tokens(patch_out, cls, pos, xbuf, B, T, D, s);
    });
  }
  for (int i = 0; i < w.vit_depth; ++i) {
    const lseg_vit_block_w& bw = w.blocks[i];
    // The residual stream lives in xbuf and both branch outputs are accumulated IN PLACE (x += proj(..),
    // x += fc2(..)): that lets the GEMM epilogue use a bulk tensor reduce-add and never read x. A hooked
    // block's output (lseg_vit.py:421-426: the hook captures the block's return value) is snapshotted into
    // its tap buffer with one device-to-device copy.
    const bool tr = i == g_trace_block;  // snapshot every intermediate of this block (lseg_debug_set_trace_block)
    const size_t x_bytes = sizeof(float) * M * D, h_bytes = sizeof(__half) * M * D;
    if (tr && add_snapshot(plan, "trace_in", xbuf, x_bytes)) return -1;
    add_layernorm(steps, xbuf, 0, bw.ln1_g, bw.ln1_b, xn, M, D, 1e-6f);
    if (tr && add_snapshot(plan, "trace_ln1", xn, h_bytes)) return -1;
    {
      GemmEpi e = epi_none();
      e.bias = bw.qkv.b;
      e.out_f16 = qkv;
      e.ldc = 3 * D;
      if (add_gemm(steps, xn, D, (int)M, (int)M, bw.qkv, e)) return -1;
    }
    if (tr && add_snapshot(plan, "trace_qkv", qkv, 3 * h_bytes)) return -1;
    {
      MhsaDesc md;
      md.qkv = qkv;
      md.out = attn;
      md.B = B;
      md.N = N;
      md.heads = heads;
      md.causal = 0;
      MhsaPlan mp;
      if (mhsa_plan(md, &mp)) return -1;
      steps.emplace_back([mp](const CallCtx&, cudaStream_t s) { return mhsa_run(mp, s); }, KIND_MHSA,
                         4.0 * B * heads * static_cast<double>(N) * N * 64);
    }
    if (tr && add_snapshot(plan, "trace_attn", attn, h_bytes)) return -1;
    for (int k = 0; k < 4 && plan->attn; ++k) {  // the hook reads this block's q, k (lseg_vit.py:22-42): qkv holds them
      if (w.hooks[k] != i) continue;             // until the next block's QKV GEMM overwrites it
      AttnProbsPlan ap;
      if (attn_probs_maps(qkv, B, N, heads, &ap)) return -1;
      steps.emplace_back(
          [ap, k](const CallCtx& c, cudaStream_t s) {
            AttnProbsPlan run = ap;
            run.p.out = c.attn[k];
            return attn_probs_run(run, s);
          },
          KIND_MHSA, 4.0 * B * heads * static_cast<double>(N) * N * 64);
    }
    {
      GemmEpi e = epi_none();
      e.bias = bw.proj.b;
      e.res_f32 = xbuf;
      e.out_f32 = xbuf;
      e.ldc = D;
      if (add_gemm(steps, attn, D, (int)M, (int)M, bw.proj, e)) return -1;
    }
    if (tr && add_snapshot(plan, "trace_x1", xbuf, x_bytes)) return -1;
    add_layernorm(steps, xbuf, 0, bw.ln2_g, bw.ln2_b, xn, M, D, 1e-6f);
    if (tr && add_snapshot(plan, "trace_ln2", xn, h_bytes)) return -1;
    {
      GemmEpi e = epi_none();
      e.bias = bw.fc1.b;
      e.act = ACT_GELU;
      e.out_f16 = hbuf;
      e.ldc = 4 * D;
      if (add_gemm(steps, xn, D, (int)M, (int)M, bw.fc1, e)) return -1;
    }
    if (tr && add_snapshot(plan, "trace_fc1", hbuf, 4 * h_bytes)) return -1;
    {
      GemmEpi e = epi_none();
      e.bias = bw.fc2.b;
      e.res_f32 = xbuf;
      e.out_f32 = xbuf;
      e.ldc = D;
      if (add_gemm(steps, hbuf, 4 * D, (int)M, (int)M, bw.fc2, e)) return -1;
    }
    if (tr && add_snapshot(plan, "trace_out", xbuf, x_bytes)) return -1;
    for (int k = 0; k < 4; ++k) {
      if (w.hooks[k] != i) continue;
      float* tap = taps[k];
      steps.emplace_back(
          [=](const CallCtx&, cudaStream_t s) {
            LSEG_CHECK_CUDA(cudaMemcpyAsync(tap, xbuf, sizeof(float) * M * D, cudaMemcpyDeviceToDevice, s));
            return 0;
          },
          KIND_MEMSET, 0.0);
    }
  }
  // final self.norm is dead code in the reference (glob unused, lseg_vit.py:108,199) -> skipped.

  // ---- readout + reassemble (lseg_vit.py:79-90, 104-146, 442-522) ----
  // Level k: 1x1 conv D -> post_channels[k], then ConvTranspose (k = s, stride s), nothing, or a 3x3 stride-2 conv
  // (lseg_vit.py:465-520 for ViT-L/16: x4, x2, -, /2; 531-586 for ViT-B/32: x8, x4, x2, -). post_channels are the
  // STORED widths: reference counts rounded up to a multiple of 64 with zero weights in the pad (96 -> 128).
  for (int k = 0; k < 4; ++k) {
    c_post[k] = w.post_channels[k];
    const int r = w.post_resample[k];
    if (c_post[k] <= 0 || c_post[k] % 64 != 0 || !(r == -2 || r == 0 || r == 2 || r == 4 || r == 8)) {
      set_error("reassemble level %d: post_channels=%d (multiple of 64), post_resample=%d (8, 4, 2, 0, -2)", k, c_post[k], r);
      return -1;
    }
    lh[k] = (r > 0) ? gh * r : (r == 0 ? gh : gh / 2);
    lw[k] = (r > 0) ? gw * r : (r == 0 ? gw : gw / 2);
  }
  for (int k = 0; k < 3; ++k)
    if (lh[k] != 2 * lh[k + 1] || lw[k] != 2 * lw[k + 1]) {
      set_error("reassemble: level %d (%dx%d) is not twice level %d (%dx%d) — the fusion decoder needs a x2 pyramid "
                "(H, W multiples of 32)", k, lh[k], lw[k], k + 1, lh[k + 1], lw[k + 1]);
      return -1;
    }
  LSEG_ALLOC(tok, __half, BT * D);
  const int cls_rows = ((B + 127) / 128) * 128;
  LSEG_ALLOC(cls16, __half, (size_t)cls_rows * D);
  LSEG_CHECK_CUDA(cudaMemsetAsync(cls16, 0, sizeof(__half) * (size_t)cls_rows * D, stream));
  LSEG_ALLOC(clsb, float, (size_t)B * D);
  LSEG_ALLOC(ro, __half, BT * D);
  plan->debug["readout3"] = ro;  // shared by the four levels: after a forward it holds the last one's
  for (int k = 0; k < 4; ++k) {
    const float* tap = taps[k];
    steps.push_back([=](const CallCtx&, cudaStream_t s) {
      return launch_readout_split(tap, tok, cls16, B, T, D, s);
    });
    {  // per-image half of the readout projection: cls * W[:,D:]^T + b
      GemmEpi e = epi_none();
      e.bias = w.readout_cls[k].b;
      e.out_f32 = clsb;
      e.ldc = D;
      if (add_gemm(steps, cls16, D, cls_rows, B, w.readout_cls[k], e)) return -1;
    }
    {  // tok * W[:,:D]^T + (per-image row) -> GELU
      GemmEpi e = epi_none();
      e.bias = clsb;
      e.bias_group_rows = T;
      e.act = ACT_GELU;
      e.out_f16 = ro;
      e.ldc = D;
      if (add_gemm(steps, tok, D, (int)BT, (int)BT, w.readout_tok[k], e)) return -1;
    }
    LSEG_ALLOC(pk, __half, BT * c_post[k]);
    char name[8];
    snprintf(name, sizeof(name), "post%d", k);
    plan->debug[name] = pk;  // [B*T, c_post[k]]
    {
      GemmEpi e = epi_none();
      e.bias = w.post_conv1x1[k].b;
      e.out_f16 = pk;
      e.ldc = c_post[k];
      if (add_gemm(steps, ro, D, (int)BT, (int)BT, w.post_conv1x1[k], e)) return -1;
    }
    const int r = w.post_resample[k];
    const lseg_linear_w& rw = w.post_resample_w[k];
    if (r > 0) {
      LSEG_ALLOC(lk, __half, BT * r * r * c_post[k]);
      GemmEpi e = epi_none();
      e.bias = rw.b;
      e.out_f16 = lk;
      e.store = STORE_D2S;
      e.d2s_s = r;
      e.d2s_cout = c_post[k];
      e.d2s_h = gh;
      e.d2s_w = gw;
      if (add_gemm(steps, pk, c_post[k], (int)BT, (int)BT, rw, e)) return -1;
      layer_in[k] = lk;
    } else if (r == 0) {
      layer_in[k] = pk;
    } else {
      const int ck = c_post[k];
      const long long rows4 = static_cast<long long>(B) * lh[k] * lw[k];
      LSEG_ALLOC(a4, __half, rows4 * 9 * ck);
      LSEG_ALLOC(l4, __half, rows4 * ck);
      steps.push_back([=](const CallCtx&, cudaStream_t s) {
        return launch_im2col_3x3_s2(pk, a4, B, gh, gw, ck, s);
      });
      GemmEpi e = epi_none();
      e.bias = rw.b;
      e.out_f16 = l4;
      e.ldc = ck;
      if (add_gemm(steps, a4, 9 * ck, (int)rows4, (int)rows4, rw, e)) return -1;
      layer_in[k] = l4;
    }
  }

  return 0;
}

// ResNet-101 trunk of the zero-shot model (lseg_net_zs.py:307-310: pretrained.layer1..4 = torchvision resnet101 stages,
// lseg_blocks_zs.py:109-119): stem 7x7 s2 (im2col + GEMM, BN + ReLU in the epilogue) -> maxpool -> 33 bottlenecks.
// Every conv is the wgmma GEMM: 1x1 = plain GEMM over the NHWC pixels, 3x3 stride 1 = implicit GEMM, 3x3 stride 2 =
// im2col rows + GEMM, 1x1 stride 2 = GEMM over the subsampled pixels; BatchNorm folded into the fp32 epilogue. The
// residual stream is fp32 (one buffer per stage, updated in place by conv3's epilogue: relu(bn3(conv3) + identity)),
// with an fp16 copy as the next conv's operand — the same split as the decoder's RCUs.
static int build_resnet_trunk(lseg_engine* eng, ImagePlan* plan, int B, int H, int W, cudaStream_t stream,
                              __half* (&layer_in)[4], int (&c_post)[4], int (&lh)[4], int (&lw)[4]) {
  (void)stream;
  const lseg_weights& w = eng->w;
  Arena& arena = plan->arena;
  std::vector<Step>& steps = plan->steps;
  const int Hs = H / 2, Ws = W / 2;  // stem output
  const long long R0 = static_cast<long long>(B) * Hs * Ws;
  LSEG_ALLOC(stem_a, __half, R0 * kStemK);
  LSEG_ALLOC(stem_o, __half, R0 * 64);
  plan->debug["stem"] = stem_o;  // NHWC fp16 [B, H/2, W/2, 64]
  steps.push_back([=](const CallCtx& c, cudaStream_t s) { return launch_stem_im2col(c.x, stem_a, B, H, W, s); });
  {
    GemmEpi e = epi_none();
    e.scale = w.rn_stem_scale;
    e.bias = w.rn_stem_shift;
    e.act = ACT_RELU;
    e.out_f16 = stem_o;
    e.ldc = 64;
    if (add_gemm(steps, stem_a, kStemK, (int)R0, (int)R0, w.rn_stem, e)) return -1;
  }
  int h = Hs / 2, ww = Ws / 2;  // after the 3x3 stride-2 max pool
  LSEG_ALLOC(pool_o, __half, static_cast<long long>(B) * h * ww * 64);
  plan->debug["pool"] = pool_o;  // NHWC fp16 [B, H/4, W/4, 64]
  steps.push_back([=](const CallCtx&, cudaStream_t s) { return launch_maxpool3x3s2_nhwc(stem_o, pool_o, B, Hs, Ws, 64, s); });
  const __half* x16 = pool_o;
  int cin = 64, blk = 0;
  for (int L = 0; L < 4; ++L) {
    const int width = 64 << L, cout = 4 * width;
    const int n = w.rn_layers[L];
    if (n <= 0 || blk + n > LSEG_RESNET_BLOCKS) {
      set_error("resnet trunk: stage %d has %d blocks", L + 1, n);
      return -1;
    }
    const int stride0 = w.rn_blocks[blk].stride;
    const int ho = h / stride0, wo = ww / stride0;
    const long long px_in = static_cast<long long>(B) * h * ww, px = static_cast<long long>(B) * ho * wo;
    LSEG_ALLOC(t1, __half, px_in * width);
    LSEG_ALLOC(t2, __half, px * width);
    LSEG_ALLOC(y32, float, px * cout);   // the stage's residual stream, updated in place
    LSEG_ALLOC(y16a, __half, px * cout);
    LSEG_ALLOC(y16b, __half, px * cout);
    for (int i = 0; i < n; ++i, ++blk) {
      const lseg_bottleneck_w& bw = w.rn_blocks[blk];
      const int stride = (i == 0) ? stride0 : 1;
      if (bw.stride != stride || (stride != 1 && stride != 2) || ((i == 0) != (bw.down.w != nullptr))) {
        set_error("resnet trunk: block %d of stage %d: stride %d / downsample do not fit a torchvision Bottleneck stage", i,
                  L + 1, bw.stride);
        return -1;
      }
      const int hi = (i == 0) ? h : ho, wi = (i == 0) ? ww : wo;
      const long long pxi = static_cast<long long>(B) * hi * wi;
      const bool tr = blk == g_trace_block;  // snapshot every intermediate of this block (lseg_debug_set_trace_block)
      if (tr && add_snapshot(plan, "trace_in", x16, sizeof(__half) * pxi * cin)) return -1;
      {  // conv1 1x1 + bn1 + relu
        GemmEpi e = epi_none();
        e.scale = bw.bn1_scale;
        e.bias = bw.bn1_shift;
        e.act = ACT_RELU;
        e.out_f16 = t1;
        e.ldc = width;
        if (add_gemm(steps, x16, cin, (int)pxi, (int)pxi, bw.conv1, e)) return -1;
      }
      if (tr && add_snapshot(plan, "trace_t1", t1, sizeof(__half) * pxi * width)) return -1;
      {  // conv2 3x3 (stride here, torchvision v1.5) + bn2 + relu
        GemmEpi e = epi_none();
        e.scale = bw.bn2_scale;
        e.bias = bw.bn2_shift;
        e.act = ACT_RELU;
        e.out_f16 = t2;
        e.ldc = width;
        if (stride == 1) {
          if (add_conv3x3(steps, t1, B, hi, wi, width, bw.conv2, e)) return -1;
        } else {
          LSEG_ALLOC(a2, __half, px * 9 * width);
          steps.push_back([=](const CallCtx&, cudaStream_t s) { return launch_im2col_3x3_s2(t1, a2, B, hi, wi, width, s); });
          if (add_gemm(steps, a2, 9 * width, (int)px, (int)px, bw.conv2, e)) return -1;
        }
      }
      if (tr && add_snapshot(plan, "trace_t2", t2, sizeof(__half) * px * width)) return -1;
      if (i == 0) {  // identity = bn_d(conv_d 1x1 stride s (x)) -> the stage's fp32 stream
        const __half* xs = x16;
        if (stride == 2) {
          LSEG_ALLOC(sub, __half, px * cin);
          const __half* xin = x16;
          steps.push_back([=](const CallCtx&, cudaStream_t s) { return launch_subsample2_nhwc(xin, sub, B, hi, wi, cin, s); });
          xs = sub;
        }
        GemmEpi e = epi_none();
        e.scale = bw.bnd_scale;
        e.bias = bw.bnd_shift;
        e.out_f32 = y32;
        e.ldc = cout;
        if (add_gemm(steps, xs, cin, (int)px, (int)px, bw.down, e)) return -1;
      }
      if (tr && add_snapshot(plan, "trace_id", y32, sizeof(float) * px * cout)) return -1;
      __half* y16 = (i & 1) ? y16b : y16a;
      {  // conv3 1x1 + bn3, + identity, relu -> fp32 stream (in place) and its fp16 copy
        GemmEpi e = epi_none();
        e.scale = bw.bn3_scale;
        e.bias = bw.bn3_shift;
        e.res_f32 = y32;
        e.out_f32 = y32;
        e.out_f16 = y16;
        e.relu_after_res = 1;
        e.ldc = cout;
        if (add_gemm(steps, t2, width, (int)px, (int)px, bw.conv3, e)) return -1;
      }
      if (tr && (add_snapshot(plan, "trace_out32", y32, sizeof(float) * px * cout) ||
                 add_snapshot(plan, "trace_out16", y16, sizeof(__half) * px * cout)))
        return -1;
      x16 = y16;
      cin = cout;
    }
    layer_in[L] = const_cast<__half*>(x16);
    c_post[L] = cout;
    lh[L] = ho;
    lw[L] = wo;
    h = ho;
    ww = wo;
  }
  if (blk != LSEG_RESNET_BLOCKS && blk <= 0) return -1;
  for (int k = 0; k < 3; ++k)
    if (lh[k] != 2 * lh[k + 1] || lw[k] != 2 * lw[k + 1]) {
      set_error("resnet trunk: stage sizes are not a x2 pyramid (H, W multiples of 32)");
      return -1;
    }
  return 0;
}

static int build_image_plan(lseg_engine* eng, int B, int H, int W, bool attn, cudaStream_t stream) {
  const lseg_weights& w = eng->w;
  std::unique_ptr<ImagePlan> plan(new ImagePlan());
  plan->B = B;
  plan->H = H;
  plan->W = W;
  plan->epoch = g_plan_epoch;
  plan->attn = attn;
  Arena& arena = plan->arena;
  t_plan_arena = &arena;
  std::vector<Step>& steps = plan->steps;
  __half* layer_in[4];  // NHWC fp16 inputs of scratch.layerN_rn
  int c_post[4], lh[4], lw[4];
  const int blocks = w.trunk == 1 ? w.rn_layers[0] + w.rn_layers[1] + w.rn_layers[2] + w.rn_layers[3] : w.vit_depth;
  if (g_trace_block >= blocks) {  // before anything is allocated or launched
    set_error("lseg_debug_set_trace_block: trace block %d is not a block of this trunk, which has %d blocks",
              g_trace_block, blocks);
    return -1;
  }
  if (w.trunk == 1) {
    if (build_resnet_trunk(eng, plan.get(), B, H, W, stream, layer_in, c_post, lh, lw)) return -1;
  } else {
    if (build_vit_trunk(eng, plan.get(), B, H, W, stream, layer_in, c_post, lh, lw)) return -1;
  }
  for (int k = 0; k < 4; ++k) {
    char name[12];
    snprintf(name, sizeof(name), "layer%d", k);
    plan->debug[name] = layer_in[k];  // NHWC fp16 [B, lh, lw, post_channels[k]]
  }

  // ---- scratch.layerN_rn (lseg_blocks.py:73-108; lseg_net.py:171-174) ----
  float* rn_f32[4];
  __half* rn_relu[4];
  for (int k = 0; k < 4; ++k) {
    const long long px = static_cast<long long>(B) * lh[k] * lw[k];
    LSEG_ALLOC(f, float, px * 256);
    LSEG_ALLOC(r, __half, px * 256);
    rn_f32[k] = f;
    rn_relu[k] = r;
    char name[12];
    snprintf(name, sizeof(name), "rn%d", k);
    plan->debug[name] = f;  // NHWC fp32 [B, lh, lw, 256]
    snprintf(name, sizeof(name), "rn%d_relu", k);
    plan->debug[name] = r;  // its ReLU, fp16
    GemmEpi e = epi_none();
    e.out_f32 = f;
    e.out_f16_relu = r;
    e.ldc = 256;
    if (add_conv3x3(steps, layer_in[k], B, lh[k], lw[k], c_post[k], w.layer_rn[k], e)) return -1;
  }

  // ---- fusion decoder (lseg_blocks.py:337-358; lseg_net.py:176-179) ----
  const float* path_prev = nullptr;  // fp32 NHWC: output of the previous refinenet + rn_f32[k] (same res as rn[k])
  __half* path1_f16 = nullptr;
  for (int k = 3; k >= 0; --k) {
    const int h = lh[k], ww = lw[k];
    const long long px = static_cast<long long>(B) * h * ww;
    LSEG_ALLOC(tmp, __half, px * 256);
    LSEG_ALLOC(r2, __half, px * 256);
    // stage buffers of this level, NHWC [B, h, ww, 256] (the _skip one at the next level's size)
    auto name_stage = [&](const char* stage, const void* p) { plan->debug["dec" + std::to_string(k) + "_" + stage] = p; };
    name_stage("tmp", tmp);  // shared by both units: after the forward it holds RCU2's conv1 output
    name_stage("rcu2", r2);
    const __half* rcu2_in_relu = rn_relu[k];
    const float* rcu2_in_f32 = rn_f32[k];
    if (path_prev) {  // output = xs[0] + resConfUnit1(xs[1])
      LSEG_ALLOC(sum_f32, float, px * 256);
      LSEG_ALLOC(sum_relu, __half, px * 256);
      name_stage("sum", sum_f32);
      name_stage("sum_relu", sum_relu);
      // path_prev already holds xs[0] + xs[1] (previous block's output + this level's layer_rn, summed by the
      // interpolation kernel below): the residual conv adds ONE fp32 operand instead of two
      if (add_rcu(steps, w.rcu1[k], rn_relu[k], path_prev, nullptr, tmp, B, h, ww, sum_f32, nullptr, sum_relu))
        return -1;
      rcu2_in_relu = sum_relu;
      rcu2_in_f32 = sum_f32;
    }
    if (add_rcu(steps, w.rcu2[k], rcu2_in_relu, rcu2_in_f32, nullptr, tmp, B, h, ww, nullptr, r2, nullptr)) return -1;
    // lseg_blocks.py:352-356: interpolate(x2, align_corners) then out_conv (1x1). Run in the other order — the 1x1 conv
    // on the low-res tensor (a quarter of the pixels), then ONE interpolation pass that writes the block's output
    // (fp32 for the next block's skip add, with that block's other input already summed in; fp16 for head1): the
    // same linear map (the interpolation weights sum to one, so the bias commutes too), 3/4 of the conv's FLOPs and
    // the hi-res fp16 intermediate gone.
    // The low-res conv result stays in fp32 by default (one fp16 rounding less than interpolating an fp16 tensor; path_1
    // measured 0.7e-3 against the oracle, 1.05e-3 with an fp16 intermediate). LSEG_OUTCONV_F16 = bit mask of levels
    // (bit k = refinenet k+1) whose result leaves through the 2.4x faster fp16 TMA-store epilogue instead (A/B).
    static const int f16_mask = getenv("LSEG_OUTCONV_F16") ? atoi(getenv("LSEG_OUTCONV_F16")) : 0;
    const bool low_f16 = (f16_mask >> k) & 1;
    __half* oc16 = nullptr;
    float* oc32 = nullptr;
    {
      GemmEpi e = epi_none();
      e.bias = w.out_conv[k].b;
      e.ldc = 256;
      if (low_f16) {
        LSEG_ALLOC(t16, __half, px * 256);
        oc16 = t16;
        e.out_f16 = t16;
      } else {
        LSEG_ALLOC(t32, float, px * 256);
        oc32 = t32;
        e.out_f32 = t32;
      }
      if (add_gemm(steps, r2, 256, (int)px, (int)px, w.out_conv[k], e)) return -1;
      name_stage("out_lr", low_f16 ? static_cast<const void*>(oc16) : oc32);
    }
    if (k > 0) {
      LSEG_ALLOC(pth, float, px * 4 * 256);
      const float* next_rn = rn_f32[k - 1];  // the next block's other input, same shape as pth
      steps.push_back([=](const CallCtx&, cudaStream_t s) {
        return low_f16 ? launch_upsample2x_nhwc256_f16<float>(oc16, pth, next_rn, B, h, ww, s)
                       : launch_upsample2x_nhwc256_f32<float>(oc32, pth, next_rn, B, h, ww, s);
      });
      path_prev = pth;
      name_stage("skip", pth);
    } else {
      LSEG_ALLOC(pth16, __half, px * 4 * 256);
      steps.push_back([=](const CallCtx&, cudaStream_t s) {
        return low_f16 ? launch_upsample2x_nhwc256_f16<__half>(oc16, pth16, nullptr, B, h, ww, s)
                       : launch_upsample2x_nhwc256_f32<__half>(oc32, pth16, nullptr, B, h, ww, s);
      });
      path1_f16 = pth16;
    }
  }
  plan->debug["path1"] = path1_f16;

  // ---- head1 + pixel normalisation (lseg_net.py:185-191) ----
  const long long BP = static_cast<long long>(B) * (H / 2) * (W / 2);
  // The pixel embedding is written once, un-normalised, in fp16, together with its fp32 squared row
  // norm (accumulated from the fp32 accumulators); the pixel x text GEMM applies logit_scale / ||row|| in
  // its epilogue. Same quantity as the reference's normalise -> half -> scale -> matmul up to where the
  // fp16 roundings fall, without the 118 MB/img fp32 feature round trip and the separate norm pass.
  const int OC = w.out_c;
  LSEG_ALLOC(featn, __half, BP * OC);
  LSEG_ALLOC(feat_sumsq, float, BP * (OC / 32));  // [row, out_c/32] partial squared norms
  {
    GemmDesc& d = plan->head1_desc;
    memset(&d, 0, sizeof(d));
    d.a = path1_f16;
    d.lda = 256;
    d.a_rows = (int)BP;
    d.w = static_cast<const __half*>(w.head1.w);
    d.w_rows = w.head1.rows;
    d.M = (int)BP;
    d.N = w.head1.out;
    d.K = w.head1.in;
    d.e = epi_none();
    d.e.bias = w.head1.b;
    d.e.out_f16 = featn;
    d.e.out_row_sumsq = feat_sumsq;
    d.e.ldc = OC;
    GemmPlan gp;
    if (gemm_plan(d, &gp)) return -1;
    if (gp.ws_bytes) {
      LSEG_ALLOC(ws, float, gp.ws_bytes / sizeof(float));
      plan->head1_ws = ws;
      gemm_set_workspace(&gp, ws);
    }
    plan->head1.emplace(std::make_pair(static_cast<const void*>(featn), static_cast<const void*>(feat_sumsq)), gp);
  }
  plan->featn = featn;
  plan->feat_sumsq = feat_sumsq;
  plan->debug["featn"] = featn;
  plan->debug["feat_sumsq"] = feat_sumsq;
  if (static_cast<int>(eng->plans.size()) >= lseg_engine::kMaxImagePlans) {
    size_t victim = 0;
    for (size_t i = 1; i < eng->plans.size(); ++i)
      if (eng->plans[i]->last_use < eng->plans[victim]->last_use) victim = i;
    LSEG_CHECK_CUDA(cudaStreamSynchronize(stream));  // the victim's buffers may still be in use by queued work
    eng->plans.erase(eng->plans.begin() + victim);
  }
  eng->plans.push_back(std::move(plan));
  eng->img = eng->plans.back().get();
  return 0;
}

// Optional per-launch timing (bench.py roofline): CUDA events recorded on the launching stream
// around every launch of one forward.
struct Profile {
  std::vector<cudaEvent_t> ev;
  std::vector<int> kind;
  std::vector<double> flops;
  int mark(cudaStream_t s) {
    cudaEvent_t e;
    LSEG_CHECK_CUDA(cudaEventCreate(&e));
    LSEG_CHECK_CUDA(cudaEventRecord(e, s));
    ev.push_back(e);
    return 0;
  }
};

// A launch of the forward or query path: counted, and timed when profiling.
static int note_launch(Profile* prof, int* launches, int kind, double flops, cudaStream_t stream) {
  ++*launches;
  if (prof) {
    if (prof->mark(stream)) return -1;
    prof->kind.push_back(kind);
    prof->flops.push_back(flops);
  }
  return 0;
}

static int check_image_shape(const char* fn, int B, int H, int W) {
  if (B <= 0) return set_error("%s: B=%d must be positive", fn, B), -1;
  if (H % 32 != 0 || W % 32 != 0 || H <= 0 || W <= 0)  // the reference fails deep inside skip_add.add
    return set_error("%s: H=%d, W=%d must be positive multiples of 32", fn, H, W), -1;  // (lseg_blocks.py:347)
  return 0;
}

// The image plan for (B, H, W), with or without the attention-recording steps, built on first use; plans built under
// other baked-in options are dropped.
static ImagePlan* image_plan(lseg_engine* eng, int B, int H, int W, cudaStream_t stream, bool attn = false) {
  eng->img = nullptr;
  for (size_t i = 0; i < eng->plans.size();) {
    ImagePlan* pl = eng->plans[i].get();
    if (pl->epoch != g_plan_epoch) {  // an option baked into the GEMM plans changed
      if (cudaStreamSynchronize(stream) != cudaSuccess) return set_error("image plan: stream sync failed"), nullptr;
      eng->plans.erase(eng->plans.begin() + i);
      continue;
    }
    if (pl->B == B && pl->H == H && pl->W == W && pl->attn == attn) eng->img = pl;
    ++i;
  }
  if (!eng->img && build_image_plan(eng, B, H, W, attn, stream)) return nullptr;
  eng->img->last_use = ++eng->use_counter;
  return eng->img;
}

// The trunk: plan.steps, then head1 into (emb, sumsq) — fp16 [B*P, out_c] un-normalised rows and their fp32 partial
// squared norms [B*P, out_c/32] — the plan's own featn / feat_sumsq for a forward, a caller's buffers for
// lseg_encode_image. Same launches and bits either way; only head1's output address differs.
static int run_trunk(lseg_engine* eng, ImagePlan& plan, const CallCtx& ctx, __half* emb, float* sumsq, cudaStream_t stream,
                     Profile* prof, int* launches) {
  auto key = std::make_pair(static_cast<const void*>(emb), static_cast<const void*>(sumsq));
  auto it = plan.head1.find(key);
  if (it == plan.head1.end()) {
    if (plan.head1.size() > 16) {  // keep the plan of the own buffers
      auto own = plan.head1.find(std::make_pair(static_cast<const void*>(plan.featn), static_cast<const void*>(plan.feat_sumsq)));
      GemmPlan keep = own->second;
      plan.head1.clear();
      plan.head1.emplace(own->first, keep);
    }
    GemmDesc d = plan.head1_desc;
    d.e.out_f16 = emb;
    d.e.out_row_sumsq = sumsq;
    GemmPlan gp;
    if (gemm_plan(d, &gp)) return -1;
    if (gp.ws_bytes) gemm_set_workspace(&gp, plan.head1_ws);
    it = plan.head1.emplace(key, gp).first;
  }
  if (prof && prof->mark(stream)) return -1;
  for (auto& st : plan.steps) {
    if (st(ctx, stream)) return -1;
    if (st.kind != KIND_MEMSET) ++*launches;  // count our kernels only
    if (prof) {
      if (prof->mark(stream)) return -1;
      prof->kind.push_back(st.kind);
      prof->flops.push_back(st.flops);
    }
  }
  const GemmDesc& d = plan.head1_desc;
  if (gemm_run(it->second, stream)) return -1;
  return note_launch(prof, launches, KIND_GEMM, 2.0 * d.M * d.N * static_cast<double>(d.K), stream);
}

// The tail workspace for (B, H, W) with room for K labels.
static TailWs* tail_ws(lseg_engine* eng, int B, int H, int W, int K, bool need_lr, cudaStream_t stream) {
  TailWs* t = nullptr;
  for (auto& p : eng->tails)
    if (p->B == B && p->H == H && p->W == W) t = p.get();
  if (!t) {
    if (static_cast<int>(eng->tails.size()) >= lseg_engine::kMaxTails) {
      size_t victim = 0;
      for (size_t i = 1; i < eng->tails.size(); ++i)
        if (eng->tails[i]->last_use < eng->tails[victim]->last_use) victim = i;
      // the victim's buffers may still be in use by queued work
      if (cudaStreamSynchronize(stream) != cudaSuccess) return set_error("tail workspace: stream sync failed"), nullptr;
      eng->tails.erase(eng->tails.begin() + victim);
    }
    eng->tails.emplace_back(new TailWs());
    t = eng->tails.back().get();
    t->B = B;
    t->H = H;
    t->W = W;
    t->epoch = g_plan_epoch;
  }
  if (t->epoch != g_plan_epoch) {  // an option baked into the GEMM plans changed
    t->corr.clear();
    t->epoch = g_plan_epoch;
  }
  t->last_use = ++eng->use_counter;
  const size_t P = static_cast<size_t>(H / 2) * (W / 2);
  if (need_lr && (!t->logits_lr || t->logits_cap_k < (size_t)K)) {
    if (t->logits_lr) {
      if (cudaStreamSynchronize(stream) != cudaSuccess) return set_error("tail workspace: stream sync failed"), nullptr;
      cudaFree(t->logits_lr);
      t->logits_lr = nullptr;
      t->corr.clear();
    }
    void* p = nullptr;
    if (cudaMalloc(&p, sizeof(__half) * (size_t)B * K * P) != cudaSuccess) {
      cudaGetLastError();
      return set_error("logits workspace allocation failed"), nullptr;
    }
    t->logits_lr = static_cast<__half*>(p);
    t->logits_cap_k = K;
  }
  const int arch = eng->w.arch_option;
  if ((arch == 1 || arch == 2) && (!t->head_ws[0] || t->head_cap_k < (size_t)K)) {
    if (cudaStreamSynchronize(stream) != cudaSuccess) return set_error("tail workspace: stream sync failed"), nullptr;
    for (int i = 0; i < 2; ++i) {
      if (t->head_ws[i]) cudaFree(t->head_ws[i]);
      t->head_ws[i] = nullptr;
      if (cudaMalloc(&t->head_ws[i], sizeof(float) * (size_t)B * K * P) != cudaSuccess) {
        cudaGetLastError();
        return set_error("head block workspace allocation failed"), nullptr;
      }
    }
    if (!t->head_cmax && cudaMalloc(&t->head_cmax, sizeof(float) * (size_t)B * P) != cudaSuccess) {
      cudaGetLastError();
      return set_error("head block workspace allocation failed"), nullptr;
    }
    t->head_cap_k = K;
  }
  return t;
}

// The label-dependent tail of LSeg.forward on a pixel embedding (emb, sumsq) of B images of H x W: the pixel x text
// GEMM, the arch_option head blocks and the x2 output stage (logits / argmax / metric counters). The one implementation
// behind every forward entry point and lseg_query. *lr_out: where the fp16 low-res logits went.
static int run_tail(lseg_engine* eng, const CallCtx& ctx, int B, int H, int W, const __half* emb, const float* sumsq,
                    cudaStream_t stream, Profile* prof, int* launches, __half** lr_out) {
  const int arch = eng->w.arch_option;
  if (ctx.out_lr && (arch == 1 || arch == 2)) {
    set_error("lseg_forward_lowres: the fp16 low-res logits are not the network output when arch_option is %d", arch);
    return -1;
  }
  const bool ragged = ctx.rag_k != nullptr;
  // a ragged batch packs sum(k) = ctx.K planes: the per-image workspaces hold B * ceil(sum / B) >= sum planes
  TailWs* t = tail_ws(eng, B, H, W, ragged ? (ctx.K + B - 1) / B : ctx.K, !ctx.out_lr, stream);
  if (!t) return -1;
  const int h2 = H / 2, w2 = W / 2;
  const long long P = static_cast<long long>(h2) * w2;
  __half* lr = ctx.out_lr ? ctx.out_lr : t->logits_lr;
  *lr_out = lr;
  // ---- pixel x text correlation (lseg_net.py:194-196): fp16 GEMM, fp16 result, NCHW store ----
  // One label set for all images (text_image_stride == 0): one GEMM over all B*P pixel rows.
  // One label block per image (zero-shot path, lseg_net_zs.py:196-210; rows [b*stride, b*stride + K) of `text`):
  // still ONE GEMM, against all B*stride text rows at once — each pixel row keeps only the K columns of its own
  // image's block (nchw_group), the other columns are computed and dropped. For K = 2 the N tile is 128 wide anyway,
  // so this costs the same tile as one image's block and replaces B launches by one. Falls back to one launch per
  // image when B*stride exceeds one 256-column tile.
  // Ragged batch (every image its own label set): ONE launch of the ragged kernel, whose work list holds only the tiles of
  // each image's own pixel rows x its own text rows; image b's columns land in planes koff[b] .. of the packed output.
  {
    TailWs::CorrKey key{ctx.text, ctx.K, ctx.text_image_stride, lr, emb, sumsq, {}};
    if (ragged) {
      key.rag.assign(1, ctx.rag_text_rows);
      key.rag.insert(key.rag.end(), ctx.rag_k, ctx.rag_k + B);
      key.rag.insert(key.rag.end(), ctx.rag_text_row, ctx.rag_text_row + B);
    }
    auto it = t->corr.find(key);
    if (it == t->corr.end() && ragged) {
      if (t->corr.size() > 16) t->corr.clear();
      const int OC = eng->w.out_c;
      GemmDesc d;
      memset(&d, 0, sizeof(d));
      d.a = emb;
      d.lda = OC;
      d.a_rows = static_cast<int>(B * P);
      d.w = ctx.text;
      d.w_rows = ctx.rag_text_rows;
      d.M = static_cast<int>(B * P);
      d.K = OC;
      d.e = epi_none();
      d.e.out_f16 = lr;
      d.e.nchw_p = static_cast<int>(P);
      d.e.row_sumsq = sumsq;
      d.e.row_sumsq_parts = OC / 32;
      d.e.row_scale = eng->w.logit_scale;
      GemmPlan gp;
      if (gemm_plan_ragged(d, B, ctx.rag_k, ctx.rag_text_row, &gp)) return -1;
      std::vector<std::pair<GemmPlan, double>> plans;
      plans.emplace_back(gp, 2.0 * P * ctx.K * static_cast<double>(OC));
      it = t->corr.emplace(key, std::move(plans)).first;
    } else if (it == t->corr.end()) {
      if (t->corr.size() > 16) t->corr.clear();
      std::vector<std::pair<GemmPlan, double>> plans;
      const long long stride = ctx.text_image_stride;
      const bool grouped = stride > 0 && static_cast<long long>(B) * stride <= 256;
      const int groups = (stride > 0 && !grouped) ? B : 1;
      for (int g = 0; g < groups; ++g) {
        GemmDesc d;
        memset(&d, 0, sizeof(d));
        const long long rows = (groups == 1) ? static_cast<long long>(B) * P : P;
        const int n_cols = grouped ? static_cast<int>(B * stride) : ctx.K;
        const int OC = eng->w.out_c;
        d.a = emb + static_cast<long long>(g) * P * OC;
        d.lda = OC;
        d.a_rows = (int)rows;
        d.w = ctx.text + static_cast<long long>(g) * stride * OC;
        d.w_rows = ((n_cols + 127) / 128) * 128;
        d.M = (int)rows;
        d.N = n_cols;
        d.K = OC;
        d.e = epi_none();
        d.e.out_f16 = lr + static_cast<long long>(g) * ctx.K * P;
        d.e.store = STORE_NCHW_T;
        d.e.nchw_p = (int)P;
        d.e.nchw_k = ctx.K;
        d.e.nchw_group = grouped ? (int)stride : 0;
        d.e.row_sumsq = sumsq + static_cast<long long>(g) * P * (OC / 32);
        d.e.row_sumsq_parts = OC / 32;
        d.e.row_scale = eng->w.logit_scale;
        GemmPlan gp;
        if (gemm_plan(d, &gp)) return -1;
        plans.emplace_back(gp, 2.0 * rows * n_cols * static_cast<double>(OC));
      }
      it = t->corr.emplace(key, std::move(plans)).first;
    }
    for (auto& pr : it->second) {
      if (gemm_run(pr.first, stream)) return -1;
      if (note_launch(prof, launches, KIND_GEMM, pr.second, stream)) return -1;
    }
  }
  // ---- optional head blocks on the fp32 view of the low-res logits (arch_option 1 / 2, lseg_net.py:198-201) ----
  const float* lr32 = nullptr;
  if (arch == 1 || arch == 2) {
    HeadBlockW hw;
    for (int i = 0; i < 9; ++i) hw.w[i] = eng->w.head_block_w[i];
    hw.bias = eng->w.head_block_b;
    const int depth = eng->w.block_depth > 1 ? eng->w.block_depth : 1;  // range(block_depth - 1) + the final call
    for (int dpt = 0; dpt < depth; ++dpt) {
      const int act = (dpt + 1 < depth) ? eng->w.head_act : HEAD_ACT_NONE;
      float* dst = t->head_ws[dpt & 1];
      if (ragged) {  // the channel max runs over each image's own labels: one launch_head_block per image
        long long koff = 0;
        for (int b = 0; b < B; ++b) {
          const long long o = koff * P;
          float* cm = t->head_cmax + b * P;
          const int kb = ctx.rag_k[b];
          int rc = (dpt == 0) ? launch_head_block(lr + o, cm, dst + o, 1, kb, h2, w2, hw, arch, act, stream)
                              : launch_head_block(static_cast<const float*>(t->head_ws[(dpt - 1) & 1]) + o, cm, dst + o, 1,
                                                  kb, h2, w2, hw, arch, act, stream);
          if (rc) return -1;
          if (arch == 1) ++*launches;
          if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
          koff += kb;
        }
        lr32 = dst;
        continue;
      }
      int rc = (dpt == 0) ? launch_head_block(lr, t->head_cmax, dst, B, ctx.K, h2, w2, hw, arch, act, stream)
                          : launch_head_block(static_cast<const float*>(t->head_ws[(dpt - 1) & 1]), t->head_cmax, dst,
                                              B, ctx.K, h2, w2, hw, arch, act, stream);
      if (rc) return -1;
      if (arch == 1) ++*launches;  // bottleneck_block: channel max + conv
      if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
      lr32 = dst;
    }
  }
  // ---- scratch.output_conv: bilinear x2, align_corners=True (lseg_net.py:203) ----
  if (ctx.out) {
    const long long planes = ragged ? ctx.K : static_cast<long long>(B) * ctx.K;
    if (lr32 ? launch_upsample2x_nchw(lr32, ctx.out, planes, h2, w2, stream)
             : launch_upsample2x_nchw(lr, ctx.out, planes, h2, w2, stream))
      return -1;
    if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
  }
  // ---- fused output_conv + torch.max(.., 1)[1] (SURVEY.md 8(f) row 2): the fp32 logits are never materialised ----
  if (ctx.xent) {  // ... with the loss (and the metric counters when ctx.seg is set) in the same kernel
    const SegStatsArgs st = ctx.seg ? *ctx.seg : SegStatsArgs{};
    if (lr32 ? launch_upsample2x_xent(lr32, ctx.out_mask, B, ctx.K, h2, w2, st, *ctx.xent, stream)
             : launch_upsample2x_xent(lr, ctx.out_mask, B, ctx.K, h2, w2, st, *ctx.xent, stream))
      return -1;
    if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;  // the loss kernel and its one-block finish
    if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
  } else if (ctx.seg) {  // ... and counted into the metric rows in the same kernel
    if (lr32 ? launch_upsample2x_segstats(lr32, ctx.out_mask, B, ctx.K, h2, w2, *ctx.seg, stream)
             : launch_upsample2x_segstats(lr, ctx.out_mask, B, ctx.K, h2, w2, *ctx.seg, stream))
      return -1;
    if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
  } else if (ctx.out_mask && ragged) {
    RaggedPlanes rp;
    memset(&rp, 0, sizeof(rp));
    for (int b = 0, koff = 0; b < B; koff += ctx.rag_k[b], ++b) {
      rp.k[b] = ctx.rag_k[b];
      rp.koff[b] = koff;
    }
    if (lr32 ? launch_upsample2x_argmax_ragged(lr32, ctx.out_mask, B, rp, h2, w2, stream)
             : launch_upsample2x_argmax_ragged(lr, ctx.out_mask, B, rp, h2, w2, stream))
      return -1;
    if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
  } else if (ctx.out_mask) {
    if (lr32 ? launch_upsample2x_argmax(lr32, ctx.out_mask, B, ctx.K, h2, w2, stream)
             : launch_upsample2x_argmax(lr, ctx.out_mask, B, ctx.K, h2, w2, stream))
      return -1;
    if (note_launch(prof, launches, KIND_EW, 0.0, stream)) return -1;
  }
  return 0;
}

static int run_forward(lseg_engine* eng, const CallCtx& ctx, int B, int H, int W, cudaStream_t stream,
                       Profile* prof = nullptr) {
  if (ensure_init()) return -1;
  if (check_image_shape("lseg_forward", B, H, W)) return -1;
  if (ctx.K <= 0) {
    set_error("lseg_forward: K=%d labels", ctx.K);
    return -1;
  }
  LSEG_CHECK_CUDA(cudaSetDevice(eng->device));
  if (ensure_init()) return -1;
  ImagePlan* plan = image_plan(eng, B, H, W, stream);
  if (!plan) return -1;
  int launches = 0;
  if (run_trunk(eng, *plan, ctx, plan->featn, plan->feat_sumsq, stream, prof, &launches)) return -1;
  __half* lr = nullptr;
  if (run_tail(eng, ctx, B, H, W, plan->featn, plan->feat_sumsq, stream, prof, &launches, &lr)) return -1;
  plan->debug["logits_lr"] = lr;
  eng->last_launches = launches;
  return 0;
}

// ------------------------------------------------------------------------------------------
// CLIP text tower (SURVEY.md Appendix A.2): fp16 residual stream, fp32 LayerNorm statistics
// ------------------------------------------------------------------------------------------
static int build_text_plan(lseg_engine* eng, int K) {
  const lseg_weights& w = eng->w;
  std::unique_ptr<TextPlan> plan(new TextPlan());
  plan->K = K;
  Arena& arena = plan->arena;
  t_plan_arena = &arena;
  const int L = 77, Wd = w.text_width, OC = w.out_c, theads = w.text_heads;
  const long long M = static_cast<long long>(K) * L;
  const int kpad = ((K + 127) / 128) * 128;
  LSEG_ALLOC(tx, __half, M * Wd);
  LSEG_ALLOC(txn, __half, M * Wd);
  LSEG_ALLOC(tqkv, __half, M * 3 * Wd);
  LSEG_ALLOC(tattn, __half, M * Wd);
  LSEG_ALLOC(th, __half, M * 4 * Wd);
  LSEG_ALLOC(teot, __half, (size_t)kpad * Wd);
  LSEG_ALLOC(tfeat, __half, (size_t)kpad * OC);
  LSEG_CHECK_CUDA(cudaMemset(teot, 0, sizeof(__half) * (size_t)kpad * Wd));

  std::vector<Step> gsteps;  // reuse the image-side builders, then adapt
  auto& steps = plan->steps;
  auto wrap = [&steps](std::vector<Step>& src) {
    for (auto& st : src) {
      Step s = st;
      steps.push_back([s](const long long*, __half*, cudaStream_t stream) {
        CallCtx c;
        memset(&c, 0, sizeof(c));
        return s(c, stream);
      });
    }
    src.clear();
  };
  const float* tok_emb = w.tok_emb;
  const float* text_pos = w.text_pos;
  steps.push_back([=](const long long* tokens, __half*, cudaStream_t s) {
    text_embed_kernel<<<static_cast<unsigned>(M), 128, 0, s>>>(tokens, tok_emb, text_pos, tx, L, Wd);
    LSEG_CHECK_CUDA(cudaGetLastError());
    return 0;
  });
  for (int i = 0; i < LSEG_TEXT_DEPTH; ++i) {
    const lseg_text_block_w& bw = w.text_blocks[i];
    add_layernorm(gsteps, tx, 1, bw.ln1_g, bw.ln1_b, txn, M, Wd, 1e-5f);
    {
      GemmEpi e = epi_none();
      e.bias = bw.in_proj.b;
      e.out_f16 = tqkv;
      e.ldc = 3 * Wd;
      if (add_gemm(gsteps, txn, Wd, (int)M, (int)M, bw.in_proj, e)) return -1;
    }
    // causal attention with torch's fp16 rounding points (text_attn.cuh), not the flash kernel of the image trunk
    gsteps.push_back([=](const CallCtx&, cudaStream_t s) { return launch_text_attn(tqkv, tattn, K, L, theads, s); });
    {
      GemmEpi e = epi_none();
      e.bias = bw.out_proj.b;
      e.res_f16 = tx;
      e.out_f16 = tx;
      e.ldc = Wd;
      if (add_gemm(gsteps, tattn, Wd, (int)M, (int)M, bw.out_proj, e)) return -1;
    }
    add_layernorm(gsteps, tx, 1, bw.ln2_g, bw.ln2_b, txn, M, Wd, 1e-5f);
    {
      GemmEpi e = epi_none();
      e.bias = bw.c_fc.b;
      e.act = ACT_QUICKGELU;
      e.out_f16 = th;
      e.ldc = 4 * Wd;
      if (add_gemm(gsteps, txn, Wd, (int)M, (int)M, bw.c_fc, e)) return -1;
    }
    {
      GemmEpi e = epi_none();
      e.bias = bw.c_proj.b;
      e.res_f16 = tx;
      e.out_f16 = tx;
      e.ldc = Wd;
      if (add_gemm(gsteps, th, 4 * Wd, (int)M, (int)M, bw.c_proj, e)) return -1;
    }
    wrap(gsteps);
  }
  add_layernorm(gsteps, tx, 1, w.lnf_g, w.lnf_b, txn, M, Wd, 1e-5f);
  wrap(gsteps);
  steps.push_back([=](const long long* tokens, __half*, cudaStream_t s) {
    text_eot_gather_kernel<<<K, 128, 0, s>>>(tokens, txn, teot, K, L, Wd);
    LSEG_CHECK_CUDA(cudaGetLastError());
    return 0;
  });
  {
    GemmEpi e = epi_none();
    e.out_f16 = tfeat;
    e.ldc = OC;
    if (add_gemm(gsteps, teot, Wd, kpad, K, w.text_proj, e)) return -1;
    wrap(gsteps);
  }
  steps.push_back([=](const long long*, __half* out, cudaStream_t s) {
    LSEG_CHECK_CUDA(cudaMemsetAsync(out, 0, sizeof(__half) * (size_t)kpad * OC, s));
    l2norm_f16_kernel<<<(K + 7) / 8, 256, 0, s>>>(tfeat, out, K, OC);
    LSEG_CHECK_CUDA(cudaGetLastError());
    return 0;
  });
  eng->txt = std::move(plan);
  return 0;
}

// Rules of a ragged batch's label table, each rejected by name: image b's k[b] >= 1 labels are rows text_row[b] ..
// text_row[b] + k[b] - 1 of a 16-byte aligned text operand with text_rows readable rows; at most kRaggedMaxImages images;
// sum(k) <= 65535 packed planes (the output stage's grid limit). *sum_k = sum(k).
static int check_ragged(const char* fn, int B, const void* text, int text_rows, const int* text_row, const int* k,
                        long long* sum_k) {
  if (!text) return set_error("%s: null text", fn), -1;
  if (reinterpret_cast<uintptr_t>(text) % 16) return set_error("%s: text must be 16-byte aligned", fn), -1;
  if (!text_row) return set_error("%s: null text_row", fn), -1;
  if (!k) return set_error("%s: null k", fn), -1;
  if (B < 1) return set_error("%s: B=%d must be positive", fn, B), -1;
  if (B > kRaggedMaxImages) return set_error("%s: B=%d images exceed the cap of %d per call", fn, B, kRaggedMaxImages), -1;
  if (text_rows < 1) return set_error("%s: text_rows=%d must be positive", fn, text_rows), -1;
  long long sum = 0;
  for (int b = 0; b < B; ++b) {
    if (k[b] < 1) return set_error("%s: k[%d]=%d labels must be positive", fn, b, k[b]), -1;
    if (text_row[b] < 0 || static_cast<long long>(text_row[b]) + k[b] > text_rows)
      return set_error("%s: text_row[%d]=%d + k[%d]=%d exceeds text_rows=%d", fn, b, text_row[b], b, k[b], text_rows), -1;
    sum += k[b];
  }
  if (sum > 65535) return set_error("%s: sum of k = %lld exceeds 65535", fn, sum), -1;
  *sum_k = sum;
  return 0;
}

// Outputs of a ragged call: logits fp32 [sum k, H, W] and / or mask int64 [B, H, W], at least one; the x2 output stage
// reads rows of at most 2 * kUpMaxW pixels.
static int check_ragged_outputs(const char* fn, const float* logits, const long long* mask, int W) {
  if (!logits && !mask) return set_error("%s: no output requested (logits or mask)", fn), -1;
  if (logits && reinterpret_cast<uintptr_t>(logits) % 16) return set_error("%s: logits must be 16-byte aligned", fn), -1;
  if (mask && reinterpret_cast<uintptr_t>(mask) % 8) return set_error("%s: mask must be 8-byte aligned", fn), -1;
  if (W > 2 * kUpMaxW) return set_error("%s: W=%d must be <= %d", fn, W, 2 * kUpMaxW), -1;
  return 0;
}

}  // namespace lseg

extern "C" {

int lseg_create(const lseg_weights* w, int device, lseg_engine** out) {
  using namespace lseg;
  if (!w || !out) {
    set_error("lseg_create: null argument");
    return -1;
  }
  if (w->trunk != 0 && w->trunk != 1) {
    set_error("lseg_create: trunk %d (0 ViT, 1 ResNet-101)", w->trunk);
    return -1;
  }
  if (w->trunk == 1) {
    int nblk = 0;
    for (int k = 0; k < 4; ++k) nblk += w->rn_layers[k] > 0 ? w->rn_layers[k] : LSEG_RESNET_BLOCKS + 1;
    if (nblk > LSEG_RESNET_BLOCKS || !w->rn_stem.w) {
      set_error("lseg_create: ResNet trunk with %d blocks (at most %d) / missing stem", nblk, LSEG_RESNET_BLOCKS);
      return -1;
    }
  } else if (w->vit_heads <= 0 || w->vit_dim != 64 * w->vit_heads || (w->vit_dim != 768 && w->vit_dim != 1024) ||
      w->vit_depth <= 0 || w->vit_depth > LSEG_VIT_DEPTH || (w->patch_size != 16 && w->patch_size != 32) ||
      w->pos_grid <= 0) {
    set_error("lseg_create: backbone geometry dim=%d depth=%d heads=%d patch=%d pos_grid=%d (dim = 64*heads in {768, "
              "1024}, depth <= %d, patch 16 | 32)", w->vit_dim, w->vit_depth, w->vit_heads, w->patch_size, w->pos_grid,
              LSEG_VIT_DEPTH);
    return -1;
  }
  if ((w->text_width != 512 && w->text_width != 768) || w->text_width != 64 * w->text_heads ||
      (w->out_c != 512 && w->out_c != 768)) {
    set_error("lseg_create: text tower width=%d heads=%d out_c=%d (width = 64*heads in {512, 768}, out_c in {512, 768})",
              w->text_width, w->text_heads, w->out_c);
    return -1;
  }
  for (int k = 0; k < 4 && w->trunk == 0; ++k)
    if (w->hooks[k] < 0 || w->hooks[k] >= w->vit_depth || (k && w->hooks[k] <= w->hooks[k - 1])) {
      set_error("lseg_create: hooks must be increasing block indices below depth %d", w->vit_depth);
      return -1;
    }
  LSEG_CHECK_CUDA(cudaSetDevice(device));
  if (ensure_init()) return -1;
  lseg_engine* e = new lseg_engine();
  e->w = *w;
  e->device = device;
  *out = e;
  return 0;
}

void lseg_destroy(lseg_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  e->plans.clear();
  e->img = nullptr;
  e->txt.reset();
  for (auto& kv : e->pos_cache) cudaFree(kv.second);
  delete e;
}

int lseg_encode_text(lseg_engine* e, const int64_t* tokens, int K, void* text_out, void* stream) {
  using namespace lseg;
  if (!e || !tokens || !text_out || K <= 0) {
    set_error("lseg_encode_text: bad argument");
    return -1;
  }
  if (ensure_init()) return -1;
  LSEG_CHECK_CUDA(cudaSetDevice(e->device));
  if (!e->txt || e->txt->K != K) {
    e->txt.reset();
    if (build_text_plan(e, K)) return -1;
  }
  int launches = 0;
  for (auto& st : e->txt->steps) {
    if (st(reinterpret_cast<const long long*>(tokens), static_cast<__half*>(text_out),
           static_cast<cudaStream_t>(stream)))
      return -1;
    ++launches;
  }
  e->last_launches = launches;
  return 0;
}

int lseg_forward(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                 long long text_image_stride, float* out, void* stream) {
  using namespace lseg;
  if (!e || !x || !text || !out || B <= 0) {
    set_error("lseg_forward: bad argument");
    return -1;
  }
  CallCtx ctx;
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = out;
  ctx.out_mask = nullptr;
  ctx.out_lr = nullptr;
  return run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_forward_lowres(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                        long long text_image_stride, void* logits_lr, float* out, void* stream) {
  using namespace lseg;
  if (!e || !x || !text || !logits_lr || B <= 0) {
    set_error("lseg_forward_lowres: bad argument");
    return -1;
  }
  CallCtx ctx;
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = out;  // optional
  ctx.out_mask = nullptr;
  ctx.out_lr = static_cast<__half*>(logits_lr);
  return run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_forward_argmax(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                        long long text_image_stride, long long* mask, float* logits, void* stream) {
  using namespace lseg;
  if (!e || !x || !text || !mask || B <= 0) {
    set_error("lseg_forward_argmax: bad argument");
    return -1;
  }
  CallCtx ctx;
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = logits;  // optional
  ctx.out_mask = mask;
  ctx.out_lr = nullptr;
  return run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_forward_segstats(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                          long long text_image_stride, const long long* target, const int* group, int nclass, int G,
                          long long* stats, long long* mask, float* logits, void* stream) {
  using namespace lseg;
  SegStatsArgs st{target, group, stats, nclass, G};
  if (!e || !text) {
    set_error("lseg_forward_segstats: null %s", e ? "text" : "engine");
    return -1;
  }
  // everything the output stage would reject is checked here, before the forward enqueues its first kernel
  if (seg_stats_check("lseg_forward_segstats", x, st, B, H, W)) return -1;
  if (H % 32 != 0 || W % 32 != 0 || W > 2 * kUpMaxW || K <= 0) {
    set_error("lseg_forward_segstats: needs H, W multiples of 32, W <= %d, K > 0 (H=%d W=%d K=%d)", 2 * kUpMaxW, H, W, K);
    return -1;
  }
  CallCtx ctx;
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = logits;  // optional
  ctx.out_mask = mask;  // optional
  ctx.out_lr = nullptr;
  ctx.seg = &st;
  return run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream));
}

// The rules the fused loss adds to a forward / query: the metric arguments (all NULL, or target and stats given), the loss
// target (NULL: the metric target), accumulator and partials, and W <= 1024. Fills st / xe on success.
static int check_fused_xent(const char* fn, const void* input, int B, int H, int W, const long long* target, const int* group,
                            int nclass, int G, long long* stats, const long long* loss_target, long long ignore_index,
                            double* loss, double* partials, long long partials_len, lseg::SegStatsArgs* st,
                            lseg::XentArgs* xe) {
  using namespace lseg;
  *st = SegStatsArgs{target, group, stats, nclass, G};
  if ((target || group || stats) && seg_stats_check(fn, input, *st, B, H, W)) return -1;
  *xe = XentArgs{loss_target ? loss_target : target, ignore_index, partials, loss};
  if (B <= 0 || B > 65535) return set_error("%s: B=%d must be in [1, 65535]", fn, B), -1;
  if (H <= 0 || W <= 0) return set_error("%s: H=%d, W=%d must be positive", fn, H, W), -1;
  if (xent_check(fn, *xe, partials_len, xent_partials_fused(B, H))) return -1;
  if (W > 2 * kUpMaxW) return set_error("%s: W=%d must be <= %d with the loss", fn, W, 2 * kUpMaxW), -1;
  return 0;
}

int lseg_forward_xent(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                      long long text_image_stride, const long long* target, const int* group, int nclass, int G,
                      long long* stats, const long long* loss_target, long long ignore_index, double* loss,
                      double* partials, long long partials_len, long long* mask, float* logits, void* stream) {
  using namespace lseg;
  const char* fn = "lseg_forward_xent";
  // every rule is checked here, before the forward enqueues its first kernel
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!x) return set_error("%s: null x", fn), -1;
  if (!text) return set_error("%s: null text", fn), -1;
  if (K <= 0) return set_error("%s: K=%d labels must be positive", fn, K), -1;
  SegStatsArgs st;
  XentArgs xe;
  if (check_fused_xent(fn, x, B, H, W, target, group, nclass, G, stats, loss_target, ignore_index, loss, partials,
                       partials_len, &st, &xe))
    return -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  CallCtx ctx;
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = logits;     // optional
  ctx.out_mask = mask;  // optional
  ctx.out_lr = nullptr;
  ctx.seg = stats ? &st : nullptr;
  ctx.xent = &xe;
  return run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_forward_profiled(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                          long long text_image_stride, float* out, void* stream, float* step_ms, int* step_kind,
                          double* step_flops, int cap, int* count) {
  using namespace lseg;
  if (!e || !x || !text || !out || B <= 0 || !step_ms || !step_kind || !step_flops || !count) {
    set_error("lseg_forward_profiled: bad argument");
    return -1;
  }
  CallCtx ctx;
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = out;
  ctx.out_mask = nullptr;
  ctx.out_lr = nullptr;
  Profile prof;
  int rc = run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream), &prof);
  if (rc == 0 && cudaStreamSynchronize(static_cast<cudaStream_t>(stream)) != cudaSuccess) {
    set_error("lseg_forward_profiled: stream sync failed");
    rc = -1;
  }
  int n = 0;
  if (rc == 0) {
    n = static_cast<int>(prof.kind.size());
    if (n > cap) n = cap;
    for (int i = 0; i < n; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, prof.ev[i], prof.ev[i + 1]);
      step_ms[i] = ms;
      step_kind[i] = prof.kind[i];
      step_flops[i] = prof.flops[i];
    }
  }
  for (cudaEvent_t ev : prof.ev) cudaEventDestroy(ev);
  *count = n;
  return rc;
}

int lseg_encode_image(lseg_engine* e, const float* x, int B, int H, int W, void* emb, float* emb_sumsq, void* stream) {
  using namespace lseg;
  const char* fn = "lseg_encode_image";
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!x) return set_error("%s: null x", fn), -1;
  if (!emb) return set_error("%s: null emb", fn), -1;
  if (!emb_sumsq) return set_error("%s: null emb_sumsq", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb) % 16) return set_error("%s: emb must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb_sumsq) % 16) return set_error("%s: emb_sumsq must be 16-byte aligned", fn), -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  if (ensure_init()) return -1;
  LSEG_CHECK_CUDA(cudaSetDevice(e->device));
  if (ensure_init()) return -1;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  ImagePlan* plan = image_plan(e, B, H, W, s);
  if (!plan) return -1;
  CallCtx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.x = x;
  int launches = 0;
  if (run_trunk(e, *plan, ctx, static_cast<__half*>(emb), emb_sumsq, s, nullptr, &launches)) return -1;
  e->last_launches = launches;
  return 0;
}

int lseg_encode_image_attention(lseg_engine* e, const float* x, int B, int H, int W, void* emb, float* emb_sumsq,
                                float* const attn[4], void* stream) {
  using namespace lseg;
  const char* fn = "lseg_encode_image_attention";
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!x) return set_error("%s: null x", fn), -1;
  if (!emb) return set_error("%s: null emb", fn), -1;
  if (!emb_sumsq) return set_error("%s: null emb_sumsq", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb) % 16) return set_error("%s: emb must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb_sumsq) % 16) return set_error("%s: emb_sumsq must be 16-byte aligned", fn), -1;
  if (!attn) return set_error("%s: null attn", fn), -1;
  for (int k = 0; k < 4; ++k) {
    if (!attn[k]) return set_error("%s: null attn[%d]", fn, k), -1;
    if (reinterpret_cast<uintptr_t>(attn[k]) % 4) return set_error("%s: attn[%d] must be 4-byte aligned", fn, k), -1;
  }
  if (e->w.trunk != 0)
    return set_error("%s: the engine has no ViT trunk (ResNet-101 weights): there are no attention maps", fn), -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  if (static_cast<long long>(B) * e->w.vit_heads > 65535)
    return set_error("%s: B*heads = %lld exceeds 65535", fn, static_cast<long long>(B) * e->w.vit_heads), -1;
  if (ensure_init()) return -1;
  LSEG_CHECK_CUDA(cudaSetDevice(e->device));
  if (ensure_init()) return -1;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  ImagePlan* plan = image_plan(e, B, H, W, s, true);
  if (!plan) return -1;
  CallCtx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.x = x;
  ctx.attn = attn;
  int launches = 0;
  if (run_trunk(e, *plan, ctx, static_cast<__half*>(emb), emb_sumsq, s, nullptr, &launches)) return -1;
  e->last_launches = launches;
  return 0;
}

int lseg_query(lseg_engine* e, const void* emb, const float* emb_sumsq, int B, int H, int W, const void* text, int K,
               long long text_image_stride, float* logits, long long* mask, const long long* target, const int* group,
               int nclass, int G, long long* stats, void* stream) {
  using namespace lseg;
  const char* fn = "lseg_query";
  // every rule is checked here, before the first launch
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!emb) return set_error("%s: null emb", fn), -1;
  if (!emb_sumsq) return set_error("%s: null emb_sumsq", fn), -1;
  if (!text) return set_error("%s: null text", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb) % 16) return set_error("%s: emb must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb_sumsq) % 16) return set_error("%s: emb_sumsq must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(text) % 16) return set_error("%s: text must be 16-byte aligned", fn), -1;
  if (logits && reinterpret_cast<uintptr_t>(logits) % 16) return set_error("%s: logits must be 16-byte aligned", fn), -1;
  if (mask && reinterpret_cast<uintptr_t>(mask) % 8) return set_error("%s: mask must be 8-byte aligned", fn), -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  if (K <= 0) return set_error("%s: K=%d labels must be positive", fn, K), -1;
  if (text_image_stride < 0 || (text_image_stride > 0 && text_image_stride < K))
    return set_error("%s: text_image_stride=%lld must be 0 or >= K=%d", fn, text_image_stride, K), -1;
  const bool seg = target || stats || group;
  if (!logits && !mask && !seg) return set_error("%s: no output requested (logits, mask or stats)", fn), -1;
  SegStatsArgs st{target, group, stats, nclass, G};
  if (seg) {
    if (seg_stats_check(fn, emb, st, B, H, W)) return -1;
    if (W > 2 * kUpMaxW) return set_error("%s: W=%d must be <= %d with stats", fn, W, 2 * kUpMaxW), -1;
  }
  if (ensure_init()) return -1;
  LSEG_CHECK_CUDA(cudaSetDevice(e->device));
  if (ensure_init()) return -1;
  CallCtx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = logits;
  ctx.out_mask = mask;
  ctx.seg = seg ? &st : nullptr;
  int launches = 0;
  __half* lr = nullptr;
  if (run_tail(e, ctx, B, H, W, static_cast<const __half*>(emb), emb_sumsq, static_cast<cudaStream_t>(stream), nullptr,
               &launches, &lr))
    return -1;
  e->last_launches = launches;
  return 0;
}

int lseg_query_xent(lseg_engine* e, const void* emb, const float* emb_sumsq, int B, int H, int W, const void* text, int K,
                    long long text_image_stride, float* logits, long long* mask, const long long* target,
                    const int* group, int nclass, int G, long long* stats, const long long* loss_target,
                    long long ignore_index, double* loss, double* partials, long long partials_len, void* stream) {
  using namespace lseg;
  const char* fn = "lseg_query_xent";
  // every rule is checked here, before the first launch
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!emb) return set_error("%s: null emb", fn), -1;
  if (!emb_sumsq) return set_error("%s: null emb_sumsq", fn), -1;
  if (!text) return set_error("%s: null text", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb) % 16) return set_error("%s: emb must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb_sumsq) % 16) return set_error("%s: emb_sumsq must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(text) % 16) return set_error("%s: text must be 16-byte aligned", fn), -1;
  if (logits && reinterpret_cast<uintptr_t>(logits) % 16) return set_error("%s: logits must be 16-byte aligned", fn), -1;
  if (mask && reinterpret_cast<uintptr_t>(mask) % 8) return set_error("%s: mask must be 8-byte aligned", fn), -1;
  if (K <= 0) return set_error("%s: K=%d labels must be positive", fn, K), -1;
  if (text_image_stride < 0 || (text_image_stride > 0 && text_image_stride < K))
    return set_error("%s: text_image_stride=%lld must be 0 or >= K=%d", fn, text_image_stride, K), -1;
  SegStatsArgs st;
  XentArgs xe;
  if (check_fused_xent(fn, emb, B, H, W, target, group, nclass, G, stats, loss_target, ignore_index, loss, partials,
                       partials_len, &st, &xe))
    return -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  if (ensure_init()) return -1;
  LSEG_CHECK_CUDA(cudaSetDevice(e->device));
  if (ensure_init()) return -1;
  CallCtx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.text = static_cast<const __half*>(text);
  ctx.K = K;
  ctx.text_image_stride = text_image_stride;
  ctx.out = logits;
  ctx.out_mask = mask;
  ctx.seg = stats ? &st : nullptr;
  ctx.xent = &xe;
  int launches = 0;
  __half* lr = nullptr;
  if (run_tail(e, ctx, B, H, W, static_cast<const __half*>(emb), emb_sumsq, static_cast<cudaStream_t>(stream), nullptr,
               &launches, &lr))
    return -1;
  e->last_launches = launches;
  return 0;
}

int lseg_forward_ragged(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int text_rows,
                        const int* text_row, const int* k, float* logits, long long* mask, void* stream) {
  using namespace lseg;
  const char* fn = "lseg_forward_ragged";
  // every rule is checked here, before the first launch
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!x) return set_error("%s: null x", fn), -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  long long sum_k = 0;
  if (check_ragged(fn, B, text, text_rows, text_row, k, &sum_k)) return -1;
  if (check_ragged_outputs(fn, logits, mask, W)) return -1;
  CallCtx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.x = x;
  ctx.text = static_cast<const __half*>(text);
  ctx.K = static_cast<int>(sum_k);
  ctx.out = logits;
  ctx.out_mask = mask;
  ctx.rag_k = k;
  ctx.rag_text_row = text_row;
  ctx.rag_text_rows = text_rows;
  return run_forward(e, ctx, B, H, W, static_cast<cudaStream_t>(stream));
}

int lseg_query_ragged(lseg_engine* e, const void* emb, const float* emb_sumsq, int B, int H, int W, const void* text,
                      int text_rows, const int* text_row, const int* k, float* logits, long long* mask, void* stream) {
  using namespace lseg;
  const char* fn = "lseg_query_ragged";
  // every rule is checked here, before the first launch
  if (!e) return set_error("%s: null engine", fn), -1;
  if (!emb) return set_error("%s: null emb", fn), -1;
  if (!emb_sumsq) return set_error("%s: null emb_sumsq", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb) % 16) return set_error("%s: emb must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb_sumsq) % 16) return set_error("%s: emb_sumsq must be 16-byte aligned", fn), -1;
  if (check_image_shape(fn, B, H, W)) return -1;
  long long sum_k = 0;
  if (check_ragged(fn, B, text, text_rows, text_row, k, &sum_k)) return -1;
  if (check_ragged_outputs(fn, logits, mask, W)) return -1;
  if (ensure_init()) return -1;
  LSEG_CHECK_CUDA(cudaSetDevice(e->device));
  if (ensure_init()) return -1;
  CallCtx ctx;
  memset(&ctx, 0, sizeof(ctx));
  ctx.text = static_cast<const __half*>(text);
  ctx.K = static_cast<int>(sum_k);
  ctx.out = logits;
  ctx.out_mask = mask;
  ctx.rag_k = k;
  ctx.rag_text_row = text_row;
  ctx.rag_text_rows = text_rows;
  int launches = 0;
  __half* lr = nullptr;
  if (run_tail(e, ctx, B, H, W, static_cast<const __half*>(emb), emb_sumsq, static_cast<cudaStream_t>(stream), nullptr,
               &launches, &lr))
    return -1;
  e->last_launches = launches;
  return 0;
}

int lseg_embedding_features(const void* emb, const float* emb_sumsq, int B, int h, int w, int C, float* out,
                            void* stream) {
  using namespace lseg;
  const char* fn = "lseg_embedding_features";
  if (!emb) return set_error("%s: null emb", fn), -1;
  if (!emb_sumsq) return set_error("%s: null emb_sumsq", fn), -1;
  if (!out) return set_error("%s: null out", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb) % 16) return set_error("%s: emb must be 16-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(emb_sumsq) % 4) return set_error("%s: emb_sumsq must be 4-byte aligned", fn), -1;
  if (reinterpret_cast<uintptr_t>(out) % 16) return set_error("%s: out must be 16-byte aligned", fn), -1;
  if (B <= 0 || h <= 0 || w <= 0) return set_error("%s: B=%d, h=%d, w=%d must be positive", fn, B, h, w), -1;
  if (C != 512 && C != 768) return set_error("%s: C=%d must be 512 or 768", fn, C), -1;
  if (ensure_init()) return -1;
  return launch_embed_features(static_cast<const __half*>(emb), emb_sumsq, out, B, static_cast<long long>(h) * w, C,
                               static_cast<cudaStream_t>(stream));
}

const void* lseg_debug_buffer(lseg_engine* e, const char* name) {
  if (!e || !e->img || !name) return nullptr;
  auto it = e->img->debug.find(name);
  return it == e->img->debug.end() ? nullptr : it->second;
}

int lseg_last_launch_count(lseg_engine* e) { return e ? e->last_launches : 0; }

}  // extern "C"
