/* lseg_b200 — C ABI of the H100-native LSeg forward path (liblseg_b200.so).
 *
 * Drop-in boundary for the hot path of isl-org/lang-seg: LSegNet.forward
 * (modules/models/lseg_net.py:160-205) and its zero-shot twin (modules/models/lseg_net_zs.py:177-214).
 * The reference has no FFI (it is pure Python over torch); the binding a maintainer adds is the ctypes
 * shim shown in INTEGRATION.md, which replaces `self.net = LSegNet(...)` in modules/lseg_module.py:76-84.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer below is a DEVICE pointer unless it says "host";
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises
 *     except where stated;
 *   - every function returns 0 on success, non-zero on failure; lseg_last_error() returns a
 *     thread-local message. There is NO CPU fallback: without a CUDA device of compute capability
 *     9.0 every compute entry point fails.
 *   - fp16 tensors are IEEE binary16 ("half"); int64 tokens match clip.tokenize's LongTensor [K,77].
 */
#ifndef LSEG_B200_H_
#define LSEG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LSEG_B200_ABI_VERSION 4

/* ---- error / info ------------------------------------------------------------------------------ */
const char* lseg_last_error(void);
int lseg_abi_version(void);
/* Reads and clears the device-side barrier watchdog: out[0] != 0 means a kernel timed out on an
 * mbarrier (out[0] = wait tag, out[1] = block, out[2] = thread, out[3] = parity). Synchronises stream.
 * When no barrier timed out it reports instead the first image whose metric group id was outside [0, G) since the last
 * read (section "segmentation metrics"): out[0] = 78, out[1] = image, out[2] = its group id, out[3] = G. When neither is
 * pending, the first loss target outside [0, K) other than ignore_index (section "cross-entropy"): out[0] = 79,
 * out[1] = image, out[2] = pixel index y * W + x, out[3] = the target value (both clamped to int). */
int lseg_read_watchdog(int out[4], void* stream);

/* ---- stage ops (each one is parity-tested on its own; SURVEY.md section 2b numbering) ------------ */

/* activation applied in the GEMM epilogue */
enum { LSEG_ACT_NONE = 0, LSEG_ACT_GELU = 1, LSEG_ACT_QUICKGELU = 2, LSEG_ACT_RELU = 3 };
/* output addressing of the GEMM epilogue */
enum { LSEG_STORE_ROWMAJOR = 0, LSEG_STORE_D2S = 1, LSEG_STORE_NCHW_T = 2 };

/* One dense contraction  C[M,N] = epi(A[M,K] * W[N,K]^T)  on wgmma (k1,k4,k6-k8,k10-k17,k19).
 * K must be a multiple of 64 and a row-major ldc a multiple of 8. bias, scale, res_f32, res2_f32, res_f16, out_f32, out_f16
 * and out_f16_relu must be 16-byte aligned (the epilogue moves them with 16-byte vector accesses); lseg_gemm rejects a
 * call that breaks one of these rules with an error naming the operand, before it touches any memory.
 * Replaces the torch Linear / Conv2d(1x1, 3x3 s1 p1) / ConvTranspose2d(k==s) calls listed in
 * SURVEY.md section 8(a): timm Block linears (lseg_vit.py:196-197), ProjectReadout (lseg_vit.py:79-90),
 * act_postprocess convs (lseg_vit.py:450-522), scratch.layerN_rn (lseg_blocks.py:73-108),
 * ResidualConvUnit_custom convs (lseg_blocks.py:265-288), out_conv (lseg_blocks.py:356),
 * head1 and the pixel x text matmul (lseg_net.py:185,194). */
typedef struct lseg_gemm_args {
  const void* a;        /* plain: fp16 [a_rows >= M, lda]; conv: fp16 NHWC [B,H,W,K] */
  long long lda;        /* plain only, elements */
  int a_rows;           /* allocated rows of a (>= M) */
  const void* w;        /* fp16 [w_rows >= N, ksize*ksize*K] row-major, tap-major for conv */
  int w_rows;
  int M, N, K;          /* conv: M = B*H*W, K = input channels */
  int conv;             /* 0 plain, 1 = ksize x ksize stride-1 conv with zero padding `pad` */
  int B, H, W, ksize, pad;
  const float* bias;    /* [N] or [groups, N]; nullable */
  int bias_group_rows;  /* >0: row r uses bias row r / bias_group_rows */
  const float* scale;   /* [N], applied before bias; nullable */
  int act;
  const float* res_f32; /* nullable, row-major ldc */
  const float* res2_f32;/* nullable, second fp32 residual (fusion skip add, lseg_blocks.py:345-347) */
  const void* res_f16;  /* nullable, fp16 residual added in fp16 after rounding (CLIP text stream) */
  float* out_f32;       /* nullable */
  void* out_f16;        /* nullable */
  void* out_f16_relu;   /* nullable: fp16 relu(result) */
  long long ldc;
  int store;
  int d2s_s, d2s_cout, d2s_h, d2s_w;
  int nchw_p, nchw_k;
  int nchw_group;       /* LSEG_STORE_NCHW_T, > 0: the N columns are per-image blocks of nchw_group columns; a row of image
                         * b stores only columns [b*nchw_group, b*nchw_group + nchw_k) as channels 0..nchw_k-1 (the
                         * zero-shot path's per-image label pair, lseg_net_zs.py:196-210, as ONE GEMM) */
  /* deferred row normalisation (head1 -> pixel x text, lseg_net.py:185-194): a GEMM can write the partial
   * squared norms of its result rows, out_row_sumsq[row, n/32] = sum over that 32-column chunk (fp32, no
   * atomics: deterministic), and an LSEG_STORE_NCHW_T GEMM can scale each row by
   * row_scale * rsqrt(sum_i row_sumsq[row, i], i < row_sumsq_parts) before rounding to fp16. */
  const float* row_sumsq;
  int row_sumsq_parts;
  float row_scale;
  float* out_row_sumsq;
  int relu_after_res;   /* 1: ReLU after the fp32 residual add, on every output (torchvision Bottleneck: relu(bn3(conv3(..)) +
                         * identity), the ResNet-101 zero-shot trunk lseg_net_zs.py:307-310); row-major store, needs res_f32 */
} lseg_gemm_args;
int lseg_gemm(const lseg_gemm_args* args, void* stream);
/* Debug: plans the GEMM lseg_gemm would run for `args` (same checks, same error messages) without launching anything or
 * allocating, and describes the plan in out[5] (host):
 *   out[0] epilogue: 0 register-direct, 1 TMA fp16 store, 2 TMA fp32 reduce-add;
 *   out[1] grid (CTAs);
 *   out[2] 1 if stream-K balancing splits tiles' K ranges over CTAs (reduce-add epilogue, lseg_set_deterministic(0));
 *   out[3] fixed split-K segment count (>= 2: raw partials + a reduce kernel), 0 otherwise;
 *   out[4] kernel instantiation: 0 register-direct, 1 TMA fp16, 2 TMA reduce-add, 3 fixed split-K, 4 grouped NCHW store
 *          (nchw_group > 0), 5 ReLU after the fp32 residual. */
int lseg_debug_gemm_plan(const lseg_gemm_args* args, int out[5]);
/* Debug: for the same plan, out[0] = its cluster size (1, or 2: pairs of CTAs computing n-tiles 2j and 2j+1 of one m-tile,
 * each loading half of the shared A tile for both) and out[1] = the number of clusters it launches (out[1] * out[0] =
 * lseg_debug_gemm_plan's grid). Pairs are possible when the n-tile count is even and tiles are not split stream-K; the
 * planner uses them when the plan has more work units (tiles, or tiles x fixed split-K segments) than the device has SMs. */
int lseg_debug_gemm_cluster(const lseg_gemm_args* args, int out[2]);
/* Debug: how GEMMs planned after this call choose their cluster size: 1 = never pair CTAs, 2 = the planner's rule
 * (default), 3 = pair CTAs in every plan where that is possible. Results are bit-identical in all three modes. Any other
 * value is rejected. */
int lseg_debug_set_gemm_cluster(int mode);
/* Debug: image plans built after this call snapshot the intermediates of trunk block `block` (ViT block, or ResNet-101
 * bottleneck counted over all four stages) into buffers that lseg_debug_buffer names after a forward:
 *   ViT     trace_in (fp32 stream before LN1), trace_ln1, trace_qkv, trace_attn (fp16), trace_x1 (fp32 stream after
 *           proj), trace_ln2, trace_fc1 (fp16, after GELU), trace_out (fp32 stream after fc2);
 *   ResNet  trace_in (fp16 block input), trace_t1, trace_t2 (fp16 conv1 / conv2 outputs), trace_id (fp32 stream before
 *           conv3: the downsample output in a stage's first block), trace_out32 (fp32 stream after conv3), trace_out16.
 * The snapshots are device-to-device copies, not kernel launches, and change no other buffer. -1 (the default) turns the
 * trace off: plans then have no extra step. A block below -1 is rejected; a block at or beyond the trunk's block count
 * makes the next forward fail before anything is launched. Cached image plans are rebuilt after a change. */
int lseg_debug_set_trace_block(int block);

/* Fused MHSA, head_dim 64 (k5; timm Attention restated at lseg_vit.py:26-39; CLIP text MHA).
 * qkv fp16 [B, N, 3*heads*64] (q|k|v thirds) -> out fp16 [B*N, heads*64].
 * B, N and heads must be positive with B*heads <= 65535; qkv must be 16-byte aligned (TMA loads) and out 4-byte aligned
 * (__half2 stores). lseg_mhsa, lseg_mhsa_variant and lseg_mhsa_trace reject a call that breaks one of these rules with an
 * error naming the argument, before anything is launched. */
int lseg_mhsa(const void* qkv, void* out, int B, int N, int heads, int causal, void* stream);
/* Same contract as lseg_mhsa with an explicit kernel choice (A/B measurements; the engine runs variant 0 unless
 * LSEG_MHSA_VARIANT overrides it). One wgmma flash-attention kernel; the variants differ in how many exponentials are
 * evaluated on the FMA pipe instead of the MUFU pipe: 0, 1, 2, 5, 6 = none; 3, 7 = one of every four score pairs;
 * 4, 8 = two of four. */
int lseg_mhsa_variant(const void* qkv, void* out, int B, int N, int heads, int causal, int variant, void* stream);
/* Attention probabilities, head_dim 64, non-causal: the tensor the reference's attention hook records (get_attention,
 * lseg_vit.py:22-42). qkv fp16 [B, N, 3*heads*64] (q|k|v thirds, as lseg_mhsa reads it) -> out fp32 [B, heads, N, N],
 * contiguous: out[b, h, i, j] = softmax_j(0.125 * q_i . k_j) of head h, with q, k the fp16 rows, the scores accumulated
 * in fp32 by the tensor cores and normalised with the row's final max and sum (two passes over the keys). Only the
 * B*heads*N*N elements are written. Same rules as lseg_mhsa: B, N and heads positive with B*heads <= 65535; qkv 16-byte
 * aligned (TMA loads); out 4-byte aligned (the row pitch 4N is generally not a multiple of 16, so the kernel stores
 * single floats). A call that breaks one of them is rejected with an error naming the argument, before anything is
 * launched. Enqueued on `stream`. */
int lseg_attn_probs(const void* qkv, float* out, int B, int N, int heads, void* stream);
/* Causal attention of the CLIP text tower with the rounding points of torch's multi_head_attention_forward on fp16
 * tensors (q*dh^-0.5, bmm -> fp16, softmax -> fp16 normalised, bmm -> fp16; SURVEY.md Appendix A.2): CUDA cores, one
 * CTA per (label, head). qkv fp16 [K, L, 3*heads*64] -> out fp16 [K*L, heads*64]. 1 <= L <= 80, 1 <= K <= 65535 and
 * 1 <= heads <= 65535; qkv and out must be 4-byte aligned (__half2 loads and stores). A call that breaks one of these
 * rules is rejected with an error naming the argument, before anything is launched. */
int lseg_text_attn(const void* qkv, void* out, int K, int L, int heads, void* stream);
/* 1 (default): every floating-point sum is formed in a fixed order (bit-reproducible across runs and batch sizes).
 * 0 (or LSEG_SPLITK=1): an in-place fp32 residual GEMM without an activation (the MLP's fc2) may split a tile's K range
 * over two CTAs whose partial sums are reduce-added in arrival order (differences at the fp32 rounding level, hence off by default). */
int lseg_set_deterministic(int on);
/* Debug: GEMMs planned after this call stamp clock64() at the epilogue / MMA hand-off points of two CTAs, blockIdx.x 0
 * and gridDim.x / 2 (in a clustered plan, rank 0 of their pair when the cluster count is even), into trace
 * ([2][20 warps][512] uint64 device memory, zeroed by the caller; NULL switches it off). Row w of a CTA is
 * warp w: rows 4-7 are consumer warpgroup 0 and rows 8-11 warpgroup 1, each stamping only the tiles it owns (every
 * other entry of the CTA's work list); the other rows stay zero. Stamp = clock64() << 8 | tag. */
int lseg_debug_gemm_trace(unsigned long long* trace);
/* Debug: same computation and rules as lseg_mhsa (variant 0), additionally stamps clock64() at the pipeline hand-off
 * points of 16 sampled CTAs into trace ([16][10 warps][256] uint64 device memory, zero-initialised by the caller,
 * not NULL). */
int lseg_mhsa_trace(const void* qkv, void* out, int B, int N, int heads, int causal, unsigned long long* trace,
                    void* stream);

/* ---- glue entries (lseg_layernorm .. lseg_text_eot_gather, and lseg_preprocess) ----------------------------------------
 * Each rejects, naming itself and the argument, before anything is launched and with its outputs untouched:
 *   - a null pointer, or one not aligned to the kernel's vector width: 16 B for the float4 / uint4 operands (layernorm
 *     x, gamma, beta, y; patchify x; assemble_tokens; readout_split tap; the NHWC kernels' x and y; the nchw upsamples'
 *     x and y except the _bg source; l2norm_scale x), 8 B for uint2 stores and int64 tokens, else the element size;
 *   - a size that is not positive;
 *   - C % 8 != 0 for the uint4 NHWC kernels (im2col_3x3_s2, upsample2x_nhwc, maxpool, subsample), D % 4 != 0 for
 *     assemble_tokens / readout_split;
 *   - a shape the kernel is not built for: layernorm C not in {512, 768, 1024}; patch not in {16, 32} or not dividing
 *     H and W; odd H or W for stem_im2col / maxpool / subsample; l2norm_scale C not a multiple of 128 or above 512;
 *     W % 8 != 0 or W > 512 for upsample2x_nchw / _f32 / argmax, odd W for _bg; add with an fp16 nhwc256 output;
 *     head_block mode not 1 / 2 or act not 0..3;
 *   - a grid beyond its limit: 65535 in y / z (B of maxpool / subsample / the NHWC upsamples / im2col_3x3_s2, 2H of the
 *     NHWC upsamples, B*H/P of patchify, ceil(h/8) and B*K of head_block, ceil(Hp/8) of preprocess, planes of the
 *     nchw upsamples, B of upsample2x_argmax), 2^31 - 1 in x
 *     (B*(H/2)*(W/2) of stem_im2col, 1 + gh*gw of pos_resize, the token rows of assemble / readout / text_embed). */

/* LayerNorm over the last dim (k3): x fp32 (in_f16=0) or fp16 (in_f16=1) [M,C] -> y fp16. */
int lseg_layernorm(const void* x, int in_f16, const float* gamma, const float* beta, void* y, long long M, int C,
                   float eps, void* stream);

/* x fp32 NCHW [B,3,H,W] -> fp16 [B*(H/P)*(W/P), 3*P*P] patch rows (k1 operand), P = patch in {16, 32}. */
int lseg_patchify(const float* x, void* a, int B, int H, int W, int patch, void* stream);
/* bilinear (align_corners=False) resize of pos_embed [1+g0*g0, D] -> [1+gh*gw, D] (k2; lseg_vit.py:149-163). */
int lseg_pos_resize(const float* pos, float* out, int g0, int gh, int gw, int D, void* stream);
/* x[b] = cat(cls, patch[b]) + pos (lseg_vit.py:188-193); fp32. */
int lseg_assemble_tokens(const float* patch, const float* cls, const float* pos, float* x, int B, int T, int D,
                         void* stream);
/* tap fp32 [B,1+T,D] -> tok fp16 [B*T,D], cls fp16 [B,D] (k10 operands; lseg_vit.py:79-90). */
int lseg_readout_split(const float* tap, void* tok, void* cls, int B, int T, int D, void* stream);
/* NHWC fp16 [B,H,W,C] -> im2col rows for the 3x3 stride-2 pad-1 conv (k13; lseg_vit.py:516-522). */
int lseg_im2col_3x3_s2(const void* x, void* a, int B, int H, int W, int C, void* stream);
/* ResNet-101 trunk glue (lseg_net_zs.py:307-310, torchvision resnet101): rows of the 7x7 stride-2 pad-3 stem conv
 * (x fp32 NCHW [B,3,H,W] -> fp16 [B*(H/2)*(W/2), 192], column c*49 + ky*7 + kx, zero beyond 147); MaxPool2d(3, 2, 1) and
 * the pixel subsampling of a 1x1 stride-2 conv on NHWC fp16 [B,H,W,C] -> [B,H/2,W/2,C]. */
int lseg_stem_im2col(const float* x, void* a, int B, int H, int W, void* stream);
int lseg_maxpool3x3s2_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream);
int lseg_subsample2_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream);
/* bilinear x2 align_corners=True, NHWC fp16 (k16; lseg_blocks.py:352-354). */
int lseg_upsample2x_nhwc(const void* x, void* y, int B, int H, int W, int C, void* stream);
/* The same interpolation for the decoder width C = 256 as the engine runs it, AFTER the 1x1 out_conv
 * (lseg_blocks.py:352-356 — the two are linear per pixel and commute; conv first touches a quarter of the pixels):
 * x fp16 (in_f16 = 1, the engine's choice) or fp32 NHWC [B,H,W,256] -> y fp16 (out_f16 = 1) or fp32 [B,2H,2W,256].
 * add (nullable, fp32, output shape, fp32 output only) is summed into the result: xs[0] + ... of the next block
 * (lseg_blocks.py:345-347). */
int lseg_upsample2x_nhwc256(const void* x, int in_f16, void* y, int out_f16, const float* add, int B, int H, int W,
                            void* stream);
/* rows fp32 [M,C] -> half(row/||row||) * logit_scale in fp16 (k19 prologue; lseg_net.py:191,194). */
int lseg_l2norm_scale(const float* x, void* y, long long M, int C, float logit_scale, void* stream);
/* text rows fp16 [M,C] -> row/||row|| in fp16 (lseg_net.py:192). */
int lseg_l2norm_f16(const void* x, void* y, int M, int C, void* stream);
/* fp16 logits [planes,H,W] -> fp32 [planes,2H,2W], bilinear align_corners=True (k20; lseg_net.py:203). */
int lseg_upsample2x_nchw(const void* x, float* y, long long planes, int H, int W, void* stream);
/* A/B switch of lseg_upsample2x_nchw's shared-memory line layout (0 interleaved, 1 split by column parity); returns the
 * previous setting. Same values either way. Default: LSEG_UPSAMPLE_SPLIT or 0. */
int lseg_debug_upsample_layout(int split);
/* The same values bit for bit from a kernel built to run BESIDE the trunk of the next step on a side stream (no shared
 * memory, 128 threads x <= 32 registers, streaming stores): the gathering rank of the multi-GPU logits gather expands all
 * shards with it (lang-seg_b200/parallel.py). Slower than lseg_upsample2x_nchw when it has the GPU to itself. */
int lseg_upsample2x_nchw_bg(const void* x, float* y, long long planes, int H, int W, void* stream);
/* same from fp32 planes (after the arch_option 1 / 2 head blocks) */
int lseg_upsample2x_nchw_f32(const float* x, float* y, long long planes, int H, int W, void* stream);
/* Interpolate (lseg_blocks.py:113-147) fused with torch.max(., 1)[1]: lr fp16 [B,K,H,W] -> mask int64 [B,2H,2W]
 * (first maximal class; the interpolated values are those of lseg_upsample2x_nchw bit for bit). */
int lseg_upsample2x_argmax(const void* lr, long long* mask, int B, int K, int H, int W, void* stream);
/* One application of scratch.head_block (arch_option 1 / 2, lseg_net.py:29-79): the SAME 3x3 kernel w9 (+ bias) over every
 * class plane of x [B,K,h,w] (fp16 if in_f16 else fp32), mode 1 adds the per-pixel maximum over the K classes of the
 * INPUT (bottleneck_block), then the activation (LSEG_HEAD_ACT_*; the reference skips it on the last application).
 * y fp32 [B,K,h,w]; cmax_ws fp32 [B,h,w] workspace (mode 1). */
enum { LSEG_HEAD_ACT_NONE = 0, LSEG_HEAD_ACT_RELU = 1, LSEG_HEAD_ACT_LRELU = 2, LSEG_HEAD_ACT_TANH = 3 };
int lseg_head_block(const void* x, int in_f16, float* cmax_ws, float* y, int B, int K, int h, int w, const float* w9_host,
                    float bias, int mode, int act, void* stream);
/* CLIP text glue (k18; SURVEY.md Appendix A.2). tokens int64 [K,L]. */
int lseg_text_embed(const int64_t* tokens, const float* tok_emb, const float* pos_emb, void* x, int K, int L, int Wd,
                    void* stream);
int lseg_text_eot_gather(const int64_t* tokens, const void* x, void* out, int K, int L, int Wd, void* stream);

/* ---- multi-scale / flip / sliding-window evaluator glue (SURVEY.md section 8(f) row 1) ------------------------------------
 * Device side of LSeg_MultiEvalModule.forward (additional_utils/models.py:55-140): the chain of interpolate / pad / slice /
 * flip calls that builds every network input and the inverse chain over every network output, as three gather kernels.
 * Window geometry (which windows exist for which scale) is integer host logic and stays in lang-seg_b200/evaluator.py. */
typedef struct lseg_eval_window {
  int height, width;  /* the scale's resized image (int(h * long_size / w + 0.5) etc., models.py:69-80) */
  int h0, w0;         /* window origin in the padded resized image (idh * stride, idw * stride, models.py:113-114) */
  int flip;           /* this network input is the horizontally flipped crop (flip_image, models.py:161-165) */
  int out_index;      /* its position in the crop batch and of its output in the logits batch */
} lseg_eval_window;
/* img fp32 [3,h,w] -> crops fp32 [n_inputs,3,crop,crop]: pixel = bilinear(align_corners=True) sample of img at the
 * scale's coordinates, or pad3_host[c] (= -mean/std, pad_image models.py:145-156) outside the resized image. wins: DEVICE. */
int lseg_eval_make_crops(const float* img, float* crops, const lseg_eval_window* wins, int n_inputs, int h, int w, int crop,
                         const float* pad3_host, void* stream);
/* outs fp32 [n,K,crop,crop] (network outputs; a window's flipped input is the entry after its plain one when flip != 0)
 * -> canvas fp32 [K,height,width]: per pixel the (plain + flipped-back) outputs of the covering windows summed in list
 * order and divided by their count (models.py:117-132); whole != 0: single padded window, no division (models.py:82-89). */
int lseg_eval_canvas(const float* outs, float* canvas, const lseg_eval_window* wins, int n_win, int K, int crop, int height,
                     int width, int flip, int whole, void* stream);
/* scores fp32 [K,h,w] += bilinear(canvas [K,height,width] -> (h,w), align_corners=True) (models.py:133-136) */
int lseg_eval_resize_add(const float* canvas, float* scores, int K, int height, int width, int h, int w, void* stream);
/* ToTensor + Normalize + Resize([Ho,Wo]) (+ constant pad to [Hp,Wp]) of an 8-bit HWC image -> fp32 [3,Hp,Wp]
 * (lseg_app.py:328-334, modules/lseg_module.py:42-53; SURVEY.md section 8(f) row 3). img: DEVICE u8 [h,w,3]. */
int lseg_preprocess(const unsigned char* img_hwc, float* out, int h, int w, int Ho, int Wo, int Hp, int Wp,
                    const float* mean3_host, const float* std3_host, const float* pad3_host, void* stream);

/* ---- segmentation metrics: the counters behind pixAcc / mIoU (PyTorch-Encoding's SegmentationMetric, test_lseg.py:314-395)
 * and the few-shot mIoU / FB-IoU (Evaluator.classify_prediction + AverageMeter, test_lseg_zs.py:290-316) -----------------
 * stats is a caller buffer of G rows of int64 counters, 3*nclass + 2 per row:
 *     [ inter(nclass) | pred(nclass) | label(nclass) | correct | labeled ]
 * For every pixel of image b, with predicted class p and int64 target t, row g = group[b] (group: int32 [B], or NULL to
 * count every image into row 0; rows may repeat and G may exceed B):
 *     t < 0            : ignored (no counter changes)
 *     otherwise        : labeled += 1
 *       p == t         : correct += 1, and inter[t] += 1 if t < nclass
 *       0 <= p < nclass: pred[p] += 1
 *       t < nclass     : label[t] += 1
 * union = pred + label - inter. The calls ADD to stats and never clear it. A target >= nclass (e.g. 255) counts as labeled
 * and adds to pred only; a prediction >= nclass (K > nclass) adds to no histogram. An image whose group id lies outside
 * [0, G) is skipped and reported by lseg_read_watchdog (tag 78). Rejected by name before any launch: NULL pointers, stats
 * or target not 8-byte aligned, group not 4-byte aligned, nclass outside [1, 2^24], G <= 0, B outside [1, 65535],
 * H or W <= 0. nclass <= 1364 counts in shared memory, larger nclass with global atomics (same result). */
/* scores fp32 [B,K,H,W]: p = first maximal class (torch.max(scores, 1)[1] on NaN-free input; a NaN score never wins, a
 * pixel whose scores are all NaN or -inf gets class 0). target int64 [B,H,W]. */
int lseg_seg_stats_scores(const float* scores, const long long* target, const int* group, int B, int K, int H, int W,
                          int nclass, int G, long long* stats, void* stream);
/* pred int64 [B,H,W] (8-byte aligned): p = pred. */
int lseg_seg_stats_mask(const long long* pred, const long long* target, const int* group, int B, int H, int W, int nclass,
                        int G, long long* stats, void* stream);

/* ---- cross-entropy ----------------------------------------------------------------------------------------------------
 * The validation loss of LSegmentationModule.validation_step (modules/lsegmentation_module.py:86-105): PyTorch-Encoding's
 * SegmentationLosses with se_loss = aux = False and no class weight, i.e. CrossEntropyLoss(ignore_index) with mean
 * reduction. Per pixel with target t and fp32 logits v_0 .. v_{K-1}:
 *     t == ignore_index : skipped
 *     t outside [0, K)  : loss NaN, counted; the first such pixel is recorded (lseg_read_watchdog tag 79: image, pixel
 *                         index y * W + x, target value) instead of torch's device-side assert
 *     otherwise         : loss = (m + log s) - v_t, m = max_k v_k, s = sum_k exp(v_k - m) (online, classes in order)
 * in fp32 (expf / logf); a NaN logit gives a NaN loss. The calls ADD {sum of losses, counted pixels} to loss double[2]
 * (8-byte aligned) and never clear it: the mean is loss[0] / loss[1] (NaN when every pixel is ignored). Each block sums
 * its pixels in fp64 in a fixed order into a slot of `partials` and one further launch adds the slots in index order,
 * without floating-point atomics: the same call gives the same bits every time.
 * lseg_xent_scores: scores fp32 [B,K,H,W] (any H, W), target int64 [B,H,W]; partials_len >= 2 * B * ceil(H*W / 1024)
 * doubles. Rejected by name before any launch: NULL or misaligned pointers, B outside [1, 65535], K <= 0, H or W <= 0,
 * partials too short. */
int lseg_xent_scores(const float* scores, const long long* target, long long ignore_index, int B, int K, int H, int W,
                     double* loss, double* partials, long long partials_len, void* stream);

/* ---- peer memory: the logits gather (SURVEY.md section 8(e)), one process per GPU over NVLink 5 / NVSwitch ----------
 * Replaces the thread-per-GPU DataParallel gather of additional_utils/models.py:35-53. A rank allocates a buffer its peers
 * can map (CUDA IPC; the 64-byte handle travels through any host channel, e.g. torch.distributed.all_gather_object);
 * peers either let lseg_forward_lowres store into the mapping or push with the copy engines (lseg_p2p_copy), then
 * publish completion with a system-scope release flag that the gathering rank's stream acquires — all enqueued on CUDA
 * streams, no host synchronisation and no NCCL call on the data path. */
int lseg_p2p_alloc(unsigned long long bytes, void** dptr, unsigned char* handle64);  /* zero-initialised; synchronises */
int lseg_p2p_open(const unsigned char* handle64, void** dptr);   /* maps a peer's buffer into this process */
int lseg_p2p_close(void* dptr);
int lseg_p2p_free(void* dptr);
int lseg_p2p_copy(void* dst, const void* src, unsigned long long bytes, void* stream);  /* async, either side may be peer */
/* *flag = value with release semantics at system scope after all earlier work of `stream` (flag: own or peer memory) */
int lseg_p2p_signal(unsigned long long* flag, unsigned long long value, void* stream);
/* blocks `stream` (a one-thread kernel) until flags[i*stride] >= value for all i < n; after timeout_ms the device
 * watchdog records tag 77 (lseg_read_watchdog) and the stream continues */
int lseg_p2p_wait(const unsigned long long* flags, int n, int stride, unsigned long long value, unsigned int timeout_ms,
                  void* stream);

/* ---- whole-model engine -------------------------------------------------------------------------- */

typedef struct lseg_linear_w {
  const void* w;       /* fp16 [rows>=out, in] row-major, rows padded to a multiple of 128 */
  const float* b;      /* fp32 [out] or NULL */
  int out, in, rows;
} lseg_linear_w;

typedef struct lseg_vit_block_w {          /* timm Block (Appendix A.1) */
  const float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  lseg_linear_w qkv, proj, fc1, fc2;
} lseg_vit_block_w;

typedef struct lseg_rcu_w {                /* ResidualConvUnit_custom, BN folded to scale/shift */
  lseg_linear_w conv1, conv2;              /* [256, 9*256] tap-major */
  const float *bn1_scale, *bn1_shift, *bn2_scale, *bn2_shift;
} lseg_rcu_w;

typedef struct lseg_text_block_w {         /* CLIP ResidualAttentionBlock (Appendix A.2) */
  const float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
  lseg_linear_w in_proj, out_proj, c_fc, c_proj;
} lseg_text_block_w;

typedef struct lseg_bottleneck_w {         /* torchvision Bottleneck v1.5, BatchNorm (eval, eps 1e-5) folded to scale/shift */
  lseg_linear_w conv1, conv2, conv3, down; /* 1x1 [w, cin] | 3x3 [w, 9*w] tap-major | 1x1 [4w, w] | 1x1 [4w, cin], w NULL if absent */
  const float *bn1_scale, *bn1_shift, *bn2_scale, *bn2_shift, *bn3_scale, *bn3_shift, *bnd_scale, *bnd_shift;
  int stride;                              /* of conv2 and of the downsample conv: 1 | 2 */
} lseg_bottleneck_w;

#define LSEG_VIT_DEPTH 24
#define LSEG_TEXT_DEPTH 12
#define LSEG_RESNET_BLOCKS 33              /* resnet101: 3 + 4 + 23 + 3 */

typedef struct lseg_weights {
  /* image trunk: a timm VisionTransformer driven by forward_flex (lseg_vit.py:166-201). The geometry travels with
   * the weights: backbone "clip_vitl16_384" = vit_large_patch16_384 (D 1024, 24 blocks, 16 heads, patch 16, hooks
   * 5/11/17/23, lseg_vit.py:442-522), "clip_vitb32_384" = vit_base_patch32_384 (D 768, 12 blocks, 12 heads, patch 32,
   * hooks 2/5/8/11, lseg_vit.py:525-589). Head dim is 64 in both. */
  int vit_dim, vit_depth, vit_heads, patch_size;
  lseg_linear_w patch;                     /* [D, 3*patch^2] */
  const float* cls_token;                  /* [D] */
  const float* pos_embed;                  /* [1+pos_grid^2, D] */
  int pos_grid;                            /* 384 / patch: 24 | 12 */
  lseg_vit_block_w blocks[LSEG_VIT_DEPTH]; /* the first vit_depth entries */
  int hooks[4];                            /* lseg_net.py:119-123 */
  /* reassemble (lseg_vit.py:442-589) */
  lseg_linear_w readout_tok[4];            /* W[:, :D]  */
  lseg_linear_w readout_cls[4];            /* W[:, D:] with the bias */
  lseg_linear_w post_conv1x1[4];           /* D -> post_channels[k] */
  int post_channels[4];                    /* STORED widths, multiples of 64: {256,512,1024,1024} | {128,192,384,768}
                                              (the reference's 96 is padded to 128 with zero weights / bias) */
  int post_resample[4];                    /* s > 0: ConvTranspose2d(k=s, stride=s); 0: none; -2: Conv2d 3x3 stride 2.
                                              {4,2,0,-2} | {8,4,2,0} */
  lseg_linear_w post_resample_w[4];        /* ConvT: [(i*s+j)*C+co, ci], bias expanded [s*s*C]; conv: [C, 9*C] tap-major;
                                              unused (w NULL) where post_resample == 0 */
  /* decoder (lseg_blocks.py:60-110, 222-358) */
  lseg_linear_w layer_rn[4];               /* [256, 9*post_channels[k]] tap-major, no bias */
  lseg_rcu_w rcu1[4], rcu2[4];             /* index i = refinenet(i+1); rcu1[3] is dead (lseg_net.py:176) */
  lseg_linear_w out_conv[4];               /* [256,256] + bias */
  lseg_linear_w head1;                     /* [out_c,256] + bias */
  float logit_scale;                       /* exp(log(1/0.07)) (lseg_net.py:141) */
  /* CLIP text tower: ViT-B/32's (width 512, 8 heads, embedding 512) for clip_vitl16_384 / clip_vitb32_384, RN50x16's
   * (width 768, 12 heads, embedding 768) for clipRN50x16_vitl16_384 (lseg_vit.py:221-257, lseg_net.py:142-146).
   * out_c = embedding width = rows of head1 = K dim of the pixel x text product. Head dim 64. */
  int text_width, text_heads, out_c;
  const float* tok_emb;                    /* [49408, text_width] fp32 */
  const float* text_pos;                   /* [77, text_width] fp32 */
  lseg_text_block_w text_blocks[LSEG_TEXT_DEPTH];
  const float *lnf_g, *lnf_b;
  lseg_linear_w text_proj;                 /* text_projection^T as [out_c(out), text_width(in)], no bias */
  /* optional head blocks over the class planes (lseg_net.py:29-79,148-154,198-201) */
  int arch_option;                         /* 0 none (default), 1 bottleneck_block, 2 depthwise_block */
  int block_depth;                         /* the block runs max(block_depth, 1) times, activation on all but the last */
  int head_act;                            /* LSEG_HEAD_ACT_* of kwargs["activation"] */
  float head_block_w[9];                   /* scratch.head_block.depthwise.depthwise.weight [1,1,3,3] */
  float head_block_b;                      /* ... .bias [1] */
  /* image trunk selector: 0 = ViT (everything above "decoder"), 1 = ResNet-101 (backbone "clip_resnet101" of the
   * zero-shot model LSegRNNetZS, lseg_net_zs.py:240-339: pretrained.layer1..4 = torchvision resnet101 stages feed
   * scratch.layerN_rn directly; post_channels = {256, 512, 1024, 2048}; the ViT / reassemble fields are ignored) */
  int trunk;
  lseg_linear_w rn_stem;                   /* conv1 7x7 s2 p3 as [64, 192]: column c*49 + ky*7 + kx, zero beyond 147 */
  const float *rn_stem_scale, *rn_stem_shift;
  int rn_layers[4];                        /* blocks per stage: 3, 4, 23, 3 */
  lseg_bottleneck_w rn_blocks[LSEG_RESNET_BLOCKS];
} lseg_weights;

typedef struct lseg_engine lseg_engine;

/* Copies the descriptor (pointers are borrowed; the caller keeps the device buffers alive). */
int lseg_create(const lseg_weights* w, int device, lseg_engine** out);
void lseg_destroy(lseg_engine* e);

/* clip_pretrained.encode_text + L2 normalisation (lseg_net.py:183,192).
 * tokens int64 [K,77] -> text fp16 [rows_padded(K), 512], rows >= K zeroed; rows_padded = ceil(K/128)*128. */
int lseg_encode_text(lseg_engine* e, const int64_t* tokens, int K, void* text_out, void* stream);

/* Stream contract of every lseg_engine call: all work is enqueued on `stream` (nothing on the legacy default stream, no
 * host synchronisation once the launch plan of a batch shape exists). An engine owns ONE set of activation buffers per
 * cached shape, so calls on the same engine must be ordered — same stream, or event-ordered across streams; two forwards
 * in flight on two streams corrupt each other. Independent concurrency = one engine per stream / thread (weights shared by
 * pointer: the descriptor only borrows them). */
/* LSeg.forward after tokenisation (lseg_net.py:166-205).
 * x fp32 NCHW [B,3,H,W] (H, W multiples of 32) -> out fp32 NCHW [B,K,H,W].
 * text fp16 [rows_padded(K),512] shared by all images (text_image_stride = 0), or one K-row block per
 * image at text + b*text_image_stride*512 halves, text_image_stride >= K, total rows padded to a multiple of 128
 * (zero-shot path, lseg_net_zs.py:196-210). */
int lseg_forward(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                 long long text_image_stride, float* out, void* stream);

/* LSeg.forward up to the fp16 matmul result (lseg_net.py:194-196): logits_lr fp16 [B,K,H/2,W/2] is written to the CALLER's
 * buffer, which may be PEER memory of another GPU (an address obtained with lseg_p2p_open): the pixel x text GEMM's
 * epilogue then stores straight into the gathering rank's buffer over NVLink — the one collective of the path
 * (SURVEY.md section 8(e)) fused into the kernel that produces the data. `out` (fp32 [B,K,H,W]) is optional (NULL: the
 * x2 upsample, lseg_net.py:203, is left to the gathering rank: lseg_upsample2x_nchw on the gathered planes is bit-identical).
 * text_image_stride > 0: rows [b*stride, b*stride + K) of `text` are image b's label block (stride >= K; any value). */
int lseg_forward_lowres(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                        long long text_image_stride, void* logits_lr, float* out, void* stream);

/* SURVEY.md 8(f) "next" row 2 — LSeg.forward fused with the torch.max(logits, 1)[1] every caller applies
 * (lseg_app.py:357-360, test_lseg.py:397, test_lseg_zs.py:301): mask int64 [B,H,W] = index of the first maximal class
 * of the (bilinearly upsampled, align_corners=True) logits, bit-identical to argmax over what lseg_forward returns.
 * The fp32 [B,K,H,W] logits are not materialised unless `logits` is non-NULL (then both are produced). */
int lseg_forward_argmax(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                        long long text_image_stride, long long* mask, float* logits, void* stream);

/* lseg_forward_argmax with the metric counters of section "segmentation metrics" fused into the same output kernel:
 * target int64 [B,H,W], group int32 [B] or NULL, stats int64 [G, 3*nclass + 2] (accumulated). The argmax p is the mask
 * lseg_forward_argmax computes; `mask` (int64 [B,H,W]) and `logits` (fp32 [B,K,H,W]) are optional outputs, NULL to skip
 * them. Needs W <= 1024 besides lseg_forward's rules; every argument is checked before the first launch. */
int lseg_forward_segstats(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                          long long text_image_stride, const long long* target, const int* group, int nclass, int G,
                          long long* stats, long long* mask, float* logits, void* stream);

/* lseg_forward_segstats with the validation cross-entropy fused into the same output kernel (section "cross-entropy"):
 * adds {sum of per-pixel losses, counted pixels} of the logits lseg_forward returns against loss_target int64 [B,H,W]
 * to loss double[2]. loss_target NULL means the metric target. The metric (target, group, nclass, G, stats as in
 * lseg_forward_segstats) is optional here: target, group and stats all NULL, or target and stats given. mask and logits
 * are optional outputs with the bits lseg_forward_argmax / lseg_forward write. partials: caller workspace of
 * partials_len >= 2 * B * ceil(H / 8) doubles, 8-byte aligned. Needs W <= 1024 besides lseg_forward's rules; every
 * argument is checked, and rejected by name, before the first launch. */
int lseg_forward_xent(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                      long long text_image_stride, const long long* target, const int* group, int nclass, int G,
                      long long* stats, const long long* loss_target, long long ignore_index, double* loss,
                      double* partials, long long partials_len, long long* mask, float* logits, void* stream);

/* Same as lseg_forward, but brackets every kernel launch with CUDA events on `stream`, synchronises,
 * and returns per-launch device time (ms), kernel class (0 elementwise, 1 wgmma GEMM, 2 MHSA,
 * 3 LayerNorm) and ALGORITHMIC flops of the launch. Used by bench.py for the roofline block. */
int lseg_forward_profiled(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int K,
                          long long text_image_stride, float* out, void* stream, float* step_ms, int* step_kind,
                          double* step_flops, int cap, int* count);

/* Encode once, query many times. LSeg.forward splits at the pixel embedding (lseg_net.py:185-191): the image path
 * (ViT or ResNet trunk, reassemble, decoder, head1) depends on the image only; the pixel x text product, the arch_option
 * head blocks and the x2 output stage depend on the labels. lseg_encode_image runs the first part into a caller's
 * buffers; lseg_query runs the second part on them, as often as wanted, with any label set.
 *
 * Embedding layout: the engine's own internal pair, for B images of H x W (h = H/2, w = W/2, P = h*w pixels per image,
 * C = out_c of the weights):
 *   emb        fp16 [B, h, w, C]     head1's output rows, NOT normalised
 *   emb_sumsq  fp32 [B, h, w, C/32]  partial squared norms of the fp32 accumulators behind those rows (column chunks of
 *                                    32), summed in index order where the norm is needed
 * This pair is what the pixel x text GEMM's epilogue consumes (it applies logit_scale / ||row|| per pixel row), so a
 * query is bit-identical to the forward of the image that produced it; exporting any other form (normalised, fp32,
 * NCHW) would round differently and break that identity. lseg_embedding_features converts the pair into the reference's
 * image_features. Both buffers are 16-byte aligned; an embedding stays valid as long as the caller keeps it (the engine
 * holds no reference to it) and only for the weights it was encoded with.
 *
 * lseg_encode_image: x fp32 NCHW [B,3,H,W] (H, W multiples of 32) -> emb, emb_sumsq. Same launches as lseg_forward's
 * image path; head1 stores straight into the caller's buffers. */
int lseg_encode_image(lseg_engine* e, const float* x, int B, int H, int W,
                      void* emb /* fp16 [B,H/2,W/2,out_c] */, float* emb_sumsq /* fp32 [B,H/2,W/2,out_c/32] */, void* stream);

/* lseg_encode_image that also records the ViT's attention maps (the reference's enable_attention_hooks, lseg_vit.py:428-441:
 * pretrained.attention["attn_1".."attn_4"]). Same launches and output bits as lseg_encode_image, plus one launch per
 * hooked block: attn[k] receives fp32 [B, heads, N, N] (N = (H/patch)*(W/patch) + 1 tokens, contiguous) = the softmax
 * probabilities of block hooks[k] (lseg_attn_probs on that block's QKV rows, run right after the block's attention, while
 * the rows are still in the workspace). The four buffers belong to the caller (no workspace grows); each must be non-NULL
 * and 4-byte aligned, and the engine must have a ViT trunk (not the ResNet-101 one). Every rule is checked, and rejected
 * by name, before the first launch. Plans that record attention are cached apart from those that do not, so a forward
 * without it runs exactly the launches it ran before. */
int lseg_encode_image_attention(lseg_engine* e, const float* x, int B, int H, int W, void* emb, float* emb_sumsq,
                                float* const attn[4], void* stream);

/* The label-dependent tail of LSeg.forward on an embedding of B images of H x W. text / K / text_image_stride as in
 * lseg_forward. Outputs, each nullable, at least one requested; each equals what the corresponding forward entry point
 * writes for the image that produced `emb`, bit for bit:
 *   logits  fp32 [B,K,H,W]  (lseg_forward)
 *   mask    int64 [B,H,W]   (lseg_forward_argmax)
 *   stats   int64 [G, 3*nclass + 2], accumulated, with target int64 [B,H,W] and group int32 [B] or NULL
 *           (lseg_forward_segstats; W <= 1024). target, group and stats are all NULL, or target and stats are given.
 * Every argument is checked, and rejected by name, before the first launch. A query at a shape the engine never ran a
 * forward at allocates only the tail's buffers (fp16 [B,K,H/2,W/2] low-res logits; fp32 head-block planes with
 * arch_option 1 / 2), never the image path's activations. */
int lseg_query(lseg_engine* e, const void* emb, const float* emb_sumsq, int B, int H, int W,
               const void* text, int K, long long text_image_stride,
               float* logits, long long* mask,
               const long long* target, const int* group, int nclass, int G, long long* stats,
               void* stream);

/* lseg_query with the cross-entropy of lseg_forward_xent: same loss arguments and rules, same result bit for bit as
 * lseg_forward_xent on the image that produced `emb`. */
int lseg_query_xent(lseg_engine* e, const void* emb, const float* emb_sumsq, int B, int H, int W,
                    const void* text, int K, long long text_image_stride,
                    float* logits, long long* mask,
                    const long long* target, const int* group, int nclass, int G, long long* stats,
                    const long long* loss_target, long long ignore_index, double* loss, double* partials,
                    long long partials_len, void* stream);

/* Ragged batch: every image brings its own label set (open-vocabulary serving: one prompt per request, batched for
 * throughput). Image b's k[b] labels are rows text_row[b] .. text_row[b] + k[b] - 1 of ONE packed text operand `text`
 * (fp16 [text_rows, out_c], L2-normalised rows as lseg_encode_text writes them, 16-byte aligned); blocks may overlap or
 * be shared. Image b's pixels meet only its own labels: the pixel x text GEMM is one launch over the tiles of each
 * image's own pixel rows x its own text rows, not over the union of the label sets. Outputs are packed by image, with
 * koff[b] = k[0] + ... + k[b-1]:
 *   logits  fp32 [sum k, H, W]  image b's logits are planes koff[b] .. koff[b] + k[b] - 1
 *   mask    int64 [B, H, W]     mask[b] indexes image b's own labels (first maximal label, as lseg_forward_argmax)
 * each nullable, at least one requested. Image b's planes and mask equal, bit for bit, what lseg_forward /
 * lseg_forward_argmax write for that image alone (B = 1) with its k[b] rows as the label set. k and text_row are HOST
 * arrays of B ints (the planner needs the tile counts; nothing is read back from the device). Rules, each checked and
 * rejected by name before the first launch: 1 <= B <= 64 images (the per-image tables travel in kernel parameters),
 * k[b] >= 1, 0 <= text_row[b] and text_row[b] + k[b] <= text_rows, sum k <= 65535, H and W positive multiples of 32,
 * W <= 1024. arch_option 1 / 2 runs the head blocks once per image (their channel max is over the image's own labels).
 * Stream contract as for the other engine calls: everything is enqueued on `stream`; the host arrays may be reused as
 * soon as the call returns. */
int lseg_forward_ragged(lseg_engine* e, const float* x, int B, int H, int W, const void* text, int text_rows,
                        const int* text_row, const int* k, float* logits, long long* mask, void* stream);

/* lseg_forward_ragged's label-dependent tail on an embedding pair (lseg_encode_image) of B images of H x W; same tables,
 * outputs and rules. Allocates only the tail's buffers, like lseg_query. */
int lseg_query_ragged(lseg_engine* e, const void* emb, const float* emb_sumsq, int B, int H, int W, const void* text,
                      int text_rows, const int* text_row, const int* k, float* logits, long long* mask, void* stream);

/* Stage op: the ragged pixel x text GEMM alone. a fp16 [B*P, C] row-major (P pixels per image, a multiple of 128; C a
 * multiple of 64), text / text_rows / text_row / k as in lseg_forward_ragged -> out fp16 [sum k, P]: plane koff[b] + j =
 * image b's pixel rows times its text row text_row[b] + j, scaled per row by row_scale * rsqrt(sum of the row's
 * row_sumsq_parts entries of row_sumsq fp32 [B*P, parts]) when row_sumsq is non-NULL (the engine's normalisation),
 * unscaled when it is NULL. Only those planes are written. Enqueued on `stream`. */
int lseg_gemm_ragged(const void* a, const float* row_sumsq, int row_sumsq_parts, float row_scale, int B, int P, int C,
                     const void* text, int text_rows, const int* text_row, const int* k, void* out, void* stream);

/* The reference's normalised pixel embedding image_features (lseg_net.py:187-191) from an embedding pair of B images
 * with an h x w grid: out fp32 NCHW [B, C, h, w] = emb * rsqrt(sum of the C/32 partials, in index order). C in
 * {512, 768}; h*w a multiple of 4; emb and out 16-byte aligned. No engine needed. */
int lseg_embedding_features(const void* emb, const float* emb_sumsq, int B, int h, int w, int C, float* out, void* stream);

/* Introspection for tests: copies of intermediate activations of the last forward (device pointers
 * into the workspace, valid until the next forward). name: "tap0".."tap3" fp32 [B,N,1024];
 * "path1" fp16 NHWC [B,H/2,W/2,256]; "logits_lr" fp16 [B,K,H/2,W/2]. Returns NULL if unknown. */
const void* lseg_debug_buffer(lseg_engine* e, const char* name);

/* Number of kernel launches issued by the last lseg_forward / lseg_encode_text call. */
int lseg_last_launch_count(lseg_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* LSEG_B200_H_ */
