"""Stage-level ops of the LSeg forward path on torch CUDA tensors (thin wrappers over the C ABI).

torch supplies device memory and the current stream only; every computation happens inside
liblseg_b200.so. Each wrapper validates dtype/contiguity (the C side takes raw pointers) and
raises LsegError with the library's message on failure.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import (ACT_GELU, ACT_NONE, ACT_QUICKGELU, ACT_RELU, STORE_D2S, STORE_NCHW_T, STORE_ROWMAJOR,  # noqa: F401
                   GemmArgs, check, load)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t, dtype=None):
    if t is None:
        return None
    if not t.is_cuda:
        raise ValueError("lseg_b200 ops take CUDA tensors (there is no CPU fallback)")
    if not t.is_contiguous():
        raise ValueError("tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise ValueError(f"expected {dtype}, got {t.dtype}")
    return C.c_void_p(t.data_ptr())


def _out(out, shape, dtype, device, what):
    """The output buffer of a glue op: a fresh torch.empty, or the caller's tensor, which must be exactly a contiguous
    `dtype` tensor of `shape` on `device` (the kernels write that many elements through a raw pointer, unchecked)."""
    shape = tuple(int(v) for v in shape)
    if out is None:
        return torch.empty(shape, dtype=dtype, device=device)
    if out.dtype != dtype or tuple(out.shape) != shape or out.device != torch.device(device) or not out.is_contiguous():
        raise _lib.LsegError(f"{what}: out must be a contiguous {dtype} {list(shape)} tensor on {device}, got "
                             f"{out.dtype} {list(out.shape)} on {out.device}{'' if out.is_contiguous() else ' (strided)'}")
    return out


def pad_rows(w, mult=128):
    """Weights are [N, K] fp16 with rows padded to a multiple of 128 (TMA box never exceeds the tensor)."""
    n = w.shape[0]
    npad = (n + mult - 1) // mult * mult
    if npad == n:
        return w.contiguous()
    out = torch.zeros((npad,) + tuple(w.shape[1:]), dtype=w.dtype, device=w.device)
    out[:n] = w
    return out


def read_watchdog():
    arr = (C.c_int * 4)()
    check(load().lseg_read_watchdog(C.byref(arr), _stream()))
    return list(arr)


def _gemm_args(a, w, N=None, *, bias=None, bias_group_rows=0, scale=None, act=ACT_NONE, res_f32=None, res2_f32=None,
               res_f16=None, out_f32=None, out_f16=None, out_f16_relu=None, ldc=None, M=None,
               conv=None, store=STORE_ROWMAJOR, d2s=None, nchw=None, row_sumsq=None, row_scale=1.0, out_row_sumsq=None,
               relu_after_res=False):
    args = GemmArgs()
    args.a = _ptr(a, torch.float16)
    args.w = _ptr(w, torch.float16)
    args.w_rows = w.shape[0]
    args.N = N if N is not None else w.shape[0]
    if conv is not None:
        B, H, W_, Cc = a.shape
        args.conv, args.B, args.H, args.W, args.ksize, args.pad = 1, B, H, W_, conv[0], conv[1]
        args.M, args.K = B * H * W_, Cc
    else:
        args.lda = a.stride(0)
        args.a_rows = a.shape[0]
        args.M = M if M is not None else a.shape[0]
        args.K = a.shape[1]
    args.bias = _ptr(bias, torch.float32)
    args.bias_group_rows = bias_group_rows
    args.scale = _ptr(scale, torch.float32)
    args.act = act
    args.res_f32 = _ptr(res_f32, torch.float32)
    args.res2_f32 = _ptr(res2_f32, torch.float32)
    args.res_f16 = _ptr(res_f16, torch.float16)
    args.out_f32 = _ptr(out_f32, torch.float32)
    args.out_f16 = _ptr(out_f16, torch.float16)
    args.out_f16_relu = _ptr(out_f16_relu, torch.float16)
    args.ldc = ldc if ldc is not None else args.N
    args.store = store
    if d2s is not None:
        args.d2s_s, args.d2s_cout, args.d2s_h, args.d2s_w = d2s
    if nchw is not None:
        args.nchw_p, args.nchw_k = nchw[0], nchw[1]
        args.nchw_group = nchw[2] if len(nchw) > 2 else 0
    args.row_sumsq = _ptr(row_sumsq, torch.float32)
    args.row_sumsq_parts = int(row_sumsq.shape[1]) if row_sumsq is not None else 0
    args.row_scale = float(row_scale)
    args.out_row_sumsq = _ptr(out_row_sumsq, torch.float32)
    args.relu_after_res = int(bool(relu_after_res))
    return args


def gemm(a, w, N=None, **kw):
    """C = epi(A W^T).  a: fp16 [M,K] (or NHWC [B,H,W,C] when conv=(ksize,pad)); w: fp16 [rows>=N, Ktot].
    Keywords: see _gemm_args and lseg_gemm_args in include/lseg_b200.h."""
    check(load().lseg_gemm(C.byref(_gemm_args(a, w, N, **kw)), _stream()))


def gemm_plan(a, w, N=None, **kw):
    """The plan gemm(a, w, N, **kw) would run, without running it (include/lseg_b200.h lseg_debug_gemm_plan):
    dict with epi (0 direct, 1 TMA fp16, 2 TMA reduce-add), grid, split_k, split_fixed and kernel (instantiation)."""
    out = (C.c_int * 5)()
    check(load().lseg_debug_gemm_plan(C.byref(_gemm_args(a, w, N, **kw)), C.byref(out)))
    return dict(zip(("epi", "grid", "split_k", "split_fixed", "kernel"), out))


def gemm_cluster(a, w, N=None, **kw):
    """Cluster layout of the plan gemm(a, w, N, **kw) would run (include/lseg_b200.h lseg_debug_gemm_cluster):
    dict with cluster (1, or 2 for CTA pairs sharing the A tile) and clusters (how many it launches)."""
    out = (C.c_int * 2)()
    check(load().lseg_debug_gemm_cluster(C.byref(_gemm_args(a, w, N, **kw)), C.byref(out)))
    return dict(zip(("cluster", "clusters"), out))


def set_gemm_cluster(mode):
    """How later GEMM plans pick their cluster size (lseg_debug_set_gemm_cluster): 1 never pair CTAs, 2 the planner's
    rule (default), 3 pair CTAs wherever possible."""
    check(load().lseg_debug_set_gemm_cluster(int(mode)))


def set_trace_block(block):
    """Snapshot the intermediates of trunk block `block` in later image plans (lseg_debug_set_trace_block: trace_* debug
    buffers after a forward); -1 turns the trace off (the default)."""
    check(load().lseg_debug_set_trace_block(int(block)))


def _attn_out(out, rows, heads, device, what):
    """A caller-given output must be fp16 [rows, heads*64]: the kernel writes exactly that much, unchecked."""
    if out is None:
        return torch.empty((rows, heads * 64), dtype=torch.float16, device=device)
    if out.dtype != torch.float16 or tuple(out.shape) != (rows, heads * 64):
        raise _lib.LsegError(f"{what}: out must be fp16 [{rows}, {heads * 64}], got {out.dtype} {list(out.shape)}")
    return out


def mhsa(qkv, B, N, heads, causal=False, variant=None, out=None):
    """variant=None: the kernel the engine runs; 0..8: see lseg_mhsa_variant in include/lseg_b200.h.
    out: optional fp16 [B*N, heads*64]."""
    out = _attn_out(out, B * N, heads, qkv.device, "mhsa")
    if variant is None:
        check(load().lseg_mhsa(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, int(causal), _stream()))
    else:
        check(load().lseg_mhsa_variant(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, int(causal), int(variant),
                                       _stream()))
    return out


def attn_probs(qkv, heads, out=None):
    """Attention probabilities softmax(0.125 * q k^T) of every head (include/lseg_b200.h lseg_attn_probs): qkv fp16
    [B, N, 3*heads*64] -> fp32 [B, heads, N, N]. out: optional contiguous fp32 [B, heads, N, N] on qkv's device."""
    if qkv.dim() != 3 or qkv.shape[2] != 3 * heads * 64:
        raise _lib.LsegError(f"attn_probs: qkv must be [B, N, {3 * heads * 64}], got {list(qkv.shape)}")
    B, N = qkv.shape[0], qkv.shape[1]
    shape = (B, heads, N, N)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=qkv.device)
    elif (out.dtype != torch.float32 or tuple(out.shape) != shape or out.device != qkv.device or
          not out.is_contiguous()):
        raise _lib.LsegError(f"attn_probs: out must be a contiguous fp32 {list(shape)} tensor on {qkv.device}, got "
                             f"{out.dtype} {list(out.shape)} on {out.device}")
    check(load().lseg_attn_probs(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, _stream()))
    return out


def text_attn(qkv, K, L, heads, out=None):
    """Causal CLIP-text attention with torch's fp16 rounding points (include/lseg_b200.h lseg_text_attn).
    out: optional fp16 [K*L, heads*64]."""
    out = _attn_out(out, K * L, heads, qkv.device, "text_attn")
    check(load().lseg_text_attn(_ptr(qkv, torch.float16), _ptr(out), K, L, heads, _stream()))
    return out


def head_block(x, weight9, bias, mode, act, out=None):
    """One application of scratch.head_block on x [B,K,h,w] (fp16 or fp32) -> fp32 (include/lseg_b200.h lseg_head_block).
    out: optional contiguous fp32 [B,K,h,w]."""
    B, K, h, w = x.shape
    y = _out(out, (B, K, h, w), torch.float32, x.device, "head_block")
    cmax = torch.empty((B, h, w), dtype=torch.float32, device=x.device)
    w9 = (C.c_float * 9)(*[float(v) for v in weight9])
    check(load().lseg_head_block(_ptr(x), int(x.dtype == torch.float16), _ptr(cmax), _ptr(y), B, K, h, w, w9, float(bias),
                                 int(mode), int(act), _stream()))
    return y


def upsample2x_nchw_f32(x, out=None):
    planes = x.numel() // (x.shape[-1] * x.shape[-2])
    H, W = x.shape[-2:]
    y = _out(out, tuple(x.shape[:-2]) + (2 * H, 2 * W), torch.float32, x.device, "upsample2x_nchw_f32")
    check(load().lseg_upsample2x_nchw_f32(_ptr(x, torch.float32), _ptr(y), planes, H, W, _stream()))
    return y


def preprocess(img_u8, size, pad_to=None, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), out=None):
    """uint8 HWC image on the GPU -> fp32 [1,3,Hp,Wp]: ToTensor + Normalize + Resize(size) (bilinear, align_corners=False,
    no antialias: torchvision's tensor resize of the reference's era) + constant pad with -mean/std (pad_image) to
    `pad_to`. One kernel (include/lseg_b200.h lseg_preprocess; lseg_app.py:328-334)."""
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise ValueError("img_u8 must be uint8 [H,W,3]")
    h, w = img_u8.shape[:2]
    Ho, Wo = size
    Hp, Wp = pad_to if pad_to is not None else (Ho, Wo)
    out = _out(out, (1, 3, Hp, Wp), torch.float32, img_u8.device, "preprocess")
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    p3 = (C.c_float * 3)(*[-float(a) / float(b) for a, b in zip(mean, std)])
    check(load().lseg_preprocess(_ptr(img_u8), _ptr(out), h, w, Ho, Wo, Hp, Wp, m3, s3, p3, _stream()))
    return out


def set_deterministic(on):
    """True (default): fixed summation order everywhere (bit-reproducible); False: the in-place residual GEMMs may
    split K across CTA pairs (include/lseg_b200.h lseg_set_deterministic)."""
    check(load().lseg_set_deterministic(int(bool(on))))


def mhsa_trace(qkv, B, N, heads, causal=False, out=None):
    """Debug: (out, trace[16 CTAs, 10 warps, 256]) with clock64 << 8 | tag stamps. out: optional fp16 [B*N, heads*64]."""
    out = _attn_out(out, B * N, heads, qkv.device, "mhsa_trace")
    trace = torch.zeros((16, 10, 256), dtype=torch.int64, device=qkv.device)
    check(load().lseg_mhsa_trace(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, int(causal), _ptr(trace), _stream()))
    return out, trace


def layernorm(x, gamma, beta, eps, out=None):
    M, Cc = x.shape
    y = _out(out, (M, Cc), torch.float16, x.device, "layernorm")
    check(load().lseg_layernorm(_ptr(x), int(x.dtype == torch.float16), _ptr(gamma, torch.float32),
                                _ptr(beta, torch.float32), _ptr(y), M, Cc, eps, _stream()))
    return y


def patchify(x, patch=16, out=None):
    B, _, H, W = x.shape
    a = _out(out, (B * (H // patch) * (W // patch), 3 * patch * patch), torch.float16, x.device, "patchify")
    check(load().lseg_patchify(_ptr(x, torch.float32), _ptr(a), B, H, W, patch, _stream()))
    return a


def pos_resize(pos, g0, gh, gw, out=None):
    D = pos.shape[-1]
    out = _out(out, (1 + gh * gw, D), torch.float32, pos.device, "pos_resize")
    check(load().lseg_pos_resize(_ptr(pos, torch.float32), _ptr(out), g0, gh, gw, D, _stream()))
    return out


def assemble_tokens(patch, cls, pos, B, T, out=None):
    D = patch.shape[-1]
    x = _out(out, (B, T + 1, D), torch.float32, patch.device, "assemble_tokens")
    check(load().lseg_assemble_tokens(_ptr(patch, torch.float32), _ptr(cls, torch.float32), _ptr(pos, torch.float32),
                                      _ptr(x), B, T, D, _stream()))
    return x


def readout_split(tap, out=None):
    """tap fp32 [B, N, D] -> (tok fp16 [B*(N-1), D], cls fp16 [B rounded up to 128, D]); the kernel writes cls rows < B
    only, the padding rows stay as the caller left them (zero when allocated here). out: optional (tok, cls) pair."""
    B, N, D = tap.shape
    tok_out, cls_out = out if out is not None else (None, None)
    tok = _out(tok_out, (B * (N - 1), D), torch.float16, tap.device, "readout_split tok")
    if cls_out is None:
        cls = torch.zeros(((B + 127) // 128 * 128, D), dtype=torch.float16, device=tap.device)
    else:
        cls = _out(cls_out, ((B + 127) // 128 * 128, D), torch.float16, tap.device, "readout_split cls")
    check(load().lseg_readout_split(_ptr(tap, torch.float32), _ptr(tok), _ptr(cls), B, N - 1, D, _stream()))
    return tok, cls


def im2col_3x3_s2(x, out=None):
    B, H, W, Cc = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    a = _out(out, (B * Ho * Wo, 9 * Cc), torch.float16, x.device, "im2col_3x3_s2")
    check(load().lseg_im2col_3x3_s2(_ptr(x, torch.float16), _ptr(a), B, H, W, Cc, _stream()))
    return a


def stem_im2col(x, out=None):
    """x fp32 NCHW [B,3,H,W] -> fp16 [B*(H/2)*(W/2), 192] rows of the ResNet stem conv (7x7 s2 p3), zero beyond column 147."""
    B, _, H, W = x.shape
    a = _out(out, (B * (H // 2) * (W // 2), 192), torch.float16, x.device, "stem_im2col")
    check(load().lseg_stem_im2col(_ptr(x, torch.float32), _ptr(a), B, H, W, _stream()))
    return a


def maxpool3x3s2_nhwc(x, out=None):
    B, H, W, Cc = x.shape
    y = _out(out, (B, H // 2, W // 2, Cc), torch.float16, x.device, "maxpool3x3s2_nhwc")
    check(load().lseg_maxpool3x3s2_nhwc(_ptr(x, torch.float16), _ptr(y), B, H, W, Cc, _stream()))
    return y


def subsample2_nhwc(x, out=None):
    B, H, W, Cc = x.shape
    y = _out(out, (B, H // 2, W // 2, Cc), torch.float16, x.device, "subsample2_nhwc")
    check(load().lseg_subsample2_nhwc(_ptr(x, torch.float16), _ptr(y), B, H, W, Cc, _stream()))
    return y


def upsample2x_nhwc(x, out_dtype=torch.float16, add=None, decoder=False, out=None):
    """bilinear x2 align_corners=True over NHWC. decoder=False: the generic fp16 -> fp16 kernel (any C);
    decoder=True (or fp32 input / fp32 output / add): the C = 256 kernels of the fusion blocks — fp16 | fp32 source,
    fp16 | fp32 result, optional fp32 skip operand summed in."""
    B, H, W, Cc = x.shape
    y = _out(out, (B, 2 * H, 2 * W, Cc), out_dtype, x.device, "upsample2x_nhwc")
    if decoder or x.dtype == torch.float32 or out_dtype == torch.float32 or add is not None:
        if Cc != 256:
            raise ValueError("the decoder interpolation kernels are built for C = 256")
        check(load().lseg_upsample2x_nhwc256(_ptr(x), int(x.dtype == torch.float16), _ptr(y),
                                             int(out_dtype == torch.float16),
                                             _ptr(add, torch.float32) if add is not None else None, B, H, W, _stream()))
    else:
        check(load().lseg_upsample2x_nhwc(_ptr(x, torch.float16), _ptr(y), B, H, W, Cc, _stream()))
    return y


def l2norm_scale(x, logit_scale, out=None):
    M, Cc = x.shape
    y = _out(out, (M, Cc), torch.float16, x.device, "l2norm_scale")
    check(load().lseg_l2norm_scale(_ptr(x, torch.float32), _ptr(y), M, Cc, float(logit_scale), _stream()))
    return y


def l2norm_f16(x, out=None):
    M, Cc = x.shape
    y = _out(out, (M, Cc), torch.float16, x.device, "l2norm_f16")
    check(load().lseg_l2norm_f16(_ptr(x, torch.float16), _ptr(y), M, Cc, _stream()))
    return y


def upsample2x_nchw(x, background=False, out=None):
    """background=True: the shared-memory-free kernel of the multi-GPU gather (same values bit for bit)."""
    B, K, H, W = x.shape
    y = _out(out, (B, K, 2 * H, 2 * W), torch.float32, x.device, "upsample2x_nchw")
    fn = load().lseg_upsample2x_nchw_bg if background else load().lseg_upsample2x_nchw
    check(fn(_ptr(x, torch.float16), _ptr(y), B * K, H, W, _stream()))
    return y


def upsample2x_argmax(x):
    """fp16 [B,K,H,W] -> int64 [B,2H,2W]: argmax over K of the align_corners=True bilinear x2 upsample (first maximum)."""
    B, K, H, W = x.shape
    m = torch.empty((B, 2 * H, 2 * W), dtype=torch.int64, device=x.device)
    check(load().lseg_upsample2x_argmax(_ptr(x, torch.float16), _ptr(m), B, K, H, W, _stream()))
    return m


def _group_ptr(group, stats, B):
    """int32 device copy of a group-id tensor of B entries (None: every image counts into row 0). Values outside int32
    are clamped into it, where they stay out of [0, G), so the device check still reports them."""
    if group is None:
        return None, None
    group = torch.as_tensor(group)
    if group.numel() != B:
        raise ValueError(f"group has {group.numel()} entries, the batch has {B} images")
    g = group.reshape(-1).to(device=stats.device, dtype=torch.int64).clamp(-2 ** 31, 2 ** 31 - 1).to(torch.int32)
    g = g.contiguous()
    return g, _ptr(g)


def _check_stats(stats, nclass):
    if stats.dtype != torch.int64 or stats.dim() != 2 or stats.shape[1] != 3 * nclass + 2:
        raise ValueError(f"stats must be int64 [G, 3*nclass+2] = [G, {3 * nclass + 2}], got {stats.dtype} "
                         f"{tuple(stats.shape)}")


def seg_stats_scores(scores, target, stats, nclass, group=None):
    """Adds the metric counters of fp32 scores [B,K,H,W] (first maximal class) against int64 target [B,H,W] to
    stats int64 [G, 3*nclass+2] (row layout and per-pixel rule: include/lseg_b200.h). group: ids [B] or None."""
    B, K, H, W = scores.shape
    _check_stats(stats, nclass)
    if tuple(target.shape) != (B, H, W):
        raise ValueError(f"target must be [B,H,W] = {(B, H, W)}, got {tuple(target.shape)}")
    g, gp = _group_ptr(group, stats, B)
    check(load().lseg_seg_stats_scores(_ptr(scores, torch.float32), _ptr(target, torch.int64), gp, B, K, H, W, nclass,
                                       stats.shape[0], _ptr(stats, torch.int64), _stream()))
    return stats


def seg_stats_mask(pred, target, stats, nclass, group=None):
    """Adds the metric counters of an int64 prediction mask [B,H,W] against int64 target [B,H,W] to stats."""
    B, H, W = pred.shape
    _check_stats(stats, nclass)
    if tuple(target.shape) != (B, H, W):
        raise ValueError(f"target must be [B,H,W] = {(B, H, W)}, got {tuple(target.shape)}")
    g, gp = _group_ptr(group, stats, B)
    check(load().lseg_seg_stats_mask(_ptr(pred, torch.int64), _ptr(target, torch.int64), gp, B, H, W, nclass,
                                     stats.shape[0], _ptr(stats, torch.int64), _stream()))
    return stats


def xent_partials(B, H, W, fused):
    """(sum, count) fp64 pairs of partials a loss call needs (include/lseg_b200.h): one per block of the loss kernel."""
    return B * ((H + 7) // 8) if fused else B * ((H * W + 1023) // 1024)


def xent_scores(scores, target, acc, ignore_index=-1):
    """Adds {sum of per-pixel cross-entropies, counted pixels} of fp32 scores [B,K,H,W] against int64 target [B,H,W]
    (pixels equal to ignore_index skipped) to acc float64 [2]. Enqueues on the current stream."""
    B, K, H, W = scores.shape
    if tuple(target.shape) != (B, H, W):
        raise ValueError(f"target must be [B,H,W] = {(B, H, W)}, got {tuple(target.shape)}")
    if acc.dtype != torch.float64 or acc.numel() != 2 or not acc.is_contiguous():
        raise ValueError("acc must be a contiguous float64 tensor of 2 elements")
    part = torch.empty((xent_partials(B, H, W, False), 2), dtype=torch.float64, device=scores.device)
    check(load().lseg_xent_scores(_ptr(scores, torch.float32), _ptr(target, torch.int64), int(ignore_index), B, K, H, W,
                                  _ptr(acc, torch.float64), _ptr(part), part.numel(), _stream()))
    return acc


def text_embed(tokens, tok_emb, pos_emb, out=None):
    K, L = tokens.shape
    Wd = tok_emb.shape[1]
    x = _out(out, (K * L, Wd), torch.float16, tok_emb.device, "text_embed")
    check(load().lseg_text_embed(_ptr(tokens, torch.int64), _ptr(tok_emb, torch.float32),
                                 _ptr(pos_emb, torch.float32), _ptr(x), K, L, Wd, _stream()))
    return x


def text_eot_gather(tokens, x, out=None):
    """Rows [K rounded up to 128, Wd]: the kernel writes rows < K, the padding rows stay as the caller left them."""
    K, L = tokens.shape
    Wd = x.shape[-1]
    if out is None:
        out = torch.zeros(((K + 127) // 128 * 128, Wd), dtype=torch.float16, device=x.device)
    else:
        out = _out(out, ((K + 127) // 128 * 128, Wd), torch.float16, x.device, "text_eot_gather")
    check(load().lseg_text_eot_gather(_ptr(tokens, torch.int64), _ptr(x, torch.float16), _ptr(out), K, L, Wd,
                                      _stream()))
    return out
