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


def gemm(a, w, N=None, *, bias=None, bias_group_rows=0, scale=None, act=ACT_NONE, res_f32=None, res2_f32=None,
         res_f16=None, out_f32=None, out_f16=None, out_f16_relu=None, ldc=None, M=None,
         conv=None, store=STORE_ROWMAJOR, d2s=None, nchw=None, row_sumsq=None, row_scale=1.0, out_row_sumsq=None,
         relu_after_res=False):
    """C = epi(A W^T).  a: fp16 [M,K] (or NHWC [B,H,W,C] when conv=(ksize,pad)); w: fp16 [rows>=N, Ktot]."""
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
    check(load().lseg_gemm(C.byref(args), _stream()))


def mhsa(qkv, B, N, heads, causal=False, variant=None, out=None):
    """variant=None: the kernel the engine runs; 0..4: see lseg_mhsa_variant in include/lseg_b200.h."""
    if out is None:
        out = torch.empty((B * N, heads * 64), dtype=torch.float16, device=qkv.device)
    if variant is None:
        check(load().lseg_mhsa(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, int(causal), _stream()))
    else:
        check(load().lseg_mhsa_variant(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, int(causal), int(variant),
                                       _stream()))
    return out


def text_attn(qkv, K, L, heads):
    """Causal CLIP-text attention with torch's fp16 rounding points (include/lseg_b200.h lseg_text_attn)."""
    out = torch.empty((K * L, heads * 64), dtype=torch.float16, device=qkv.device)
    check(load().lseg_text_attn(_ptr(qkv, torch.float16), _ptr(out), K, L, heads, _stream()))
    return out


def head_block(x, weight9, bias, mode, act):
    """One application of scratch.head_block on x [B,K,h,w] (fp16 or fp32) -> fp32 (include/lseg_b200.h lseg_head_block)."""
    B, K, h, w = x.shape
    y = torch.empty((B, K, h, w), dtype=torch.float32, device=x.device)
    cmax = torch.empty((B, h, w), dtype=torch.float32, device=x.device)
    w9 = (C.c_float * 9)(*[float(v) for v in weight9])
    check(load().lseg_head_block(_ptr(x), int(x.dtype == torch.float16), _ptr(cmax), _ptr(y), B, K, h, w, w9, float(bias),
                                 int(mode), int(act), _stream()))
    return y


def upsample2x_nchw_f32(x):
    planes = x.numel() // (x.shape[-1] * x.shape[-2])
    H, W = x.shape[-2:]
    y = torch.empty(tuple(x.shape[:-2]) + (2 * H, 2 * W), dtype=torch.float32, device=x.device)
    check(load().lseg_upsample2x_nchw_f32(_ptr(x, torch.float32), _ptr(y), planes, H, W, _stream()))
    return y


def preprocess(img_u8, size, pad_to=None, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    """uint8 HWC image on the GPU -> fp32 [1,3,Hp,Wp]: ToTensor + Normalize + Resize(size) (bilinear, align_corners=False,
    no antialias: torchvision's tensor resize of the reference's era) + constant pad with -mean/std (pad_image) to
    `pad_to`. One kernel (include/lseg_b200.h lseg_preprocess; lseg_app.py:328-334)."""
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise ValueError("img_u8 must be uint8 [H,W,3]")
    h, w = img_u8.shape[:2]
    Ho, Wo = size
    Hp, Wp = pad_to if pad_to is not None else (Ho, Wo)
    out = torch.empty((1, 3, Hp, Wp), dtype=torch.float32, device=img_u8.device)
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    p3 = (C.c_float * 3)(*[-float(a) / float(b) for a, b in zip(mean, std)])
    check(load().lseg_preprocess(_ptr(img_u8), _ptr(out), h, w, Ho, Wo, Hp, Wp, m3, s3, p3, _stream()))
    return out


def set_deterministic(on):
    """True (default): fixed summation order everywhere (bit-reproducible); False: the in-place residual GEMMs may
    split K across CTA pairs (include/lseg_b200.h lseg_set_deterministic)."""
    check(load().lseg_set_deterministic(int(bool(on))))


def mhsa_trace(qkv, B, N, heads, causal=False):
    """Debug: (out, trace[16 CTAs, 10 warps, 256]) with clock64 << 8 | tag stamps."""
    out = torch.empty((B * N, heads * 64), dtype=torch.float16, device=qkv.device)
    trace = torch.zeros((16, 10, 256), dtype=torch.int64, device=qkv.device)
    check(load().lseg_mhsa_trace(_ptr(qkv, torch.float16), _ptr(out), B, N, heads, int(causal), _ptr(trace), _stream()))
    return out, trace


def layernorm(x, gamma, beta, eps):
    M, Cc = x.shape
    y = torch.empty((M, Cc), dtype=torch.float16, device=x.device)
    check(load().lseg_layernorm(_ptr(x), int(x.dtype == torch.float16), _ptr(gamma, torch.float32),
                                _ptr(beta, torch.float32), _ptr(y), M, Cc, eps, _stream()))
    return y


def patchify(x, patch=16):
    B, _, H, W = x.shape
    a = torch.empty((B * (H // patch) * (W // patch), 3 * patch * patch), dtype=torch.float16, device=x.device)
    check(load().lseg_patchify(_ptr(x, torch.float32), _ptr(a), B, H, W, patch, _stream()))
    return a


def pos_resize(pos, g0, gh, gw):
    D = pos.shape[-1]
    out = torch.empty((1 + gh * gw, D), dtype=torch.float32, device=pos.device)
    check(load().lseg_pos_resize(_ptr(pos, torch.float32), _ptr(out), g0, gh, gw, D, _stream()))
    return out


def assemble_tokens(patch, cls, pos, B, T):
    D = patch.shape[-1]
    x = torch.empty((B, T + 1, D), dtype=torch.float32, device=patch.device)
    check(load().lseg_assemble_tokens(_ptr(patch, torch.float32), _ptr(cls, torch.float32), _ptr(pos, torch.float32),
                                      _ptr(x), B, T, D, _stream()))
    return x


def readout_split(tap):
    B, N, D = tap.shape
    tok = torch.empty((B * (N - 1), D), dtype=torch.float16, device=tap.device)
    cls = torch.zeros(((B + 127) // 128 * 128, D), dtype=torch.float16, device=tap.device)
    check(load().lseg_readout_split(_ptr(tap, torch.float32), _ptr(tok), _ptr(cls), B, N - 1, D, _stream()))
    return tok, cls


def im2col_3x3_s2(x):
    B, H, W, Cc = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    a = torch.empty((B * Ho * Wo, 9 * Cc), dtype=torch.float16, device=x.device)
    check(load().lseg_im2col_3x3_s2(_ptr(x, torch.float16), _ptr(a), B, H, W, Cc, _stream()))
    return a


def stem_im2col(x):
    """x fp32 NCHW [B,3,H,W] -> fp16 [B*(H/2)*(W/2), 192] rows of the ResNet stem conv (7x7 s2 p3), zero beyond column 147."""
    B, _, H, W = x.shape
    a = torch.empty((B * (H // 2) * (W // 2), 192), dtype=torch.float16, device=x.device)
    check(load().lseg_stem_im2col(_ptr(x, torch.float32), _ptr(a), B, H, W, _stream()))
    return a


def maxpool3x3s2_nhwc(x):
    B, H, W, Cc = x.shape
    y = torch.empty((B, H // 2, W // 2, Cc), dtype=torch.float16, device=x.device)
    check(load().lseg_maxpool3x3s2_nhwc(_ptr(x, torch.float16), _ptr(y), B, H, W, Cc, _stream()))
    return y


def subsample2_nhwc(x):
    B, H, W, Cc = x.shape
    y = torch.empty((B, H // 2, W // 2, Cc), dtype=torch.float16, device=x.device)
    check(load().lseg_subsample2_nhwc(_ptr(x, torch.float16), _ptr(y), B, H, W, Cc, _stream()))
    return y


def upsample2x_nhwc(x, out_dtype=torch.float16, add=None, decoder=False):
    """bilinear x2 align_corners=True over NHWC. decoder=False: the generic fp16 -> fp16 kernel (any C);
    decoder=True (or fp32 input / fp32 output / add): the C = 256 kernels of the fusion blocks — fp16 | fp32 source,
    fp16 | fp32 result, optional fp32 skip operand summed in."""
    B, H, W, Cc = x.shape
    y = torch.empty((B, 2 * H, 2 * W, Cc), dtype=out_dtype, device=x.device)
    if decoder or x.dtype == torch.float32 or out_dtype == torch.float32 or add is not None:
        if Cc != 256:
            raise ValueError("the decoder interpolation kernels are built for C = 256")
        check(load().lseg_upsample2x_nhwc256(_ptr(x), int(x.dtype == torch.float16), _ptr(y),
                                             int(out_dtype == torch.float16),
                                             _ptr(add, torch.float32) if add is not None else None, B, H, W, _stream()))
    else:
        check(load().lseg_upsample2x_nhwc(_ptr(x, torch.float16), _ptr(y), B, H, W, Cc, _stream()))
    return y


def l2norm_scale(x, logit_scale):
    M, Cc = x.shape
    y = torch.empty((M, Cc), dtype=torch.float16, device=x.device)
    check(load().lseg_l2norm_scale(_ptr(x, torch.float32), _ptr(y), M, Cc, float(logit_scale), _stream()))
    return y


def l2norm_f16(x):
    M, Cc = x.shape
    y = torch.empty_like(x)
    check(load().lseg_l2norm_f16(_ptr(x, torch.float16), _ptr(y), M, Cc, _stream()))
    return y


def upsample2x_nchw(x, background=False):
    """background=True: the shared-memory-free kernel of the multi-GPU gather (same values bit for bit)."""
    B, K, H, W = x.shape
    y = torch.empty((B, K, 2 * H, 2 * W), dtype=torch.float32, device=x.device)
    fn = load().lseg_upsample2x_nchw_bg if background else load().lseg_upsample2x_nchw
    check(fn(_ptr(x, torch.float16), _ptr(y), B * K, H, W, _stream()))
    return y


def upsample2x_argmax(x):
    """fp16 [B,K,H,W] -> int64 [B,2H,2W]: argmax over K of the align_corners=True bilinear x2 upsample (first maximum)."""
    B, K, H, W = x.shape
    m = torch.empty((B, 2 * H, 2 * W), dtype=torch.int64, device=x.device)
    check(load().lseg_upsample2x_argmax(_ptr(x, torch.float16), _ptr(m), B, K, H, W, _stream()))
    return m


def text_embed(tokens, tok_emb, pos_emb):
    K, L = tokens.shape
    Wd = tok_emb.shape[1]
    x = torch.empty((K * L, Wd), dtype=torch.float16, device=tok_emb.device)
    check(load().lseg_text_embed(_ptr(tokens, torch.int64), _ptr(tok_emb, torch.float32),
                                 _ptr(pos_emb, torch.float32), _ptr(x), K, L, Wd, _stream()))
    return x


def text_eot_gather(tokens, x):
    K, L = tokens.shape
    Wd = x.shape[-1]
    out = torch.zeros(((K + 127) // 128 * 128, Wd), dtype=torch.float16, device=x.device)
    check(load().lseg_text_eot_gather(_ptr(tokens, torch.int64), _ptr(x, torch.float16), _ptr(out), K, L, Wd,
                                      _stream()))
    return out
