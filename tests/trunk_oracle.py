"""Float64 references and error bounds for every op of one image-trunk block (csrc/engine.cuh build_vit_trunk and
build_resnet_trunk), each op fed the engine's own input of that op: the trace_* buffers that
lseg_debug_set_trace_block snapshots, plus patch_out, stem and pool, which the plan keeps anyway.

Shared by tests/test_trunk_stages_gpu.py (against one traced forward) and tests/test_trunk_stages_cpu.py (float32
emulations of each op's recipe must pass both tiers, planted defects must fail the tier named for them). Plain torch:
CPU or CUDA. Every bound is built from the existing pieces, with the notation of their docstrings:
stage_oracle.linear_terms / conv_terms / epilogue (tensor-core accumulation gamma_n mag, folded BN, bias, ReLU,
gelu_erf, residual adds, fp16 stores), glue_oracle.layernorm_ref and attention_oracle.mhsa_oracle.

ViT block (timm Block, lseg_vit.py:166-201; x the fp32 residual stream of one image, [N, D]):

    patch      rn16(patchify(x)) W_p^T + b_p -> fp32            conv_terms (stride P) + epilogue(bias)
    LN1        trace_in -> trace_ln1 (fp16, eps 1e-6)           layernorm_ref
    QKV        trace_ln1 W_qkv^T + b -> trace_qkv (fp16)        linear_terms + epilogue(bias, fp16)
    MHSA       trace_qkv -> trace_attn (fp16)                   mhsa_oracle with the exponential of the engine's
                                                                variant (g_mhsa_variant: 0 = MUFU ex2, EPS_EX2)
    proj       trace_in + (trace_attn W_o^T + b) -> trace_x1    linear_terms + epilogue(bias, res = trace_in) + reduce
    LN2        trace_x1 -> trace_ln2                            layernorm_ref
    fc1        gelu(trace_ln2 W_1^T + b) -> trace_fc1 (fp16)    linear_terms + epilogue(bias, gelu, fp16)
    fc2        trace_x1 + (trace_fc1 W_2^T + b) -> trace_out    as proj

Reduce-add. proj and fc2 update the stream in place through the bulk-tensor reduce-add epilogue: the GEMM's epilogue
forms v = fl(acc + b) and the TMA unit stores fl(x + v), which is the one residual rounding epilogue charges
(u (|y| + E)). Under stream-K balancing (LSEG_SPLITK) a tile's K range is split over up to S CTAs; each reduce-adds its
own partial sum (only the segment that starts at k = 0 adds the bias), so the running value is rounded S times, not
once. The accumulation itself is unchanged: a segment sums fewer terms, and gamma_n mag bounds the sum of the
segments' gamma_{n_s} mag_s. Every running value is bounded by |x| + mag + |b| + E, so each extra segment adds
u (|x| + mag + |b| + E). S is the largest number of CTAs whose unit ranges meet one tile:
ceil(k_iters / (units / grid - 4)) + 1, the -4 for the 4-chunk rounding of the range boundaries (gemm_tc.cuh Sched).

ResNet-101 bottleneck (torchvision v1.5: the stride sits on conv2; x16 the fp16 block input, NHWC):

    stem       relu(bn(conv7x7 s2 p3 (rn16(x)))) -> fp16        conv_terms + epilogue(scale, shift, relu, fp16)
    conv1      relu(bn1(conv1x1(trace_in))) -> trace_t1        conv_terms + epilogue(scale, shift, relu, fp16)
    conv2      relu(bn2(conv3x3 at the block's stride          conv_terms (stride, pad 1) + epilogue(..., fp16)
               (trace_t1))) -> trace_t2
    downsample bn_d(conv1x1(trace_in[:, ::s, ::s])) -> fp32    conv_terms + epilogue(scale, shift), the stage's stream
               (the first block of a stage: trace_id)
    out32      relu(trace_id + bn3(conv3x3(trace_t2)))          epilogue(scale, shift, res = trace_id), then relu:
               -> trace_out32 (fp32)                            1-Lipschitz, the bound carries over
    out16      rn16(out32) -> trace_out16                       out32's bound + half an fp16 ulp

Tiers (stage_oracle.check). A: every element within its bound. B: fp16 outputs bit-identical to rn16(ref) on at least
FP16_IDENTICAL of their elements (fc1: of those with |GELU| >= 2^-7, where gelu_erf is documented accurate to half an
fp16 ulp, as for the readout); fp32 outputs with an RMS error below FP32_RMS half fp16 ulps. The MHSA output is judged
as tests/test_attention_gpu.py judges the kernel, by its bound alone (mhsa_oracle's bound already holds a full fp16
ulp): its bit-identical fraction is reported, not required.
"""
import torch

import attention_oracle as A
import glue_oracle as G
import stage_oracle as S
from glue_oracle import U, r16, ulp16

F64 = torch.float64
LN_EPS = 1e-6
BM, BN, BK = 128, 128, 64  # gemm_tc.cuh kGemmBM / kGemmBN / kGemmBK


def stream_k_segments(M, N, K, grid):
    """Most CTAs that can reduce-add into one tile of an M x N x K stream-K GEMM on `grid` CTAs (module docstring)."""
    tiles, k_iters = -(-M // BM) * -(-N // BN), K // BK
    per_cta = max(1, tiles * k_iters // grid - 4)
    return -(-k_iters // per_cta) + 1


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def _reduce_add(acc, mag, n, b, x, segments):
    """x + (acc + b) through the reduce-add epilogue with `segments` reduce-adds per tile."""
    ref, E = S.epilogue(acc, mag, n, bias=b, res=(x,))
    for _ in range(segments - 1):
        E = E + U * (x.to(F64).abs() + mag + S._dev(b, acc).abs() + E)
    return ref, E


# ------------------------------------------------------------------------------------------------------------------
# ViT
# ------------------------------------------------------------------------------------------------------------------
def patch_embed(x, w, b):
    """patch_out fp32 [B*T, D] of the image x fp32 NCHW: rn16(x) (patchify rounds) x w16(W) [D, 3, P, P] + b."""
    P = w.shape[-1]
    acc, mag, n, _ = S.conv_terms(_nhwc(r16(x)), S.w16(w), stride=P, pad=0)
    ref, E = S.epilogue(acc, mag, n, bias=b)
    D = w.shape[0]
    return {"ref": ref.reshape(-1, D), "bound": E.reshape(-1, D)}


def layernorm(x, g, b):
    ref, E = G.layernorm_ref(x, g, b, LN_EPS)
    return {"ref": ref, "bound": E}


def linear(a, w, b, *, act=None, out_f16=True):
    """act(a w16(w)^T + b), fp16 or fp32; a GELU output is judged in tier B where |GELU| >= 2^-7."""
    acc, mag, n, _ = S.linear_terms(a, S.w16(w))
    ref, E = S.epilogue(acc, mag, n, bias=b, act=act, out_f16=out_f16)
    st = {"ref": ref, "bound": E}
    if act == "gelu":
        st["b_mask"] = ref.abs() >= 2.0 ** -7
    return st


def residual_linear(a, w, b, x, segments=1):
    """x + (a w16(w)^T + b), fp32, through the reduce-add epilogue (`segments` reduce-adds per tile)."""
    acc, mag, n, _ = S.linear_terms(a, S.w16(w))
    ref, E = _reduce_add(acc, mag, n, b, x, segments)
    return {"ref": ref, "bound": E}


def mhsa(qkv, N, heads, eps_exp=A.EPS_EX2):
    """The attention output fp16 [N, D] of one image's qkv fp16 [N, 3D]: bound only (module docstring)."""
    ref, E = A.mhsa_oracle(qkv.reshape(1, N, -1), 1, N, heads, False, eps_exp)
    return {"ref": ref, "bound": E, "b_min": 0.0}


def vit_block_params(sd, i, device=None):
    """Block i's weights from the state dict (float64 tensors; GEMM weights are rounded by the oracle)."""
    q = f"pretrained.model.blocks.{i}."
    names = {"ln1_g": "norm1.weight", "ln1_b": "norm1.bias", "ln2_g": "norm2.weight", "ln2_b": "norm2.bias",
             "qkv_w": "attn.qkv.weight", "qkv_b": "attn.qkv.bias", "proj_w": "attn.proj.weight",
             "proj_b": "attn.proj.bias", "fc1_w": "mlp.fc1.weight", "fc1_b": "mlp.fc1.bias", "fc2_w": "mlp.fc2.weight",
             "fc2_b": "mlp.fc2.bias"}
    return {k: sd[q + v].to(device=device, dtype=F64) for k, v in names.items()}


def vit_block(tr, p, heads, *, eps_exp=A.EPS_EX2, seg_proj=1, seg_fc2=1):
    """op -> (got, stage dict, fp16?) for one image's trace tensors tr (trace_in .. trace_out, [N, .]) of a block with
    weights p (vit_block_params)."""
    N = tr["trace_in"].shape[0]
    return {
        "ln1": (tr["trace_ln1"], layernorm(tr["trace_in"], p["ln1_g"], p["ln1_b"]), True),
        "qkv": (tr["trace_qkv"], linear(tr["trace_ln1"], p["qkv_w"], p["qkv_b"]), True),
        "mhsa": (tr["trace_attn"], mhsa(tr["trace_qkv"], N, heads, eps_exp), True),
        "proj": (tr["trace_x1"], residual_linear(tr["trace_attn"], p["proj_w"], p["proj_b"], tr["trace_in"], seg_proj),
                 False),
        "ln2": (tr["trace_ln2"], layernorm(tr["trace_x1"], p["ln2_g"], p["ln2_b"]), True),
        "fc1": (tr["trace_fc1"], linear(tr["trace_ln2"], p["fc1_w"], p["fc1_b"], act="gelu"), True),
        "fc2": (tr["trace_out"], residual_linear(tr["trace_fc1"], p["fc2_w"], p["fc2_b"], tr["trace_x1"], seg_fc2),
                False),
    }


# ------------------------------------------------------------------------------------------------------------------
# ResNet-101
# ------------------------------------------------------------------------------------------------------------------
def conv_bn(x, w, bn, *, stride=1, pad=0, relu=True, out_f16=True):
    """act(bn(conv(x))) of NHWC x with w [Cout, Cin, k, k] (rounded to fp16) and bn = (scale, shift) folded."""
    acc, mag, n, _ = S.conv_terms(x, S.w16(w), stride=stride, pad=pad)
    ref, E = S.epilogue(acc, mag, n, scale=bn[0], bias=bn[1], act="relu" if relu else None, out_f16=out_f16)
    return {"ref": ref, "bound": E}


def stem(x, w, bn):
    """relu(bn(conv7x7 s2 p3)) of the image x fp32 NCHW, fp16 NHWC: stem_im2col rounds x to fp16."""
    return conv_bn(_nhwc(r16(x)), w, bn, stride=2, pad=3)


def out32(t2, w3, bn3, ident):
    """relu(ident + bn3(conv3(t2))), fp32: the relu_after_res epilogue."""
    acc, mag, n, _ = S.conv_terms(t2, S.w16(w3), pad=0)
    ref, E = S.epilogue(acc, mag, n, scale=bn3[0], bias=bn3[1], res=(ident,))
    return {"ref": ref.clamp_min(0), "bound": E}


def out16(st32):
    """rn16 of the fp32 stream, from its reference: + half an fp16 ulp."""
    return {"ref": st32["ref"], "bound": st32["bound"] + ulp16(st32["ref"].abs() + st32["bound"]) / 2}


def bottleneck_params(sd, blk, layers=(3, 4, 23, 3), device=None):
    """(params, stride) of global bottleneck blk under the state dict names of packing._pack_resnet."""
    from lseg_b200.packing import fold_bn
    L, i = 0, blk
    while i >= layers[L]:
        i -= layers[L]
        L += 1
    q = f"pretrained.layer1.4.{i}." if L == 0 else f"pretrained.layer{L + 1}.{i}."

    def bn(prefix):
        s, t = fold_bn(sd, prefix)
        return s.to(device=device, dtype=F64), t.to(device=device, dtype=F64)

    p = {f"w{j}": sd[f"{q}conv{j}.weight"].to(device=device, dtype=F64) for j in (1, 2, 3)}
    p.update({f"bn{j}": bn(f"{q}bn{j}.") for j in (1, 2, 3)})
    if i == 0:
        p["wd"] = sd[q + "downsample.0.weight"].to(device=device, dtype=F64)
        p["bnd"] = bn(q + "downsample.1.")
    return p, (2 if L > 0 and i == 0 else 1)


def bottleneck(tr, p, stride):
    """op -> (got, stage dict, fp16?) for one image's trace tensors (NHWC) of a bottleneck with params p."""
    ops = {
        "conv1": (tr["trace_t1"], conv_bn(tr["trace_in"], p["w1"], p["bn1"]), True),
        "conv2": (tr["trace_t2"], conv_bn(tr["trace_t1"], p["w2"], p["bn2"], stride=stride, pad=1), True),
    }
    if "wd" in p:
        xs = tr["trace_in"][:, ::stride, ::stride]
        ops["downsample"] = (tr["trace_id"], conv_bn(xs, p["wd"], p["bnd"], relu=False, out_f16=False), False)
    st = out32(tr["trace_t2"], p["w3"], p["bn3"], tr["trace_id"])
    ops["out32"] = (tr["trace_out32"], st, False)
    ops["out16"] = (tr["trace_out16"], out16(st), True)
    return ops


def judge(ops):
    """-> ({op: {worst, tier_b}}, [failure messages]) over the ops of vit_block / bottleneck."""
    report, fails = {}, []
    for name, (got, st, f16) in ops.items():
        report[name], f = S.check(got, st, f16)
        fails += [f"{name}: {m}" for m in f]
    return report, fails
