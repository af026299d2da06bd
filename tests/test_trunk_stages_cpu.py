"""The per-op bounds of tests/trunk_oracle.py are neither too loose nor too tight: on CPU, a float32 emulation of each
trunk op's recipe in the engine (fp16 operands, fp32 accumulation, the engine's rounding points) passes both tiers, and
an emulation with one planted defect fails the tier named for it. Small shapes (a ViT block at D = 128, 2 heads, N = 37,
B = 2; a bottleneck at 8 x 8 -> 4 x 4) at the scales of the seeded synthetic networks (oracle/synth.py).
"""
import json
import math

import pytest
import torch
import torch.nn.functional as F

import glue_oracle as G
import trunk_oracle as T
from test_image_stages_cpu import gelu_erf32

F32 = torch.float32
B, N, D, HEADS = 2, 37, 128, 2


def _randn(shape, seed, scale=1.0, mean=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale + mean).float()


def _w32(w):
    return w.half().float()


# ------------------------------------------------------------------------------------------------------------------
# float32 emulations of the engine's recipe; keyword flags plant one defect each
# ------------------------------------------------------------------------------------------------------------------
def emu_linear(a, w, b, *, act=None, gelu_tanh=False):
    y = a.float() @ _w32(w).t() + b.float()
    if act == "gelu":
        y = F.gelu(y, approximate="tanh") if gelu_tanh else gelu_erf32(y)
    return y.half()


def emu_residual(a, w, b, x, *, segments=1, bias_every_segment=False, x_f16=False):
    """x += a w^T + b as reduce-adds of `segments` K-slices (only the first adds b, unless bias_every_segment)."""
    x = x.half().float() if x_f16 else x.clone()
    K = a.shape[1]
    for s in range(segments):
        k0, k1 = s * K // segments, (s + 1) * K // segments
        v = a[:, k0:k1].float() @ _w32(w[:, k0:k1]).t()
        if s == 0 or bias_every_segment:
            v = v + b.float()
        x = x + v
    return x


def emu_mhsa(qkv, *, swap_qk_head=None, tail_keys_from_neighbour=False):
    """Flash attention's rounding points in float32: S = q k^T, p = exp(0.125 (S - max)), O = fp16(p) v / sum p.
    qkv fp16 [B, N, 3D] -> fp16 [B*N, D]."""
    x = qkv.float().reshape(B, N, 3, HEADS, 64).permute(2, 0, 3, 1, 4)  # [3, B, heads, N, 64]
    q, k, v = x[0].clone(), x[1].clone(), x[2]
    if swap_qk_head is not None:
        q[:, swap_qk_head], k[:, swap_qk_head] = x[1][:, swap_qk_head], x[0][:, swap_qk_head]
    s = q @ k.transpose(-1, -2)
    if tail_keys_from_neighbour:  # the last (partial) 64-row query tile reads the next image's keys
        t0 = (N - 1) // 64 * 64
        s[:, :, t0:] = q[:, :, t0:] @ k.roll(1, 0).transpose(-1, -2)
    p = torch.exp(0.125 * (s - s.amax(-1, keepdim=True)))
    o = (p.half().float() @ v) / p.sum(-1, keepdim=True)
    return o.half().permute(0, 2, 1, 3).reshape(B * N, D)


def _vit_params(seed):
    g = lambda i, shape, std, mean=0.0: _randn(shape, seed * 100 + i, std, mean).double()  # noqa: E731
    return {"ln1_g": g(1, (D,), 0.1, 1.0), "ln1_b": g(2, (D,), 0.05), "ln2_g": g(3, (D,), 0.1, 1.0),
            "ln2_b": g(4, (D,), 0.05), "qkv_w": g(5, (3 * D, D), 0.1), "qkv_b": g(6, (3 * D,), 0.02),
            "proj_w": g(7, (D, D), 0.02), "proj_b": g(8, (D,), 0.02), "fc1_w": g(9, (4 * D, D), 0.05),
            "fc1_b": g(10, (4 * D,), 0.02), "fc2_w": g(11, (D, 4 * D), 0.02), "fc2_b": g(12, (D,), 0.02)}


def emu_vit_block(x, p, prev=None, **defect):
    """The trace of one block on the fp32 stream x [B*N, D]. Defects: gelu_tanh, swap_qk_head, tail_keys_from_neighbour,
    ln2_prev (LN2 with `prev`'s weights), proj_x_f16, fc2_segments + bias_every_segment."""
    tr = {"trace_in": x}
    tr["trace_ln1"] = G.layernorm_emulate(x, p["ln1_g"], p["ln1_b"], T.LN_EPS)
    tr["trace_qkv"] = emu_linear(tr["trace_ln1"], p["qkv_w"], p["qkv_b"])
    tr["trace_attn"] = emu_mhsa(tr["trace_qkv"], swap_qk_head=defect.get("swap_qk_head"),
                                tail_keys_from_neighbour=defect.get("tail_keys_from_neighbour", False))
    tr["trace_x1"] = emu_residual(tr["trace_attn"], p["proj_w"], p["proj_b"], x, x_f16=defect.get("proj_x_f16", False))
    ln2 = prev if defect.get("ln2_prev") else p
    tr["trace_ln2"] = G.layernorm_emulate(tr["trace_x1"], ln2["ln2_g"], ln2["ln2_b"], T.LN_EPS)
    tr["trace_fc1"] = emu_linear(tr["trace_ln2"], p["fc1_w"], p["fc1_b"], act="gelu",
                                 gelu_tanh=defect.get("gelu_tanh", False))
    tr["trace_out"] = emu_residual(tr["trace_fc1"], p["fc2_w"], p["fc2_b"], tr["trace_x1"],
                                   segments=defect.get("fc2_segments", 1),
                                   bias_every_segment=defect.get("bias_every_segment", False))
    return tr


def vit_ops(tr, p, **kw):
    """trunk_oracle.vit_block per image, the images' outputs concatenated (one report per op over the batch)."""
    per = [T.vit_block({k: v[b * N:(b + 1) * N] for k, v in tr.items()}, p, HEADS, **kw) for b in range(B)]
    out = {}
    for op in per[0]:
        st = {k: torch.cat([q[op][1][k] for q in per]) for k in per[0][op][1] if k != "b_min"}
        if "b_min" in per[0][op][1]:
            st["b_min"] = per[0][op][1]["b_min"]
        out[op] = (torch.cat([q[op][0] for q in per]), st, per[0][op][2])
    return out


# ResNet: one stride-2 first block of a stage (cin 64 -> width 32 -> cout 128) and one stride-1 block
CIN, WIDTH, COUT, HW = 64, 32, 128, 8


def _conv_w(cout, cin, k, seed):
    return _randn((cout, cin, k, k), seed, math.sqrt(2.0 / (cout * k * k))).double()


def _bn(c, seed, damp=1.0):
    g = torch.Generator().manual_seed(seed)
    sd = {"bn.weight": (1.0 + 0.3 * torch.randn(c, generator=g)) * damp, "bn.bias": 0.1 * torch.randn(c, generator=g),
          "bn.running_mean": 0.1 * torch.randn(c, generator=g), "bn.running_var": 0.5 + torch.rand(c, generator=g)}
    from stage_oracle import fold_bn
    return fold_bn(sd, "bn.")


def _rn_params(seed, cin, down):
    p = {"w1": _conv_w(WIDTH, cin, 1, seed), "w2": _conv_w(WIDTH, WIDTH, 3, seed + 1),
         "w3": _conv_w(COUT, WIDTH, 1, seed + 2), "bn1": _bn(WIDTH, seed + 3), "bn2": _bn(WIDTH, seed + 4),
         "bn3": _bn(COUT, seed + 5, 0.12)}
    if down:
        p["wd"], p["bnd"] = _conv_w(COUT, cin, 1, seed + 6), _bn(COUT, seed + 7)
    return p


def _conv32(x, w, bn, stride=1, pad=0, relu=True):
    y = F.conv2d(x.float().permute(0, 3, 1, 2), _w32(w.float()), stride=stride, padding=pad).permute(0, 2, 3, 1)
    y = y * bn[0].float() + bn[1].float()
    return y.clamp_min(0) if relu else y


def emu_bottleneck(x16, p, stride, ident=None, **defect):
    """The trace of one bottleneck on the fp16 NHWC input. Defects: stride_on_conv1, down_no_subsample,
    relu_before_residual, out16_from_f16."""
    tr = {"trace_in": x16}
    if defect.get("stride_on_conv1"):  # torchvision v1: 1x1 stride s, then 3x3 stride 1
        tr["trace_t1"] = _conv32(x16[:, ::stride, ::stride], p["w1"], p["bn1"]).half()
        tr["trace_t2"] = _conv32(tr["trace_t1"], p["w2"], p["bn2"], pad=1).half()
    else:
        tr["trace_t1"] = _conv32(x16, p["w1"], p["bn1"]).half()
        tr["trace_t2"] = _conv32(tr["trace_t1"], p["w2"], p["bn2"], stride=stride, pad=1).half()
    if "wd" in p:
        if defect.get("down_no_subsample"):  # the downsample GEMM reads the first rows of the full-resolution input
            ho, wo = x16.shape[1] // stride, x16.shape[2] // stride
            rows = x16.reshape(-1, 1, 1, CIN)[:B * ho * wo]
            ident = _conv32(rows, p["wd"], p["bnd"], relu=False).reshape(B, ho, wo, COUT)
        else:
            ident = _conv32(x16[:, ::stride, ::stride], p["wd"], p["bnd"], relu=False)
    tr["trace_id"] = ident
    branch = _conv32(tr["trace_t2"], p["w3"], p["bn3"], relu=False)
    if defect.get("relu_before_residual"):
        tr["trace_out32"] = branch.clamp_min(0) + ident
    else:
        tr["trace_out32"] = (branch + ident).clamp_min(0)
    if defect.get("out16_from_f16"):  # the branch rounded to fp16 before the residual add
        tr["trace_out16"] = (branch.half().float() + ident).clamp_min(0).half()
    else:
        tr["trace_out16"] = tr["trace_out32"].half()
    return tr


# ------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------
def _cases():
    """name -> {op: (got, stage dict, fp16?)} for the faithful emulations; defect -> (tier, op, got, stage dict, fp16?)."""
    cases, defects = {}, {}
    # ViT: a block on a stream of order one, its predecessor's weights for the LN2 defect
    x = _randn((B * N, D), 1, 1.0)
    p, prev = _vit_params(2), _vit_params(3)
    good = emu_vit_block(x, p)
    cases["vit"] = vit_ops(good, p)
    split = emu_vit_block(x, p, fc2_segments=2)
    cases["vit_split"] = {"fc2": vit_ops(split, p, seg_fc2=2)["fc2"]}

    def defect(name, tier, op, tr, **kw):
        got, st, f16 = vit_ops(tr, p, **kw)[op]
        defects[name] = (tier, got, st, f16)

    defect("gelu_tanh", "A", "fc1", emu_vit_block(x, p, gelu_tanh=True))
    defect("qk_swapped_in_one_head", "A", "mhsa", emu_vit_block(x, p, swap_qk_head=1))
    defect("tail_query_tile_reads_neighbour_keys", "A", "mhsa", emu_vit_block(x, p, tail_keys_from_neighbour=True))
    defect("ln2_with_previous_block_weights", "A", "ln2", emu_vit_block(x, p, prev, ln2_prev=True))
    defect("proj_residual_from_fp16_x", "B", "proj", emu_vit_block(x, p, proj_x_f16=True))
    defect("split_bias_added_by_every_segment", "A", "fc2",
           emu_vit_block(x, p, fc2_segments=2, bias_every_segment=True), seg_fc2=2)

    # ResNet: a stride-2 first block of a stage (downsample into the stream), then a stride-1 block on its output
    x16 = _randn((B, HW, HW, CIN), 4, 1.0).clamp_min(0).half()
    p0, p1 = _rn_params(10, CIN, True), _rn_params(20, COUT, False)
    t0 = emu_bottleneck(x16, p0, 2)
    t1 = emu_bottleneck(t0["trace_out16"], p1, 1, ident=t0["trace_out32"])
    cases["rn_first"] = T.bottleneck(t0, p0, 2)
    cases["rn_next"] = T.bottleneck(t1, p1, 1)

    def rn_defect(name, tier, op, **kw):
        got, st, f16 = T.bottleneck(emu_bottleneck(x16, p0, 2, **kw), p0, 2)[op]
        defects[name] = (tier, got, st, f16)

    rn_defect("relu_before_residual", "A", "out32", relu_before_residual=True)
    rn_defect("downsample_without_subsample", "A", "downsample", down_no_subsample=True)
    rn_defect("out16_from_fp16_intermediate", "B", "out16", out16_from_f16=True)
    # torchvision v1 (stride on conv1): its conv2 output against the v1.5 reference fed the same block input
    v1 = emu_bottleneck(x16, p0, 2, stride_on_conv1=True)
    st = T.conv_bn(t0["trace_t1"], p0["w2"], p0["bn2"], stride=2, pad=1)
    defects["stride_on_conv1_torchvision_v1"] = ("A", v1["trace_t2"], st, True)
    return cases, defects


@pytest.fixture(scope="module")
def trunk_cases():
    return _cases()


def test_emulated_ops_pass(trunk_cases):
    cases, _ = trunk_cases
    report, bad = {}, {}
    for name, ops in cases.items():
        report[name], fails = T.judge(ops)
        if fails:
            bad[name] = fails
    print("TRUNK_CPU " + json.dumps(report))
    assert not bad, bad


def test_planted_defects_are_caught(trunk_cases):
    _, defects = trunk_cases
    import stage_oracle as S
    report, missed = {}, []
    for name, (tier, got, st, f16) in defects.items():
        rep, fails = S.check(got, st, f16)
        caught = [f for f in fails if f.startswith(f"tier {tier}")]
        report[name] = {**rep, "tier": tier, "caught": bool(caught)}
        if not caught:
            missed.append(name)
    print("TRUNK_DEFECTS_CPU " + json.dumps(report))
    assert not missed, (missed, report)


def test_stream_k_segments():
    """fc2 of ViT-L/16 at B = 8, 480 x 480 on 132 CTAs: 456 tiles of 64 k-chunks, ~221 per CTA -> at most 2 per tile;
    a tile longer than a CTA's range spans more."""
    assert T.stream_k_segments(8 * 901, 1024, 4096, 132) == 2
    assert T.stream_k_segments(1000, 256, 64 * 64, 132) >= 3
