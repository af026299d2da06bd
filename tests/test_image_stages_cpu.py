"""The image-path stage bounds of tests/stage_oracle.py are neither too loose nor too tight: on CPU, a float32 emulation of
each stage's recipe in the engine (fp16 operands, fp32 accumulation, the engine's rounding points) passes both tiers,
and an emulation with one planted defect fails the tier named for it. Small shapes; the weight and activation scales
are those of the seeded synthetic network (outputs of order one, kaiming-scaled weights, BatchNorm scales away from 1).
"""
import json
import math

import pytest
import torch
import torch.nn.functional as F

import glue_oracle as G
import stage_oracle as S

LS = math.exp(math.log(1 / 0.07))
F32 = torch.float32


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64) * scale


def _conv_w(cout, cin, k, seed):
    return _randn((cout, cin, k, k), seed, 1.0 / math.sqrt(cin * k * k)).float()


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    sd = {"bn.weight": 1.0 + 0.3 * torch.randn(c, generator=g), "bn.bias": 0.2 * torch.randn(c, generator=g),
          "bn.running_mean": 0.2 * torch.randn(c, generator=g), "bn.running_var": 0.5 + torch.rand(c, generator=g)}
    return S.fold_bn(sd, "bn.")


def _f16(t):
    return t.to(torch.float16)


def _w32(w):
    return S.w16(w).float()


# ------------------------------------------------------------------------------------------------------------------
# float32 emulations of the engine's recipe; keyword flags plant one defect each
# ------------------------------------------------------------------------------------------------------------------
def gelu_erf32(x):
    """common.cuh gelu_erf in fp32: x / (1 + 2^(x P(x^2))) with its degree-4 fit P (exact exp2 and reciprocal here)."""
    u = x * x
    p = ((((u * -3.228989445e-06 + 8.823814435e-05) * u + 3.602744768e-04) * u - 1.052266877e-01) * u
         - 2.302045391e+00)
    return x * (1.0 / (1.0 + torch.exp2(x * p)))


def emu_readout(tap, w, b, *, cls_neighbour=False):
    x = tap.half().float()
    D = x.shape[-1]
    tok, cls = x[:, 1:], x[:, 0]
    if cls_neighbour:
        cls = cls.roll(1, 0)
    clsb = cls @ _w32(w[:, D:]).t() + b.float()
    pre = tok @ _w32(w[:, :D]).t() + clsb[:, None]
    return gelu_erf32(pre).reshape(-1, D).half()


def emu_linear(x, w, b, *, out_f16=True, extra_f16=False):
    y = x.float() @ _w32(w.reshape(w.shape[0], -1)).t() + b.float()
    if extra_f16:
        y = y.half().float()
    return y.half() if out_f16 else y


def _conv(x, w, stride=1, pad=1, leak_rows=False):
    """fp32 conv of NHWC x; leak_rows: the images stacked into one tall image, so the zero padding rows of image b read
    the neighbouring image's border row."""
    xc = x.float().permute(0, 3, 1, 2)
    if leak_rows:
        B, C, h, wd = xc.shape
        y = F.conv2d(xc.permute(1, 0, 2, 3).reshape(1, C, B * h, wd), _w32(w), stride=stride, padding=pad)
        return y.reshape(-1, B, h, wd).permute(1, 2, 3, 0)
    return F.conv2d(xc, _w32(w), stride=stride, padding=pad).permute(0, 2, 3, 1)


def emu_resample(x, r, w, b, *, transpose_taps=False):
    xc = x.float().permute(0, 3, 1, 2)
    if r > 0:
        wt = w.transpose(2, 3) if transpose_taps else w
        y = F.conv_transpose2d(xc, _w32(wt), b.float(), stride=r)
    else:
        y = F.conv2d(xc, _w32(w), b.float(), stride=2, padding=1)
    return y.permute(0, 2, 3, 1).half()


def emu_conv3x3(x, w, scale=None, shift=None, act=None, res=(), *, out_f16=False, shift_first=False, leak_rows=False):
    y = _conv(x, w, leak_rows=leak_rows)
    if scale is not None:
        y = (y + shift.float()) * scale.float() if shift_first else y * scale.float() + shift.float()
    if act == "relu":
        y = y.clamp_min(0)
    for r in res:
        y = y + r
    return y.half() if out_f16 else y


def emu_rcu1(x_relu, skip, w1, bn1, w2, bn2, *, skip_f16=False):
    h = emu_conv3x3(x_relu, w1, *bn1, act="relu", out_f16=True)
    return emu_conv3x3(h, w2, *bn2, res=(skip.half().float() if skip_f16 else skip,))


def emu_upsample(x, add=None, *, out_f16=False, align_false=False):
    xc = x.float().permute(0, 3, 1, 2)
    if align_false:
        y = F.interpolate(xc, scale_factor=2, mode="bilinear", align_corners=False)
    else:
        y = G.upsample2x_emulate(xc)
    y = y.permute(0, 2, 3, 1)
    if add is not None:
        y = y + add
    return y.half() if out_f16 else y


def emu_head1(p1, w, b, *, sumsq_from_f16=False):
    f = p1.float() @ _w32(w.reshape(w.shape[0], -1)).t() + b.float()
    featn = f.half()
    src = featn.float() if sumsq_from_f16 else f
    ss = (src * src).reshape(f.shape[:-1] + (f.shape[-1] // 32, 32)).sum(-1)
    return featn, ss


def emu_pixel_text(featn, sumsq, text, K, stride=0):
    B = featn.shape[0]
    mul = torch.tensor(LS, dtype=F32) * torch.rsqrt(sumsq.sum(-1, keepdim=True))
    out = []
    for b in range(B):
        t = text[b * stride:b * stride + K] if stride else text[:K]
        out.append((featn[b].float() @ t.float().t() * mul[b]).half().t())
    return torch.stack(out)


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
B, h, w = 2, 4, 6  # a decoder level: B >= 2 for the cross-image defects


def _act(shape, seed, scale=1.0):
    return _randn(shape, seed, scale).float()


def _stage_cases():
    """name -> (got, stage dict, fp16?) for the faithful emulation and every planted defect; defects list which tier
    must catch them."""
    cases, defects = {}, {}
    # 1. readout (ViT-B/32 width, T = 2x3 tokens)
    D = 768
    tap = _act((B, 7, D), 1, 2.0)
    wr, br = _act((D, 2 * D), 2, 1.0 / math.sqrt(2 * D)), _act((D,), 3, 0.1)
    st = S.readout(tap, wr, br)
    cases["readout"] = (emu_readout(tap, wr, br), st, True)
    defects["readout_cls_from_neighbour_image"] = ("A", emu_readout(tap, wr, br, cls_neighbour=True), st, True)
    # 2. post, from the observable readout and from the tap through the unobservable one
    c = 128
    wp, bp = _conv_w(c, D, 1, 4), _act((c,), 5, 0.1)
    ro = emu_readout(tap, wr, br)
    cases["post"] = (emu_linear(ro, wp, bp), S.post(ro, wp, bp), True)
    ro_ref = S.readout(tap, wr, br)
    cases["tap_to_post"] = (emu_linear(ro, wp, bp), S.post(ro_ref["ref"], wp, bp, e_in=ro_ref["bound"]), True)
    # 3. resample: ConvTranspose x4, 3x3 stride 2
    pk = _f16(_act((B, 2, 3, c), 6))
    wt, bt = _randn((c, c, 4, 4), 7, 1.0 / math.sqrt(c)).float(), _act((c,), 8, 0.1)
    st = S.resample(pk, 4, wt, bt)
    cases["resample_convT"] = (emu_resample(pk, 4, wt, bt), st, True)
    defects["convT_taps_transposed"] = ("A", emu_resample(pk, 4, wt, bt, transpose_taps=True), st, True)
    pk2 = _f16(_act((B, 2 * h, 2 * w, c), 9))
    ws, bs = _conv_w(c, c, 3, 10), _act((c,), 11, 0.1)
    cases["resample_conv_s2"] = (emu_resample(pk2, -2, ws, bs), S.resample(pk2, -2, ws, bs), True)
    # 4. layer_rn (fp32)
    lay = _f16(_act((B, h, w, c), 12))
    wl = _conv_w(256, c, 3, 13)
    st = S.conv3x3(lay, wl)
    cases["layer_rn"] = (emu_conv3x3(lay, wl), st, False)
    defects["conv_pad_row_from_neighbour_image"] = ("A", emu_conv3x3(lay, wl, leak_rows=True), st, False)
    rn = emu_conv3x3(lay, wl)
    rn_relu = rn.clamp_min(0).half()
    # 5. RCU1: conv2(relu(bn1(conv1(rn_relu)))) + skip
    w1, w2 = _conv_w(256, 256, 3, 14), _conv_w(256, 256, 3, 15)
    bn1, bn2 = _bn(256, 16), _bn(256, 17)
    skip = _act((B, h, w, 256), 18, 1.5)
    st = S.rcu1(rn_relu, skip, w1, bn1, w2, bn2)
    cases["rcu1"] = (emu_rcu1(rn_relu, skip, w1, bn1, w2, bn2), st, False)
    defects["skip_from_wrong_level"] = ("A", emu_rcu1(rn_relu, rn, w1, bn1, w2, bn2), st, False)
    defects["rcu1_residual_from_fp16_copy"] = ("B", emu_rcu1(rn_relu, skip, w1, bn1, w2, bn2, skip_f16=True), st,
                                               False)
    # 6. RCU2 conv1 (fp16 out), 7. RCU2 conv2 + fp32 residual (fp16 out)
    sm = emu_rcu1(rn_relu, skip, w1, bn1, w2, bn2)
    sm_relu = sm.clamp_min(0).half()
    st = S.conv3x3(sm_relu, w1, scale=bn1[0], shift=bn1[1], act="relu", out_f16=True)
    cases["rcu2_conv1"] = (emu_conv3x3(sm_relu, w1, *bn1, act="relu", out_f16=True), st, True)
    defects["bn_shift_before_scale"] = ("A", emu_conv3x3(sm_relu, w1, *bn1, act="relu", out_f16=True,
                                                         shift_first=True), st, True)
    tmp = emu_conv3x3(sm_relu, w1, *bn1, act="relu", out_f16=True)
    st = S.conv3x3(tmp, w2, scale=bn2[0], shift=bn2[1], res=(sm,), out_f16=True)
    cases["rcu2_conv2"] = (emu_conv3x3(tmp, w2, *bn2, res=(sm,), out_f16=True), st, True)
    defects["rcu2_residual_from_fp16_copy"] = ("B", emu_conv3x3(tmp, w2, *bn2, res=(sm.half().float(),),
                                                                out_f16=True), st, True)
    # 8. out_conv (fp32; fp16 under LSEG_OUTCONV_F16)
    r2 = emu_conv3x3(tmp, w2, *bn2, res=(sm,), out_f16=True)
    wo, bo = _conv_w(256, 256, 1, 19), _act((256,), 20, 0.1)
    st = S.out_conv(r2, wo, bo)
    oc = emu_linear(r2, wo, bo, out_f16=False)
    cases["out_conv"] = (oc, st, False)
    cases["out_conv_f16"] = (emu_linear(r2, wo, bo), S.out_conv(r2, wo, bo, out_f16=True), True)
    defects["out_lr_extra_fp16_rounding"] = ("B", emu_linear(r2, wo, bo, out_f16=False, extra_f16=True), st, False)
    # 9. upsample + skip (fp32), the level-0 path1 (fp16), and the out_conv reorder against interpolate-then-conv
    rn_next = _act((B, 2 * h, 2 * w, 256), 21)
    st = S.upsample_skip(oc, rn_next)
    cases["upsample_skip"] = (emu_upsample(oc, rn_next), st, False)
    defects["upsample_align_corners_false"] = ("A", emu_upsample(oc, rn_next, align_false=True), st, False)
    cases["upsample_path1"] = (emu_upsample(oc, out_f16=True), S.upsample_skip(oc, out_f16=True), True)
    cases["out_conv_reorder"] = (emu_upsample(oc, rn_next), S.out_conv_upsampled(r2, wo, bo, rn_next), False)
    # 10. head1 -> featn (fp16), feat_sumsq (fp32)
    p1 = emu_upsample(oc, out_f16=True)
    wh, bh = _conv_w(512, 256, 1, 22), _act((512,), 23, 0.1)
    featn, ss = emu_head1(p1, wh, bh)
    st_f, st_s = S.head1(p1, wh, bh)
    cases["head1_featn"] = (featn, st_f, True)
    cases["head1_sumsq"] = (ss, st_s, False)
    defects["sumsq_from_fp16_featn"] = ("B", emu_head1(p1, wh, bh, sumsq_from_f16=True)[1], st_s, False)
    # 11. pixel x text: one label set with K > 256 (more than one N tile), and the grouped zero-shot layout
    fr, sr = featn.reshape(B, -1, 512), ss.reshape(B, -1, 16)
    text = _act((300, 512), 24)
    text = _f16(text / text.norm(dim=-1, keepdim=True))
    cases["pixel_text"] = (emu_pixel_text(fr, sr, text, 300), S.pixel_text(fr, sr, text, 300, LS), True)
    cases["pixel_text_grouped"] = (emu_pixel_text(fr, sr, text, 2, stride=5),
                                   S.pixel_text(fr, sr, text, 2, LS, stride=5), True)
    # 12. head blocks (arch_option 1 / 2, block_depth 2) + output interpolation
    lr = cases["pixel_text"][0][:, :7].reshape(B, 7, h * 2, w * 2)
    w9 = [0.1, -0.2, 0.05, 0.3, 0.4, -0.1, 0.2, 0.0, -0.3]
    for mode, act in ((1, 2), (2, 3)):
        y = G.head_block_emulate(G.head_block_emulate(lr, w9, 0.05, mode, act), w9, 0.05, mode, 0)
        cases[f"head_blocks_opt{mode}"] = (G.upsample2x_emulate(y), S.head_blocks(lr, w9, 0.05, mode, act, 2), False)
    return cases, defects


@pytest.fixture(scope="module")
def stage_cases():
    return _stage_cases()


def test_emulated_stages_pass(stage_cases):
    cases, _ = stage_cases
    report, bad = {}, {}
    for name, (got, st, f16) in cases.items():
        report[name], fails = S.check(got, st, f16)
        if fails:
            bad[name] = fails
    print("STAGES_CPU " + json.dumps(report))
    assert not bad, bad


def test_planted_defects_are_caught(stage_cases):
    _, defects = stage_cases
    report, missed = {}, []
    for name, (tier, got, st, f16) in defects.items():
        rep, fails = S.check(got, st, f16)
        caught = [f for f in fails if f.startswith(f"tier {tier}")]
        report[name] = {**rep, "tier": tier, "caught": bool(caught)}
        if not caught:
            missed.append(name)
    print("DEFECTS_CPU " + json.dumps(report))
    assert not missed, (missed, report)
