"""Every stage of the engine's image path, element by element, fed the engine's own input of that stage.

One forward per case; then, per image (float64 references on the device stay at a few GB), each stage buffer the engine
names (`Engine.debug_tensor`: readout3, post{k}, layer{k}, rn{k}, dec{k}_*, path1, featn, feat_sumsq, logits_lr) is
checked against the float64 reference of tests/stage_oracle.py computed from the engine's buffer that feeds it: tier A
(every element within the derived bound) and tier B (fp16 outputs mostly bit-identical to the rounded reference, fp32
outputs free of hidden fp16 roundings). Exact contracts on top: the ReLU'd fp16 copies equal relu(fp32) rounded once,
the channel pad of ViT-B/32's first level (96 -> 128) is exactly zero, and the identity level is the post buffer itself.
Each case prints one STAGES json line: per stage the worst err / bound ratio and the tier-B figure (worst image).

The A/B switches LSEG_OUTCONV_F16 and LSEG_SPLITK_FIXED are read once per process: a subprocess runs one small case
under each setting and saves its stage buffers; this process checks them.
"""
import json
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import stage_oracle as S
from parity_util import state_dict, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F16, F32 = torch.float16, torch.float32

_ENGINES = {}


def _engine(bb, **kw):
    """One engine resident at a time (weights + plans: a few GB of a shared card)."""
    key = (bb, tuple(sorted(kw.items())))
    if key not in _ENGINES:
        from lseg_b200.engine import Engine
        _ENGINES.clear()
        torch.cuda.empty_cache()
        sd = synth.make_state_dict(0, head_block=True) if kw else state_dict(0, bb)
        _ENGINES[key] = (Engine(sd, torch.device("cuda:0"), backbone=bb, **kw), sd)
    return _ENGINES[key]


def _text(rows, out_c, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.randn((rows, out_c), generator=g)
    return (t / t.norm(dim=-1, keepdim=True)).half()


def _pad(t, dim, n):
    if t.shape[dim] == n:
        return t
    shape = list(t.shape)
    shape[dim] = n - t.shape[dim]
    return torch.cat([t, torch.zeros(shape, dtype=t.dtype)], dim=dim)


def _geometry(bb, H, W):
    from lseg_b200.packing import BACKBONES, stored_channels
    cfg = BACKBONES[bb]
    if cfg.get("trunk") == "resnet101":
        return cfg, [H // 4 >> k for k in range(4)], [W // 4 >> k for k in range(4)], list(cfg["features"])
    P = cfg["patch"]
    gh, gw = H // P, W // P
    f = [gh * r if r > 0 else (gh if r == 0 else gh // 2) for r in cfg["resample"]]
    g = [gw * r if r > 0 else (gw if r == 0 else gw // 2) for r in cfg["resample"]]
    return cfg, f, g, [stored_channels(c) for c in cfg["features"]]


def buffer_specs(bb, out_c, B, H, W, K, lr_f16_mask=0):
    """name -> (shape, dtype) of every stage buffer a forward of this shape leaves behind."""
    cfg, lh, lw, cp = _geometry(bb, H, W)
    spec = {}
    if "patch" in cfg:
        P, D = cfg["patch"], cfg["dim"]
        T = (H // P) * (W // P)
        spec["readout3"] = ((B * T, D), F16)
        for k in range(4):
            spec[f"tap{k}"] = ((B, T + 1, D), F32)
            spec[f"post{k}"] = ((B * T, cp[k]), F16)
    for k in range(4):
        px = (B, lh[k], lw[k])
        spec[f"layer{k}"] = (px + (cp[k],), F16)
        spec[f"rn{k}"] = (px + (256,), F32)
        spec[f"rn{k}_relu"] = (px + (256,), F16)
        if k < 3:
            spec[f"dec{k}_sum"] = (px + (256,), F32)
            spec[f"dec{k}_sum_relu"] = (px + (256,), F16)
        spec[f"dec{k}_tmp"] = (px + (256,), F16)
        spec[f"dec{k}_rcu2"] = (px + (256,), F16)
        spec[f"dec{k}_out_lr"] = (px + (256,), F16 if (lr_f16_mask >> k) & 1 else F32)
        if k > 0:
            spec[f"dec{k}_skip"] = ((B, 2 * lh[k], 2 * lw[k], 256), F32)
    spec["path1"] = ((B, H // 2, W // 2, 256), F16)
    spec["featn"] = ((B, H // 2, W // 2, out_c), F16)
    spec["feat_sumsq"] = ((B, H // 2, W // 2, out_c // 32), F32)
    spec["logits_lr"] = ((B, K, H // 2, W // 2), F16)
    return spec


class Report:
    def __init__(self):
        self.stages, self.fails = {}, []

    def check(self, name, got, st, f16):
        rep, fails = S.check(got, st, f16)
        old = self.stages.get(name)
        if old:  # worst image: largest ratio, smallest identical fraction / largest RMS
            rep = {"worst": max(old["worst"], rep["worst"]),
                   "tier_b": min(old["tier_b"], rep["tier_b"]) if f16 else max(old["tier_b"], rep["tier_b"])}
        self.stages[name] = rep
        self.fails += [f"{name}: {f}" for f in fails]

    def exact(self, name, ok):
        if not ok:
            self.fails.append(f"{name}: not exact")


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _dec(sd, k, unit):
    q = f"scratch.refinenet{k + 1}.{unit}."
    return sd[q + "conv1.weight"], S.fold_bn(sd, q + "bn1."), sd[q + "conv2.weight"], S.fold_bn(sd, q + "bn2.")


def check_stages(get, sd, bb, out_c, B, H, W, K, text, stride=0, lr_f16_mask=0, logit_scale=None):
    """get(name) -> the stage buffer (cuda, shaped by buffer_specs). Returns a Report."""
    from lseg_b200.packing import reference_logit_scale
    cfg, lh, lw, cp = _geometry(bb, H, W)
    rep = Report()
    vit = "patch" in cfg
    for b in range(B):
        one = slice(b, b + 1)
        if vit:
            P, D = cfg["patch"], cfg["dim"]
            gh, gw = H // P, W // P
            T = gh * gw
            rows = slice(b * T, (b + 1) * T)
            for k in range(4):
                q = f"pretrained.act_postprocess{k + 1}."
                c = cfg["features"][k]
                ro = S.readout(get(f"tap{k}")[one], sd[q + "0.project.0.weight"], sd[q + "0.project.0.bias"])
                wp, bp = _pad(sd[q + "3.weight"], 0, cp[k]), _pad(sd[q + "3.bias"], 0, cp[k])
                post = get(f"post{k}")[rows]
                if k == 3:  # stage 1: tap -> readout; stage 2: readout -> post
                    rep.check("readout3", get("readout3")[rows], ro, True)
                    rep.check("post3", post, S.post(get("readout3")[rows], wp, bp), True)
                else:  # the readout of levels 0-2 is overwritten: tap -> post through both GEMMs
                    rep.check(f"post{k}", post, S.post(ro["ref"], wp, bp, e_in=ro["bound"]), True)
                rep.exact(f"post{k}_pad_zero", bool((post[:, c:] == 0).all()))
                # stage 3: resample
                r = cfg["resample"][k]
                lay = get(f"layer{k}")[one]
                x = post.reshape(1, gh, gw, cp[k])
                if r == 0:
                    rep.exact(f"layer{k}_is_post{k}", _bits_equal(lay, x))
                else:
                    wr = _pad(_pad(sd[q + "4.weight"], 0, cp[k]), 1, cp[k])
                    rep.check(f"layer{k}", lay, S.resample(x, r, wr, _pad(sd[q + "4.bias"], 0, cp[k])), True)
                rep.exact(f"layer{k}_pad_zero", bool((lay[..., c:] == 0).all()))
        # stage 4: layer_rn, fp32 + its ReLU'd fp16 copy
        for k in range(4):
            w = _pad(sd[f"scratch.layer{k + 1}_rn.weight"], 1, cp[k])
            rn = get(f"rn{k}")[one]
            rep.check(f"rn{k}", rn, S.conv3x3(get(f"layer{k}")[one], w), False)
            rep.exact(f"rn{k}_relu", _bits_equal(get(f"rn{k}_relu")[one], rn.clamp_min(0).half()))
        for k in range(3, -1, -1):
            if k < 3:  # stage 5: RCU1 + the skip sum
                w1, bn1, w2, bn2 = _dec(sd, k, "resConfUnit1")
                sm = get(f"dec{k}_sum")[one]
                rep.check(f"dec{k}_sum", sm, S.rcu1(get(f"rn{k}_relu")[one], get(f"dec{k + 1}_skip")[one], w1, bn1,
                                                    w2, bn2), False)
                rep.exact(f"dec{k}_sum_relu", _bits_equal(get(f"dec{k}_sum_relu")[one], sm.clamp_min(0).half()))
                x16, x32 = get(f"dec{k}_sum_relu")[one], sm
            else:
                x16, x32 = get("rn3_relu")[one], get("rn3")[one]
            w1, bn1, w2, bn2 = _dec(sd, k, "resConfUnit2")
            tmp = get(f"dec{k}_tmp")[one]  # stage 6: RCU2 conv1; stage 7: conv2 + fp32 residual
            rep.check(f"dec{k}_tmp", tmp, S.conv3x3(x16, w1, scale=bn1[0], shift=bn1[1], act="relu", out_f16=True), True)
            r2 = get(f"dec{k}_rcu2")[one]
            rep.check(f"dec{k}_rcu2", r2, S.conv3x3(tmp, w2, scale=bn2[0], shift=bn2[1], res=(x32,), out_f16=True), True)
            # stage 8: out_conv at low res; stage 9: x2 interpolation (+ the next level's layer_rn), fed that buffer; and
            # the two together against the reference module's order (interpolate, then out_conv)
            q = f"scratch.refinenet{k + 1}.out_conv."
            lr16 = bool((lr_f16_mask >> k) & 1)
            oc = get(f"dec{k}_out_lr")[one]
            rep.check(f"dec{k}_out_lr", oc, S.out_conv(r2, sd[q + "weight"], sd[q + "bias"], out_f16=lr16), lr16)
            add = get(f"rn{k - 1}")[one] if k > 0 else None
            out = get(f"dec{k}_skip")[one] if k > 0 else get("path1")[one]
            name = f"dec{k}_skip" if k > 0 else "path1"
            rep.check(name, out, S.upsample_skip(oc, add, out_f16=k == 0), k == 0)
            rep.check(name + "_vs_interpolate_then_conv", out,
                      S.out_conv_upsampled(r2, sd[q + "weight"], sd[q + "bias"], add, lr_f16=lr16, out_f16=k == 0),
                      k == 0)
        # stage 10: head1 -> featn + partial squared norms; stage 11: pixel x text
        featn, ss = get("featn")[one], get("feat_sumsq")[one]
        st_f, st_s = S.head1(get("path1")[one], sd["scratch.head1.weight"], sd["scratch.head1.bias"])
        rep.check("featn", featn, st_f, True)
        rep.check("feat_sumsq", ss, st_s, False)
        P2 = (H // 2) * (W // 2)
        tb = text[b * stride:] if stride else text
        st = S.pixel_text(featn.reshape(1, P2, out_c), ss.reshape(1, P2, -1), tb, K,
                          logit_scale if logit_scale is not None else reference_logit_scale(), stride)
        rep.check("logits_lr", get("logits_lr")[one].reshape(1, K, P2), st, True)
    return rep


def _report(name, rep):
    print("STAGES " + json.dumps({"case": name, **rep.stages}))


def _run_case(bb, B, H, W, K, zs=False):
    eng, sd = _engine(bb)
    x = synth.make_image(B, H, W, seed=B * 1000 + H + 7).cuda()
    stride = 0
    if zs:  # LSegRNNetZS's operand: image b's pair of labels at rows [2b, 2b + 2)
        stride, K = 2, 2
        text = _text(eng.padded_rows(B * 2), eng.out_c, H + W)
    else:
        text = _text(eng.padded_rows(K), eng.out_c, H + W)
    text = text.cuda()
    eng.forward(x, text, K, text_image_stride=stride)
    torch.cuda.synchronize()
    spec = buffer_specs(bb, eng.out_c, B, H, W, K)
    rep = check_stages(lambda n: eng.debug_tensor(n, *spec[n]), sd, bb, eng.out_c, B, H, W, K, text, stride)
    _report(f"{bb}_B{B}_{H}x{W}_K{K}" + ("_zs" if zs else ""), rep)
    assert not rep.fails, rep.fails


# (1, 32, 32): the deepest level is 1x1, so 8 of the 9 taps of its 3x3 convs read padding; (2, 160, 224, 300): more
# than one N tile of the pixel x text GEMM; 480^2 at B = 1 / 8: the benchmark shapes
@pytest.mark.parametrize("B,H,W,K", [(1, 32, 32, 3), (2, 64, 96, 7), (2, 160, 224, 300), (2, 480, 480, 150),
                                     (8, 480, 480, 150)])
def test_stages_vitl16(B, H, W, K):
    _run_case("clip_vitl16_384", B, H, W, K)


@pytest.mark.parametrize("B,H,W,K", [(3, 160, 224, 7), (1, 32, 32, 2)])
def test_stages_vitb32(B, H, W, K):
    """ConvT x8 / x4 / x2 and the identity level; the 96 -> 128 channel pad of level 0."""
    _run_case("clip_vitb32_384", B, H, W, K)


def test_stages_rn50x16():
    """out_c = 768: 24 partial squared norms per pixel."""
    _run_case("clipRN50x16_vitl16_384", 2, 64, 96, 5)


def test_stages_rn101_zero_shot():
    """ResNet-101 stages into layer_rn (2048 channels at level 3: K = 18432), the grouped zero-shot pixel x text."""
    _run_case("clip_resnet101", 3, 96, 128, 2, zs=True)


@pytest.mark.parametrize("arch,act", [(1, "lrelu"), (2, "tanh")])
def test_stages_head_blocks(arch, act):
    """Stage 12 (arch_option 1 / 2, block_depth 2): the fp16 low-res logits -> head blocks -> x2 -> the fp32 logits."""
    from lseg_b200._lib import HEAD_ACT
    eng, sd = _engine("clip_vitl16_384", arch_option=arch, block_depth=2, activation=act)
    B, H, W, K = 2, 64, 96, 5
    x = synth.make_image(B, H, W, seed=2064).cuda()
    text = _text(eng.padded_rows(K), eng.out_c, 5).cuda()
    out = eng.forward(x, text, K)
    torch.cuda.synchronize()
    lr = eng.debug_tensor("logits_lr", (B, K, H // 2, W // 2), F16)
    w9 = sd["scratch.head_block.depthwise.depthwise.weight"].reshape(9).tolist()
    bias = float(sd["scratch.head_block.depthwise.depthwise.bias"].reshape(-1)[0])
    rep = Report()
    rep.check("logits", out, S.head_blocks(lr, w9, bias, arch, HEAD_ACT[act], 2), False)
    _report(f"head_blocks_opt{arch}_{act}", rep)
    assert not rep.fails, rep.fails


_SWITCH_SCRIPT = """
import sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import lseg_b200
import test_image_stages_gpu as T
bb, B, H, W, K, mask = "clip_vitl16_384", 2, 64, 96, 7, int(sys.argv[3])
eng, sd = T._engine(bb)
x = T.synth.make_image(B, H, W, seed=B * 1000 + H + 7).cuda()
text = T._text(eng.padded_rows(K), eng.out_c, H + W).cuda()
eng.forward(x, text, K)
spec = T.buffer_specs(bb, eng.out_c, B, H, W, K, mask)
torch.save({n: eng.debug_tensor(n, *s).cpu() for n, s in spec.items()}, sys.argv[2])
"""


@pytest.mark.parametrize("env", [{"LSEG_OUTCONV_F16": "15"}, {"LSEG_SPLITK_FIXED": "0"}, {"LSEG_SPLITK_FIXED": "3"}])
def test_stages_under_switches(env):
    """LSEG_OUTCONV_F16=15: every dec{k}_out_lr is fp16 (its stage moves to the fp16 tier; the interpolation stage keeps
    its bound, being fed that buffer). LSEG_SPLITK_FIXED=0 / 3: no / three-way split-K of the decoder convs; every bound
    and tier holds unchanged."""
    mask = int(env.get("LSEG_OUTCONV_F16", "0"))
    B, H, W, K = 2, 64, 96, 7
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "stages.pt")
        subprocess.run([sys.executable, "-c", _SWITCH_SCRIPT, ROOT, path, str(mask)], env=dict(os.environ, **env),
                       check=True, timeout=1200)
        bufs = torch.load(path)
    sd = state_dict(0)
    text = _text(((K + 127) // 128) * 128, 512, H + W)
    text = text.cuda()
    rep = check_stages(lambda n: bufs[n].cuda(), sd, "clip_vitl16_384", 512, B, H, W, K, text, lr_f16_mask=mask)
    _report("switch_" + "_".join(f"{k}={v}" for k, v in env.items()), rep)
    assert not rep.fails, rep.fails
