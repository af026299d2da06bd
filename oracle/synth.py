"""TEST INFRASTRUCTURE (oracle side) — seeded synthetic weights, tokens and images for LSeg.

No checkpoints, CLIP BPE vocabulary or datasets exist offline (SURVEY.md Appendix B), so every
parity/bench run uses this deterministic stand-in data. Weights come from numpy's PCG64 stream
(bit-reproducible across machines for the same numpy version), with the state-dict key names and
shapes of SURVEY.md Appendix C so the same dict loads into the reference modules, the oracle and
the H100 build. Init scales mirror the constructors (timm trunc_normal .02, torch Conv2d default
kaiming-uniform, CLIP initialize_parameters); LayerNorm/BatchNorm statistics and biases are
perturbed so that folding and bias paths are actually exercised.
"""
import zlib

import numpy as np
import torch

VIT_DEPTH = 24
VIT_DIM = 1024
TEXT_DEPTH = 12
TEXT_WIDTH = 512
CONTEXT = 77
VOCAB = 49408
SOT, EOT = 49406, 49407


class _Gen:
    def __init__(self, seed):
        self.rng = np.random.Generator(np.random.PCG64(seed))

    def normal(self, shape, std, mean=0.0):
        a = self.rng.standard_normal(size=shape, dtype=np.float32)
        a *= np.float32(std)
        if mean:
            a += np.float32(mean)
        return torch.from_numpy(a)

    def uniform(self, shape, lo, hi):
        a = self.rng.random(size=shape, dtype=np.float32)
        return torch.from_numpy(a * np.float32(hi - lo) + np.float32(lo))

    def kaiming(self, shape):
        fan_in = int(np.prod(shape[1:]))
        b = 1.0 / np.sqrt(fan_in)
        return self.uniform(shape, -b, b)


# image backbones (modules/models/lseg_vit.py:221-238 + 408-532; 259-405): trunk geometry, reassemble channels and
# the resampling op behind each 1x1 conv (s > 0 ConvTranspose2d k=s stride=s, -2 Conv2d 3x3 stride 2, 0 none)
# `text`: (transformer_width, embed_dim) of the CLIP text tower — ViT-B/32's or RN50x16's (lseg_vit.py:224, 243, 260)
BACKBONE_SHAPES = {
    "clip_vitl16_384": dict(dim=1024, depth=24, patch=16, feats=(256, 512, 1024, 1024), resample=(4, 2, 0, -2),
                            text=(512, 512)),
    "clipRN50x16_vitl16_384": dict(dim=1024, depth=24, patch=16, feats=(256, 512, 1024, 1024), resample=(4, 2, 0, -2),
                                   text=(768, 768)),
    "clip_vitb32_384": dict(dim=768, depth=12, patch=32, feats=(96, 192, 384, 768), resample=(8, 4, 2, 0),
                            text=(512, 512)),
    # zero-shot ResNet trunk (lseg_net_zs.py:240-339): no ViT, the scratch decoder takes resnet101's four stages
    "clip_resnet101": dict(feats=(256, 512, 1024, 2048), text=(512, 512)),
}


def _resnet101_state(g, sd):
    """torchvision resnet101 parameters under the key names of _make_resnet_backbone (lseg_blocks_zs.py:109-119):
    pretrained.layer1 = Sequential(conv1, bn1, relu, maxpool, layer1), pretrained.layer2..4 = resnet.layer2..4."""
    def bn(prefix, c):
        sd[prefix + "weight"] = g.uniform((c,), 0.5, 1.5)
        sd[prefix + "bias"] = g.normal((c,), 0.1)
        sd[prefix + "running_mean"] = g.normal((c,), 0.1)
        sd[prefix + "running_var"] = g.uniform((c,), 0.5, 1.5)
        sd[prefix + "num_batches_tracked"] = torch.tensor(100, dtype=torch.int64)

    def conv(shape):  # kaiming-normal fan_out like torchvision's ResNet init, damped so 33 blocks stay O(1)
        fan_out = shape[0] * shape[2] * shape[3]
        return g.normal(shape, (2.0 / fan_out) ** 0.5)

    sd["pretrained.layer1.0.weight"] = conv((64, 3, 7, 7))
    bn("pretrained.layer1.1.", 64)
    inplanes = 64
    for layer, (planes, n) in enumerate(zip((64, 128, 256, 512), (3, 4, 23, 3)), start=1):
        for i in range(n):
            p = f"pretrained.layer1.4.{i}." if layer == 1 else f"pretrained.layer{layer}.{i}."
            sd[p + "conv1.weight"] = conv((planes, inplanes, 1, 1))
            bn(p + "bn1.", planes)
            sd[p + "conv2.weight"] = conv((planes, planes, 3, 3))
            bn(p + "bn2.", planes)
            sd[p + "conv3.weight"] = conv((planes * 4, planes, 1, 1))
            bn(p + "bn3.", planes * 4)
            sd[p + "bn3.weight"] *= 0.12  # keep the residual branches from multiplying the stream over 33 blocks
            if i == 0:
                sd[p + "downsample.0.weight"] = conv((planes * 4, inplanes, 1, 1))
                bn(p + "downsample.1.", planes * 4)
            inplanes = planes * 4


def make_state_dict(seed=0, with_clip_visual_stub=False, head_block=False, backbone="clip_vitl16_384"):
    """fp32 state dict of LSegNet(backbone=...) — keys per SURVEY.md Appendix C. The draw order for the default
    backbone is frozen (the committed golden fixtures were generated from it)."""
    g = _Gen(seed)
    sd = {}
    shp = BACKBONE_SHAPES[backbone]
    if backbone == "clip_resnet101":
        _resnet101_state(g, sd)
        return _decoder_and_text_state(g, sd, shp, with_clip_visual_stub, head_block)
    D, P, depth = shp["dim"], shp["patch"], shp["depth"]
    p = "pretrained.model."
    sd[p + "cls_token"] = g.normal((1, 1, D), 0.02)
    sd[p + "pos_embed"] = g.normal((1, 1 + (384 // P) ** 2, D), 0.02)
    sd[p + "patch_embed.proj.weight"] = g.normal((D, 3, P, P), 0.02)
    sd[p + "patch_embed.proj.bias"] = g.normal((D,), 0.02)
    for i in range(depth):
        b = f"{p}blocks.{i}."
        for n in ("norm1", "norm2"):
            sd[b + n + ".weight"] = g.normal((D,), 0.1, 1.0)
            sd[b + n + ".bias"] = g.normal((D,), 0.05)
        sd[b + "attn.qkv.weight"] = g.normal((3 * D, D), 0.02)
        sd[b + "attn.qkv.bias"] = g.normal((3 * D,), 0.02)
        sd[b + "attn.proj.weight"] = g.normal((D, D), 0.02)
        sd[b + "attn.proj.bias"] = g.normal((D,), 0.02)
        sd[b + "mlp.fc1.weight"] = g.normal((4 * D, D), 0.02)
        sd[b + "mlp.fc1.bias"] = g.normal((4 * D,), 0.02)
        sd[b + "mlp.fc2.weight"] = g.normal((D, 4 * D), 0.02)
        sd[b + "mlp.fc2.bias"] = g.normal((D,), 0.02)
    sd[p + "norm.weight"] = g.normal((D,), 0.1, 1.0)
    sd[p + "norm.bias"] = g.normal((D,), 0.05)
    feats = list(shp["feats"])
    for k in range(4):
        q = f"pretrained.act_postprocess{k + 1}."
        sd[q + "0.project.0.weight"] = g.kaiming((D, 2 * D))
        sd[q + "0.project.0.bias"] = g.uniform((D,), -0.02, 0.02)
        sd[q + "3.weight"] = g.kaiming((feats[k], D, 1, 1))
        sd[q + "3.bias"] = g.uniform((feats[k],), -0.03, 0.03)
    for k in range(4):
        r, c = shp["resample"][k], feats[k]
        q = f"pretrained.act_postprocess{k + 1}.4."
        if r > 0:
            sd[q + "weight"] = g.kaiming((c, c, r, r))
            sd[q + "bias"] = g.uniform((c,), -0.03, 0.03)
        elif r == -2:
            sd[q + "weight"] = g.kaiming((c, c, 3, 3))
            sd[q + "bias"] = g.uniform((c,), -0.01, 0.01)
    return _decoder_and_text_state(g, sd, shp, with_clip_visual_stub, head_block)


def _decoder_and_text_state(g, sd, shp, with_clip_visual_stub, head_block):
    feats = list(shp["feats"])
    for k in range(4):
        sd[f"scratch.layer{k + 1}_rn.weight"] = g.kaiming((256, feats[k], 3, 3))
    for k in range(1, 5):
        q = f"scratch.refinenet{k}."
        sd[q + "out_conv.weight"] = g.kaiming((256, 256, 1, 1))
        sd[q + "out_conv.bias"] = g.uniform((256,), -0.06, 0.06)
        for u in ("resConfUnit1", "resConfUnit2"):
            for c in ("1", "2"):
                sd[f"{q}{u}.conv{c}.weight"] = g.kaiming((256, 256, 3, 3))
                sd[f"{q}{u}.bn{c}.weight"] = g.uniform((256,), 0.5, 1.5)
                sd[f"{q}{u}.bn{c}.bias"] = g.normal((256,), 0.1)
                sd[f"{q}{u}.bn{c}.running_mean"] = g.normal((256,), 0.1)
                sd[f"{q}{u}.bn{c}.running_var"] = g.uniform((256,), 0.5, 1.5)
                sd[f"{q}{u}.bn{c}.num_batches_tracked"] = torch.tensor(100, dtype=torch.int64)
    Wd, out_c = shp["text"]
    sd["scratch.head1.weight"] = g.kaiming((out_c, 256, 1, 1))
    sd["scratch.head1.bias"] = g.uniform((out_c,), -0.06, 0.06)
    # CLIP ViT-B/32 text tower (CLIP.initialize_parameters scales)
    c = "clip_pretrained."
    sd[c + "positional_embedding"] = g.normal((CONTEXT, Wd), 0.01)
    sd[c + "text_projection"] = g.normal((Wd, out_c), Wd ** -0.5)
    sd[c + "logit_scale"] = torch.tensor(float(np.log(1 / 0.07)))
    sd[c + "token_embedding.weight"] = g.normal((VOCAB, Wd), 0.02)
    proj_std = (Wd ** -0.5) * ((2 * TEXT_DEPTH) ** -0.5)
    for i in range(TEXT_DEPTH):
        b = f"{c}transformer.resblocks.{i}."
        sd[b + "attn.in_proj_weight"] = g.normal((3 * Wd, Wd), Wd ** -0.5)
        sd[b + "attn.in_proj_bias"] = g.normal((3 * Wd,), 0.02)
        sd[b + "attn.out_proj.weight"] = g.normal((Wd, Wd), proj_std)
        sd[b + "attn.out_proj.bias"] = g.normal((Wd,), 0.02)
        sd[b + "ln_1.weight"] = g.normal((Wd,), 0.1, 1.0)
        sd[b + "ln_1.bias"] = g.normal((Wd,), 0.05)
        sd[b + "mlp.c_fc.weight"] = g.normal((4 * Wd, Wd), (2 * Wd) ** -0.5)
        sd[b + "mlp.c_fc.bias"] = g.normal((4 * Wd,), 0.02)
        sd[b + "mlp.c_proj.weight"] = g.normal((Wd, 4 * Wd), proj_std)
        sd[b + "mlp.c_proj.bias"] = g.normal((Wd,), 0.02)
        sd[b + "ln_2.weight"] = g.normal((Wd,), 0.1, 1.0)
        sd[b + "ln_2.bias"] = g.normal((Wd,), 0.05)
    sd[c + "ln_final.weight"] = g.normal((Wd,), 0.1, 1.0)
    sd[c + "ln_final.bias"] = g.normal((Wd,), 0.05)
    if with_clip_visual_stub:  # real checkpoints also carry the (unused) CLIP visual tower
        sd[c + "visual.conv1.weight"] = g.normal((8, 3, 32, 32), 0.02)
    if head_block:  # arch_option 1 / 2 (lseg_net.py:148-154); drawn last so every other tensor keeps its value
        sd["scratch.head_block.depthwise.depthwise.weight"] = g.uniform((1, 1, 3, 3), -0.4, 0.4)
        sd["scratch.head_block.depthwise.depthwise.bias"] = g.uniform((1,), -0.2, 0.2)
    return sd


def tokenize(labels, context_length=CONTEXT):
    """Deterministic stand-in for clip.tokenize (same shape/dtype/SOT/EOT/padding contract):
    lower-cased whitespace words -> 1000 + crc32(word) % 40000. int64 [K, 77]."""
    if isinstance(labels, str):
        labels = [labels]
    out = torch.zeros((len(labels), context_length), dtype=torch.int64)
    for i, text in enumerate(labels):
        words = text.lower().strip().split()
        ids = [SOT] + [1000 + (zlib.crc32(w.encode("utf-8")) % 40000) for w in words] + [EOT]
        if len(ids) > context_length:
            raise RuntimeError(f"Input {text} is too long for context length {context_length}")
        out[i, : len(ids)] = torch.tensor(ids, dtype=torch.int64)
    return out


def synthetic_prompts(k, seed=0):
    """K synthetic token rows for the open-vocab stress config (SURVEY.md section 8(d) config 5)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = torch.zeros((k, CONTEXT), dtype=torch.int64)
    for i in range(k):
        n = int(rng.integers(1, 7))
        ids = [SOT] + [int(v) for v in rng.integers(1000, 40001, size=n)] + [EOT]
        out[i, : len(ids)] = torch.tensor(ids, dtype=torch.int64)
    return out


def make_image(batch, h, w, seed=0):
    """Normalised-image stand-in: N(0,1) clamped to [-1,1] (Normalize(.5,.5) range, lseg_module.py:37-50)."""
    rng = np.random.Generator(np.random.PCG64(1000 + seed))
    a = rng.standard_normal(size=(batch, 3, h, w), dtype=np.float32)
    # low-frequency structure so neighbouring pixels are correlated like a real image
    a = torch.from_numpy(a)
    low = torch.nn.functional.interpolate(a[:, :, ::16, ::16], size=(h, w), mode="bilinear", align_corners=False)
    return (0.6 * low + 0.4 * a).clamp_(-1, 1).contiguous()


ADE20K_150 = None


def ade20k_labels(path=None):
    """ADE20K-150 names parsed as modules/lseg_module.py:97-109 (last CSV field, first ';' synonym,
    header dropped). The label file is an input fixture copied verbatim to tests/golden/."""
    import os
    if path is None:
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden",
                            "ade20k_objectInfo150.txt")
    labels = []
    with open(path, "r") as f:
        for line in f.readlines():
            labels.append(line.strip().split(",")[-1].split(";")[0])
    return labels[1:]
