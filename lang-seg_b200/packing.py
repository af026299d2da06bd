"""State-dict -> packed device buffers for the sm_90a engine (host-side, one-off per weight load).

Input: the reference's state dict (key names of SURVEY.md Appendix C, fp32). Output: the
`lseg_weights` descriptor of include/lseg_b200.h plus the tensors that back its pointers.

Layouts
  * every GEMM weight is fp16 [N, K] row-major (K contiguous = "K-major" wgmma operand), rows padded
    with zeros to a multiple of 128 so a TMA box never exceeds the tensor;
  * 3x3 convs are tap-major: [N, (ky, kx, c)]  (the implicit-GEMM K loop walks taps, then channels);
  * ConvTranspose2d with kernel == stride becomes a GEMM with N = (i, j, co) and a depth-to-space
    store; its bias is expanded to [s*s*cout];
  * ProjectReadout's Linear(2D->D) is split into the token half W[:, :D] and the cls half
    W[:, D:] (+bias) — exact up to summation order (SURVEY.md section 2b k10);
  * eval-mode BatchNorm is folded to per-channel (scale, shift) applied in the GEMM epilogue in fp32.
"""
import math

import numpy as np
import torch

from . import _lib

VIT_DEPTH = _lib.VIT_DEPTH
TEXT_DEPTH = _lib.TEXT_DEPTH
HOOKS = (5, 11, 17, 23)  # modules/models/lseg_net.py:119-123 (clip_vitl16_384)

# Image backbones of LSeg.__init__ (lseg_net.py:119-123) and how modules/models/lseg_vit.py builds them:
# _make_pretrained_clip_vitl16_384 (:221-238 + _make_vit_b16_backbone :408-532) and _make_pretrained_clip_vitb32_384
# (:259-273 + _make_vit_b32_backbone :275-405). `resample` per level: s > 0 ConvTranspose2d(k=s, stride=s), 0 nothing,
# -2 Conv2d 3x3 stride 2. Both use the CLIP ViT-B/32 text tower.
# `text`: (transformer_width, heads, embed_dim) of the CLIP model whose text tower is used — ViT-B/32 or RN50x16
# (lseg_vit.py:224, 243, 260); embed_dim is LSeg's out_c (lseg_net.py:142-146).
BACKBONES = {
    "clip_vitl16_384": dict(dim=1024, depth=24, heads=16, patch=16, hooks=(5, 11, 17, 23),
                            features=(256, 512, 1024, 1024), resample=(4, 2, 0, -2), timm="vit_large_patch16_384",
                            clip="ViT-B/32", text=(512, 8, 512)),
    "clipRN50x16_vitl16_384": dict(dim=1024, depth=24, heads=16, patch=16, hooks=(5, 11, 17, 23),
                                   features=(256, 512, 1024, 1024), resample=(4, 2, 0, -2), timm="vit_large_patch16_384",
                                   clip="RN50x16", text=(768, 12, 768)),
    "clip_vitb32_384": dict(dim=768, depth=12, heads=12, patch=32, hooks=(2, 5, 8, 11),
                            features=(96, 192, 384, 768), resample=(8, 4, 2, 0), timm="vit_base_patch32_384",
                            clip="ViT-B/32", text=(512, 8, 512)),
    # zero-shot model LSegRNNetZS only (lseg_net_zs.py:240-378; lseg_blocks_zs.py:42-48, lseg_vit_zs.py:742-748): a
    # torchvision resnet101 whose four stages feed scratch.layerN_rn directly — no ViT, no reassemble
    "clip_resnet101": dict(trunk="resnet101", layers=(3, 4, 23, 3), features=(256, 512, 1024, 2048),
                           clip="ViT-B/32", text=(512, 8, 512)),
}


def stored_channels(c):
    """Channel count as the engine stores it: the next multiple of 64 (TMA boxes of the implicit-GEMM convs and the K
    loop work in 64-channel chunks); the pad carries zero weights and zero bias, so it stays exactly zero."""
    return (c + 63) // 64 * 64


def _pad_to(t, dim, n):
    if t.shape[dim] == n:
        return t
    shape = list(t.shape)
    shape[dim] = n - t.shape[dim]
    return torch.cat([t, torch.zeros(shape, dtype=t.dtype, device=t.device)], dim=dim)


def _pad_rows(w, mult=128):
    n = w.shape[0]
    npad = (n + mult - 1) // mult * mult
    if npad == n:
        return w.contiguous()
    out = torch.zeros((npad,) + tuple(w.shape[1:]), dtype=w.dtype, device=w.device)
    out[:n] = w
    return out


def conv3x3_to_gemm(w):
    """[Cout, Cin, 3, 3] -> [Cout, 9*Cin] tap-major (ky, kx, c)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def deconv_to_gemm(w):
    """ConvTranspose2d weight [Cin, Cout, s, s] (kernel == stride) -> [(i, j, co), ci]."""
    cin, cout, s, _ = w.shape
    return w.permute(2, 3, 1, 0).reshape(s * s * cout, cin)


def fold_bn(sd, prefix, eps=1e-5):
    """BatchNorm2d eval -> y = x*scale + shift (modules/models/lseg_blocks.py:265-288, eps 1e-5)."""
    g, b = sd[prefix + "weight"].float(), sd[prefix + "bias"].float()
    m, v = sd[prefix + "running_mean"].float(), sd[prefix + "running_var"].float()
    scale = g / torch.sqrt(v + eps)
    return scale, b - m * scale


def reference_logit_scale():
    """exp(log(1/0.07)) evaluated in fp32 like `nn.Parameter(torch.ones([]) * np.log(1 / 0.07)).exp()`
    (modules/models/lseg_net.py:141)."""
    return float((torch.ones([]) * np.log(1 / 0.07)).exp())


class PackedWeights:
    """Owns the packed tensors and the ctypes descriptor that points into them."""

    def __init__(self, state_dict, device, arch_option=0, block_depth=0, activation="lrelu", backbone="clip_vitl16_384"):
        if backbone not in BACKBONES:
            raise ValueError(f"backbone {backbone!r}: this engine builds {sorted(BACKBONES)}")
        self.device = torch.device(device)
        self.backbone = backbone
        self._keep = []
        self.desc = _lib.Weights()
        self._pack(state_dict, BACKBONES[backbone])
        d = self.desc
        d.arch_option, d.block_depth = int(arch_option or 0), int(block_depth or 0)
        d.head_act = _lib.HEAD_ACT[activation] if d.arch_option else 0
        if d.arch_option in (1, 2):  # scratch.head_block (lseg_net.py:148-154): one shared 3x3 kernel + bias
            w = state_dict["scratch.head_block.depthwise.depthwise.weight"].detach().float().reshape(9).tolist()
            for i in range(9):
                d.head_block_w[i] = w[i]
            d.head_block_b = float(state_dict["scratch.head_block.depthwise.depthwise.bias"].detach().float().reshape(-1)[0])

    # -- helpers -------------------------------------------------------------------------------
    def _f32(self, t):
        t = t.detach().to(self.device, torch.float32).contiguous()
        self._keep.append(t)
        return t.data_ptr()

    def _f16_rows(self, t):
        t = _pad_rows(t.detach().to(self.device, torch.float32).to(torch.float16).contiguous())
        self._keep.append(t)
        return t

    def _linear(self, slot, w2d, bias, round_bias_f16=False):
        wt = self._f16_rows(w2d)
        slot.w = wt.data_ptr()
        slot.out, slot.in_ = int(w2d.shape[0]), int(w2d.shape[1])
        slot.rows = int(wt.shape[0])
        if bias is not None:
            b = bias.detach().float()
            if round_bias_f16:  # CLIP's Linear biases are fp16 tensors after convert_weights
                b = b.half().float()
            slot.b = self._f32(b)
        else:
            slot.b = None

    # -- packing -------------------------------------------------------------------------------
    def _pack_resnet(self, sd, cfg):
        """torchvision resnet101 under the key names of _make_resnet_backbone (lseg_blocks_zs.py:109-119): the stem is
        pretrained.layer1.{0,1}, stage 1 pretrained.layer1.4.*, stages 2-4 pretrained.layer{2,3,4}.*."""
        d = self.desc
        d.trunk = 1
        stem = sd["pretrained.layer1.0.weight"]
        if tuple(stem.shape) != (64, 3, 7, 7):
            raise ValueError(f"{self.backbone}: stem conv is {tuple(stem.shape)}, expected (64, 3, 7, 7)")
        self._linear(d.rn_stem, _pad_to(stem.reshape(64, 147), 1, 192), None)
        s, t = fold_bn(sd, "pretrained.layer1.1.")
        d.rn_stem_scale, d.rn_stem_shift = self._f32(s), self._f32(t)
        blk = 0
        for layer, n in enumerate(cfg["layers"], start=1):
            d.rn_layers[layer - 1] = n
            for i in range(n):
                q = f"pretrained.layer1.4.{i}." if layer == 1 else f"pretrained.layer{layer}.{i}."
                b = d.rn_blocks[blk]
                w1, w2, w3 = sd[q + "conv1.weight"], sd[q + "conv2.weight"], sd[q + "conv3.weight"]
                self._linear(b.conv1, w1.reshape(w1.shape[0], w1.shape[1]), None)
                self._linear(b.conv2, conv3x3_to_gemm(w2), None)
                self._linear(b.conv3, w3.reshape(w3.shape[0], w3.shape[1]), None)
                for j, slot in ((1, "bn1"), (2, "bn2"), (3, "bn3")):
                    s, t = fold_bn(sd, f"{q}bn{j}.")
                    setattr(b, slot + "_scale", self._f32(s))
                    setattr(b, slot + "_shift", self._f32(t))
                b.stride = 2 if (layer > 1 and i == 0) else 1
                if i == 0:
                    wd = sd[q + "downsample.0.weight"]
                    self._linear(b.down, wd.reshape(wd.shape[0], wd.shape[1]), None)
                    s, t = fold_bn(sd, q + "downsample.1.")
                    b.bnd_scale, b.bnd_shift = self._f32(s), self._f32(t)
                blk += 1
        for k in range(4):
            d.post_channels[k] = cfg["features"][k]

    def _pack(self, sd, cfg):
        d = self.desc
        if cfg.get("trunk") == "resnet101":
            self._pack_resnet(sd, cfg)
            return self._pack_decoder_and_text(sd, cfg)
        p = "pretrained.model."
        D, P = cfg["dim"], cfg["patch"]
        d.vit_dim, d.vit_depth, d.vit_heads, d.patch_size = D, cfg["depth"], cfg["heads"], P
        pw = sd[p + "patch_embed.proj.weight"]
        if tuple(pw.shape) != (D, 3, P, P):
            raise ValueError(f"{self.backbone}: patch_embed.proj.weight is {tuple(pw.shape)}, expected {(D, 3, P, P)}")
        self._linear(d.patch, pw.reshape(D, 3 * P * P), sd[p + "patch_embed.proj.bias"])
        d.cls_token = self._f32(sd[p + "cls_token"].reshape(D))
        pos = sd[p + "pos_embed"].reshape(-1, D)
        d.pos_embed = self._f32(pos)
        d.pos_grid = int(round(math.sqrt(pos.shape[0] - 1)))
        for i in range(cfg["depth"]):
            b = f"{p}blocks.{i}."
            blk = d.blocks[i]
            blk.ln1_g, blk.ln1_b = self._f32(sd[b + "norm1.weight"]), self._f32(sd[b + "norm1.bias"])
            blk.ln2_g, blk.ln2_b = self._f32(sd[b + "norm2.weight"]), self._f32(sd[b + "norm2.bias"])
            self._linear(blk.qkv, sd[b + "attn.qkv.weight"], sd[b + "attn.qkv.bias"])
            self._linear(blk.proj, sd[b + "attn.proj.weight"], sd[b + "attn.proj.bias"])
            self._linear(blk.fc1, sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"])
            self._linear(blk.fc2, sd[b + "mlp.fc2.weight"], sd[b + "mlp.fc2.bias"])
        for k in range(4):
            d.hooks[k] = cfg["hooks"][k]
            q = f"pretrained.act_postprocess{k + 1}."
            w = sd[q + "0.project.0.weight"]
            self._linear(d.readout_tok[k], w[:, :D], None)
            self._linear(d.readout_cls[k], w[:, D:], sd[q + "0.project.0.bias"])
            c, cp = cfg["features"][k], stored_channels(cfg["features"][k])
            d.post_channels[k], d.post_resample[k] = cp, cfg["resample"][k]
            cw = sd[q + "3.weight"]
            if cw.shape[0] != c:
                raise ValueError(f"{self.backbone}: act_postprocess{k + 1}.3 has {cw.shape[0]} channels, expected {c}")
            self._linear(d.post_conv1x1[k], _pad_to(cw.reshape(c, D), 0, cp), _pad_to(sd[q + "3.bias"], 0, cp))
            r = cfg["resample"][k]
            if r > 0:    # ConvTranspose2d [cin, cout, r, r]
                w = _pad_to(_pad_to(sd[q + "4.weight"], 0, cp), 1, cp)
                self._linear(d.post_resample_w[k], deconv_to_gemm(w), _pad_to(sd[q + "4.bias"], 0, cp).repeat(r * r))
            elif r == -2:  # Conv2d 3x3 stride 2 [cout, cin, 3, 3]
                w = _pad_to(_pad_to(sd[q + "4.weight"], 0, cp), 1, cp)
                self._linear(d.post_resample_w[k], conv3x3_to_gemm(w), _pad_to(sd[q + "4.bias"], 0, cp))
        self._pack_decoder_and_text(sd, cfg)

    def _pack_decoder_and_text(self, sd, cfg):
        d = self.desc
        for k in range(4):
            self._linear(d.layer_rn[k], conv3x3_to_gemm(_pad_to(sd[f"scratch.layer{k + 1}_rn.weight"], 1,
                                                                stored_channels(cfg["features"][k]))), None)
            q = f"scratch.refinenet{k + 1}."
            for slot, unit in ((d.rcu1[k], "resConfUnit1."), (d.rcu2[k], "resConfUnit2.")):
                self._linear(slot.conv1, conv3x3_to_gemm(sd[q + unit + "conv1.weight"]), None)
                self._linear(slot.conv2, conv3x3_to_gemm(sd[q + unit + "conv2.weight"]), None)
                s1, t1 = fold_bn(sd, q + unit + "bn1.")
                s2, t2 = fold_bn(sd, q + unit + "bn2.")
                slot.bn1_scale, slot.bn1_shift = self._f32(s1), self._f32(t1)
                slot.bn2_scale, slot.bn2_shift = self._f32(s2), self._f32(t2)
            oc = sd[q + "out_conv.weight"]
            self._linear(d.out_conv[k], oc.reshape(oc.shape[0], oc.shape[1]), sd[q + "out_conv.bias"])
        h1 = sd["scratch.head1.weight"]
        d.text_width, d.text_heads, d.out_c = cfg["text"]
        if h1.shape[0] != d.out_c or tuple(sd["clip_pretrained.text_projection"].shape) != (d.text_width, d.out_c):
            raise ValueError(f"{self.backbone}: head1 has {h1.shape[0]} channels / text_projection is "
                             f"{tuple(sd['clip_pretrained.text_projection'].shape)}, expected out_c {d.out_c}, "
                             f"text width {d.text_width} (CLIP {cfg['clip']})")
        self._linear(d.head1, h1.reshape(h1.shape[0], h1.shape[1]), sd["scratch.head1.bias"])
        d.logit_scale = reference_logit_scale()
        # CLIP text tower: Linear / MHA weights are fp16 in the reference (clip.load on cuda)
        c = "clip_pretrained."
        d.tok_emb = self._f32(sd[c + "token_embedding.weight"])
        d.text_pos = self._f32(sd[c + "positional_embedding"])
        for i in range(TEXT_DEPTH):
            b = f"{c}transformer.resblocks.{i}."
            blk = d.text_blocks[i]
            blk.ln1_g, blk.ln1_b = self._f32(sd[b + "ln_1.weight"]), self._f32(sd[b + "ln_1.bias"])
            blk.ln2_g, blk.ln2_b = self._f32(sd[b + "ln_2.weight"]), self._f32(sd[b + "ln_2.bias"])
            self._linear(blk.in_proj, sd[b + "attn.in_proj_weight"], sd[b + "attn.in_proj_bias"], True)
            self._linear(blk.out_proj, sd[b + "attn.out_proj.weight"], sd[b + "attn.out_proj.bias"], True)
            self._linear(blk.c_fc, sd[b + "mlp.c_fc.weight"], sd[b + "mlp.c_fc.bias"], True)
            self._linear(blk.c_proj, sd[b + "mlp.c_proj.weight"], sd[b + "mlp.c_proj.bias"], True)
        d.lnf_g, d.lnf_b = self._f32(sd[c + "ln_final.weight"]), self._f32(sd[c + "ln_final.bias"])
        self._linear(d.text_proj, sd[c + "text_projection"].t(), None)
