"""TEST INFRASTRUCTURE — CPU oracle of the ViT's recorded attention maps (enable_attention_hooks).

The reference's hook (get_attention, modules/models/lseg_vit.py:22-42) recomputes softmax((q @ k^T) * scale) from
module.qkv(x) on the input of blocks[h].attn and stores the fp32 [B, heads, N, N] tensor as "attn_1".."attn_4" in
pretrained.attention (:428-441). This module runs the trunk of oracle/lseg_oracle.py (same functions, same order, so
the taps are those of lseg_oracle.vit_forward_flex bit for bit) and keeps those probabilities at the hooked blocks.
Pinned against the reference itself by oracle/make_golden_attention.py (tests/golden/ref_attention.npz).
"""
import torch
import torch.nn.functional as F

from oracle import lseg_oracle as O


def attention_probs(x, sd, prefix, num_heads, qk_out=None):
    """softmax((q @ k^T) * dh^-0.5) of timm Attention at `prefix` on its input x [B, N, C] -> fp32 [B, heads, N, N].
    qk_out: a list that receives q and k, fp32 [B, heads, N, dh]."""
    B, N, C = x.shape
    qkv = F.linear(x, sd[prefix + "qkv.weight"], sd[prefix + "qkv.bias"])
    qkv = qkv.reshape(B, N, 3, num_heads, C // num_heads).permute(2, 0, 3, 1, 4)
    q, k = qkv[0], qkv[1]
    if qk_out is not None:
        qk_out.extend((q, k))
    return ((q @ k.transpose(-2, -1)) * ((C // num_heads) ** -0.5)).softmax(dim=-1)


@torch.no_grad()
def vit_attention_maps(x, sd, backbone="clip_vitl16_384", taps_out=None, qk_out=None):
    """{"attn_1".."attn_4": fp32 [B, heads, N, N]}: the dict the reference's pretrained.attention holds after a forward
    of x fp32 [B,3,H,W] with enable_attention_hooks=True. Runs the trunk up to the last hooked block only; taps_out (a
    list) receives the four taps as lseg_oracle.vit_forward_flex returns them; qk_out (a dict) receives the hooked
    blocks' q and k as "attn_k": (q, k), fp32 [B, heads, N, dh]."""
    cfg = O.BACKBONES[backbone]
    hooks, heads = cfg["hooks"], cfg["heads"]
    p = "pretrained.model."
    b, c, h, w = x.shape
    patch = sd[p + "patch_embed.proj.weight"].shape[-1]
    pos_embed = O.resize_pos_embed(sd[p + "pos_embed"], h // patch, w // patch)
    x = F.conv2d(x, sd[p + "patch_embed.proj.weight"], sd[p + "patch_embed.proj.bias"], stride=patch)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat((sd[p + "cls_token"].expand(b, -1, -1), x), dim=1)
    x = x + pos_embed
    out = {}
    for i in range(max(hooks) + 1):
        prefix = f"{p}blocks.{i}."
        if i in hooks:
            hn = F.layer_norm(x, (x.shape[-1],), sd[prefix + "norm1.weight"], sd[prefix + "norm1.bias"], 1e-6)
            name = f"attn_{list(hooks).index(i) + 1}"
            qk = [] if qk_out is not None else None
            out[name] = attention_probs(hn, sd, prefix + "attn.", heads, qk)
            if qk is not None:
                qk_out[name] = tuple(qk)
        x = O.vit_block(x, sd, prefix, heads)
        if i in hooks and taps_out is not None:
            taps_out.append(x)
    return out
