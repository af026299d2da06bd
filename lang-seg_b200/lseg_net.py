"""Drop-in `LSegNet` / `LSegNetZS` whose forward runs on the sm_90a engine.

Mirrors the reference interface for the hot path (SURVEY.md section 8(b)):
  * constructor signatures of modules/models/lseg_net.py:208-226 and lseg_net_zs.py:219-239;
  * `forward(x, labelset='')` (lseg_net.py:160) / `forward(x, class_info)` (lseg_net_zs.py:177); beyond the reference,
    `x` may be a PixelEmbedding from `encode_image(x)`: only the label-dependent tail then runs, with the same result;
  * attributes the callers touch: `.pretrained.model.patch_embed.img_size` (lseg_module.py:86-89),
    `.scratch`, `.clip_pretrained` (with `.encode_text`), `.labels`, `.text`, `.crop_size`, `.out_c`,
    `.arch_option`, `.logit_scale`;
  * `enable_attention_hooks=True` (the `_make_encoder` argument, lseg_blocks.py:22) on a ViT-L/16 backbone: every call
    that runs the image path records the hooked blocks' attention probabilities in `.pretrained.attention`
    (lseg_vit.py:428-441), and `get_mean_attention_map` (lseg_vit.py:45-54) turns one token's row into an image map;
  * state-dict key names and shapes of SURVEY.md Appendix C, so `BaseModel.load` / Lightning's
    `load_from_checkpoint` (prefix `net.`) keep working; the unused `clip_pretrained.visual.*` and timm
    `head.*` entries of real checkpoints are accepted and ignored.
The torch sub-modules below are parameter holders only (they give the reference's names, shapes and
default inits); no torch op runs in forward. There is no CPU path: a non-CUDA input raises.
"""
import itertools
import threading
import weakref
from collections import OrderedDict

import torch
import torch.nn as nn

from .packing import BACKBONES, reference_logit_scale
from .tokenizer import tokenize


# ---------------------------------------------------------------------------------------------
# parameter holders (names == reference / timm / CLIP module names)
# ---------------------------------------------------------------------------------------------
def _vit_holder(cfg):
    """timm VisionTransformer parameter holder (vit_large_patch16_384 / vit_base_patch32_384)."""
    D, P, depth, heads = cfg["dim"], cfg["patch"], cfg["depth"], cfg["heads"]
    m = nn.Module()
    m.patch_embed = nn.Module()
    m.patch_embed.proj = nn.Conv2d(3, D, kernel_size=P, stride=P)
    m.patch_embed.img_size = (384, 384)
    m.cls_token = nn.Parameter(torch.zeros(1, 1, D))
    m.pos_embed = nn.Parameter(torch.zeros(1, 1 + (384 // P) ** 2, D))
    nn.init.normal_(m.cls_token, std=0.02)
    nn.init.normal_(m.pos_embed, std=0.02)
    blocks = []
    for _ in range(depth):
        b = nn.Module()
        b.norm1 = nn.LayerNorm(D, eps=1e-6)
        b.attn = nn.Module()
        b.attn.qkv = nn.Linear(D, 3 * D)
        b.attn.proj = nn.Linear(D, D)
        b.attn.num_heads = heads
        b.norm2 = nn.LayerNorm(D, eps=1e-6)
        b.mlp = nn.Module()
        b.mlp.fc1 = nn.Linear(D, 4 * D)
        b.mlp.fc2 = nn.Linear(4 * D, D)
        blocks.append(b)
    m.blocks = nn.ModuleList(blocks)
    m.norm = nn.LayerNorm(D, eps=1e-6)  # present in checkpoints; dead in forward (lseg_vit.py:108,199)
    m.patch_size = [P, P]
    m.start_index = 1
    return m


def _readout_holder(D):
    r = nn.Module()
    r.project = nn.Sequential(nn.Linear(2 * D, D), nn.GELU())
    return r


def _bottleneck_holder(inplanes, planes, downsample):
    """torchvision.models.resnet.Bottleneck parameter names (conv1/bn1/conv2/bn2/conv3/bn3[/downsample.{0,1}])."""
    b = nn.Module()
    b.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
    b.bn1 = nn.BatchNorm2d(planes)
    b.conv2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False)
    b.bn2 = nn.BatchNorm2d(planes)
    b.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
    b.bn3 = nn.BatchNorm2d(planes * 4)
    if downsample:
        b.downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, bias=False), nn.BatchNorm2d(planes * 4))
    return b


def _resnet_holder(cfg):
    """pretrained.layer1..4 as _make_resnet_backbone builds them (lseg_blocks_zs.py:109-119): layer1 = Sequential(conv1,
    bn1, relu, maxpool, resnet.layer1), layer2..4 = the torchvision stages."""
    p = nn.Module()
    inplanes = 64
    for layer, (planes, n) in enumerate(zip((64, 128, 256, 512), cfg["layers"]), start=1):
        blocks = []
        for i in range(n):
            blocks.append(_bottleneck_holder(inplanes, planes, i == 0))
            inplanes = planes * 4
        stage = nn.Sequential(*blocks)
        if layer == 1:
            stage = nn.Sequential(nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False), nn.BatchNorm2d(64), nn.Identity(),
                                  nn.Identity(), stage)
        setattr(p, f"layer{layer}", stage)
    return p


def _pretrained_holder(cfg):
    """act_postprocess1..4 with the reference's Sequential indices (0 readout, 3 the 1x1 conv, 4 the resampling op;
    lseg_vit.py:309-398 for ViT-B/32, :445-520 for ViT-L/16)."""
    if cfg.get("trunk") == "resnet101":
        return _resnet_holder(cfg)
    D = cfg["dim"]
    p = nn.Module()
    p.model = _vit_holder(cfg)
    for k in range(4):
        c, r = cfg["features"][k], cfg["resample"][k]
        mods = [_readout_holder(D), nn.Identity(), nn.Identity(), nn.Conv2d(D, c, 1)]
        if r > 0:
            mods.append(nn.ConvTranspose2d(c, c, r, stride=r))
        elif r == -2:
            mods.append(nn.Conv2d(c, c, 3, stride=2, padding=1))
        setattr(p, f"act_postprocess{k + 1}", nn.Sequential(*mods))
    return p


def _rcu_holder():
    u = nn.Module()
    u.conv1 = nn.Conv2d(256, 256, 3, padding=1, bias=False)
    u.conv2 = nn.Conv2d(256, 256, 3, padding=1, bias=False)
    u.bn1 = nn.BatchNorm2d(256)
    u.bn2 = nn.BatchNorm2d(256)
    return u


def _scratch_holder(out_c, features=(256, 512, 1024, 1024)):
    s = nn.Module()
    for k, cin in enumerate(features):
        setattr(s, f"layer{k + 1}_rn", nn.Conv2d(cin, 256, 3, padding=1, bias=False))
    for k in range(1, 5):
        f = nn.Module()
        f.out_conv = nn.Conv2d(256, 256, 1)
        f.resConfUnit1 = _rcu_holder()
        f.resConfUnit2 = _rcu_holder()
        setattr(s, f"refinenet{k}", f)
    s.head1 = nn.Conv2d(256, out_c, 1)
    s.output_conv = nn.Sequential()  # Interpolate(x2, bilinear, align_corners=True): no parameters
    return s


class _ClipTextHolder(nn.Module):
    """CLIP text tower parameters (ViT-B/32: width 512, 8 heads, embedding 512; RN50x16: 768, 12, 768); `encode_text` runs
    on the engine of the owning net."""

    def __init__(self, width=512, heads=8, embed_dim=512):
        super().__init__()
        self.positional_embedding = nn.Parameter(torch.empty(77, width).normal_(std=0.01))
        self.text_projection = nn.Parameter(torch.empty(width, embed_dim).normal_(std=width ** -0.5))
        self.logit_scale = nn.Parameter(torch.ones([]) * 2.6592600)
        self.token_embedding = nn.Embedding(49408, width)
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        blocks = []
        for _ in range(12):
            b = nn.Module()
            b.attn = nn.MultiheadAttention(width, heads)
            b.ln_1 = nn.LayerNorm(width)
            b.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(width, 4 * width)), ("gelu", nn.Identity()),
                                               ("c_proj", nn.Linear(4 * width, width))]))
            b.ln_2 = nn.LayerNorm(width)
            blocks.append(b)
        self.transformer = nn.Module()
        self.transformer.resblocks = nn.Sequential(*blocks)
        self.ln_final = nn.LayerNorm(width)
        self._owner = None

    def encode_text(self, text):
        owner = self._owner() if self._owner is not None else None
        if owner is None:
            raise RuntimeError("clip_pretrained is detached from its LSegNet")
        feats = owner._engine_for(text.device).encode_text(text)
        # un-normalised features are not kept by the engine; callers on this path (lseg_net.py:183-192)
        # normalise immediately, and normalisation is idempotent.
        return feats[: text.shape[0]]


_IGNORED_PREFIXES = ("clip_pretrained.visual.", "pretrained.model.head.", "pretrained.model.pre_logits.")

_WEIGHTS_GENERATION = itertools.count(1)  # process-wide: an embedding of another net never matches either


def get_mean_attention_map(attn, token, shape):
    """modules/models/lseg_vit.py:45-54 in plain torch: the attention row of query `token` over the patch keys of attn
    [B, heads, N, N] (as `.pretrained.attention["attn_k"]` holds it), unflattened to the token grid of an image of
    shape[2:] (H, W), upsampled bicubically (align_corners=False) to H x W, then averaged over dim 0.

    The reference's quirks are kept, so results match it call for call:
      * the grid is shape[2] // 16 x shape[3] // 16 whatever the backbone's patch size (both ViT-L/16 backbones record);
      * `.squeeze(0)` then `mean(0)`: for B = 1 the squeeze drops the batch and the mean runs over the heads -> [H, W];
        for B > 1 nothing is squeezed and the mean runs over the IMAGES -> [heads, H, W].
    Not on the hot path: no CUDA needed (CPU or CUDA tensors)."""
    attn = attn[:, :, token, 1:]
    attn = attn.unflatten(2, torch.Size([shape[2] // 16, shape[3] // 16])).float()
    attn = torch.nn.functional.interpolate(attn, size=shape[2:], mode="bicubic", align_corners=False).squeeze(0)
    all_attn = torch.mean(attn, 0)
    return all_attn


def is_ragged(labelset):
    """True for a per-image list of label lists (list[list[str]]): every image of the batch has its own label set."""
    return isinstance(labelset, (list, tuple)) and any(isinstance(l, (list, tuple)) for l in labelset)


def ragged_label_table(labelsets):
    """Host tables of a batch in which image b has its own labels labelsets[b] -> (union, rows, k, koff):
      union  the distinct labels of the batch in first-appearance order: each is tokenized and encoded once
      rows   the union index of every row of the packed text operand; image b's labels are rows koff[b] .. koff[b]+k[b]-1
      k      label count of every image
      koff   first packed text row of every image, which is also its first plane of the packed logits (prefix sum of k)"""
    index, union, rows, k, koff = {}, [], [], [], []
    for b, labels in enumerate(labelsets):
        if not isinstance(labels, (list, tuple)) or not labels or not all(isinstance(n, str) for n in labels):
            raise ValueError(f"labelsets[{b}] must be a non-empty list of label strings, got {labels!r}")
        koff.append(len(rows))
        k.append(len(labels))
        for name in labels:
            if name not in index:
                index[name] = len(union)
                union.append(name)
            rows.append(index[name])
    return union, rows, k, koff


class PixelEmbedding:
    """LSeg's pixel embedding of B images, as `LSegNet.encode_image` returns it: the output of the image path (trunk,
    decoder, head1; lseg_net.py:166-185) that every label set is then queried against. Pass it wherever the net takes
    `x` — forward / predict / update_metric run only the label-dependent tail on it and return what they return for the
    images themselves, bit for bit.

    Holds the engine's own pair (include/lseg_b200.h): `emb` fp16 [B,H/2,W/2,out_c] un-normalised rows and `sumsq` fp32
    [B,H/2,W/2,out_c/32] partial squared norms. `features()` gives the reference's normalised image_features. 62.7 MB
    per 480x480 image (out_c 512)."""

    def __init__(self, emb, sumsq, size, backbone, out_c, generation):
        self.emb = emb
        self.sumsq = sumsq
        self.size = tuple(size)  # (H, W) of the encoded images
        self.backbone = backbone
        self.out_c = out_c
        self.generation = generation

    @property
    def device(self):
        return self.emb.device

    @property
    def shape(self):
        """(B, 3, H, W): the shape of the images it encodes, where code reads x.shape."""
        return (self.emb.shape[0], 3) + self.size

    def __len__(self):
        return self.emb.shape[0]

    def __getitem__(self, idx):
        if not isinstance(idx, slice) or idx.step not in (None, 1):
            raise TypeError("PixelEmbedding supports contiguous batch slices emb[i:j]")
        return PixelEmbedding(self.emb[idx], self.sumsq[idx], self.size, self.backbone, self.out_c, self.generation)

    @staticmethod
    def cat(embs):
        """Concatenate along the batch: same net, weights and image size."""
        embs = list(embs)
        if not embs:
            raise ValueError("PixelEmbedding.cat of nothing")
        e0 = embs[0]
        for e in embs[1:]:
            if (e.size, e.backbone, e.out_c, e.generation, e.device) != (e0.size, e0.backbone, e0.out_c, e0.generation,
                                                                         e0.device):
                raise ValueError("PixelEmbedding.cat: embeddings of different image sizes, nets, weights or devices")
        return PixelEmbedding(torch.cat([e.emb for e in embs]), torch.cat([e.sumsq for e in embs]), e0.size, e0.backbone,
                              e0.out_c, e0.generation)

    def features(self):
        """The reference's normalised per-pixel embedding image_features (lseg_net.py:187-191, before `@ text.t()`) as
        fp32 [B, out_c, H/2, W/2]."""
        from .engine import embedding_features
        return embedding_features(self.emb, self.sumsq)


class _LSegBase(nn.Module):
    def _init_common(self, **kwargs):
        backbone = kwargs.get("backbone", "clip_vitl16_384")
        if backbone not in BACKBONES:
            # same failure mode as lseg_blocks.py:53-55. Built here: the three backbones of lseg_net.py:119-123
            # (clip_vitl16_384, clipRN50x16_vitl16_384, clip_vitb32_384); clip_resnet101 (lseg_blocks.py:46-52) is not.
            print(f"Backbone '{backbone}' not implemented")
            assert False
        self.backbone = backbone
        cfg = BACKBONES[backbone]
        self.arch_option = kwargs.get("arch_option", 0) or 0
        if self.arch_option not in (0, 1, 2):
            raise ValueError(f"arch_option {self.arch_option}: the reference defines 0, 1 (bottleneck_block) and 2 "
                             f"(depthwise_block) (lseg_net.py:148-154)")
        self.block_depth = kwargs.get("block_depth", 0) or 0
        self.activation = kwargs.get("activation", "lrelu")
        if self.arch_option and self.activation not in ("relu", "lrelu", "tanh"):
            raise ValueError(f"activation '{self.activation}': relu, lrelu or tanh (lseg_net.py:45-50)")
        self.channels_last = False
        self.out_c = cfg["text"][2]  # lseg_net.py:142-146: 768 with the RN50x16 text tower, else 512
        # holders are built on the meta device (no per-module default init: 400 M parameters would take
        # ~11 s of single-threaded CPU RNG) and then materialised with one cheap pass, see _fast_init
        with torch.device("meta"):
            self.clip_pretrained = _ClipTextHolder(*cfg["text"])
            self.pretrained = _pretrained_holder(cfg)
            self.scratch = _scratch_holder(self.out_c, cfg["features"])
            if self.arch_option in (1, 2):  # scratch.head_block.depthwise.depthwise = Conv2d(1, 1, 3, padding=1)
                hb = nn.Module()
                hb.depthwise = nn.Module()
                hb.depthwise.depthwise = nn.Conv2d(1, 1, kernel_size=3, stride=1, padding=1)
                self.scratch.head_block = hb
        self.logit_scale = torch.tensor(reference_logit_scale())
        # enable_attention_hooks (lseg_blocks.py:22): only the ViT-L/16 encoders honour it; _make_pretrained_clip_vitb32_384
        # forces it off (lseg_vit.py:270) and the ResNet trunk has no attention
        self._records_attention = bool(kwargs.get("enable_attention_hooks", False)) and cfg.get("patch") == 16
        if self._records_attention:
            self.pretrained.attention = {}  # per net (the reference's dict is module-global, lseg_vit.py:19)
        self.clip_pretrained._owner = weakref.ref(self)
        self._install_load_hooks()
        self._shared = {"engines": {}, "text_cache": {}, "lock": threading.Lock(), "master": weakref.ref(self),
                        "generation": next(_WEIGHTS_GENERATION)}
        self._fast_init()

    def _fast_init(self):
        """Materialise parameters on CPU: weights ~ U(+-1/sqrt(fan_in)) (torch's Linear/Conv default),
        LayerNorm/BatchNorm at identity, biases zero, embeddings/tokens small. Real use loads a checkpoint
        over this (load_state_dict / BaseModel.load); benchmarks run on it as 'random init'."""
        self.to_empty(device="cpu")
        # CPU RNG is ~25 M values/s; draw one block of U(-1,1) with a prime length and tile it (memcpy
        # speed) with a moving offset — rows of a weight never line up with the period
        period = 4194301
        base = torch.rand(period, generator=torch.Generator().manual_seed(0)) * 2.0 - 1.0
        cursor = 0
        norm_like = set()
        for name, mod in self.named_modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.reset_running_stats()
            if isinstance(mod, (nn.BatchNorm2d, nn.LayerNorm)):
                norm_like.add(name)
        with torch.no_grad():
            for name, p in self.named_parameters():
                owner = name.rsplit(".", 1)[0]
                if owner in norm_like:
                    p.fill_(1.0 if name.endswith("weight") else 0.0)
                elif name.endswith("logit_scale"):
                    p.fill_(2.6592600)
                elif p.dim() >= 2:
                    fan_in = p[0].numel() if p.dim() > 1 else p.numel()
                    if name.endswith(("cls_token", "pos_embed", "positional_embedding", "token_embedding.weight")):
                        bound = 0.03
                    else:
                        bound = fan_in ** -0.5
                    n = p.numel()
                    flat = p.view(-1)
                    done = 0
                    while done < n:
                        take = min(n - done, period - cursor)
                        flat[done:done + take] = base[cursor:cursor + take]
                        done += take
                        cursor = (cursor + take) % period
                    p.mul_(bound)
                else:
                    p.zero_()

    # -- weight management -------------------------------------------------------------------
    def _invalidate(self):
        if hasattr(self, "_shared"):
            with self._shared["lock"]:
                self._shared["engines"].clear()
                self._shared["text_cache"].clear()
                self._shared["generation"] = next(_WEIGHTS_GENERATION)  # embeddings encoded so far are stale

    def refresh(self):
        """Re-pack weights after in-place parameter edits."""
        self._invalidate()

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._invalidate()
        return out

    # Checkpoint loading goes through torch's recursive _load_from_state_dict when this net is a CHILD of the module
    # being loaded (Lightning's load_from_checkpoint loads `net.*` keys on the LightningModule), which never calls a
    # child's load_state_dict override. So the two things that must happen on every load are hooks on this module:
    #   pre : drop the entries of real checkpoints that have no holder here (CLIP visual tower, timm head) — they
    #         would otherwise be 'unexpected keys' under strict=True;
    #   post: drop the packed device weights / text-feature cache so the next forward re-packs.
    def _install_load_hooks(self):
        def pre(module, state_dict, prefix, *unused):
            for k in [k for k in state_dict if k.startswith(prefix) and k[len(prefix):].startswith(_IGNORED_PREFIXES)]:
                del state_dict[k]

        def post(module, incompatible_keys):
            module._invalidate()

        self.register_load_state_dict_pre_hook(pre)
        self.register_load_state_dict_post_hook(post)

    def load(self, path):
        """BaseModel.load (modules/models/lseg_net.py:81-92)."""
        parameters = torch.load(path, map_location=torch.device("cpu"))
        if "optimizer" in parameters:
            parameters = parameters["model"]
        self.load_state_dict(parameters)

    def _engine_for(self, device):
        from .engine import Engine
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("lseg_b200.LSegNet runs on CUDA (H100, sm_90a) only; there is no CPU fallback")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        shared = self._shared
        with shared["lock"]:
            eng = shared["engines"].get(device)
            if eng is None:
                sd = self.state_dict()
                if not sd:  # DataParallel replica: parameters live on the master copy
                    master = shared["master"]()
                    sd = master.state_dict() if master is not None else sd
                eng = Engine(sd, device, arch_option=self.arch_option, block_depth=self.block_depth,
                             activation=self.activation, backbone=self.backbone)
                shared["engines"][device] = eng
            return eng

    def _text_features(self, engine, tokens):
        key = (engine.device, tokens.shape[0], tokens.cpu().numpy().tobytes())
        cache = self._shared["text_cache"]
        feats = cache.get(key)
        if feats is None:
            feats = engine.encode_text(tokens)
            if len(cache) > 64:
                cache.clear()
            cache[key] = feats
        return feats

    @torch.no_grad()
    def encode_image(self, x):
        """The image path of forward (trunk, decoder, head1; lseg_net.py:166-185) of x fp32 [B,3,H,W] -> a
        PixelEmbedding to pass to forward / predict / update_metric in place of x, with any label set. Records the
        attention maps when the net was built with enable_attention_hooks."""
        self._check_eval()
        engine = self._engine_for(x.device)
        if self._records_attention:
            emb, sumsq, attn = engine.encode_image_attention(x.float())
            for k, a in enumerate(attn):  # fresh tensors: ones a caller kept from an earlier call stay as they were
                self.pretrained.attention[f"attn_{k + 1}"] = a
        else:
            emb, sumsq = engine.encode_image(x.float())
        return PixelEmbedding(emb, sumsq, x.shape[2:], self.backbone, self.out_c, self._shared["generation"])

    def _image_path(self, x):
        """x as it goes to the engine: with enable_attention_hooks, images are encoded here (recording the attention
        maps) and the call continues on the embedding, whose tail (lseg_query) is bit-identical to the fused forward; a
        PixelEmbedding, or any input of a net that does not record, is returned as it is."""
        if self._records_attention and not isinstance(x, PixelEmbedding):
            return self.encode_image(x)
        return x

    def _ragged_text(self, engine, labelsets, b):
        """Packed text operand of a ragged batch: the union of its labels encoded once (through the text-feature cache),
        then one device gather into image order, rows padded to a multiple of 128. -> (text, k, koff)."""
        if len(labelsets) != b:
            raise ValueError(f"{len(labelsets)} label sets for a batch of {b} images: one list of labels per image")
        union, rows, k, koff = ragged_label_table(labelsets)
        feats = self._text_features(engine, tokenize(union))
        text = torch.zeros((engine.padded_rows(len(rows)), self.out_c), dtype=torch.float16, device=engine.device)
        text[: len(rows)] = feats.index_select(0, torch.tensor(rows, dtype=torch.int64).to(engine.device))
        return text, k, koff

    def _run_ragged(self, x, labelsets, want_logits):
        """Forward (want_logits) or predict of a batch whose image b has its own labels labelsets[b]."""
        emb = x if isinstance(x, PixelEmbedding) else None
        engine = self._embedding_engine(emb) if emb is not None else self._engine_for(x.device)
        b, h, w = x.shape[0], x.shape[2], x.shape[3]
        text, k, koff = self._ragged_text(engine, labelsets, b)
        logits = torch.empty((sum(k), h, w), dtype=torch.float32, device=x.device) if want_logits else None
        mask = None if want_logits else torch.empty((b, h, w), dtype=torch.int64, device=x.device)
        if emb is not None:
            engine.query_ragged(emb.emb, emb.sumsq, text, koff, k, logits=logits, mask=mask)
        else:
            engine.forward_ragged(x.float(), text, koff, k, logits=logits, mask=mask)
        if not want_logits:
            return mask
        return [logits[o:o + n].unsqueeze(0) for o, n in zip(koff, k)]

    def _embedding_engine(self, emb):
        """The engine that queries `emb`, after checking that this net's current weights produced it."""
        if emb.backbone != self.backbone or emb.out_c != self.out_c:
            raise ValueError(f"embedding of backbone {emb.backbone!r} (out_c {emb.out_c}); this net is {self.backbone!r} "
                             f"(out_c {self.out_c})")
        if emb.generation != self._shared["generation"]:
            raise ValueError("embedding was encoded by another net, or with weights that have changed since "
                             "(load_state_dict / refresh / .to()): encode the images again")
        if emb.device.type != "cuda":
            raise ValueError(f"embedding is on {emb.device}; lseg_b200 runs on CUDA only")
        return self._engine_for(emb.device)

    def _check_eval(self):
        if self.training:
            raise NotImplementedError("lseg_b200.LSegNet is inference-only (BatchNorm running stats, no autograd); "
                                      "call .eval() first")


class LSegNet(_LSegBase):
    """Network for semantic segmentation — H100-native forward (reference: lseg_net.py:208-226)."""

    def __init__(self, labels, path=None, scale_factor=0.5, crop_size=480, **kwargs):
        super().__init__()
        self.crop_size = crop_size
        self.scale_factor = scale_factor
        self.labels = labels
        if BACKBONES.get(kwargs.get("backbone", "clip_vitl16_384"), {}).get("trunk") == "resnet101":
            # lseg_blocks.py:53-55: the ViT model's _make_encoder does not know this backbone (it belongs to LSegRNNetZS)
            print(f"Backbone '{kwargs['backbone']}' not implemented")
            assert False
        self._init_common(**kwargs)
        self.text = tokenize(self.labels)
        if path is not None:
            self.load(path)

    supports_out = True  # forward(..., out=) writes into a caller tensor (the evaluator's output batch)

    @torch.no_grad()
    def forward(self, x, labelset="", out=None):
        """`out` (optional, beyond the reference signature): a contiguous fp32 [B,K,H,W] CUDA tensor to write into.
        `labelset` may also be a list of B label lists, one per image: the result is then a list of B fp32 tensors
        [1, k_b, H, W] (views of one packed buffer), each what forward(x[b:b+1], labelset[b]) returns."""
        self._check_eval()
        if is_ragged(labelset):
            if out is not None:
                raise ValueError("out= is not supported with per-image label sets: the result is one tensor per image")
            return self._run_ragged(self._image_path(x), labelset, want_logits=True)
        if isinstance(labelset, torch.Tensor):
            text = labelset
        elif isinstance(labelset, str) and labelset == "":
            text = self.text
        else:
            text = tokenize(labelset)
        if not isinstance(x, PixelEmbedding) and out is not None and (
                out.dtype != torch.float32 or not out.is_contiguous() or
                tuple(out.shape) != (x.shape[0], text.shape[0], x.shape[2], x.shape[3])):
            raise ValueError("out must be a contiguous float32 [B,K,H,W] tensor")
        x = self._image_path(x)
        if isinstance(x, PixelEmbedding):
            engine = self._embedding_engine(x)
            feats = self._text_features(engine, text)
            b, (h, w), k = len(x), x.size, text.shape[0]
            if out is None:
                out = torch.empty((b, k, h, w), dtype=torch.float32, device=x.device)
            engine.query(x.emb, x.sumsq, feats, k, logits=out)
            return out
        engine = self._engine_for(x.device)
        feats = self._text_features(engine, text)
        return engine.forward(x.float(), feats, text.shape[0], out=out)

    def _labelset_tokens(self, labelset):
        if isinstance(labelset, torch.Tensor):
            return labelset
        if isinstance(labelset, str) and labelset == "":
            return self.text
        return tokenize(labelset)

    @torch.no_grad()
    def predict(self, x, labelset=""):
        """torch.max(self.forward(x, labelset), 1)[1] — what every caller of the reference does with the logits
        (lseg_app.py:357-360, test_lseg.py:397) — fused on the device: int64 [B,H,W], the fp32 [B,K,H,W] logits are
        never written (SURVEY.md 8(f) row 2). With a list of B label lists, mask[b] indexes labelset[b]."""
        self._check_eval()
        if is_ragged(labelset):
            return self._run_ragged(self._image_path(x), labelset, want_logits=False)
        text = self._labelset_tokens(labelset)
        x = self._image_path(x)
        if isinstance(x, PixelEmbedding):
            engine = self._embedding_engine(x)
            mask = torch.empty((len(x),) + x.size, dtype=torch.int64, device=x.device)
            engine.query(x.emb, x.sumsq, self._text_features(engine, text), text.shape[0], mask=mask)
            return mask
        engine = self._engine_for(x.device)
        feats = self._text_features(engine, text)
        return engine.forward_argmax(x.float(), feats, text.shape[0])

    @torch.no_grad()
    def update_metric(self, metric, x, target, labelset=""):
        """metric.update(target, self.forward(x, labelset)) for a lseg_b200.metrics.SegmentationMetric, fused into the
        output kernel: the counters of torch.max(logits, 1)[1] against target (int64 [B,H,W], or [H,W] for B = 1; -1 =
        ignored) are added on the device. Neither logits nor mask are written, and nothing synchronises."""
        from .metrics import _as_target
        self._check_eval()
        if is_ragged(labelset):
            raise ValueError("update_metric does not take per-image label sets: the class ids of the metric would differ "
                             "from image to image")
        text = self._labelset_tokens(labelset)
        x = self._image_path(x)
        emb = x if isinstance(x, PixelEmbedding) else None
        engine = self._embedding_engine(emb) if emb is not None else self._engine_for(x.device)
        feats = self._text_features(engine, text)
        stats = metric._buffer(x.device)
        t = _as_target(target, x.device, (x.shape[0], x.shape[2], x.shape[3]))
        if emb is not None:
            engine.query(emb.emb, emb.sumsq, feats, text.shape[0], target=t, stats=stats, nclass=metric.nclass)
        else:
            engine.forward_stats(x.float(), feats, text.shape[0], t, stats, metric.nclass)


    @torch.no_grad()
    def loss(self, x, target, labelset="", ignore_index=-1, metric=None):
        """F.cross_entropy(self.forward(x, labelset), target, ignore_index=ignore_index) — the validation loss of
        LSegmentationModule.validation_step — fused into the output kernel: a 0-d fp32 CUDA tensor, computed without
        writing the logits and without synchronising. target int64 [B,H,W] (or [H,W] for B = 1). A target outside
        [0, K) other than ignore_index makes the loss NaN and is recorded on the device (lseg_read_watchdog tag 79, which
        FewShotMeter.compute_iou raises on) where torch would assert. With `metric` (a lseg_b200.metrics.SegmentationMetric), its counters are added in the
        same kernel, exactly as update_metric adds them."""
        from .metrics import _as_target, _mean_loss
        self._check_eval()
        if is_ragged(labelset):
            raise ValueError("loss does not take per-image label sets: the class ids of the target would differ from "
                             "image to image")
        text = self._labelset_tokens(labelset)
        x = self._image_path(x)
        emb = x if isinstance(x, PixelEmbedding) else None
        engine = self._embedding_engine(emb) if emb is not None else self._engine_for(x.device)
        feats = self._text_features(engine, text)
        t = _as_target(target, x.device, (x.shape[0], x.shape[2], x.shape[3]))
        acc = torch.zeros(2, dtype=torch.float64, device=x.device)
        kw = dict(ignore_index=ignore_index)
        if metric is not None:
            kw.update(target=t, stats=metric._buffer(x.device), nclass=metric.nclass)
        if emb is not None:
            engine.query_loss(emb.emb, emb.sumsq, feats, text.shape[0], t, acc, **kw)
        else:
            engine.forward_loss(x.float(), feats, text.shape[0], t, acc, **kw)
        return _mean_loss(acc)


class LSegNetZS(_LSegBase):
    """Zero-shot variant (reference: lseg_net_zs.py:219-239; forward :177-214): one ['others', name]
    prompt pair per image, selected by class_info."""

    def __init__(self, label_list, path=None, scale_factor=0.5, aux=False, use_relabeled=False, use_pretrained=True,
                 **kwargs):
        super().__init__()
        self.scale_factor = scale_factor
        self.aux = aux
        self.use_relabeled = use_relabeled
        self.label_list = label_list
        self.use_pretrained = use_pretrained
        self._init_common(**kwargs)
        self._check_backbone()
        self.texts = [tokenize(["others", name]) for name in self.label_list]  # lseg_net_zs.py:169-175
        if path is not None:
            self.load(path)

    def _pair_features(self, engine):
        """L2-normalised fp16 features of every ['others', name] pair, [2 * n_labels, out_c], encoded in ONE text-tower
        call per device (the reference re-encodes the pair of every image on every forward, lseg_net_zs.py:196)."""
        tokens = torch.cat(self.texts, 0)
        return self._text_features(engine, tokens)

    def _image_text(self, engine, class_info, device):
        """text operand of the zero-shot forward: image b's pair at rows [2b, 2b+2) (text_image_stride = 2), rows padded
        to a multiple of 128 — one gather, no per-image Python loop."""
        ids = torch.as_tensor(class_info).to(device=device, dtype=torch.int64).reshape(-1)
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= len(self.label_list)):
            raise IndexError("class_info out of range")
        pairs = self._pair_features(engine)
        rows = torch.stack((2 * ids, 2 * ids + 1), 1).reshape(-1)
        # > 256 text rows: the engine falls back to one 128-row weight tile per image starting at that image's
        # block, so the last blocks need 128 readable rows behind them
        extra = 128 if rows.numel() > 256 else 0
        text = torch.zeros((engine.padded_rows(rows.numel()) + extra, self.out_c), dtype=torch.float16, device=device)
        text[: rows.numel()] = pairs.index_select(0, rows)
        return text

    @torch.no_grad()
    def forward(self, x, class_info):
        self._check_eval()
        x = self._image_path(x)
        if isinstance(x, PixelEmbedding):
            engine = self._embedding_engine(x)
            out = torch.empty((len(x), 2) + x.size, dtype=torch.float32, device=x.device)
            engine.query(x.emb, x.sumsq, self._image_text(engine, class_info, x.device), 2, text_image_stride=2,
                         logits=out)
            return out
        engine = self._engine_for(x.device)
        return engine.forward(x.float(), self._image_text(engine, class_info, x.device), 2, text_image_stride=2)

    def _check_backbone(self):
        if BACKBONES[self.backbone].get("trunk") == "resnet101":
            # the reference keeps the two apart the same way: LSegNetZS asserts out in _make_encoder's ViT branch
            raise ValueError("backbone 'clip_resnet101' is the trunk of LSegRNNetZS (lseg_net_zs.py:345), not LSegNetZS")

    @torch.no_grad()
    def predict(self, x, class_info):
        """argmax over the ['others', name] pair per pixel (test_lseg_zs.py:301), fused on the device."""
        self._check_eval()
        x = self._image_path(x)
        if isinstance(x, PixelEmbedding):
            engine = self._embedding_engine(x)
            mask = torch.empty((len(x),) + x.size, dtype=torch.int64, device=x.device)
            engine.query(x.emb, x.sumsq, self._image_text(engine, class_info, x.device), 2, text_image_stride=2,
                         mask=mask)
            return mask
        engine = self._engine_for(x.device)
        return engine.forward_argmax(x.float(), self._image_text(engine, class_info, x.device), 2, text_image_stride=2)

    @torch.no_grad()
    def update_metric(self, meter, x, class_info, target, query_ignore_idx=None):
        """Evaluator.classify_prediction(self.predict(x, class_info), target, query_ignore_idx) followed by
        meter.update(..., class_info) for a lseg_b200.metrics.FewShotMeter, fused into the output kernel: image b's
        counters go straight to the meter's row class_info[b]. Neither logits nor mask are written; the one host
        synchronisation is forward()'s class_info range check. A padded input takes a target padded with -1."""
        from .metrics import _as_target, _fewshot_target
        self._check_eval()
        x = self._image_path(x)
        emb = x if isinstance(x, PixelEmbedding) else None
        engine = self._embedding_engine(emb) if emb is not None else self._engine_for(x.device)
        text = self._image_text(engine, class_info, x.device)
        t = _as_target(target, x.device, (x.shape[0], x.shape[2], x.shape[3]))
        t = _fewshot_target(t, query_ignore_idx)
        group = torch.as_tensor(class_info).to(x.device)
        if emb is not None:
            engine.query(emb.emb, emb.sumsq, text, 2, text_image_stride=2, target=t, stats=meter.stats, nclass=2,
                         group=group)
        else:
            engine.forward_stats(x.float(), text, 2, t, meter.stats, 2, group=group, text_image_stride=2)


    @torch.no_grad()
    def loss(self, x, class_info, target, ignore_index=-1, meter=None, query_ignore_idx=None):
        """criterion(self.forward(x, class_info), target) of the zero-shot validation step (CrossEntropyLoss with
        ignore_index over the raw target), fused into the output kernel: a 0-d fp32 CUDA tensor. With `meter` (a
        lseg_b200.metrics.FewShotMeter), the same kernel also adds the update_metric counters (the metric target gets
        query_ignore_idx applied, the loss target does not) and the loss is appended to meter.loss_buf. A target outside
        [0, 2) other than ignore_index (e.g. 255 with ignore_index=-1) gives NaN and a device record instead of torch's
        assert."""
        from .metrics import _as_target, _fewshot_target, _mean_loss
        self._check_eval()
        x = self._image_path(x)
        emb = x if isinstance(x, PixelEmbedding) else None
        engine = self._embedding_engine(emb) if emb is not None else self._engine_for(x.device)
        text = self._image_text(engine, class_info, x.device)
        t = _as_target(target, x.device, (x.shape[0], x.shape[2], x.shape[3]))
        acc = torch.zeros(2, dtype=torch.float64, device=x.device)
        kw = dict(ignore_index=ignore_index, text_image_stride=2)
        if meter is not None:
            kw.update(target=_fewshot_target(t, query_ignore_idx), stats=meter.stats, nclass=2,
                      group=torch.as_tensor(class_info).to(x.device))
        if emb is not None:
            engine.query_loss(emb.emb, emb.sumsq, text, 2, t, acc, **kw)
        else:
            engine.forward_loss(x.float(), text, 2, t, acc, **kw)
        loss = _mean_loss(acc)
        if meter is not None:
            meter.loss_buf.append(loss)
        return loss


class LSegRNNetZS(LSegNetZS):
    """Zero-shot model on the ResNet-101 trunk (reference: lseg_net_zs.py:240-378, `LSegRN` / `LSegRNNetZS`; backbone
    "clip_resnet101" = torchvision resnet101 + the CLIP ViT-B/32 text tower, lseg_vit_zs.py:742-748): the four ResNet stages
    feed scratch.layerN_rn directly (lseg_net_zs.py:307-315); decoder, per-image ['others', name] head and x2 output as in
    LSegNetZS. Same constructor and state-dict keys (pretrained.layer1.{0,1,4.*}, pretrained.layer{2,3,4}.*, scratch.*,
    clip_pretrained.*)."""

    def __init__(self, label_list, path=None, scale_factor=0.5, aux=False, use_relabeled=False, use_pretrained=True,
                 **kwargs):
        kwargs.setdefault("backbone", "clip_resnet101")
        super().__init__(label_list, path=path, scale_factor=scale_factor, aux=aux, use_relabeled=use_relabeled,
                         use_pretrained=use_pretrained, **kwargs)

    def _check_backbone(self):
        if BACKBONES[self.backbone].get("trunk") != "resnet101":
            raise ValueError(f"LSegRNNetZS runs the ResNet trunk (backbone 'clip_resnet101'), got {self.backbone!r}")
