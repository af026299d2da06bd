"""Drop-in `LSegNet` / `LSegNetZS` whose forward runs on the sm_90a engine.

Mirrors the reference interface for the hot path (SURVEY.md section 8(b)):
  * constructor signatures of modules/models/lseg_net.py:208-226 and lseg_net_zs.py:219-239;
  * `forward(x, labelset='')` (lseg_net.py:160) / `forward(x, class_info)` (lseg_net_zs.py:177);
  * attributes the callers touch: `.pretrained.model.patch_embed.img_size` (lseg_module.py:86-89),
    `.scratch`, `.clip_pretrained` (with `.encode_text`), `.labels`, `.text`, `.crop_size`, `.out_c`,
    `.arch_option`, `.logit_scale`;
  * state-dict key names and shapes of SURVEY.md Appendix C, so `BaseModel.load` / Lightning's
    `load_from_checkpoint` (prefix `net.`) keep working; the unused `clip_pretrained.visual.*` and timm
    `head.*` entries of real checkpoints are accepted and ignored.
The torch sub-modules below are parameter holders only (they give the reference's names, shapes and
default inits); no torch op runs in forward. There is no CPU path: a non-CUDA input raises.
"""
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
        self.clip_pretrained._owner = weakref.ref(self)
        self._install_load_hooks()
        self._shared = {"engines": {}, "text_cache": {}, "lock": threading.Lock(), "master": weakref.ref(self)}
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
        """`out` (optional, beyond the reference signature): a contiguous fp32 [B,K,H,W] CUDA tensor to write into."""
        self._check_eval()
        if isinstance(labelset, torch.Tensor):
            text = labelset
        elif isinstance(labelset, str) and labelset == "":
            text = self.text
        else:
            text = tokenize(labelset)
        engine = self._engine_for(x.device)
        feats = self._text_features(engine, text)
        if out is not None and (out.dtype != torch.float32 or not out.is_contiguous() or
                                tuple(out.shape) != (x.shape[0], text.shape[0], x.shape[2], x.shape[3])):
            raise ValueError("out must be a contiguous float32 [B,K,H,W] tensor")
        return engine.forward(x.float(), feats, text.shape[0], out=out)

    @torch.no_grad()
    def predict(self, x, labelset=""):
        """torch.max(self.forward(x, labelset), 1)[1] — what every caller of the reference does with the logits
        (lseg_app.py:357-360, test_lseg.py:397) — fused on the device: int64 [B,H,W], the fp32 [B,K,H,W] logits are
        never written (SURVEY.md 8(f) row 2)."""
        self._check_eval()
        if isinstance(labelset, torch.Tensor):
            text = labelset
        elif isinstance(labelset, str) and labelset == "":
            text = self.text
        else:
            text = tokenize(labelset)
        engine = self._engine_for(x.device)
        feats = self._text_features(engine, text)
        return engine.forward_argmax(x.float(), feats, text.shape[0])


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
        engine = self._engine_for(x.device)
        return engine.forward_argmax(x.float(), self._image_text(engine, class_info, x.device), 2, text_image_stride=2)


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
