"""Python handle over the C engine (lseg_create / lseg_encode_text / lseg_forward)."""
import ctypes as C

import torch

from . import _lib
from .packing import PackedWeights


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check_embedding(emb, sumsq, device=None, out_c=None):
    """Validates an embedding pair (include/lseg_b200.h) -> (B, H, W) of the images it encodes."""
    if not isinstance(emb, torch.Tensor) or not isinstance(sumsq, torch.Tensor):
        raise ValueError("emb and sumsq must be tensors")
    device = emb.device if device is None else device
    if emb.device != device or sumsq.device != device or device.type != "cuda":
        raise ValueError(f"embedding is on {emb.device} / {sumsq.device}, expected {device} (CUDA)")
    c = emb.shape[-1] if out_c is None else out_c
    if (emb.dtype != torch.float16 or emb.dim() != 4 or emb.shape[3] != c or c not in (512, 768) or
            not emb.is_contiguous()):
        raise ValueError(f"emb must be a contiguous float16 [B,H/2,W/2,{c}] tensor (out_c 512 or 768), got {emb.dtype} "
                         f"{tuple(emb.shape)}")
    want = tuple(emb.shape[:3]) + (c // 32,)
    if sumsq.dtype != torch.float32 or tuple(sumsq.shape) != want or not sumsq.is_contiguous():
        raise ValueError(f"sumsq must be a contiguous float32 {want} tensor, got {sumsq.dtype} {tuple(sumsq.shape)}")
    b, h2, w2, _ = emb.shape
    if b == 0 or h2 % 16 or w2 % 16:
        raise ValueError(f"emb grid {h2}x{w2} of {b} images: not the embedding of H, W multiples of 32")
    return b, 2 * h2, 2 * w2


def embedding_features(emb, sumsq, out=None):
    """The reference's normalised image_features fp32 [B,C,H/2,W/2] (lseg_net.py:187-191) of an embedding pair: the
    export kernel of liblseg_b200.so, no engine needed. Enqueues on the current stream."""
    b, h, w = check_embedding(emb, sumsq)
    c = emb.shape[3]
    shape = (b, c, h // 2, w // 2)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=emb.device)
    elif out.device != emb.device or out.dtype != torch.float32 or tuple(out.shape) != shape or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous float32 {shape} tensor on {emb.device}")
    lib = _lib.load()
    with torch.cuda.device(emb.device):
        _lib.check(lib.lseg_embedding_features(C.c_void_p(emb.data_ptr()), C.c_void_p(sumsq.data_ptr()), b, h // 2,
                                               w // 2, c, C.c_void_p(out.data_ptr()), _stream()))
    return out


class Engine:
    """Owns the packed weights and the native engine for one CUDA device."""

    def __init__(self, state_dict, device, arch_option=0, block_depth=0, activation="lrelu", backbone="clip_vitl16_384"):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("lseg_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        self.device = device
        self.lib = _lib.load()
        with torch.cuda.device(device):
            self.weights = PackedWeights(state_dict, device, arch_option=arch_option, block_depth=block_depth,
                                         activation=activation, backbone=backbone)
            self.out_c = int(self.weights.desc.out_c)
            torch.cuda.synchronize()
            handle = C.c_void_p()
            idx = device.index if device.index is not None else torch.cuda.current_device()
            _lib.check(self.lib.lseg_create(C.byref(self.weights.desc), idx, C.byref(handle)))
        self.handle = handle

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.lseg_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    @staticmethod
    def padded_rows(k):
        return (k + 127) // 128 * 128

    def encode_text(self, tokens):
        """tokens int64 [K,77] (any device) -> L2-normalised text features fp16 [rows_padded(K), out_c]."""
        tokens = tokens.to(self.device, torch.int64).contiguous()
        k = tokens.shape[0]
        if tokens.dim() != 2 or tokens.shape[1] != 77:
            raise ValueError("tokens must be int64 [K, 77]")
        out = torch.empty((self.padded_rows(k), self.out_c), dtype=torch.float16, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_encode_text(self.handle, C.c_void_p(tokens.data_ptr()), k,
                                                 C.c_void_p(out.data_ptr()), _stream()))
        return out

    def forward(self, x, text, k, text_image_stride=0, out=None):
        """x fp32 [B,3,H,W] cuda; text fp16 [rows,out_c] (or [B*stride,out_c] per-image blocks) -> fp32 [B,K,H,W]."""
        if x.device != self.device:
            raise RuntimeError(f"input is on {x.device}, engine is on {self.device}")
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("x must be float32 [B,3,H,W]")
        x = x.contiguous()
        b, _, h, w = x.shape
        if h % 32 or w % 32:
            raise ValueError(f"H={h}, W={w} must be multiples of 32 (the reference fails on odd token grids)")
        if out is None:
            out = torch.empty((b, k, h, w), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                             C.c_void_p(text.data_ptr()), k, text_image_stride,
                                             C.c_void_p(out.data_ptr()), _stream()))
        return out

    def forward_lowres(self, x, text, k, text_image_stride=0, logits_lr=None, out=None):
        """LSeg.forward up to the reference's fp16 matmul result: fp16 [B,K,H/2,W/2]. `logits_lr` may be a tensor of
        this device or a raw device address (int) — e.g. a peer GPU's gather slot opened with lseg_p2p_open: the
        pixel x text GEMM then stores straight over NVLink. `out` (fp32 [B,K,H,W]) is optional."""
        self._check_input(x)
        x = x.contiguous()
        b, _, h, w = x.shape
        if logits_lr is None:
            logits_lr = torch.empty((b, k, h // 2, w // 2), dtype=torch.float16, device=self.device)
        lr_ptr = logits_lr if isinstance(logits_lr, int) else logits_lr.data_ptr()
        op = C.c_void_p(out.data_ptr()) if out is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward_lowres(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                    C.c_void_p(text.data_ptr()), k, text_image_stride,
                                                    C.c_void_p(lr_ptr), op, _stream()))
        return logits_lr

    def _check_input(self, x):
        if x.device != self.device:
            raise RuntimeError(f"input is on {x.device}, engine is on {self.device}")
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("x must be float32 [B,3,H,W]")
        if x.shape[2] % 32 or x.shape[3] % 32:
            raise ValueError(f"H={x.shape[2]}, W={x.shape[3]} must be multiples of 32 (the reference fails on odd token "
                             f"grids)")

    def forward_argmax(self, x, text, k, text_image_stride=0, out=None, logits=None):
        """Like forward, but returns torch.max(logits, 1)[1] as int64 [B,H,W] without materialising the fp32 logits
        (they are also written when a `logits` tensor is passed)."""
        if x.device != self.device:
            raise RuntimeError(f"input is on {x.device}, engine is on {self.device}")
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("x must be float32 [B,3,H,W]")
        x = x.contiguous()
        b, _, h, w = x.shape
        if h % 32 or w % 32:
            raise ValueError(f"H={h}, W={w} must be multiples of 32 (the reference fails on odd token grids)")
        if out is None:
            out = torch.empty((b, h, w), dtype=torch.int64, device=self.device)
        lp = C.c_void_p(logits.data_ptr()) if logits is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward_argmax(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                    C.c_void_p(text.data_ptr()), k, text_image_stride,
                                                    C.c_void_p(out.data_ptr()), lp, _stream()))
        return out

    def forward_stats(self, x, text, k, target, stats, nclass, group=None, text_image_stride=0, mask=None, logits=None):
        """Forward + argmax + metric counters in one output kernel: adds the counters of torch.max(logits, 1)[1] against
        target int64 [B,H,W] to stats int64 [G, 3*nclass+2] (include/lseg_b200.h), in row group[b] for image b (row 0
        without a group). Writes the mask / logits only into the tensors passed; enqueues on the current stream and does
        not synchronise."""
        from .ops import _check_stats, _group_ptr
        self._check_input(x)
        x = x.contiguous()
        b, _, h, w = x.shape
        _check_stats(stats, nclass)
        if target.device != self.device or target.dtype != torch.int64 or tuple(target.shape) != (b, h, w):
            raise ValueError(f"target must be int64 [B,H,W] = {(b, h, w)} on {self.device}")
        if stats.device != self.device or not stats.is_contiguous():
            raise ValueError(f"stats must be a contiguous tensor on {self.device}")
        for name, t, dt, shape in (("mask", mask, torch.int64, (b, h, w)), ("logits", logits, torch.float32, (b, k, h, w))):
            if t is not None and (t.device != self.device or t.dtype != dt or tuple(t.shape) != shape or
                                  not t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous {dt} {shape} tensor on {self.device}")
        target = target.contiguous()
        g, gp = _group_ptr(group, stats, b)
        mp = C.c_void_p(mask.data_ptr()) if mask is not None else None
        lp = C.c_void_p(logits.data_ptr()) if logits is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward_segstats(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                      C.c_void_p(text.data_ptr()), k, text_image_stride,
                                                      C.c_void_p(target.data_ptr()), gp, nclass, stats.shape[0],
                                                      C.c_void_p(stats.data_ptr()), mp, lp, _stream()))
        return stats

    def _loss_args(self, b, h, w, k, loss_target, acc, ignore_index, target, stats, nclass, group, mask, logits):
        """ctypes arguments of lseg_forward_xent / lseg_query_xent from `target` to `partials_len`, after checking the
        tensors; the partials workspace comes back too, so that it outlives the call's enqueue."""
        from .ops import _check_stats, _group_ptr, xent_partials
        if loss_target.device != self.device or loss_target.dtype != torch.int64 or tuple(loss_target.shape) != (b, h, w):
            raise ValueError(f"loss target must be int64 [B,H,W] = {(b, h, w)} on {self.device}")
        if acc.device != self.device or acc.dtype != torch.float64 or acc.numel() != 2 or not acc.is_contiguous():
            raise ValueError(f"acc must be a contiguous float64 tensor of 2 elements on {self.device}")
        for name, t, dt, shape in (("mask", mask, torch.int64, (b, h, w)), ("logits", logits, torch.float32, (b, k, h, w))):
            if t is not None and (t.device != self.device or t.dtype != dt or tuple(t.shape) != shape or
                                  not t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous {dt} {shape} tensor on {self.device}")
        tp = gp = sp = g = None
        if stats is not None or target is not None:
            if stats is None or target is None:
                raise ValueError("target and stats go together")
            _check_stats(stats, nclass)
            if target.device != self.device or target.dtype != torch.int64 or tuple(target.shape) != (b, h, w):
                raise ValueError(f"target must be int64 [B,H,W] = {(b, h, w)} on {self.device}")
            if stats.device != self.device or not stats.is_contiguous():
                raise ValueError(f"stats must be a contiguous tensor on {self.device}")
            target = target.contiguous()
            g, gp = _group_ptr(group, stats, b)
            tp, sp = C.c_void_p(target.data_ptr()), C.c_void_p(stats.data_ptr())
        loss_target = loss_target.contiguous()
        part = torch.empty((xent_partials(b, h, w, True), 2), dtype=torch.float64, device=self.device)
        args = [tp, gp, nclass, stats.shape[0] if stats is not None else 0, sp, C.c_void_p(loss_target.data_ptr()),
                int(ignore_index), C.c_void_p(acc.data_ptr()), C.c_void_p(part.data_ptr()), part.numel()]
        return args, (target, g, loss_target, part)

    def forward_loss(self, x, text, k, loss_target, acc, ignore_index=-1, text_image_stride=0, target=None, stats=None,
                     nclass=0, group=None, mask=None, logits=None):
        """Forward with the cross-entropy fused into the output kernel: adds {sum of per-pixel losses, counted pixels} of
        the logits against loss_target int64 [B,H,W] (pixels equal to ignore_index skipped) to acc float64 [2]. With
        target and stats, also the metric counters as forward_stats adds them; mask / logits are written when passed.
        Enqueues on the current stream and does not synchronise."""
        self._check_input(x)
        x = x.contiguous()
        b, _, h, w = x.shape
        args, keep = self._loss_args(b, h, w, k, loss_target, acc, ignore_index, target, stats, nclass, group, mask,
                                     logits)
        mp = C.c_void_p(mask.data_ptr()) if mask is not None else None
        lp = C.c_void_p(logits.data_ptr()) if logits is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward_xent(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                  C.c_void_p(text.data_ptr()), k, text_image_stride, *args, mp, lp,
                                                  _stream()))
        return acc

    def query_loss(self, emb, sumsq, text, k, loss_target, acc, ignore_index=-1, text_image_stride=0, target=None,
                   stats=None, nclass=0, group=None, mask=None, logits=None):
        """forward_loss's label-dependent tail on a stored embedding pair: the same bits as forward_loss on the images
        that produced it."""
        b, h, w = check_embedding(emb, sumsq, self.device, self.out_c)
        args, keep = self._loss_args(b, h, w, k, loss_target, acc, ignore_index, target, stats, nclass, group, mask,
                                     logits)
        mp = C.c_void_p(mask.data_ptr()) if mask is not None else None
        lp = C.c_void_p(logits.data_ptr()) if logits is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_query_xent(self.handle, C.c_void_p(emb.data_ptr()), C.c_void_p(sumsq.data_ptr()),
                                                b, h, w, C.c_void_p(text.data_ptr()), k, text_image_stride, lp, mp,
                                                *args, _stream()))
        return acc

    def encode_image(self, x):
        """The image path of forward (trunk, decoder, head1) -> the pixel embedding pair (emb fp16 [B,H/2,W/2,out_c],
        sumsq fp32 [B,H/2,W/2,out_c/32]); layout in include/lseg_b200.h. Enqueues on the current stream."""
        self._check_input(x)
        x = x.contiguous()
        b, _, h, w = x.shape
        emb = torch.empty((b, h // 2, w // 2, self.out_c), dtype=torch.float16, device=self.device)
        sumsq = torch.empty((b, h // 2, w // 2, self.out_c // 32), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_encode_image(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                  C.c_void_p(emb.data_ptr()), C.c_void_p(sumsq.data_ptr()), _stream()))
        return emb, sumsq

    def attention_shape(self, b, h, w):
        """Shape of one hooked block's attention probabilities for B images of H x W: [B, heads, N, N] with N the
        token count (patch grid + class token)."""
        d = self.weights.desc
        if d.trunk != 0:
            raise ValueError("attention maps need a ViT trunk; this engine runs the ResNet-101 one")
        p = int(d.patch_size)
        n = (h // p) * (w // p) + 1
        return (b, int(d.vit_heads), n, n)

    def encode_image_attention(self, x):
        """encode_image that also records the attention probabilities of the four hooked blocks: returns (emb, sumsq,
        [attn_1, .., attn_4]), each attn_k a fresh fp32 [B, heads, N, N] tensor. The embedding pair has the same bits as
        encode_image's. Enqueues on the current stream."""
        self._check_input(x)
        x = x.contiguous()
        b, _, h, w = x.shape
        shape = self.attention_shape(b, h, w)
        emb = torch.empty((b, h // 2, w // 2, self.out_c), dtype=torch.float16, device=self.device)
        sumsq = torch.empty((b, h // 2, w // 2, self.out_c // 32), dtype=torch.float32, device=self.device)
        attn = [torch.empty(shape, dtype=torch.float32, device=self.device) for _ in range(4)]
        ptrs = (C.c_void_p * 4)(*[a.data_ptr() for a in attn])
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_encode_image_attention(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                            C.c_void_p(emb.data_ptr()), C.c_void_p(sumsq.data_ptr()),
                                                            ptrs, _stream()))
        return emb, sumsq, attn

    def query(self, emb, sumsq, text, k, text_image_stride=0, logits=None, mask=None, target=None, stats=None,
              nclass=0, group=None):
        """The label-dependent tail of forward on a stored embedding: writes the fp32 logits [B,K,H,W] (as forward), the
        int64 mask [B,H,W] (as forward_argmax) and / or adds the metric counters of the mask against target to stats (as
        forward_stats) — whichever tensors are passed, at least one. Enqueues on the current stream."""
        from .ops import _check_stats, _group_ptr
        b, h, w = check_embedding(emb, sumsq, self.device, self.out_c)
        if logits is None and mask is None and stats is None:
            raise ValueError("query: no output requested (logits, mask or stats)")
        for name, t, dt, shape in (("mask", mask, torch.int64, (b, h, w)), ("logits", logits, torch.float32, (b, k, h, w))):
            if t is not None and (t.device != self.device or t.dtype != dt or tuple(t.shape) != shape or
                                  not t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous {dt} {shape} tensor on {self.device}")
        tp = gp = sp = None
        g = 0
        if stats is not None or target is not None:
            if stats is None or target is None:
                raise ValueError("query: target and stats go together")
            _check_stats(stats, nclass)
            if target.device != self.device or target.dtype != torch.int64 or tuple(target.shape) != (b, h, w):
                raise ValueError(f"target must be int64 [B,H,W] = {(b, h, w)} on {self.device}")
            if stats.device != self.device or not stats.is_contiguous():
                raise ValueError(f"stats must be a contiguous tensor on {self.device}")
            target = target.contiguous()
            g, gp = _group_ptr(group, stats, b)
            tp, sp = C.c_void_p(target.data_ptr()), C.c_void_p(stats.data_ptr())
        lp = C.c_void_p(logits.data_ptr()) if logits is not None else None
        mp = C.c_void_p(mask.data_ptr()) if mask is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_query(self.handle, C.c_void_p(emb.data_ptr()), C.c_void_p(sumsq.data_ptr()), b, h, w,
                                           C.c_void_p(text.data_ptr()), k, text_image_stride, lp, mp, tp, gp,
                                           nclass, stats.shape[0] if stats is not None else 0, sp, _stream()))

    def _ragged_args(self, text, text_row, k, b, h, w, logits, mask):
        """ctypes arguments of a ragged call (include/lseg_b200.h), after checking the output tensors' shapes."""
        if len(text_row) != b or len(k) != b:
            raise ValueError(f"text_row and k need one entry per image ({b}), got {len(text_row)} and {len(k)}")
        if text.device != self.device or text.dtype != torch.float16 or text.dim() != 2 or not text.is_contiguous():
            raise ValueError(f"text must be a contiguous float16 [rows, out_c] tensor on {self.device}")
        if logits is None and mask is None:
            raise ValueError("ragged call: no output requested (logits or mask)")
        for name, t, dt, shape in (("mask", mask, torch.int64, (b, h, w)), ("logits", logits, torch.float32,
                                                                            (sum(k), h, w))):
            if t is not None and (t.device != self.device or t.dtype != dt or tuple(t.shape) != shape or
                                  not t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous {dt} {shape} tensor on {self.device}")
        ints = C.c_int * b
        return [C.c_void_p(text.data_ptr()), text.shape[0], ints(*text_row), ints(*k),
                C.c_void_p(logits.data_ptr()) if logits is not None else None,
                C.c_void_p(mask.data_ptr()) if mask is not None else None, _stream()]

    def forward_ragged(self, x, text, text_row, k, logits=None, mask=None):
        """Forward of a batch in which image b has its own k[b] labels, rows text_row[b] .. of `text` (fp16 [rows,
        out_c]). Writes the packed fp32 logits [sum k, H, W] (image b's planes follow those of images 0 .. b-1) and / or
        the int64 mask [B, H, W] (mask[b] indexes image b's labels) into the tensors passed. Enqueues on the current
        stream."""
        self._check_input(x)
        x = x.contiguous()
        b, _, h, w = x.shape
        args = self._ragged_args(text, text_row, k, b, h, w, logits, mask)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward_ragged(self.handle, C.c_void_p(x.data_ptr()), b, h, w, *args))

    def query_ragged(self, emb, sumsq, text, text_row, k, logits=None, mask=None):
        """forward_ragged's label-dependent tail on a stored embedding pair."""
        b, h, w = check_embedding(emb, sumsq, self.device, self.out_c)
        args = self._ragged_args(text, text_row, k, b, h, w, logits, mask)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_query_ragged(self.handle, C.c_void_p(emb.data_ptr()), C.c_void_p(sumsq.data_ptr()),
                                                  b, h, w, *args))

    def forward_profiled(self, x, text, k, text_image_stride=0, out=None):
        """One forward with CUDA events around every launch. Returns (out, [(ms, kind, flops), ...])."""
        x = x.contiguous()
        b, _, h, w = x.shape
        if out is None:
            out = torch.empty((b, k, h, w), dtype=torch.float32, device=self.device)
        cap = 2048
        ms = (C.c_float * cap)()
        kind = (C.c_int * cap)()
        flops = (C.c_double * cap)()
        n = C.c_int(0)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.lseg_forward_profiled(self.handle, C.c_void_p(x.data_ptr()), b, h, w,
                                                      C.c_void_p(text.data_ptr()), k, text_image_stride,
                                                      C.c_void_p(out.data_ptr()), _stream(), ms, kind, flops, cap,
                                                      C.byref(n)))
        return out, [(ms[i], kind[i], flops[i]) for i in range(n.value)]

    def last_launch_count(self):
        return int(self.lib.lseg_last_launch_count(self.handle))

    def debug_tensor(self, name, shape, dtype):
        """View of an intermediate activation of the last forward (valid until the next forward)."""
        ptr = self.lib.lseg_debug_buffer(self.handle, name.encode())
        if not ptr:
            raise KeyError(name)
        # build a tensor aliasing device memory through the cuda array interface
        class _Holder:
            pass
        h = _Holder()
        typestr = {torch.float32: "<f4", torch.float16: "<f2"}[dtype]
        h.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}
        return torch.as_tensor(h, device=self.device)
