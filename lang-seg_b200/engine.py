"""Python handle over the C engine (lseg_create / lseg_encode_text / lseg_forward)."""
import ctypes as C

import torch

from . import _lib
from .packing import PackedWeights


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


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
