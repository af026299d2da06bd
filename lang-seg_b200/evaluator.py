"""Batched multi-scale / flip / sliding-window evaluator (SURVEY.md 8(f) "next" row 1).

Mirror of `LSeg_MultiEvalModule.forward` (reference `additional_utils/models.py:55-140`; helpers `:142-170`): for
every scale the image is resized (bilinear, align_corners=True), padded to the crop size with the normalised-zero
value, cut into crop_size x crop_size windows with stride int(crop_size * 2/3), every window is evaluated plain and
horizontally flipped, the window outputs are summed into a canvas that is divided by the per-pixel window count,
cropped, resized back and summed over scales.

The reference evaluates the windows ONE AT A TIME (batch 1, 2 forwards per window — 36+ forwards per image at the
default six scales, each re-encoding the label set). Here every window of every scale (and its flip) is collected
first and pushed through the network in large batches — all windows have the same crop_size x crop_size shape — and
only then are the reference's accumulations replayed, in the reference's order, on the precomputed outputs. With a
batch-invariant network (lseg_b200 in its default deterministic mode) the result is bit-identical to the sequential
algorithm; `tests/test_evaluator_cpu.py` checks that against the unmodified reference class on CPU.

Two implementations of the glue around `net(batch, label_set)` = `LSegNet.forward`:
  * `fused=True` (default on a CUDA image): three gather kernels of liblseg_b200.so (csrc/evaluator.cuh) — every network
    input of a scale is sampled straight from the original image (resize + pad + slice + pad + flip in one launch), the
    window outputs are overlap-averaged into the scale's canvas and the canvas is resized back and added to the scores;
    the resized / padded images and the per-window torch slices never exist;
  * `fused=False`: the same algorithm as torch calls (runs on CPU too: tests/test_evaluator_cpu.py pins it bit for bit
    against the unmodified reference class).
Both keep the reference's order of floating-point operations. One process per GPU handles its own images
(lang-seg_b200/parallel.py) instead of the reference's thread-per-GPU `parallel_forward`
(`additional_utils/models.py:35-53`).
"""
import math

import torch
import torch.nn.functional as F

UP_KWARGS = {"mode": "bilinear", "align_corners": True}  # additional_utils/models.py:18


def resize_image(img, h, w, **up_kwargs):  # additional_utils/models.py:142-143
    return F.interpolate(img, (h, w), **up_kwargs)


def pad_image(img, mean, std, crop_size):  # additional_utils/models.py:145-156
    b, c, h, w = img.shape
    assert c == 3
    padh = crop_size - h if h < crop_size else 0
    padw = crop_size - w if w < crop_size else 0
    out = img.new_empty((b, c, h + padh, w + padw))
    for i in range(c):
        out[:, i] = F.pad(img[:, i], (0, padw, 0, padh), value=-float(mean[i]) / float(std[i]))
    return out


def flip_image(img):  # additional_utils/models.py:161-165
    return img.flip(3)


class MultiScaleEvaluator:
    """`MultiScaleEvaluator(net, base_size, crop_size)(image[1,3,h,w], label_set) -> scores fp32 [1,K,h,w]`.

    net(x[B,3,crop,crop], label_set) -> [B,K,crop,crop] is `LSegNet.forward` (or the Lightning module's
    `evaluate_random`, reference modules/lsegmentation_module.py:54-59). crop_size must be a multiple of 32.
    """

    def __init__(self, net, base_size=520, crop_size=480, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), flip=True,
                 scales=(0.5, 0.75, 1.0, 1.25, 1.5, 1.75), up_kwargs=None, max_batch=16, fused=None):
        self.net = net
        self.base_size = base_size
        self.crop_size = crop_size
        self.mean = mean
        self.std = std
        self.flip = flip
        self.scales = list(scales)
        self.up_kwargs = dict(UP_KWARGS if up_kwargs is None else up_kwargs)
        self.max_batch = max_batch
        self.fused = fused  # None: fused kernels whenever the image is on a CUDA device

    # ---- integer geometry of one scale (additional_utils/models.py:67-114), shared by both implementations ----
    def _geometry(self, h, w, scale):
        crop = self.crop_size
        stride = int(crop * (2.0 / 3.0))
        long_size = int(math.ceil(self.base_size * scale))
        if h > w:
            height = long_size
            width = int(1.0 * w * long_size / h + 0.5)
            short_size = width
        else:
            width = long_size
            height = int(1.0 * h * long_size / w + 0.5)
            short_size = height
        if long_size <= crop:
            return {"height": height, "width": width, "whole": True, "origins": [(0, 0)]}
        ph = max(height, crop) if short_size < crop else height
        pw = max(width, crop) if short_size < crop else width
        h_grids = int(math.ceil(1.0 * (ph - crop) / stride)) + 1
        w_grids = int(math.ceil(1.0 * (pw - crop) / stride)) + 1
        origins = [(idh * stride, idw * stride) for idh in range(h_grids) for idw in range(w_grids)]
        return {"height": height, "width": width, "whole": False, "origins": origins}

    # ---- fused device path: csrc/evaluator.cuh through the C ABI ----
    def _windows(self, h, w):
        """Per-scale geometry, the window list of every network input (plain and flipped, scale by scale) and the first
        row of each scale in it."""
        geo = [self._geometry(h, w, scale) for scale in self.scales]
        rows, first = [], []
        for g in geo:
            first.append(len(rows))
            for (h0, w0) in g["origins"]:
                rows.append([g["height"], g["width"], h0, w0, 0, len(rows)])
                if self.flip:
                    rows.append([g["height"], g["width"], h0, w0, 1, len(rows)])
        return geo, rows, first

    def _crops(self, image, rows):
        """Every network input of every scale, built by ONE launch: crops fp32 [len(rows),3,crop,crop]."""
        import ctypes as C
        from . import _lib
        dev = image.device
        _, _, h, w = image.shape
        crop = self.crop_size
        img = image[0].contiguous().float()
        pad = (C.c_float * 3)(*[-float(m) / float(s) for m, s in zip(self.mean, self.std)])
        wins = torch.tensor(rows, dtype=torch.int32).to(dev)
        crops = torch.empty((len(rows), 3, crop, crop), dtype=torch.float32, device=dev)
        _lib.check(_lib.load().lseg_eval_make_crops(C.c_void_p(img.data_ptr()), C.c_void_p(crops.data_ptr()),
                                                    C.c_void_p(wins.data_ptr()), len(rows), h, w, crop, pad,
                                                    C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        return crops, wins

    def _settings(self):
        return (self.base_size, self.crop_size, tuple(self.mean), tuple(self.std), self.flip, tuple(self.scales),
                self.max_batch)

    @torch.no_grad()
    def encode(self, image):
        """The image-dependent part of `self(image, label_set)`: every crop and flip of every scale through
        `net.encode_image`, in the batches the fused path uses. `self(encoded, label_set)` / `.predict(encoded,
        label_set)` then run only the label-dependent tails and the canvas / resize-add glue, and return what they return
        for the image, bit for bit. Holds one pixel embedding per network input: 36 of 62.7 MB each (2.3 GB) for a
        683x512 image at the default scales."""
        if not callable(getattr(self.net, "encode_image", None)):
            raise TypeError(f"{type(self.net).__name__} has no encode_image: the evaluator cannot store its image path")
        if self.fused is False or not image.is_cuda:
            raise TypeError("encode() runs the fused device path: fused=False and CPU images have no stored embeddings")
        batch, _, h, w = image.shape
        assert batch == 1, "only single image is supported for evaluation (additional_utils/models.py:62)"
        with torch.cuda.device(image.device):
            _, rows, _ = self._windows(h, w)
            crops, _ = self._crops(image, rows)
            embs = [self.net.encode_image(crops[i:i + self.max_batch]) for i in range(0, len(rows), self.max_batch)]
        return EncodedImage(embs, (h, w), image.device, self._settings())

    @torch.no_grad()
    def _forward_fused(self, image, label_set):
        import ctypes as C
        from . import _lib
        lib = _lib.load()
        dev = image.device
        crop = self.crop_size
        per = 2 if self.flip else 1

        def stream():
            return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

        with torch.cuda.device(dev):
            if isinstance(image, EncodedImage):
                if image.settings != self._settings():
                    raise ValueError("EncodedImage was encoded by an evaluator with other sizes, scales or batching")
                h, w = image.size
                geo, rows, first = self._windows(h, w)
                wins = torch.tensor(rows, dtype=torch.int32).to(dev)
                inputs = image.batches
            else:
                _, _, h, w = image.shape
                geo, rows, first = self._windows(h, w)
                # evaluated in fixed-size batches (the engine caches one launch plan per batch shape: per-scale batches
                # of 2, 2, 8, 12, ... would rebuild it every time)
                crops, wins = self._crops(image, rows)
                inputs = [crops[i:i + self.max_batch] for i in range(0, len(rows), self.max_batch)]
            outs = None
            direct = getattr(self.net, "supports_out", False)  # LSegNet writes straight into the output batch
            for i, x in zip(range(0, len(rows), self.max_batch), inputs):
                if direct and outs is not None:
                    self.net(x, label_set, out=outs[i:i + self.max_batch])
                    continue
                o = self.net(x, label_set).float()
                if outs is None:
                    outs = torch.empty((len(rows),) + tuple(o.shape[1:]), dtype=torch.float32, device=dev)
                outs[i:i + o.shape[0]] = o
            K = outs.shape[1]
            scores = torch.zeros((1, K, h, w), dtype=torch.float32, device=dev)
            for g, f0 in zip(geo, first):
                n_win = len(g["origins"])
                plain = wins[f0:f0 + per * n_win:per].contiguous()  # one entry per window of this scale
                canvas = torch.empty((K, g["height"], g["width"]), dtype=torch.float32, device=dev)
                _lib.check(lib.lseg_eval_canvas(C.c_void_p(outs.data_ptr()), C.c_void_p(canvas.data_ptr()),
                                                C.c_void_p(plain.data_ptr()), n_win, K, crop, g["height"], g["width"],
                                                int(self.flip), int(g["whole"]), stream()))
                _lib.check(lib.lseg_eval_resize_add(C.c_void_p(canvas.data_ptr()), C.c_void_p(scores.data_ptr()), K,
                                                    g["height"], g["width"], h, w, stream()))
        return scores

    # ---- phase 1: geometry + windows of one scale (additional_utils/models.py:67-123, no network calls) ----
    def _plan_scale(self, image, scale):
        _, _, h, w = image.shape
        crop = self.crop_size
        stride = int(crop * (2.0 / 3.0))
        long_size = int(math.ceil(self.base_size * scale))
        if h > w:
            height = long_size
            width = int(1.0 * w * long_size / h + 0.5)
            short_size = width
        else:
            width = long_size
            height = int(1.0 * h * long_size / w + 0.5)
            short_size = height
        cur_img = resize_image(image, height, width, **self.up_kwargs)
        plan = {"height": height, "width": width, "windows": []}
        if long_size <= crop:
            plan["whole"] = True
            plan["windows"].append((0, height, 0, width, pad_image(cur_img, self.mean, self.std, crop)))
            return plan
        plan["whole"] = False
        pad_img = pad_image(cur_img, self.mean, self.std, crop) if short_size < crop else cur_img
        ph, pw = pad_img.shape[2:]
        assert ph >= height and pw >= width
        plan["ph"], plan["pw"] = ph, pw
        h_grids = int(math.ceil(1.0 * (ph - crop) / stride)) + 1
        w_grids = int(math.ceil(1.0 * (pw - crop) / stride)) + 1
        for idh in range(h_grids):
            for idw in range(w_grids):
                h0, w0 = idh * stride, idw * stride
                h1, w1 = min(h0 + crop, ph), min(w0 + crop, pw)
                win = pad_image(pad_img[:, :, h0:h1, w0:w1], self.mean, self.std, crop)
                plan["windows"].append((h0, h1, w0, w1, win))
        return plan

    # ---- phase 2: every window (and its flip) through the network in large batches ----
    def _run_windows(self, windows, label_set):
        xs = []
        for win in windows:
            xs.append(win)
            if self.flip:
                xs.append(flip_image(win))
        outs = []
        for i in range(0, len(xs), self.max_batch):
            outs.append(self.net(torch.cat(xs[i:i + self.max_batch], 0), label_set).float())
        outs = torch.cat(outs, 0)
        per = 2 if self.flip else 1
        res = []
        for i in range(len(windows)):
            o = outs[per * i:per * i + 1].clone()  # module_inference, additional_utils/models.py:134-140
            if self.flip:
                o += flip_image(outs[per * i + 1:per * i + 2])
            res.append(o)
        return res

    @torch.no_grad()
    def forward(self, image, label_set=""):
        if isinstance(image, EncodedImage):
            if self.fused is False:
                raise TypeError("an EncodedImage is evaluated by the fused device path; this evaluator has fused=False")
            return self._forward_fused(image, label_set)
        batch, _, h, w = image.shape
        assert batch == 1, "only single image is supported for evaluation (additional_utils/models.py:62)"
        fused = image.is_cuda if self.fused is None else self.fused
        if fused:
            if not image.is_cuda:
                raise RuntimeError("the fused evaluator kernels need a CUDA image (fused=False runs the torch glue)")
            return self._forward_fused(image, label_set)
        plans = [self._plan_scale(image, s) for s in self.scales]
        windows = [win[4] for p in plans for win in p["windows"]]
        outs = self._run_windows(windows, label_set)
        nclass = outs[0].shape[1]
        scores = image.new_zeros((batch, nclass, h, w), dtype=torch.float32)
        k = 0
        for p in plans:  # phase 3: the reference's accumulation order, on the precomputed window outputs
            height, width = p["height"], p["width"]
            if p["whole"]:
                outputs = outs[k][:, :, 0:height, 0:width]
                k += 1
            else:
                outputs = image.new_zeros((batch, nclass, p["ph"], p["pw"]), dtype=torch.float32)
                count_norm = image.new_zeros((batch, 1, p["ph"], p["pw"]), dtype=torch.float32)
                for (h0, h1, w0, w1, _) in p["windows"]:
                    outputs[:, :, h0:h1, w0:w1] += outs[k][:, :, 0:h1 - h0, 0:w1 - w0]
                    count_norm[:, :, h0:h1, w0:w1] += 1
                    k += 1
                assert (count_norm == 0).sum() == 0
                outputs = outputs / count_norm
                outputs = outputs[:, :, :height, :width]
            scores += resize_image(outputs, h, w, **self.up_kwargs)
        return scores

    __call__ = forward

    @torch.no_grad()
    def predict(self, image, label_set=""):
        """torch.max(scores, 1)[1] (test_lseg.py:397)."""
        return torch.max(self.forward(image, label_set), 1)[1]

    def num_forwards(self, image):
        """(network forwards the reference would issue, crop-sized images we batch) for this image size."""
        h, w = image.shape[2:]
        n = sum(len(self._geometry(h, w, s)["origins"]) for s in self.scales)
        return (n * (2 if self.flip else 1), n * (2 if self.flip else 1))


class EncodedImage:
    """`MultiScaleEvaluator.encode(image)`: the pixel embeddings of every network input of one image (one
    PixelEmbedding per batch of the fused path), the image size and the evaluator settings they were made with."""

    def __init__(self, batches, size, device, settings):
        self.batches = batches
        self.size = tuple(size)
        self.device = device
        self.settings = settings
