"""Device-side test-time transform: decoded uint8 RGB frame -> the tensor the reference's CPU pipeline produces
(data/transforms/transforms.py:27-63 Resize, :117-119 ToTensor, :122-135 Normalize), bit for bit.

The host part below is the float arithmetic of Pillow's `precompute_coeffs` / `normalize_coeffs_8bpc`
(src/libImaging/Resample.c, Pillow 12.2 -- third-party code the reference reaches through
torchvision.transforms.functional.resize and does not pin): Python floats are C doubles, so the tables are the ones
Pillow computes; the per-pixel integer work runs in `mega_image_transform_u8` (csrc/image_ops.cu). Tables depend only on
(source size, output size) and are cached on the device."""
import math

import numpy as np
import torch

from ... import _lib
from .jpeg import EncodedImage, decode_jpeg_exact

PRECISION_BITS = 32 - 8 - 2


def get_size(image_size, min_size, max_size):
    """Resize.get_size (data/transforms/transforms.py:36-56) for a single test-time min_size: (w, h) -> (oh, ow)"""
    w, h = image_size
    size = min_size
    if max_size is not None:
        lo, hi = float(min((w, h))), float(max((w, h)))
        if hi / lo * size > max_size:
            size = int(round(max_size * lo / hi))
    if (w <= h and w == size) or (h <= w and h == size):
        return (h, w)
    if w < h:
        return (int(size * h / w), size)
    return (size, int(size * w / h))


def resample_tables(in_size, out_size):
    """bilinear (support 1.0) coefficient tables of one axis: (bounds int32 [2*out], kk int32 [out*ksize], ksize)"""
    scale = filterscale = float(in_size) / out_size          # box = (0, in_size)
    if filterscale < 1.0:
        filterscale = 1.0
    support = 1.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros(2 * out_size, dtype=np.int32)
    kk = np.zeros(out_size * ksize, dtype=np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        xmin = int(center - support + 0.5)                   # C cast: truncation (the operand is >= -0.5 + ...)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        ws = []
        ww = 0.0
        for x in range(xmax):
            a = (x + xmin - center + 0.5) * ss
            if a < 0.0:
                a = -a
            wgt = 1.0 - a if a < 1.0 else 0.0
            ws.append(wgt)
            ww += wgt
        for x in range(xmax):
            k = ws[x] / ww if ww != 0.0 else ws[x]
            kk[xx * ksize + x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        bounds[2 * xx], bounds[2 * xx + 1] = xmin, xmax
    return bounds, kk, ksize


def decode_jpeg(data, device="cuda"):
    """encoded JPEG bytes (bytes / uint8 tensor) -> planar uint8 RGB [3, H, W] on the device through nvJPEG
    (torchvision.io.decode_jpeg: a library decoder, like PIL's libjpeg in the reference's data loader; their IDCTs
    differ in the last bit, so pixel values are not bit-identical across decoders -- the transform after it is)"""
    import torchvision
    if not torch.is_tensor(data):
        data = torch.frombuffer(bytearray(data), dtype=torch.uint8)
    return torchvision.io.decode_jpeg(data, device=device, mode=torchvision.io.ImageReadMode.RGB)


class DeviceTestTransform(object):
    """callable with the reference's transform signature `(image, target=None) -> (tensor, target)`.
    image: PIL.Image (RGB), uint8 ndarray / tensor [H, W, 3] on the host or on the device, or a planar uint8 [3, H, W]
    tensor (what `decode_jpeg` below / torchvision.io.decode_jpeg(device="cuda") returns: nvJPEG output is consumed in
    place, no re-layout), or an `EncodedImage` (JPEG bytes, decoded on the device by `decode_jpeg_exact` to PIL's
    pixels). Returns a float32 [3, H', W'] device tensor.
    `jpeg_decode` ("pil" / "device", MODEL.B200.JPEG_DECODE) tells whoever opens the files -- the datasets and the
    detectors' look-ahead reads -- what to hand over: a decoded PIL image, or the file's bytes through `decode_batch`."""

    def __init__(self, min_size, max_size, mean, std, to_bgr255=True, device="cuda", hflip=False, jpeg_decode="pil"):
        if jpeg_decode not in ("pil", "device"):
            raise ValueError("MODEL.B200.JPEG_DECODE must be \"pil\" or \"device\", got %r" % (jpeg_decode,))
        self.jpeg_decode = jpeg_decode
        if isinstance(min_size, (list, tuple)):
            assert len(min_size) == 1, "test-time transform: a single MIN_SIZE_TEST"
            min_size = min_size[0]
        self.min_size, self.max_size = int(min_size), max_size
        self.mean = np.asarray(mean, dtype=np.float32)
        self.std = np.asarray(std, dtype=np.float32)
        self.to_bgr255 = bool(to_bgr255)
        self.hflip = bool(hflip)          # RandomHorizontalFlip(1.0) after Resize: the flipped test-time augmentation passes
        self.device = torch.device(device)
        self._tables = {}

    def _axis(self, in_size, out_size):
        key = (in_size, out_size)
        t = self._tables.get(key)
        if t is None:
            if in_size == out_size:
                t = (None, None, 0)
            else:
                b, k, ks = resample_tables(in_size, out_size)
                t = (torch.from_numpy(b).to(self.device), torch.from_numpy(k).to(self.device), ks)
            self._tables[key] = t
        return t

    def decode_batch(self, images):
        """list of EncodedImage -> list of planar uint8 [3, H, W] tensors on the device, decoded as one batch (one
        copy, two launches); an object that appears several times in the list is decoded once"""
        uniq = list({id(e): e for e in images}.values())
        decoded = dict(zip((id(e) for e in uniq), decode_jpeg_exact([e.data for e in uniq], device=self.device)))
        return [decoded[id(e)] for e in images]

    def __call__(self, image, target=None, out=None):
        if isinstance(image, EncodedImage):
            image = decode_jpeg_exact(image.data, device=self.device)
        if not torch.is_tensor(image) and hasattr(image, "convert"):         # PIL.Image
            image = np.asarray(image.convert("RGB"))
        if isinstance(image, np.ndarray):
            image = torch.from_numpy(np.array(image, copy=True))
        if image.dtype != torch.uint8 or image.dim() != 3 or 3 not in (image.shape[0], image.shape[2]):
            raise ValueError("expected a uint8 [H, W, 3] or [3, H, W] RGB image, got %s %s" % (image.dtype, tuple(image.shape)))
        src = image.to(self.device, non_blocking=True).contiguous()
        _lib.require_cuda(src)
        planar = src.shape[2] != 3                      # [3, H, W]; a [3, W, 3] strip counts as interleaved
        if planar:
            h, w = src.shape[1], src.shape[2]
            row, pix, ch = src.stride(1), 1, src.stride(0)
        else:
            h, w = src.shape[0], src.shape[1]
            row, pix, ch = src.stride(0), 3, 1
        oh, ow = get_size((w, h), self.min_size, self.max_size)
        bh, kh, ksh = self._axis(w, ow)
        bv, kv, ksv = self._axis(h, oh)
        if out is None:
            out = torch.empty(3, oh, ow, device=self.device)
        assert out.shape == (3, oh, ow) and out.dtype == torch.float32 and out.is_contiguous()
        args = (_lib.ptr(src), h, w, row, pix, ch, _lib.ptr(bh), _lib.ptr(kh), ksh, _lib.ptr(bv), _lib.ptr(kv), ksv, oh,
                ow, self.mean.ctypes.data, self.std.ctypes.data, int(self.to_bgr255))
        if self.hflip:
            _lib.check(_lib.lib.mega_image_transform_u8_ex(*args, 1, _lib.ptr(out), _lib.stream_ptr()),
                       "mega_image_transform_u8_ex")
        else:
            _lib.check(_lib.lib.mega_image_transform_u8(*args, _lib.ptr(out), _lib.stream_ptr()), "mega_image_transform_u8")
        if target is not None and hasattr(target, "resize"):
            target = target.resize((ow, oh))
        return out, target

    def __repr__(self):
        return "DeviceTestTransform(min_size=%s, max_size=%s, to_bgr255=%s, hflip=%s)" % (
            self.min_size, self.max_size, self.to_bgr255, self.hflip)
