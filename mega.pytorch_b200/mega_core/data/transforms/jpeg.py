"""`decode_jpeg_exact`: encoded JPEG bytes -> planar uint8 RGB [3, H, W] on the device with the pixels
`PIL.Image.open(...).convert("RGB")` gives (SURVEY.md section 8f row 1). The serial half of the format -- markers and
Huffman codes -- runs on the host in the library (mega_jpeg_entropy_decode; ctypes releases the GIL, so the frames of
a batch are decoded by a small thread pool); coefficients and the descriptor table cross to the device in ONE copy from
a pinned staging buffer, and two kernels finish the whole batch (mega_jpeg_decode_batch: IDCT, then chroma upsampling
+ colour conversion). A stream the library refuses (progressive, CMYK, damaged, ...) is decoded by PIL itself and
uploaded: identical pixels by definition, counted in `decode_jpeg_exact.fallbacks`.
There is no prefetch: a call decodes its own batch and returns once the device work is queued, so the host stage of
the next item overlaps the GPU only as far as the caller's loop leaves the device busy."""
import concurrent.futures
import contextlib
import ctypes
import io
import logging
import os

import numpy as np
import torch

from ... import _lib

_pool = None
_staging = {}          # device -> (pinned uint8 tensor, event recorded after the copy that last read it)


class EncodedImage(object):
    """encoded JPEG bytes on their way to DeviceTestTransform (a holder, so that `bytes` is never sniffed)"""
    __slots__ = ("data",)

    def __init__(self, data):
        self.data = bytes(data)


def _workers():
    global _pool
    if _pool is None:                              # non-daemon threads, joined by concurrent.futures at interpreter exit
        _pool = concurrent.futures.ThreadPoolExecutor(max_workers=max(1, min(4, os.cpu_count() or 1)),
                                                      thread_name_prefix="mega_jpeg")
    return _pool


def _stage(nbytes, device):
    """host staging buffer of at least nbytes, safe to overwrite: pinned and reused (grown by doubling) for a CUDA
    device, once the copy that last read it has completed"""
    if device.type != "cuda":
        return torch.empty(nbytes, dtype=torch.uint8), None
    buf, event = _staging.get(device, (None, None))
    if event is not None:
        event.synchronize()
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 2 * (buf.numel() if buf is not None else 0)), dtype=torch.uint8).pin_memory()
    event = torch.cuda.Event()
    _staging[device] = (buf, event)
    return buf, event


def _pil_pixels(data, device):
    from PIL import Image
    rgb = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
    return torch.from_numpy(np.ascontiguousarray(rgb.transpose(2, 0, 1))).to(device)


def _fallback(data, device, status):
    if decode_jpeg_exact.fallbacks == 0:
        logging.getLogger("mega_core.data").warning(
            "decode_jpeg_exact: a stream is outside the baseline subset or damaged (status %d); such frames are decoded "
            "by PIL on the host (decode_jpeg_exact.fallbacks counts them)", status)
    decode_jpeg_exact.fallbacks += 1
    return _pil_pixels(data, device)


def decode_jpeg_exact(data, device="cuda"):
    """bytes -> uint8 [3, H, W] device tensor; a list of bytes -> a list of such tensors, decoded as ONE batch (one
    host-to-device copy, two kernel launches, whatever the sizes). Work is queued on torch's current stream."""
    single = isinstance(data, (bytes, bytearray, memoryview))
    items = [bytes(d) for d in ([data] if single else data)]
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    lib = _lib.lib
    results = [None] * len(items)
    infos, live = [], []
    for i, d in enumerate(items):
        info = _lib.JpegInfo()
        st = lib.mega_jpeg_probe(d, len(d), ctypes.byref(info))
        if st != 0:
            results[i] = _fallback(d, device, st)
        else:
            infos.append(info)
            live.append(i)
    if live:
        # the stream the kernels are queued on is the current stream of the tensors' device
        with torch.cuda.device(device) if device.type == "cuda" else contextlib.nullcontext():
            _decode_live(items, live, infos, results, device)
    return results[0] if single else results


def _decode_live(items, live, infos, results, device):
    """host entropy stage of the probed streams, one upload, the two kernels; fills results[i] for i in live"""
    lib = _lib.lib
    n = len(live)
    starts = np.concatenate([[0], np.cumsum([f.total_blocks for f in infos])]).astype(np.int64)
    desc_bytes = (ctypes.sizeof(_lib.JpegDesc) * n + 63) // 64 * 64
    coef_bytes = int(starts[-1]) * 128
    stage, event = _stage(desc_bytes + coef_bytes, device)
    base = stage.data_ptr()

    def entropy(k):
        info = _lib.JpegInfo()
        d = items[live[k]]
        st = lib.mega_jpeg_entropy_decode(d, len(d), ctypes.byref(info), base + desc_bytes + int(starts[k]) * 128,
                                          infos[k].total_blocks)
        return st, info

    done = list(_workers().map(entropy, range(n))) if n > 1 else [entropy(0)]
    failed = {}
    arr = (_lib.JpegInfo * n)()
    for k, (st, info) in enumerate(done):
        if st == 0 and info.total_blocks == infos[k].total_blocks:
            arr[k] = info
        else:                                   # keeps its (unused) place in the batch; PIL supplies the pixels
            failed[k] = st
            arr[k] = infos[k]
    descs = (_lib.JpegDesc * n).from_address(base)
    totals = (_lib.c_ll * 3)()
    _lib.check(lib.mega_jpeg_plan_batch(arr, n, descs, totals), "mega_jpeg_plan_batch")
    assert totals[0] == starts[-1]
    staged = stage[:desc_bytes + coef_bytes]
    if device.type == "cuda":
        dev = torch.empty(desc_bytes + coef_bytes, dtype=torch.uint8, device=device)
        dev.copy_(staged, non_blocking=True)
        event.record()
    else:
        dev = staged
    planes = torch.empty(int(totals[0]) * 64, dtype=torch.uint8, device=device)
    out = torch.empty(int(totals[2]), dtype=torch.uint8, device=device)
    _lib.require_cuda(dev, planes, out)
    _lib.check(lib.mega_jpeg_decode_batch(base, _lib.ptr(dev), n, dev.data_ptr() + desc_bytes, _lib.ptr(planes),
                                          planes.numel(), _lib.ptr(out), out.numel(), _lib.stream_ptr()),
               "mega_jpeg_decode_batch")
    for k, i in enumerate(live):
        if k in failed:
            results[i] = _fallback(items[i], device, failed[k])
        else:
            d = descs[k]
            results[i] = out[d.out_off:d.out_off + 3 * d.width * d.height].view(3, d.height, d.width)


decode_jpeg_exact.fallbacks = 0
