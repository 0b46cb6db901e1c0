"""CPU checks of the exact JPEG decoder (SURVEY.md section 8f row 1; oracle/jpeg_oracle.py, csrc/jpeg_host.cuh,
csrc/jpeg_decode.cuh, mega_core/data/transforms/jpeg.py):
  1. the numpy restatement of the decode equals PIL.Image.open(...).convert("RGB") bit for bit;
  2. the library's host entropy decoder (the real libmega_b200.so; it needs no driver) gives the restatement's
     coefficients and descriptors;
  3. the kernels' bodies, built for the host and driven by the product's own decode_jpeg_exact, give PIL's pixels, and
     through DeviceTestTransform the reference pipeline's tensor;
  4. unsupported and damaged streams end in a status under an address/undefined-behaviour-sanitised build of the host
     decoder, the wrapper falls back to PIL and counts it, and whatever damaged stream the decoder does accept gives
     Pillow's pixels;
  5. MODEL.B200.JPEG_DECODE = "device" leaves every dataset class's items, and the detector's look-ahead frames,
     bit-identical to "pil";
  6. a committed fixture pins the pixels independently of the Pillow installed here.
The GPU test (tests/test_jpeg_decode_gpu.py) repeats 3 on the device."""
import ctypes
import hashlib
import io
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import image_oracle  # noqa: E402
import jpeg_oracle as jo  # noqa: E402

MEAN, STD = [102.9801, 115.9465, 122.7717], [1.0, 1.0, 1.0]
SIZES = [(16, 16), (17, 23), (8, 8), (1, 1), (53, 37), (250, 333), (3, 5), (2, 4)]
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "jpeg_decode.pt"), weights_only=False)


def frame(seed, h, w, kind="blocks"):
    g = np.random.default_rng(seed)
    if kind == "saturated":                                    # overshoots 0..255 after the IDCT
        return (g.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)
    if kind == "contrast":
        img = np.zeros((h, w, 3), np.uint8)
        img[::2, ::3] = 255
        img[:, w // 2:, 0] = 255
        return img
    base = g.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3), dtype=np.uint8)
    img = np.kron(base, np.ones((8, 8, 1), dtype=np.uint8))[:h, :w]
    return np.clip(img.astype(np.int16) + g.integers(0, 40, (h, w, 3), dtype=np.int16) - 20, 0, 255).astype(np.uint8)


def encode(img, sub, quality, **kw):
    pil = Image.fromarray(img[..., 0]) if sub == "L" else Image.fromarray(img, "RGB")
    if sub != "L":
        kw["subsampling"] = sub
    from PIL import ImageFile
    buf = io.BytesIO()
    block, ImageFile.MAXBLOCK = ImageFile.MAXBLOCK, 1 << 24    # room for an optimised pass over a large, noisy frame
    try:
        pil.save(buf, "JPEG", quality=quality, **kw)
    finally:
        ImageFile.MAXBLOCK = block
    return buf.getvalue()


def pil_pixels(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def matrix(sizes=SIZES, big=True):
    """(label, bytes): subsampling x quality x content x encoder options over the sizes, plus one 720p frame each"""
    out = []
    for h, w in sizes:
        for si, sub in enumerate((0, 1, 2, "L")):
            for qi, q in enumerate((30, 75, 95, 100)):
                kind = ("blocks", "saturated", "contrast")[(si + qi) % 3]
                kw = ({}, {"optimize": True}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1})[(si * 4 + qi + h) % 4]
                out.append(("%dx%d-%s-q%d-%s-%s" % (h, w, sub, q, kind, "".join(kw)), encode(frame(h * w + q, h, w, kind), sub, q, **kw)))
    if big:
        for sub in (2, 1, 0, "L"):
            out.append(("720x1280-%s" % sub, encode(frame(7, 720, 1280), sub, 90)))
    return out


def test_numpy_restatement_equals_pil():
    for label, data in matrix():
        assert np.array_equal(jo.decode(data), pil_pixels(data)), label


def test_optimised_tables_reach_codes_longer_than_the_fast_lookup():
    """a large noisy frame with optimize=True carries Huffman codes of 11..16 bits: the host decoder's slow path"""
    from mega_core import _lib
    data = encode(frame(11, 250, 333), 2, 95, optimize=True)
    i, longest = 2, 0
    while data[i + 1] != 0xDA:
        ln = data[i + 2] << 8 | data[i + 3]
        if data[i + 1] == 0xC4:
            j = i + 4
            while j < i + 2 + ln:
                counts = data[j + 1:j + 17]
                longest = max(longest, max(k + 1 for k in range(16) if counts[k]))
                j += 17 + sum(counts)
        i += 2 + ln
    assert longest > 10
    ref = jo.parse(data)
    info = _lib.JpegInfo()
    coef = np.zeros((sum(c["bw"] * c["bh"] for c in ref["comps"]), 64), np.int16)
    assert _lib.lib.mega_jpeg_entropy_decode(data, len(data), ctypes.byref(info), coef.ctypes.data, len(coef)) == 0
    assert np.array_equal(coef, np.concatenate([c["coef"] for c in ref["comps"]]))
    assert np.array_equal(jo.pixels(ref), pil_pixels(data))


def test_golden_fixture_pins_the_pixels(host_decoder):
    live = all(np.array_equal(pil_pixels(c["jpeg"]), c["rgb"].numpy()) for c in GOLD["cases"])
    for c in GOLD["cases"]:
        assert np.array_equal(jo.decode(c["jpeg"]), c["rgb"].numpy())
        assert torch.equal(host_decoder.decode_jpeg_exact(c["jpeg"], device="cpu").permute(1, 2, 0), c["rgb"])
    if not live:
        pytest.skip("the Pillow installed here decodes the fixture differently from Pillow %s: live comparisons "
                    "in this module compare against another decoder" % GOLD["pillow"])


def test_host_entropy_decoder_equals_restatement():
    from mega_core import _lib
    for label, data in matrix(big=False) + matrix(sizes=[], big=True)[:1]:
        ref = jo.parse(data)
        info = _lib.JpegInfo()
        assert _lib.lib.mega_jpeg_probe(data, len(data), ctypes.byref(info)) == 0, label
        assert info.total_blocks == sum(c["bw"] * c["bh"] for c in ref["comps"])
        coef = np.full((info.total_blocks, 64), 7, np.int16)
        info2 = _lib.JpegInfo()
        assert _lib.lib.mega_jpeg_entropy_decode(data, len(data), ctypes.byref(info2), coef.ctypes.data, info.total_blocks) == 0
        assert (info2.width, info2.height, info2.ncomp, info2.hmax, info2.vmax, info2.color, info2.mcus_x, info2.mcus_y) == tuple(
            ref[k] for k in ("width", "height", "ncomp", "hmax", "vmax", "color", "mcus_x", "mcus_y")), label
        for i, c in enumerate(ref["comps"]):
            assert (info2.comp_dw[i], info2.comp_dh[i], info2.comp_bw[i], info2.comp_bh[i]) == (c["dw"], c["dh"], c["bw"], c["bh"])
            assert np.array_equal(np.array(info2.quant[i][:]), c["quant"])
        assert np.array_equal(coef, np.concatenate([c["coef"] for c in ref["comps"]])), label
        assert _lib.lib.mega_jpeg_entropy_decode(data, len(data), ctypes.byref(info2), coef.ctypes.data, info.total_blocks - 1) == 1


def _build(flags, tag):
    """g++ build of tests/native/jpeg_decode_host.cpp, cached in the temp directory under the digest of its sources"""
    src = os.path.join(ROOT, "tests", "native", "jpeg_decode_host.cpp")
    deps = [src] + [os.path.join(ROOT, "mega.pytorch_b200", "csrc", n) for n in ("jpeg_decode.cuh", "jpeg_host.cuh")] + [
        os.path.join(ROOT, "include", "mega_b200.h")]
    digest = hashlib.sha256(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
    path = os.path.join(tempfile.gettempdir(), "mega_jpeg_decode_host_%s_%s_%d.so" % (tag, digest, os.getuid()))
    if not os.path.exists(path):
        tmp = path + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17"] + flags + [
            "-I", os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"), "-o", tmp, src])
        os.replace(tmp, path)
    return path


@pytest.fixture
def host_decoder(monkeypatch):
    """the product's decode path with the device stage replaced by the host build of the kernels' bodies"""
    from mega_core import _lib
    from mega_core.data import transforms as T
    host = ctypes.CDLL(_build([], "plain"))
    fn, real = host.mega_jpeg_decode_batch, _lib.lib.mega_jpeg_decode_batch
    fn.argtypes, fn.restype = real.argtypes, real.restype
    monkeypatch.setattr(_lib.lib, "mega_jpeg_decode_batch", fn)
    so = os.path.join(tempfile.gettempdir(), "mega_image_ops_host_%d.so" % os.getuid())
    if not os.path.exists(so):
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-I",
                               os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               "-o", tmp, os.path.join(ROOT, "tests", "native", "image_ops_host.cpp")])
        os.replace(tmp, so)
    fn, real = ctypes.CDLL(so).mega_image_transform_u8, _lib.lib.mega_image_transform_u8
    fn.argtypes, fn.restype = real.argtypes, real.restype
    monkeypatch.setattr(_lib.lib, "mega_image_transform_u8", fn)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    monkeypatch.setattr(_lib, "require_cuda", lambda *a: None)
    monkeypatch.setattr(T.decode_jpeg_exact, "fallbacks", 0)
    return T


def test_kernel_bodies_give_pil_pixels_and_the_reference_tensor(host_decoder):
    T = host_decoder
    cases = matrix()
    for label, data in cases:
        out = T.decode_jpeg_exact(data, device="cpu")
        assert out.dtype == torch.uint8 and np.array_equal(out.permute(1, 2, 0).numpy(), pil_pixels(data)), label
    batch = [d for _, d in cases[5:28]]                        # 23 images of mixed sizes and samplings: one batch
    for out, data in zip(T.decode_jpeg_exact(batch, device="cpu"), batch):
        assert np.array_equal(out.permute(1, 2, 0).numpy(), pil_pixels(data))
    assert T.decode_jpeg_exact.fallbacks == 0
    tr = T.DeviceTestTransform(60, 100, MEAN, STD, True, device="cpu")
    for label, data in cases[20:24] + cases[-2:]:
        ref = image_oracle.reference_pipeline(pil_pixels(data), 60, 100, MEAN, STD, True)
        out, _ = tr(T.EncodedImage(data))
        assert torch.equal(out, ref), label


def test_unsupported_and_damaged_streams(host_decoder):
    T = host_decoder
    img = frame(3, 40, 56)
    good = encode(img, 2, 80, restart_marker_blocks=2)
    prog = encode(img, 2, 80, progressive=True)
    buf = io.BytesIO()
    Image.fromarray(img, "RGB").convert("CMYK").save(buf, "JPEG", quality=80)
    cmyk = buf.getvalue()
    damaged = [good[:k] for k in range(0, len(good), 8)]
    g = np.random.default_rng(0)
    for _ in range(150):
        b = bytearray(good)
        b[int(g.integers(2, len(b)))] = int(g.integers(0, 256))
        damaged.append(bytes(b))
    # the sanitised build runs in a child process (the sanitiser runtime must be loaded first); a finding aborts it
    child = ("import ctypes, sys, pickle\n"
             "lib = ctypes.CDLL(sys.argv[1]); streams = pickle.load(open(sys.argv[2], 'rb'))\n"
             "out = []\n"
             "for d in streams:\n"
             "    info = ctypes.create_string_buffer(1024)\n"
             "    coef = ctypes.create_string_buffer(128 * 128)\n"
             "    a = lib.mega_jpeg_probe(d, ctypes.c_longlong(len(d)), info)\n"
             "    b = lib.mega_jpeg_entropy_decode(d, ctypes.c_longlong(len(d)), info, coef, ctypes.c_longlong(128))\n"
             "    out.append((a, b))\n"
             "pickle.dump(out, open(sys.argv[3], 'wb'))\n")
    import pickle
    so = _build(["-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"], "asan")
    with tempfile.TemporaryDirectory() as tmp:
        pickle.dump([prog, cmyk, good] + damaged, open(os.path.join(tmp, "in.pkl"), "wb"))
        libasan = subprocess.check_output(["g++", "-print-file-name=libasan.so"], text=True).strip()
        env = dict(os.environ, LD_PRELOAD=libasan, ASAN_OPTIONS="detect_leaks=0")
        res = subprocess.run([sys.executable, "-c", child, so, os.path.join(tmp, "in.pkl"), os.path.join(tmp, "out.pkl")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-3000:]
        status = pickle.load(open(os.path.join(tmp, "out.pkl"), "rb"))
    assert status[0] == (16, 16) and status[1] == (16, 16) and status[2] == (0, 0)
    assert all(b in (0, 16, 17) for _, b in status) and sum(b == 17 for _, b in status) > len(damaged) // 2
    assert all(b == 17 for (_, b), d in zip(status[3:], damaged) if len(d) < len(good) - 2)      # every truncation
    # every damaged stream the decoder accepts must give Pillow's pixels (and Pillow must accept it too): single-byte
    # corruptions of four files, headers and entropy data alike
    files = [good, encode(frame(2, 33, 47), 1, 90), encode(frame(3, 24, 24), 0, 95, optimize=True), encode(frame(4, 40, 40), "L", 75)]
    accepted = 0
    for fi, f in enumerate(files):
        g = np.random.default_rng(100 + fi)
        for _ in range(700):
            b = bytearray(f)
            pos = int(g.integers(2, len(b)))
            b[pos] = int(g.integers(0, 256))
            b = bytes(b)
            before = T.decode_jpeg_exact.fallbacks
            try:
                out = T.decode_jpeg_exact(b, device="cpu")
            except Exception:
                assert T.decode_jpeg_exact.fallbacks == before + 1      # PIL's exception, from the fallback
                continue
            if T.decode_jpeg_exact.fallbacks == before:
                accepted += 1
                assert np.array_equal(out.permute(1, 2, 0).numpy(), pil_pixels(b)), (fi, pos, b[pos])
    assert accepted > 1000
    T.decode_jpeg_exact.fallbacks = 0
    # the wrapper: PIL's pixels or PIL's exception, counted
    for data in (prog, cmyk):
        assert np.array_equal(T.decode_jpeg_exact(data, device="cpu").permute(1, 2, 0).numpy(), pil_pixels(data))
    assert T.decode_jpeg_exact.fallbacks == 2
    outs = T.decode_jpeg_exact([good, prog, good], device="cpu")
    assert T.decode_jpeg_exact.fallbacks == 3 and all(np.array_equal(o.permute(1, 2, 0).numpy(), pil_pixels(good)) for o in outs[::2])
    with pytest.raises(Exception):
        T.decode_jpeg_exact(good[:len(good) // 2], device="cpu")
    assert T.decode_jpeg_exact.fallbacks == 4


def test_datasets_and_lookahead_are_identical_with_device_decoding(host_decoder, tmp_path):
    T = host_decoder
    from test_datasets_cpu import make_tree
    from mega_core.data import datasets as D
    from mega_core.modeling.detector.generalized_rcnn import GeneralizedRCNNMEGA
    make_tree(str(tmp_path))
    ils = os.path.join(str(tmp_path), "ILSVRC2015")
    items = {}
    for mode in ("pil", "device"):
        tr = T.DeviceTestTransform(60, 100, MEAN, STD, True, device="cpu", jpeg_decode=mode)
        args = dict(image_set="VID_val_videos", data_dir=str(tmp_path), img_dir=os.path.join(ils, "Data", "VID"),
                    anno_path=os.path.join(ils, "Annotations", "VID"),
                    img_index=os.path.join(ils, "ImageSets", "VID_val_videos.txt"), transforms=tr, is_train=False)
        if mode == "pil":                                       # today's path reaches none of the new calls
            tr.decode_batch = lambda *a: pytest.fail("decode_batch on the PIL path")
        for cls in (D.VIDDataset, D.VIDRDNDataset, D.VIDFGFADataset, D.VIDMEGADataset, D.VIDDFFDataset):
            np.random.seed(0)
            ds = cls(**args)
            items[mode, cls.__name__] = [ds[i] for i in (0, 5, 13, 14, 22)]
        det = GeneralizedRCNNMEGA.__new__(GeneralizedRCNNMEGA)
        det.end_id, det.seg_len = 0, 14
        infos = {"pattern": "val/vidA/%06d", "img_dir": os.path.join(ils, "Data", "VID", "%s.JPEG"), "transforms": tr}
        items[mode, "lookahead"] = det._read_lookahead(infos, 5)

    def same(a, b):
        if torch.is_tensor(a):
            return torch.equal(a, b)
        if isinstance(a, dict):
            return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a if k != "transforms")
        if isinstance(a, (list, tuple)):
            return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
        if hasattr(a, "bbox"):
            return torch.equal(a.bbox, b.bbox) and a.size == b.size
        return a == b

    for (mode, name), got in items.items():
        if mode == "device":
            assert same(items["pil", name], got), name
