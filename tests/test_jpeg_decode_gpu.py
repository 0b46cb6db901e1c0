"""GPU checks of the exact JPEG decoder (csrc/jpeg_decode.cu through mega_core.data.transforms.decode_jpeg_exact): the
matrix of tests/test_jpeg_decode_cpu.py on the device, single images and one mixed batch of 23, equal to
PIL.Image.open(...).convert("RGB") bit for bit; the tensor after DeviceTestTransform equal to the reference pipeline;
the same under a non-default current stream with the pinned staging buffer reused from call to call; and a MEGA
video through make_data_loader and the detector with MODEL.B200.JPEG_DECODE = "device" against "pil": identical
detections."""
import io
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import image_oracle  # noqa: E402

pytestmark = pytest.mark.gpu
MEAN, STD = [102.9801, 115.9465, 122.7717], [1.0, 1.0, 1.0]


def frame(seed, h, w, saturated=False):
    g = np.random.default_rng(seed)
    if saturated:
        return (g.integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)
    base = g.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3), dtype=np.uint8)
    img = np.kron(base, np.ones((8, 8, 1), dtype=np.uint8))[:h, :w]
    return np.clip(img.astype(np.int16) + g.integers(0, 40, (h, w, 3), dtype=np.int16) - 20, 0, 255).astype(np.uint8)


def encode(img, sub, quality, **kw):
    buf = io.BytesIO()
    if sub == "L":
        Image.fromarray(img[..., 0]).save(buf, "JPEG", quality=quality, **kw)
    else:
        Image.fromarray(img, "RGB").save(buf, "JPEG", quality=quality, subsampling=sub, **kw)
    return buf.getvalue()


def pil_pixels(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def matrix():
    out = []
    for h, w in [(16, 16), (17, 23), (8, 8), (1, 1), (53, 37), (250, 333), (3, 5), (2, 4)]:
        for si, sub in enumerate((0, 1, 2, "L")):
            for qi, q in enumerate((30, 75, 95, 100)):
                kw = ({}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1})[(si + qi + h) % 3]
                out.append(encode(frame(h * w + q, h, w, saturated=(si + qi) % 3 == 1), sub, q, **kw))
    for sub in (2, 1, 0, "L"):
        out.append(encode(frame(7, 720, 1280), sub, 90))
    return out


def test_device_decode_equals_pil_single_and_batched():
    from mega_core.data import transforms as T
    before = T.decode_jpeg_exact.fallbacks
    cases = matrix()
    for data in cases:
        out = T.decode_jpeg_exact(data)
        assert out.is_cuda and out.dtype == torch.uint8
        assert np.array_equal(out.permute(1, 2, 0).cpu().numpy(), pil_pixels(data))
    batch = cases[9:29] + cases[-3:]                               # 23 frames: mixed sizes and samplings, 720p among them
    outs = T.decode_jpeg_exact(batch)
    assert len(outs) == 23
    for out, data in zip(outs, batch):
        assert np.array_equal(out.permute(1, 2, 0).cpu().numpy(), pil_pixels(data))
    assert T.decode_jpeg_exact.fallbacks == before
    tr = T.DeviceTestTransform(600, 1000, MEAN, STD, True)
    for data in (cases[-4], cases[-3], cases[21]):
        ref = image_oracle.reference_pipeline(pil_pixels(data), 600, 1000, MEAN, STD, True)
        out, _ = tr(T.EncodedImage(data))
        assert torch.equal(out.cpu(), ref)


def test_device_decode_on_a_side_stream_reuses_its_staging_buffer():
    from mega_core.data import transforms as T
    cases = [encode(frame(s, 360, 640), 2, 85) for s in range(6)]
    refs = [pil_pixels(d) for d in cases]
    side = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(side):
        for data in cases:                                           # back to back: each call overwrites the pinned buffer
            outs.append(T.decode_jpeg_exact(data))
        outs.append(T.decode_jpeg_exact(cases))
    side.synchronize()
    for out, ref in zip(outs[:6], refs):
        assert np.array_equal(out.permute(1, 2, 0).cpu().numpy(), ref)
    for out, ref in zip(outs[6], refs):
        assert np.array_equal(out.permute(1, 2, 0).cpu().numpy(), ref)


def test_mega_video_detections_are_identical_with_device_decoding(cuda_dev, tmp_path):
    """MODEL.B200.JPEG_DECODE as the config key exposes it: make_data_loader (VIDMEGADataset reading bytes, one decode
    batch per item), the detector's own look-ahead reads of frame 0, the tiny MEGA R-101 body in the strict mode. The
    decoded frames are bit-equal, so the detections are."""
    from mega_core.b200 import synth
    from mega_core.config import cfg as base
    from mega_core.config.paths_catalog import DatasetCatalog
    from mega_core.data import make_data_loader
    from mega_core.data import transforms as T
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from test_datasets_cpu import make_tree
    make_tree(str(tmp_path), videos=(("val/vidA", 16, 160, 96), ("val/vidB", 9, 144, 96)))

    class Catalog(DatasetCatalog):
        DATA_DIR = str(tmp_path)

    sd = synth.make_state_dict("mega_r101_tiny", seed=3)
    before = T.decode_jpeg_exact.fallbacks
    results = {}
    for mode in ("pil", "device"):
        cfg = base.clone()
        cfg.merge_from_dict({"DATASETS": {"TEST": ("VID_val_videos",)}, "TEST": {"IMS_PER_BATCH": 1},
                             "MODEL": {"VID": {"METHOD": "mega"}, "B200": {"JPEG_DECODE": mode}},
                             "INPUT": {"MIN_SIZE_TEST": 96, "MAX_SIZE_TEST": 160}, "DATALOADER": {"NUM_WORKERS": 0}})
        np.random.seed(0)
        (loader,) = make_data_loader(cfg, is_train=False, dataset_catalog=Catalog)
        assert loader.dataset.transforms.jpeg_decode == mode
        model = build_detection_model_from_state_dict(sd, method="mega", device=cuda_dev, precision="fp32x3")
        dets, inputs = [], []
        with torch.no_grad():
            for images, _, _ in loader:
                inputs.append(images["cur"].tensors.clone())
                dets.append(model(images)[0].to("cpu"))
        results[mode] = (dets, inputs)
    assert T.decode_jpeg_exact.fallbacks == before
    assert len(results["pil"][0]) == 25 and sum(len(d) for d in results["pil"][0]) > 0
    for a, b in zip(results["pil"][1], results["device"][1]):
        assert torch.equal(a, b)
    for a, b in zip(*(results[m][0] for m in ("pil", "device"))):
        assert torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("scores"), b.get_field("scores"))
        assert torch.equal(a.get_field("labels"), b.get_field("labels"))
