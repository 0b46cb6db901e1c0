"""Writes tests/golden/jpeg_decode.pt: a handful of tiny JPEG byte strings with the pixels Pillow (12.2.0,
libjpeg-turbo) decodes them to, so that the decoder's result stays pinned wherever another Pillow is installed.
Usage: python oracle/make_golden_jpeg.py"""
import io
import os

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frame(seed, h, w):
    g = np.random.default_rng(seed)
    base = g.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3), dtype=np.uint8)
    img = np.kron(base, np.ones((8, 8, 1), dtype=np.uint8))[:h, :w]
    return np.clip(img.astype(np.int16) + g.integers(0, 40, (h, w, 3), dtype=np.int16) - 20, 0, 255).astype(np.uint8)


def main():
    cases = []
    for seed, (h, w, sub, q, kw) in enumerate([(17, 23, 2, 75, {}), (16, 16, 0, 95, {}), (37, 53, 1, 30, {}),
                                               (24, 40, "L", 90, {}), (33, 21, 2, 100, {"restart_marker_blocks": 2}),
                                               (9, 5, 2, 85, {"optimize": True})]):
        img = frame(seed, h, w)
        buf = io.BytesIO()
        if sub == "L":
            Image.fromarray(img[..., 0]).save(buf, "JPEG", quality=q, **kw)
        else:
            Image.fromarray(img, "RGB").save(buf, "JPEG", quality=q, subsampling=sub, **kw)
        data = buf.getvalue()
        rgb = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        cases.append({"jpeg": data, "rgb": torch.from_numpy(rgb.copy())})
    import PIL
    torch.save({"pillow": PIL.__version__, "cases": cases}, os.path.join(ROOT, "tests", "golden", "jpeg_decode.pt"))
    print("wrote %d cases, %d bytes of JPEG" % (len(cases), sum(len(c["jpeg"]) for c in cases)))


if __name__ == "__main__":
    main()
