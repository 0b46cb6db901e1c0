"""Measures the three ways a JPEG frame can reach the model's input tensor, on one GPU, alternating in one process:
(a) PIL decode + upload + device transform, (b) nvJPEG (torchvision.io.decode_jpeg) + device transform, (c) the exact
decoder (host entropy stage + mega_jpeg_decode_batch) + device transform, on seeded synthetic 720p JPEGs (4:2:0,
quality 75 and 90) made in memory. Also: host entropy-decode time per image (host clock), bytes copied to the device,
time of the two kernels per image from CUDA events over many launches, single and in batches of 23, next to the
floors bytes / HBM bandwidth. Prints one JSON line; fails without a GPU.
Usage: python tools/bench_jpeg_decode.py [--images 16] [--rounds 5]"""
import argparse
import ctypes
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "mega.pytorch_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def frames(n, quality):
    from PIL import Image
    out = []
    for s in range(n):
        g = np.random.default_rng(1000 * quality + s)
        base = g.integers(0, 256, (92, 162, 3), dtype=np.uint8)
        img = np.kron(base, np.ones((8, 8, 1), dtype=np.uint8))[:720, :1280]
        img = np.clip(img.astype(np.int16) + g.integers(0, 24, (720, 1280, 3), dtype=np.int16) - 12, 0, 255).astype(np.uint8)
        buf = io.BytesIO()
        Image.fromarray(img, "RGB").save(buf, "JPEG", quality=quality, subsampling=2)
        out.append(buf.getvalue())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_jpeg_decode needs a GPU"
    from PIL import Image
    from mega_core import _lib
    from mega_core.data import transforms as T
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                   text=True).strip().splitlines()[0]
    tr = T.DeviceTestTransform(600, 1000, [102.9801, 115.9465, 122.7717], [1.0, 1.0, 1.0], True)
    result = {"card": card, "host_cpus": os.cpu_count(), "images": args.images, "size": "1280x720 4:2:0"}
    for quality in (75, 90):
        data = frames(args.images, quality)
        res = {"mean_file_bytes": int(np.mean([len(d) for d in data]))}

        def run_pil():
            for d in data:
                tr(Image.open(io.BytesIO(d)).convert("RGB"))

        def run_nvjpeg():
            for d in data:
                tr(T.decode_jpeg(d))

        def run_exact_single():
            for d in data:
                tr(T.EncodedImage(d))

        def run_exact_batch():
            for img in T.decode_jpeg_exact(data):
                tr(img)

        paths = {"pil": run_pil, "nvjpeg": run_nvjpeg, "exact_single": run_exact_single, "exact_batch": run_exact_batch}
        times = {k: [] for k in paths}
        for r in range(args.rounds + 1):                            # round 0 warms every path up
            for k, fn in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if r:
                    times[k].append((time.perf_counter() - t0) / len(data))
        res["end_to_end_images_per_s"] = {k: round(1.0 / float(np.median(v)), 1) for k, v in times.items()}
        res["end_to_end_ms_spread"] = {k: [round(1e3 * min(v), 3), round(1e3 * max(v), 3)] for k, v in times.items()}
        # host stage alone, 1 / 2 / 4 threads
        info = _lib.JpegInfo()
        _lib.lib.mega_jpeg_probe(data[0], len(data[0]), ctypes.byref(info))
        bufs = [np.zeros((info.total_blocks, 64), np.int16) for _ in data]

        def entropy(i):
            f = _lib.JpegInfo()
            assert _lib.lib.mega_jpeg_entropy_decode(data[i], len(data[i]), ctypes.byref(f), bufs[i].ctypes.data, info.total_blocks) == 0

        import concurrent.futures
        host = {}
        for threads in (1, 2, 4):
            with concurrent.futures.ThreadPoolExecutor(threads) as pool:
                list(pool.map(entropy, range(len(data))))
                t0 = time.perf_counter()
                for _ in range(args.rounds):
                    list(pool.map(entropy, range(len(data))))
                host[str(threads)] = round(1e3 * (time.perf_counter() - t0) / (args.rounds * len(data)), 3)
        res["host_entropy_ms_per_image_by_threads"] = host
        res["h2d_bytes_per_image"] = int(info.total_blocks) * 128 + ctypes.sizeof(_lib.JpegDesc)
        # the two kernels: CUDA events around repeated launches of the device stage alone
        for n in (1, 23):
            batch = (data * 2)[:n]
            infos = (_lib.JpegInfo * n)()
            coef = np.zeros((n * info.total_blocks, 64), np.int16)
            for i, d in enumerate(batch):
                f = _lib.JpegInfo()
                _lib.lib.mega_jpeg_entropy_decode(d, len(d), ctypes.byref(f), coef[i * info.total_blocks:].ctypes.data, info.total_blocks)
                infos[i] = f
            descs = (_lib.JpegDesc * n)()
            totals = (_lib.c_ll * 3)()
            _lib.check(_lib.lib.mega_jpeg_plan_batch(infos, n, descs, totals))
            d_desc = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
            d_coef = torch.from_numpy(coef).cuda()
            planes = torch.empty(totals[0] * 64, dtype=torch.uint8, device="cuda")
            out = torch.empty(totals[2], dtype=torch.uint8, device="cuda")
            launch = lambda: _lib.check(_lib.lib.mega_jpeg_decode_batch(  # noqa: E731
                ctypes.addressof(descs), _lib.ptr(d_desc), n, _lib.ptr(d_coef), _lib.ptr(planes), planes.numel(),
                _lib.ptr(out), out.numel(), _lib.stream_ptr()))
            for _ in range(10):
                launch()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 200
            e0.record()
            for _ in range(reps):
                launch()
            e1.record()
            torch.cuda.synchronize()
            us = 1e3 * e0.elapsed_time(e1) / reps
            pixels = sum(d.width * d.height for d in descs)
            # IDCT: 2 B of coefficient in, 1 B of sample out per sample; colour: every sample in, 3 B per pixel out
            moved = totals[0] * 64 * (2 + 1) + totals[0] * 64 + 3 * pixels
            res["device_stage_us_batch_%d" % n] = {"both_kernels": round(us, 2), "per_image": round(us / n, 2),
                                                   "floor_us_at_3.35TB/s": round(moved / 3.35e6, 2)}
        result["q%d" % quality] = res
    print(json.dumps(result))


if __name__ == "__main__":
    main()
