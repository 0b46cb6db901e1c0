"""Device time of Seq-NMS (csrc/seq_nms.cu) on a seeded synthetic workload shaped like the ImageNet VID val set: 555
videos with lengths from a fixed seeded distribution, 300 detections per frame, 30 classes, most scores just above the
0.001 test threshold (the junk-heavy case: many short chains, many iterations per (video, class)). Launches run as
mega_core.engine.seq_nms runs them (whole videos, at most FRAMES_PER_LAUNCH frames per launch) with the inputs resident
on the device; CUDA events around all launches, after a warm-up pass. Also times the NumPy oracle
(tests/seq_nms_oracle.py) on a stated subset and checks the device result on that subset against it bit for bit.
Prints the card name and power limit of the run.

    python tools/bench_seq_nms.py [--videos 555] [--repeats 3] [--oracle-videos 2] [--oracle-frames 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mega.pytorch_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_DET, N_CLASSES = 300, 30


def video_lengths(n, seed=0):
    """lengths of n videos: log-normal around ~300 frames, 6..2000 (the val set: 555 videos, 176,126 frames)"""
    rng = np.random.default_rng(seed)
    return np.clip(np.round(rng.lognormal(np.log(250), 0.75, n)), 6, 2000).astype(int)


def make_video_packed(rng, T, W=1000, H=600):
    """[T, 300] boxes / scores / labels of one video, class-major per frame: 8 objects drifting through the video with 6
    noisy boxes each (scores 0.05..1), the other 252 detections junk (uniform boxes, scores 0.001 + Exp(0.01))."""
    n_obj, k = 8, 6
    cls = rng.integers(1, N_CLASSES + 1, n_obj)
    p0 = rng.uniform([0, 0], [W * 0.7, H * 0.7], (n_obj, 2))
    wh = rng.uniform(30, 300, (n_obj, 2))
    vel = rng.normal(0, 6, (n_obj, 2))
    pos = p0[None] + vel[None] * np.arange(1, T + 1)[:, None, None]                       # [T, n_obj, 2]
    base = np.concatenate([pos, pos + wh[None]], -1)                                      # [T, n_obj, 4]
    obj = base[:, :, None, :] + rng.normal(0, 0.06, (T, n_obj, k, 4)) * np.concatenate([wh, wh], -1)[None, :, None, :]
    obj_s = np.clip(rng.beta(5, 2, (T, n_obj, k)) * rng.uniform(0.3, 1.0, (T, n_obj, 1)), 1e-3, 1)
    n_junk = N_DET - n_obj * k
    xy = rng.uniform([0, 0], [W, H], (T, n_junk, 2))
    junk = np.concatenate([xy, xy + rng.uniform(8, 400, (T, n_junk, 2))], -1)
    boxes = np.concatenate([obj.reshape(T, n_obj * k, 4), junk], 1).astype(np.float32)
    boxes[..., 2:] = np.maximum(boxes[..., 2:], boxes[..., :2])
    scores = np.concatenate([obj_s.reshape(T, -1), 1e-3 + rng.exponential(0.01, (T, n_junk))], 1).astype(np.float32)
    labels = np.concatenate([np.repeat(cls, k)[None].repeat(T, 0), rng.integers(1, N_CLASSES + 1, (T, n_junk))], 1)
    o = np.argsort(labels, 1, kind="stable")
    take = lambda a: np.take_along_axis(a, o[..., None] if a.ndim == 3 else o, 1)        # noqa: E731
    return take(boxes), take(scores), take(labels).astype(np.int32)


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        power = "unknown (%s)" % e
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=555)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-videos", type=int, default=2)
    ap.add_argument("--oracle-frames", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_seq_nms.py times the CUDA kernels: it needs a GPU"
    from mega_core.b200 import ops
    from mega_core.engine import seq_nms as sn
    import seq_nms_oracle as so
    dev = torch.device("cuda")
    lengths = video_lengths(args.videos)
    rng = np.random.default_rng(1)
    t0 = time.time()
    vids = [make_video_packed(rng, int(T)) for T in lengths]
    gen_s = time.time() - t0
    # launches of whole videos, <= FRAMES_PER_LAUNCH frames each, inputs on the device
    chunks, v0 = [], 0
    while v0 < len(vids):
        v1, n = v0, 0
        while v1 < len(vids) and (v1 == v0 or n + lengths[v1] <= sn.FRAMES_PER_LAUNCH):
            n += lengths[v1]
            v1 += 1
        part = vids[v0:v1]
        chunks.append((torch.from_numpy(np.concatenate([p[0] for p in part])).to(dev),
                       torch.from_numpy(np.concatenate([p[1] for p in part])).to(dev),
                       torch.from_numpy(np.concatenate([p[2] for p in part])).to(dev),
                       torch.full((n,), N_DET, dtype=torch.int32, device=dev),
                       torch.tensor(np.cumsum([0] + list(lengths[v0:v1])), dtype=torch.int32, device=dev)))
        v0 = v1

    def run():
        return [ops.seq_nms(*c, N_CLASSES + 1) for c in chunks]

    run()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        outs = run()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    kept = sum(int(k.sum()) for _, k in outs)
    # the oracle on a subset: the first --oracle-frames frames of the first --oracle-videos videos, one launch
    sub = [[(v[0][t], v[1][t], v[2][t].astype(np.int64)) for t in range(min(args.oracle_frames, len(v[0])))]
           for v in vids[:args.oracle_videos]]
    boxes, scores, labels, counts, offsets, nc = so.pack(sub)
    dargs = [torch.from_numpy(x).to(dev) for x in (boxes, scores, labels, counts, offsets)]
    ops.seq_nms(*dargs, nc)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    ns, kp = ops.seq_nms(*dargs, nc)
    b.record()
    torch.cuda.synchronize()
    sub_dev_ms = a.elapsed_time(b)
    t0 = time.time()
    want = [so.seq_nms_video(v) for v in sub]
    oracle_s = time.time() - t0
    got = so.unpack(sub, kp.cpu().numpy(), ns.cpu().numpy())
    identical = all(np.array_equal(kg, kw) and np.array_equal(sg.view(np.uint32), sw.view(np.uint32))
                    for gv, wv in zip(got, want) for (kg, sg), (kw, sw) in zip(gv, wv))
    name, power = card()
    print(json.dumps({
        "card": name, "power_limit": power,
        "workload": {"videos": len(vids), "frames": int(lengths.sum()), "detections_per_frame": N_DET,
                     "classes": N_CLASSES, "launches": len(chunks), "frames_per_launch_max": sn.FRAMES_PER_LAUNCH,
                     "kept": kept, "junk_per_frame": N_DET - 48},
        "device_ms": {"best": min(times), "all": times},
        "oracle_subset": {"videos": len(sub), "frames_each": [len(v) for v in sub], "oracle_s": oracle_s,
                          "device_ms": sub_dev_ms, "bit_identical": identical},
        "host_generation_s": gen_s,
    }))


if __name__ == "__main__":
    main()
