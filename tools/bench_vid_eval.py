"""Time VID detection evaluation on a seeded workload shaped like ImageNet VID val: 555 videos, 176,126 frames, 300
detections per frame (scores >= 0.001), 30 classes, 1-3 GT per frame with motion IoUs spread over the three ranges.

  * host: eval_detection_vid with the four motion ranges (all / fast / medium / slow), as do_vid_evaluation runs them
    with --motion-specific; on the first --host-frames frames (the host path is linear in the frames; the per-frame
    time is reported with the extrapolation to the whole set);
  * device: the same four ranges in one pass of csrc/vid_eval.cu -- kernel time (CUDA events around mega_vid_eval,
    inputs already on the device) and end to end (packing, copies, kernels, AP sums on the host) on all frames, with
    the predictions resized in the kernel;
  * the per-image host work that stays in do_vid_evaluation either way: BoxList.resize (host path) and building the
    GT BoxList (the synthetic stand-in for dataset.get_groundtruth, which parses an XML file on a real dataset).
On the first --check-frames frames the device APs are checked against the host evaluator with stable_ties=True (bit for
bit); the difference to the host's default tie order is reported as max |dAP|. Prints one JSON line; GPU only.

usage: python tools/bench_vid_eval.py [--frames 176126] [--videos 555] [--dets 300] [--host-frames 4000]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mega.pytorch_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def workload(frames, videos, dets, classes=30, seed=0):
    """-> (preds in a 600 x 1000 input size, gts, image sizes, motion lists); one class per video for its GT"""
    from mega_core.structures.bounding_box import BoxList
    g = np.random.default_rng(seed)
    sizes = [(500, 375), (1280, 720), (640, 360), (960, 540)]
    vid_len = np.full(videos, frames // videos)
    vid_len[:frames - vid_len.sum()] += 1
    vid_of = np.repeat(np.arange(videos), vid_len)
    n_gt = g.integers(1, 4, frames)
    gt_tot = int(n_gt.sum())
    vsize = np.array([sizes[v % len(sizes)] for v in range(videos)], np.float32)
    wh = vsize[vid_of]                                           # [F, 2]
    gw = np.repeat(wh, n_gt, 0)
    x1 = g.uniform(0, 0.6, gt_tot) * gw[:, 0]
    y1 = g.uniform(0, 0.6, gt_tot) * gw[:, 1]
    gt = np.stack([x1, y1, x1 + g.uniform(0.1, 0.4, gt_tot) * gw[:, 0],
                   y1 + g.uniform(0.1, 0.4, gt_tot) * gw[:, 1]], 1).round().astype(np.float32)
    vcls = g.integers(1, classes + 1, (videos, 3))
    gl = vcls[np.repeat(vid_of, n_gt), np.concatenate([np.arange(k) for k in n_gt])]
    motion = g.choice([0.5, 0.65, 0.75, 0.85, 0.92, 0.97], gt_tot)
    # detections: 1/4 jittered copies of the frame's GT, the rest clutter; in the 600 x 1000 network input size
    p = frames * dets
    first_gt = np.concatenate([[0], np.cumsum(n_gt)[:-1]])
    img = np.repeat(np.arange(frames), dets)
    src = first_gt[img] + (g.integers(0, 1 << 30, p) % n_gt[img])
    near = g.random(p) < 0.25
    scale_in = np.minimum(600.0 / wh.min(1), 1000.0 / wh.max(1)).astype(np.float32)
    iw = np.repeat(wh, dets, 0)
    clutter_x = g.uniform(0, 0.8, p) * iw[:, 0]
    clutter_y = g.uniform(0, 0.8, p) * iw[:, 1]
    clutter = np.stack([clutter_x, clutter_y, clutter_x + g.uniform(0.05, 0.2, p) * iw[:, 0],
                        clutter_y + g.uniform(0.05, 0.2, p) * iw[:, 1]], 1)
    boxes = np.where(near[:, None], gt[src] + g.normal(0, 8, (p, 4)), clutter)
    boxes = (boxes * np.repeat(scale_in, dets)[:, None]).astype(np.float32)
    labels = np.where(near & (g.random(p) < 0.8), gl[src], g.integers(1, classes + 1, p)).astype(np.int64)
    scores = (0.001 + 0.999 * g.random(p) ** np.where(near, 0.3, 3.0)).astype(np.float32)
    order = np.lexsort((-scores, labels, img))                   # class-major inside a frame, as the engines return them
    boxes, labels, scores = torch.from_numpy(boxes[order]), torch.from_numpy(labels[order]), torch.from_numpy(scores[order])
    gtt, glt = torch.from_numpy(gt), torch.from_numpy(gl.astype(np.int64))
    preds, gts, img_sizes, motions = [], [], [], []
    for f, (b, l, s) in enumerate(zip(boxes.split(dets), labels.split(dets), scores.split(dets))):
        w, h = int(wh[f, 0]), int(wh[f, 1])
        pr = BoxList(b, (int(round(w * scale_in[f])), int(round(h * scale_in[f]))), mode="xyxy")
        pr.add_field("scores", s)
        pr.add_field("labels", l)
        preds.append(pr)
        img_sizes.append((w, h))
    off = 0
    for f in range(frames):
        k = int(n_gt[f])
        gts.append((gtt[off:off + k], glt[off:off + k], img_sizes[f]))
        motions.append(motion[off:off + k].tolist())
        off += k
    return preds, gts, img_sizes, motions


def make_gt(entry):
    from mega_core.structures.bounding_box import BoxList
    b, l, size = entry
    gt = BoxList(b, size, mode="xyxy")
    gt.add_field("labels", l)
    return gt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=176126)
    ap.add_argument("--videos", type=int, default=555)
    ap.add_argument("--dets", type=int, default=300)
    ap.add_argument("--host-frames", type=int, default=4000)
    ap.add_argument("--check-frames", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vid_eval needs a GPU"
    from mega_core.b200 import ops
    from mega_core.data.datasets.evaluation.vid.vid_eval import _VidEvalInputs, eval_detection_vid
    ranges = [[0.0, 1.0], [0.0, 0.7], [0.7, 0.9], [0.9, 1.0]]
    dev = torch.device("cuda", 0)
    t0 = time.perf_counter()
    preds, gt_src, sizes, motion = workload(args.frames, args.videos, args.dets)
    gen_s = time.perf_counter() - t0
    # per-image host work that stays in do_vid_evaluation
    t0 = time.perf_counter()
    gts = [make_gt(e) for e in gt_src]
    gt_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    resized = [p.resize(s) for p, s in zip(preds, sizes)]
    resize_s = time.perf_counter() - t0
    # host path, 4 ranges, on the first host-frames frames
    hf = min(args.host_frames, args.frames)
    t0 = time.perf_counter()
    host = eval_detection_vid(resized[:hf], gts[:hf], 0.5, ranges, True, motion_ious=motion[:hf])
    host_s = time.perf_counter() - t0
    sub = eval_detection_vid(preds[:hf], gts[:hf], 0.5, ranges, True, motion_ious=motion[:hf], device=True,
                             image_sizes=sizes[:hf])
    tie_dap = max(float(np.nanmax(np.abs(host[r]["ap"] - sub[r]["ap"]))) for r in host)
    cf = min(args.check_frames, hf)
    stable = eval_detection_vid(resized[:cf], gts[:cf], 0.5, ranges, True, motion_ious=motion[:cf], stable_ties=True)
    dev_cf = eval_detection_vid(preds[:cf], gts[:cf], 0.5, ranges, True, motion_ious=motion[:cf], device=True,
                                image_sizes=sizes[:cf])
    same = all(np.array_equal(stable[r]["ap"], dev_cf[r]["ap"], equal_nan=True) for r in stable)
    # device path end to end, all frames
    e2e = []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = eval_detection_vid(preds, gts, 0.5, ranges, True, motion_ious=motion, device=True, image_sizes=sizes)
        e2e.append(time.perf_counter() - t0)
    # kernel time: mega_vid_eval alone on inputs already on the device
    x = _VidEvalInputs(preds, gts, motion, ranges, sizes, pin=True)
    buf = x.host.to(dev)
    nr = len(x.ranges)
    stats = torch.empty(x.stats_count(), dtype=torch.int64, device=dev)
    steps = torch.empty(nr, 3, x.num_steps, dtype=torch.float64, device=dev)
    curves = torch.empty(2, nr, x.p_tot, dtype=torch.float64, device=dev)
    run = lambda: ops.vid_eval(*[x.view(buf, i) for i in range(9)], x.num_classes, x.ranges, 0.5,   # noqa: E731
                               x.view(buf, 9), x.num_steps, curves[0], curves[1], stats, steps)
    run()
    torch.cuda.synchronize()
    kern = []
    for _ in range(args.repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        kern.append(a.elapsed_time(b) / 1e3)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out = {"gpu": smi[0] if smi else None, "frames": args.frames, "videos": args.videos, "dets_per_frame": args.dets,
           "detections": x.p_tot, "gt": x.g_tot, "classes": x.num_classes - 1, "ranges": nr,
           "workload_gen_s": round(gen_s, 2),
           "host_frames": hf, "host_4ranges_s": round(host_s, 3),
           "host_4ranges_ms_per_frame": round(1e3 * host_s / hf, 4),
           "host_4ranges_extrapolated_s": round(host_s / hf * args.frames, 1),
           "check_frames": cf, "device_equals_host_stable_ties": bool(same),
           "max_abs_dap_vs_host_default_ties": tie_dap,
           "device_kernel_s": [round(v, 4) for v in kern], "device_e2e_s": [round(v, 3) for v in e2e],
           "resize_s": round(resize_s, 2), "resize_ms_per_frame": round(1e3 * resize_s / args.frames, 4),
           "gt_boxlist_s": round(gt_s, 2),
           "map": {r: round(float(res[r]["map"]), 6) for r in res}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
