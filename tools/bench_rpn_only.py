"""MODEL.RPN_ONLY on the GPU, timed with CUDA events (prints one JSON line, with the card and its power limit).

1. Frames per second of the single-frame and FGFA R-101-C4 detectors (synthetic weights) on 600 x 1000 frames, the
   full detector against its RPN-only configuration, in the strict (fp32x3) and throughput (f16) arithmetic. FGFA is
   timed in its steady state (one new frame per step, FlowNetS over the 19-frame window).
2. Proposal recall of a seeded workload the size of ImageNet-VID val (synth.synthetic_proposal_dataset: 176,126 frames
   of up to 300 proposals and up to 4 GT boxes, plus 64 frames of up to 1000 proposals and 200 GT boxes): the device
   kernel (host-to-device copy, launch and copy back, as eval_proposals_vid runs it) against a torch restatement of the
   reference's per-image, per-round loop (vid_eval.py:72-119) on the CPU, which is timed on the first --ref-images
   frames and reported per frame.

Usage: python tools/bench_rpn_only.py [--iters N] [--ref-images N] [--out FILE]
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


def card():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        power = "unknown (%s)" % e
    return name, power


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def detector_fps(arch, precision, rpn_only, iters, dev, h=600, w=1000):
    from mega_core.b200 import engine, synth
    sd = synth.make_state_dict(arch, seed=1)
    if rpn_only:
        sd = {k: v for k, v in sd.items() if not k.startswith("roi_heads.")}
    frames = [synth.synthetic_frame(i, h, w).to(dev) for i in range(24)]
    if arch.startswith("base"):
        eng = engine.BaseEngine(sd, engine.EngineConfig(precision=precision, rpn_only=rpn_only), device=dev)
        ms = timed(lambda: eng.forward(frames[0], w, h), iters)
    else:
        eng = engine.FgfaEngine(sd, engine.EngineConfig(all_frame_interval=19, key_frame_location=9, precision=precision,
                                                        rpn_only=rpn_only), device=dev)
        eng.start_video(frames[0], frames[1:10], w, h)
        step = [10]

        def fn():
            eng.step(frames[step[0] % len(frames)], w, h)
            step[0] += 1
        ms = timed(fn, iters)
    del eng
    torch.cuda.empty_cache()
    return 1000.0 / ms


def reference_loop(pb, ps, gb, po, go, n, iou_thresh=0.5, limit=300):
    """vid_eval.py:72-119 restated with the reference's torch calls, on the CPU, images [0, n)"""
    hits, num_pos = 0, 0
    for i in range(n):
        b = torch.from_numpy(pb[po[i]:po[i + 1]])
        s = torch.from_numpy(ps[po[i]:po[i + 1]])
        g = torch.from_numpy(gb[go[i]:go[i + 1]])
        b = b[s.sort(descending=True)[1]][:limit]
        num_pos += len(g)
        if len(g) == 0 or len(b) == 0:
            continue
        a1 = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
        a2 = (g[:, 2] - g[:, 0] + 1) * (g[:, 3] - g[:, 1] + 1)
        wh = (torch.min(b[:, None, 2:], g[:, 2:]) - torch.max(b[:, None, :2], g[:, :2]) + 1).clamp(min=0)
        inter = wh[:, :, 0] * wh[:, :, 1]
        overlaps = inter / (a1[:, None] + a2 - inter)
        o = torch.zeros(len(g))
        for j in range(min(len(b), len(g))):
            max_overlaps, argmax_overlaps = overlaps.max(dim=0)
            gt_ovr, gt_ind = max_overlaps.max(dim=0)
            box_ind = argmax_overlaps[gt_ind]
            o[j] = overlaps[box_ind, gt_ind]
            overlaps[box_ind, :] = -1
            overlaps[:, gt_ind] = -1
        hits += int((o >= iou_thresh).sum())
    return hits, num_pos


def recall_timing(dev, ref_images):
    from mega_core.b200 import ops, synth
    pb, ps, gb, po, go = synth.synthetic_proposal_dataset(seed=5)
    n = len(po) - 1
    host = [torch.from_numpy(a).pin_memory() for a in (pb, ps, gb, po, go)]
    mp, mg = int(np.diff(po).max()), int(np.diff(go).max())
    ov = torch.empty(len(gb), device=dev)
    stats = torch.empty(3, dtype=torch.int64, device=dev)
    res = {}

    def run():
        d = [t.to(dev, non_blocking=True) for t in host]
        ops.proposal_recall(d[0], d[1], d[3], d[2], d[4], mp, mg, 300, 0.5, ov, stats)
        res["stats"] = stats.cpu()

    ms = timed(run, 5, warmup=1)
    kernel_only = [t.to(dev) for t in host]
    ms_kernel = timed(lambda: ops.proposal_recall(kernel_only[0], kernel_only[1], kernel_only[3], kernel_only[2],
                                                  kernel_only[4], mp, mg, 300, 0.5, ov, stats), 5, warmup=1)
    t0 = time.perf_counter()
    ref_hits, ref_pos = reference_loop(pb, ps, gb, po, go, ref_images)
    ref_s = time.perf_counter() - t0
    ops.proposal_recall(*[t.to(dev) for t in (torch.from_numpy(pb[:po[ref_images]]), torch.from_numpy(ps[:po[ref_images]]),
                                              torch.from_numpy(po[:ref_images + 1]), torch.from_numpy(gb[:go[ref_images]]),
                                              torch.from_numpy(go[:ref_images + 1]))],
                        int(np.diff(po[:ref_images + 1]).max()), int(np.diff(go[:ref_images + 1]).max()), 300, 0.5,
                        ov, stats)
    sub = stats.cpu().tolist()
    hits, num_pos, rejected = res["stats"].tolist()
    return {"images": n, "proposals": int(po[-1]), "gt": int(go[-1]), "recall": hits / num_pos, "rejected": rejected,
            "device_ms_with_copies": ms, "device_ms_kernel": ms_kernel,
            "torch_loop_images": ref_images, "torch_loop_ms_per_image": 1000 * ref_s / ref_images,
            "torch_loop_projected_s_for_all": ref_s / ref_images * n,
            "subset_counts_equal": [sub[0], sub[1]] == [ref_hits, ref_pos]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-images", type=int, default=2000)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_rpn_only measures on the GPU"
    dev = torch.device("cuda:0")
    name, power = card()
    out = {"gpu": name, "power_limit": power, "fps_600x1000": {}}
    for arch in ("base_r101", "fgfa_r101"):
        for precision in ("fp32x3", "f16"):
            full = detector_fps(arch, precision, False, args.iters, dev)
            rpn = detector_fps(arch, precision, True, args.iters, dev)
            out["fps_600x1000"]["%s_%s" % (arch, precision)] = {"full": round(full, 2), "rpn_only": round(rpn, 2),
                                                                 "speedup": round(rpn / full, 3)}
    out["proposal_recall"] = recall_timing(dev, args.ref_images)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
