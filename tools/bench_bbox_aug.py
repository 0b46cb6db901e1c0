"""Test-time box augmentation on the GPU, timed with CUDA events (prints one JSON line, with the card and its power
limit).

1. Per-image time of the single-frame R-101-C4 detector (synthetic weights) on a 600 x 1000 image through
   BaseEngine.forward_bbox_aug, for two plans: H_FLIP only (2 passes), and the reference's TTA configuration
   (test_time_aug/e2e_mask_rcnn_R_50_FPN_1x.yaml: H_FLIP, SCALES 400..1200, MAX_SIZE 2000, SCALE_H_FLIP: 20 passes on
   a 600-pixel image with MIN_SIZE_TEST 600 -- identity, its flip, then 9 scales and their flips; the 1200 scale runs
   a 1200 x 2000 image). Input transforms included; the plain single-pass forward is timed for comparison.
2. The merge alone, on the raw per-pass tensors of 18 passes x 300 proposals x 31 classes: the collect + merge
   kernels against the reference's host loop of filter_results (box_head/inference.py:108-149: threshold, 30 _C.nms
   calls with a host sync each, kthvalue on the CPU), run here on the same device tensors with this package's _C.nms.

Usage: python tools/bench_bbox_aug.py [--iters N] [--precision f16|tf32|fp32x3]
"""
import argparse
import json
import os
import subprocess
import sys

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


def timed(fn, iters, warmup=2):
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


def filter_results_host_loop(boxes, scores, num_classes, score_thresh, nms, max_det):
    """box_head/inference.py:108-149 as the reference runs it, on device tensors: boxes [N, C*4], scores [N, C]"""
    from mega_core import _C
    inds_all = scores > score_thresh
    res_b, res_s, res_l = [], [], []
    for j in range(1, num_classes):
        inds = inds_all[:, j].nonzero().squeeze(1)
        s_j, b_j = scores[inds, j], boxes[inds, j * 4:(j + 1) * 4]
        keep = _C.nms(b_j, s_j, nms)
        res_b.append(b_j[keep])
        res_s.append(s_j[keep])
        res_l.append(torch.full((keep.numel(),), j, dtype=torch.int64, device=boxes.device))
    b, s, l = torch.cat(res_b), torch.cat(res_s), torch.cat(res_l)
    n = b.shape[0]
    if n > max_det > 0:
        thr, _ = torch.kthvalue(s.cpu(), n - max_det + 1)
        keep = torch.nonzero(s >= thr.item()).squeeze(1)
        b, s, l = b[keep], s[keep], l[keep]
    return b, s, l


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--precision", default="f16")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_bbox_aug measures on the GPU"
    from mega_core.b200 import engine, ops, synth
    from mega_core.data.transforms import DeviceTestTransform
    from mega_core.engine.bbox_aug import aug_plan
    dev = torch.device("cuda:0")
    name, power = card()
    mean, std = [102.9801, 115.9465, 122.7717], [1.0, 1.0, 1.0]
    eng = engine.BaseEngine(synth.make_state_dict("base_r101", seed=0), engine.EngineConfig(precision=args.precision),
                            device=dev)
    g = torch.Generator().manual_seed(0)
    image = torch.randint(0, 256, (600, 1000, 3), generator=g, dtype=torch.uint8).to(dev)
    transforms = {}

    def run(plan):
        def passes():
            for p in plan:
                key = (p.min_size, p.max_size, p.hflip)
                if key not in transforms:
                    transforms[key] = DeviceTestTransform(p.min_size, p.max_size, mean, std, True, device=dev,
                                                          hflip=p.hflip)
                yield transforms[key](image)[0][None], p.size[0], p.size[1], p.hflip
        return eng.forward_bbox_aug(passes(), len(plan), plan[0].size[0], plan[0].size[1])

    out = {"card": name, "power_limit": power, "precision": args.precision, "image": "600x1000"}
    plain = DeviceTestTransform(600, 1000, mean, std, True, device=dev)
    out["single_pass_ms"] = timed(lambda: eng.forward(plain(image)[0][None], 1000, 600), args.iters)
    plans = {"hflip_only": aug_plan((1000, 600), 600, 1000, True, (), 4000, False),
             "reference_tta": aug_plan((1000, 600), 600, 1000, True, tuple(range(400, 1201, 100)), 2000, True)}
    for label, plan in plans.items():
        out[label + "_passes"] = len(plan)
        out[label + "_ms_per_image"] = timed(lambda: run(plan), args.iters)

    # merge alone: 18 passes x 300 proposals x 31 classes of raw per-pass output
    A, R, C = 18, 300, 31
    logits = torch.randn(A, R, C, generator=g).mul_(2).to(dev)
    deltas = torch.randn(A, R, 4 * C, generator=g).mul_(0.5).to(dev)
    xy = torch.rand(A, R, 2, generator=g) * 900
    props = torch.cat([xy, xy + torch.rand(A, R, 2, generator=g) * 200 + 8], 2).to(dev)
    cnt = torch.full((1,), R, dtype=torch.int32, device=dev)
    ws = torch.zeros(ops.bbox_aug_workspace_bytes(A, R, C), dtype=torch.uint8, device=dev)
    cap = (C - 1) * A * R
    dets = (torch.zeros(cap, 4, device=dev), torch.zeros(cap, device=dev), torch.zeros(cap, dtype=torch.int64, device=dev),
            torch.zeros(1, dtype=torch.int32, device=dev))
    wts = (10.0, 10.0, 5.0, 5.0)

    def collect_merge():
        for a in range(A):
            ops.bbox_aug_collect(logits[a], deltas[a], props[a], cnt, C, a, A, 1000, 600, a & 1, 1.0, 1.0, 0.001, wts, ws)
        ops.bbox_aug_merge(A, R, C, 0.5, 300, ws, dets)

    collect_merge()
    torch.cuda.synchronize()
    # the same raw boxes / scores the reference's host loop would see: [A*R, C*4] / [A*R, C] from the staging
    slots = A * R * C
    nb = (16 * slots + 255) // 256 * 256
    raw_b = ws[:16 * slots].view(torch.float32).view(C, A * R, 4).permute(1, 0, 2).reshape(A * R, C * 4).contiguous()
    raw_s = ws[nb:nb + 4 * slots].view(torch.float32).view(C, A * R).t().contiguous()
    out["collect_merge_ms"] = timed(collect_merge, 50)
    # collect rewrites the candidate flags the merge consumes, so the merge alone is timed as collect+merge minus collect
    out["collect_ms"] = timed(lambda: [ops.bbox_aug_collect(logits[a], deltas[a], props[a], cnt, C, a, A, 1000, 600,
                                                            a & 1, 1.0, 1.0, 0.001, wts, ws) for a in range(A)], 50)
    out["merge_ms"] = out["collect_merge_ms"] - out["collect_ms"]
    out["reference_host_loop_filter_results_ms"] = timed(
        lambda: filter_results_host_loop(raw_b, raw_s, C, 0.001, 0.5, 300), 10)
    collect_merge()
    n = int(dets[3].item())
    rb, _, rl = filter_results_host_loop(raw_b, raw_s, C, 0.001, 0.5, 300)
    out["merge_dets"], out["host_loop_dets"] = n, int(rb.shape[0])
    out["labels_per_class_equal"] = bool(torch.equal(torch.bincount(dets[2][:n], minlength=C),
                                                     torch.bincount(rl, minlength=C)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
