"""Generate tests/golden/rpn_only.pt from the UNMODIFIED reference -- TEST INFRASTRUCTURE.

1. Proposal recall: the reference's eval_proposals_vid (data/datasets/evaluation/vid/vid_eval.py:72-119) on seeded
   synthetic cases. The fixture keeps the inputs, the recall and the per-image greedy-round overlaps the function
   concatenates (read through an instrumented `torch` namespace of the loaded file whose `cat` records its argument;
   the evaluator's code is not touched). The cases hold objectness ties, images with more proposals than `limit`,
   images with fewer proposals than GT boxes, images without GT or without proposals, and proposals with exactly equal
   IoU to a GT box (duplicates, and boxes shifted by the same amount to either side).
2. The state_dict layout (key -> shape) of the reference detectors built with MODEL.RPN_ONLY True for
   configs/vid_R_50_C4_1x.yaml, configs/DFF/vid_R_101_C4_DFF_1x.yaml and configs/FGFA/vid_R_101_C4_FGFA_1x.yaml.

Usage: python oracle/make_golden_rpn_only.py   (needs the reference checkout; a fresh process, because it imports the
reference's `mega_core`)."""
import contextlib
import importlib.util
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402

W, H = 640, 360
CONFIGS = {"base_r50": "configs/vid_R_50_C4_1x.yaml", "dff_r101": "configs/DFF/vid_R_101_C4_DFF_1x.yaml",
           "fgfa_r101": "configs/FGFA/vid_R_101_C4_FGFA_1x.yaml"}


def _gt(g, n):
    x1, y1 = g.integers(0, W - 120, n), g.integers(0, H - 100, n)
    return np.stack([x1, y1, x1 + g.integers(15, 110, n), y1 + g.integers(15, 90, n)], 1).astype(np.float32)


def _image(g, n_props, n_gt, score_decimals=1, tie_shifts=True):
    """proposals around the GT boxes (jittered, duplicated, and shifted by +-d to either side -- equal IoU) plus clutter;
    objectness rounded to `score_decimals` so that ties occur"""
    gt = _gt(g, n_gt) if n_gt else np.zeros((0, 4), np.float32)
    props = []
    for k in range(n_gt):
        b = gt[k]
        if tie_shifts and g.random() < 0.7:
            d = float(g.integers(1, 6))
            props += [b + [-d, 0, -d, 0], b + [d, 0, d, 0]]           # same IoU with b
        if g.random() < 0.5:
            props += [b.copy(), b.copy()]                             # duplicates
        props += [b + g.normal(0, 4, 4).astype(np.float32).round(1) for _ in range(int(g.integers(0, 4)))]
    while len(props) < n_props:
        a, c = g.uniform(0, W - 60), g.uniform(0, H - 60)
        props.append(np.asarray([a, c, a + g.uniform(8, 200), c + g.uniform(8, 150)], np.float32))
    props = np.asarray(props[:n_props], np.float32).reshape(-1, 4)
    order = g.permutation(len(props))
    props = props[order]
    scores = np.round(g.uniform(0, 1, len(props)), score_decimals).astype(np.float32)
    return props, scores, gt


def synth_cases():
    cases = []
    g = np.random.default_rng(11)
    cases.append({"name": "ties", "iou_thresh": 0.5, "limit": 300,
                  "images": [_image(g, int(g.integers(5, 60)), int(g.integers(1, 6))) for _ in range(40)]})
    g = np.random.default_rng(12)
    cases.append({"name": "limit_bites", "iou_thresh": 0.5, "limit": 300,
                  "images": [_image(g, int(g.integers(301, 700)), int(g.integers(1, 12)), 2) for _ in range(12)]})
    g = np.random.default_rng(13)
    cases.append({"name": "fewer_proposals_than_gt", "iou_thresh": 0.5, "limit": 300,
                  "images": [_image(g, int(g.integers(1, 4)), int(g.integers(4, 9)), 1, False) for _ in range(15)]})
    g = np.random.default_rng(14)
    imgs = []
    for i in range(24):
        kind = i % 4               # 0: no GT, 1: no proposals, 2: neither, 3: both
        imgs.append(_image(g, 0 if kind in (1, 2) else int(g.integers(1, 40)), 0 if kind in (0, 2) else int(g.integers(1, 5))))
    cases.append({"name": "empty_images", "iou_thresh": 0.5, "limit": 300, "images": imgs})
    g = np.random.default_rng(15)
    cases.append({"name": "small_limit_thresh_0.7", "iou_thresh": 0.7, "limit": 7,
                  "images": [_image(g, int(g.integers(3, 30)), int(g.integers(1, 10))) for _ in range(30)]})
    return cases


def run_recall(cases):
    ref_import.setup()
    spec = importlib.util.spec_from_file_location(
        "ref_vid_eval", os.path.join(ref_import.REFERENCE, "mega_core", "data", "datasets", "evaluation", "vid", "vid_eval.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    from mega_core.structures.bounding_box import BoxList
    seen = []

    def cat(tensors, *a, **k):
        seen.append([t.clone() for t in tensors])
        return torch.cat(tensors, *a, **k)

    ref.torch = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    ref.torch.cat = cat
    out = []
    for case in cases:
        preds, gts = [], []
        for props, scores, gt in case["images"]:
            p = BoxList(torch.from_numpy(props), (W, H), mode="xyxy")
            p.add_field("objectness", torch.from_numpy(scores))
            preds.append(p)
            gts.append(BoxList(torch.from_numpy(gt).reshape(-1, 4), (W, H), mode="xyxy"))
        seen.clear()
        with contextlib.redirect_stdout(io.StringIO()):
            res = ref.eval_proposals_vid(preds, gts, iou_thresh=case["iou_thresh"], limit=case["limit"])
        assert len(seen) == 1
        out.append({"name": case["name"], "iou_thresh": case["iou_thresh"], "limit": case["limit"],
                    "images": [{"boxes": torch.from_numpy(p), "objectness": torch.from_numpy(s), "gt": torch.from_numpy(gt)}
                               for p, s, gt in case["images"]],
                    "recall": res["recall"].clone(), "gt_overlaps": seen[0]})
        print("  %-24s %3d images  recall %.6f  (%d images with GT and proposals)" % (
            case["name"], len(case["images"]), res["recall"].item(), len(seen[0])))
    return out


def state_dict_layouts():
    from mega_core.modeling.detector import build_detection_model
    layouts = {}
    for name, path in CONFIGS.items():
        cfg = ref_import.build_cfg(path, ["MODEL.RPN_ONLY", True])
        model = build_detection_model(cfg)
        layouts[name] = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        assert not any(k.startswith("roi_heads") for k in layouts[name])
        print("  %-10s %s: %d entries" % (name, path, len(layouts[name])))
    return layouts


def main():
    torch.manual_seed(0)
    gold = {"recall_cases": run_recall(synth_cases()), "state_dicts": state_dict_layouts(), "image_size": (W, H)}
    path = os.path.join(os.path.dirname(HERE), "tests", "golden", "rpn_only.pt")
    torch.save(gold, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
