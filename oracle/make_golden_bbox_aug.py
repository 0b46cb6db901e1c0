"""Generate tests/golden/bbox_aug_r50_240x400.pt by running the UNMODIFIED reference's test-time box augmentation
(engine/bbox_aug.py:11-68, im_detect_bbox_aug) on the CPU, with the synthetic single-frame R-50-C4 weights and one
synthetic uint8 RGB image.

Needs a checkout of the reference (ref_import.REFERENCE, overridable with MEGA_REFERENCE):
    python oracle/make_golden_bbox_aug.py

Passes: identity at MIN_SIZE_TEST 192, its horizontal flip, then scales 144 and 288 with MAX_SIZE 448, each also
flipped. On the 240 x 400 image the 144 pass has equal x / y ratios to the identity frame (the single-ratio branch of
BoxList.resize) and the 288 pass hits MAX_SIZE (269 x 448, per-axis ratios). Per pass the fixture holds the transformed
image size, the RPN proposals, the predictor's logits and deltas, and the post-processor's raw BoxList (all K x C rows,
softmax + decode + clip, before any threshold); then the merged detections filter_results returns. The image is
regenerated from its seed (mega_core.b200.synth.synthetic_image_u8; the fixture keeps a digest of its bytes), and
POST_NMS_TOP_N_TEST is 32 so that the raw rows of six passes stay small.
"""
import hashlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
GOLD = os.path.join(ROOT, "tests", "golden")

import ref_import  # noqa: E402
from make_golden import synth  # noqa: E402

H, W, IMAGE_SEED, PROPOSALS = 240, 400, 5, 32
SETTINGS = ["INPUT.MIN_SIZE_TEST", 192, "MODEL.RPN.POST_NMS_TOP_N_TEST", PROPOSALS, "TEST.BBOX_AUG.ENABLED", True, "TEST.BBOX_AUG.H_FLIP", True,
            "TEST.BBOX_AUG.SCALES", (144, 288), "TEST.BBOX_AUG.MAX_SIZE", 448, "TEST.BBOX_AUG.SCALE_H_FLIP", True]


def golden_bbox_aug():
    cfg = ref_import.build_cfg("configs/vid_R_50_C4_1x.yaml", SETTINGS)
    from mega_core.config import cfg as global_cfg           # what im_detect_bbox_aug reads
    global_cfg.merge_from_other_cfg(cfg)
    global_cfg.freeze()
    import types
    from PIL import Image
    import mega_core.engine.bbox_aug as ref_aug
    from mega_core.data import transforms as ref_T
    from mega_core.modeling.detector import build_detection_model
    # engine/bbox_aug.py:73-79 puts the package's Resize and Normalize, which return (image, target) tuples
    # (data/transforms/transforms.py:58-63, :130-135), into a torchvision Compose whose next step takes an image, so the
    # reference's TTA path raises as shipped. Only that return convention is adapted here: the same classes compute.
    first = lambda cls: (lambda *a, **k: (lambda t: (lambda img: t(img)[0]))(cls(*a, **k)))  # noqa: E731
    ref_aug.T = types.SimpleNamespace(Resize=first(ref_T.Resize), Normalize=first(ref_T.Normalize))
    im_detect_bbox_aug = ref_aug.im_detect_bbox_aug
    model = build_detection_model(cfg).eval()
    sd = synth.make_state_dict("base_r50", seed=1)
    full = dict(sd)
    full["rpn.anchor_generator.cell_anchors.0"] = model.state_dict()["rpn.anchor_generator.cell_anchors.0"]
    model.load_state_dict(full, strict=True)
    assert model.roi_heads.box.post_processor.bbox_aug_enabled

    passes = []
    pred = model.roi_heads.box.predictor
    post = model.roi_heads.box.post_processor
    orig_pred, orig_post = pred.forward, post.forward

    def pf(x):
        r = orig_pred(x)
        passes.append({"class_logits": r[0].clone(), "box_regression": r[1].clone()})
        return r

    def pp(x, boxes):
        res = orig_post(x, boxes)
        assert len(res) == 1
        passes[-1].update({"proposals": boxes[0].bbox.clone(), "size": tuple(int(v) for v in res[0].size),
                           "raw_boxes": res[0].bbox.clone(), "raw_scores": res[0].get_field("scores").clone()})
        return res

    pred.forward, post.forward = pf, pp
    img = synth.synthetic_image_u8(H, W, IMAGE_SEED)
    with torch.no_grad():
        out = im_detect_bbox_aug(model, [Image.fromarray(img.numpy())], torch.device("cpu"))[0]
    assert len(passes) == 6, len(passes)
    flips = [False, True, False, True, False, True]
    for p, f in zip(passes, flips):
        p["hflip"] = f
        print("  pass %s flip=%d proposals %d raw rows %d" % (p["size"], f, p["proposals"].shape[0], p["raw_boxes"].shape[0]))
    print("  merged detections:", out.bbox.shape[0], "image size", out.size)
    return {"arch": "base_r50", "seed": 1, "image_hw": (H, W), "image_seed": IMAGE_SEED,
            "image_sha256": hashlib.sha256(img.numpy().tobytes()).hexdigest(), "post_nms_top_n": PROPOSALS,
            "settings": SETTINGS, "min_size_test": 192,
            "max_size_test": int(cfg.INPUT.MAX_SIZE_TEST), "scales": [144, 288], "aug_max_size": 448,
            "score_thresh": float(cfg.MODEL.ROI_HEADS.SCORE_THRESH), "nms": float(cfg.MODEL.ROI_HEADS.NMS),
            "detections_per_img": int(cfg.MODEL.ROI_HEADS.DETECTIONS_PER_IMG), "num_classes": 31,
            "bbox_reg_weights": tuple(float(v) for v in cfg.MODEL.ROI_HEADS.BBOX_REG_WEIGHTS),
            "passes": passes, "size": tuple(int(v) for v in out.size), "boxes": out.bbox.clone(),
            "scores": out.get_field("scores").clone(), "labels": out.get_field("labels").clone()}


# (source (w, h), MIN_SIZE_TEST, MAX_SIZE_TEST, H_FLIP, SCALES, BBOX_AUG.MAX_SIZE, SCALE_H_FLIP)
PLAN_CASES = [((400, 240), 192, 1000, True, (144, 288), 448, True),
              ((1000, 600), 600, 1000, True, (400, 500, 600, 700, 800, 900, 1000, 1100, 1200), 2000, True),
              ((333, 500), 192, 300, False, (100, 250), 320, True),
              ((640, 480), 480, 640, True, (), 4000, False),
              ((500, 375), 300, 1000, False, (200, 600), 700, False),
              ((1280, 720), 600, 1000, True, (480, 720), 1100, True)]


def reference_plans():
    """the passes im_detect_bbox_aug makes (order, Resize.get_size, flip) for PLAN_CASES, recorded from its own control
    flow: the per-pass detectors are replaced by stubs that return an empty BoxList of the resized size"""
    from PIL import Image
    import mega_core.engine.bbox_aug as ref_aug
    from mega_core.config import cfg as global_cfg
    from mega_core.data import transforms as ref_T
    from mega_core.structures.bounding_box import BoxList
    calls = []

    def stub(hflip):
        def run(model, images, target_scale, target_max_size, device):
            oh, ow = ref_T.Resize(target_scale, target_max_size).get_size(images[0].size)
            calls.append({"min_size": target_scale, "max_size": target_max_size, "hflip": hflip, "size": (ow, oh)})
            b = BoxList(torch.zeros(0, 4), (ow, oh), mode="xyxy")
            b.add_field("scores", torch.zeros(0))
            return [b]
        return run

    ref_aug.im_detect_bbox, ref_aug.im_detect_bbox_hflip = stub(False), stub(True)
    out = []
    for size, mn, mx, hf, scales, amx, shf in PLAN_CASES:
        global_cfg.defrost()
        global_cfg.merge_from_list(["INPUT.MIN_SIZE_TEST", mn, "INPUT.MAX_SIZE_TEST", mx, "TEST.BBOX_AUG.H_FLIP", hf,
                                    "TEST.BBOX_AUG.SCALES", scales, "TEST.BBOX_AUG.MAX_SIZE", amx,
                                    "TEST.BBOX_AUG.SCALE_H_FLIP", shf])
        global_cfg.freeze()
        del calls[:]
        ref_aug.im_detect_bbox_aug(None, [Image.new("RGB", size)], torch.device("cpu"))
        out.append({"image_size": size, "min_size_test": mn, "max_size_test": mx, "h_flip": hf, "scales": scales,
                    "max_size": amx, "scale_h_flip": shf, "passes": [dict(c) for c in calls]})
        print("  plan", size, [c["size"] for c in calls])
    return out


def main():
    torch.set_num_threads(8)
    os.makedirs(GOLD, exist_ok=True)
    path = os.path.join(GOLD, "bbox_aug_r50_240x400.pt")
    gold = golden_bbox_aug()
    gold["plans"] = reference_plans()
    torch.save(gold, path)
    print("  wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
