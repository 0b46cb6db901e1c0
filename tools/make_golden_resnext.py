"""Generate tests/golden/mega_x101_192x320.pt and tests/golden/base_x101_192x320.pt by running the UNMODIFIED reference with
MODEL.RESNETS.NUM_GROUPS 32 / WIDTH_PER_GROUP 8 (ResNeXt-101 32x8d) on the seeded synthetic "x101" weights
(mega_core.b200.synth), and check the oracle (with grouped bottlenecks, tests/resnext_oracle.py) against it on the way.
Same protocol as oracle/make_golden.py for mega_r101_192x320.pt / base_r50_192x320.pt: only outputs are stored, plus the
reference model's parameter / buffer list, which the package's module tree must equal.

Run where the reference checkout exists:   python tools/make_golden_resnext.py
"""
import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
GOLD = os.path.join(ROOT, "tests", "golden")

import make_golden as mg  # noqa: E402
import mega_oracle as mo  # noqa: E402
import ref_import  # noqa: E402
from resnext_oracle import grouped_bottlenecks  # noqa: E402

X101_OPTS = ("MODEL.RESNETS.NUM_GROUPS", 32, "MODEL.RESNETS.WIDTH_PER_GROUP", 8)


@contextlib.contextmanager
def x101_configs():
    """every reference config built inside gets the ResNeXt-101 32x8d keys on top of its YAML"""
    saved = ref_import.build_cfg

    def build_cfg(config_file, opts=()):
        return saved(config_file, tuple(opts) + X101_OPTS)
    ref_import.build_cfg = build_cfg
    try:
        yield
    finally:
        ref_import.build_cfg = saved


def ref_state_dict_shapes(config_file, opts=()):
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(ref_import.build_cfg(config_file, opts))
    return [(k, tuple(v.shape)) for k, v in model.state_dict().items()]


def golden_mega_x101(h=192, w=320, n_frames=4, total=40):
    print("  MEGA X-101 32x8d @%dx%d: reference vs oracle, %d frames" % (h, w, n_frames))
    sd = mg.synth.make_state_dict("mega_x101", seed=0)
    frames = [mg.synth.synthetic_frame(i, h, w) for i in range(total)]
    gidx = mg.synth.global_frame_indices(total, seed=0)
    globals_per_frame = [gidx[:10]] + [[gidx[(10 + t - 1) % total]] for t in range(1, n_frames)]
    ref = mg.run_reference_mega(sd, frames, globals_per_frame, n_frames)
    orc = mo.MegaOracle(sd, record=True)
    gold = []
    for t in range(n_frames):
        infos = {"frame_category": 0 if t == 0 else 1,
                 "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                 "ref_g": [frames[j] for j in globals_per_frame[t]]}
        b, s, l = orc.forward(frames[t], infos)
        r = ref[t]
        assert r["class_logits"].shape == orc.trace["class_logits"].shape, "proposal count differs"
        mg.close(orc.trace["class_logits"], r["class_logits"], 2e-5, "frame %d class_logits" % t)
        mg.close(orc.trace["box_regression"], r["box_regression"], 2e-5, "frame %d box_regression" % t)
        assert torch.equal(l, r["labels"]) and b.shape == r["boxes"].shape, "detections differ (frame %d)" % t
        mg.close(b, r["boxes"], 1e-4, "frame %d det boxes" % t)
        mg.close(s, r["scores"], 1e-5, "frame %d det scores" % t)
        gold.append({"class_logits": r["class_logits"], "box_regression": r["box_regression"],
                     "proposals": orc.trace["proposals"], "boxes": r["boxes"], "scores": r["scores"],
                     "labels": r["labels"]})
    return {"arch": "mega_x101", "seed": 0, "h": h, "w": w, "total": total, "globals_per_frame": globals_per_frame,
            "frames": gold, "state_dict_shapes": ref_state_dict_shapes("configs/MEGA/vid_R_101_C4_MEGA_1x.yaml")}


def golden_base_x101(h=192, w=320):
    """the single-frame config (configs/vid_R_50_C4_1x.yaml) with the X-101 body: CONV_BODY R-101-C4 + the grouped keys"""
    print("  single-frame X-101 32x8d @%dx%d: reference vs oracle" % (h, w))
    opts = ("MODEL.BACKBONE.CONV_BODY", "R-101-C4")
    cfg = ref_import.build_cfg("configs/vid_R_50_C4_1x.yaml", opts)
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(cfg).eval()
    sd = mg.synth.make_state_dict("base_x101", seed=1)
    full = dict(sd)
    full["rpn.anchor_generator.cell_anchors.0"] = model.state_dict()["rpn.anchor_generator.cell_anchors.0"]
    model.load_state_dict(full, strict=True)
    img = mg.synth.synthetic_frame(3, h, w)
    hooks = {}
    pred = model.roi_heads.box.predictor
    orig = pred.forward

    def pf(x):
        r = orig(x)
        hooks["class_logits"], hooks["box_regression"] = r[0].clone(), r[1].clone()
        return r

    pred.forward = pf
    with torch.no_grad():
        res = model([img[0].clone()])[0]
    orc = mo.BaseOracle(sd, record=True)
    b, s, l = orc.forward(img)
    mg.close(orc.trace["class_logits"], hooks["class_logits"], 2e-5, "base class_logits")
    assert torch.equal(l, res.get_field("labels"))
    mg.close(b, res.bbox, 1e-4, "base det boxes")
    return {"arch": "base_x101", "seed": 1, "h": h, "w": w, "frame_index": 3,
            "class_logits": hooks["class_logits"], "box_regression": hooks["box_regression"],
            "proposals": orc.trace["proposals"], "boxes": res.bbox.clone(),
            "scores": res.get_field("scores").clone(), "labels": res.get_field("labels").clone(),
            "state_dict_shapes": ref_state_dict_shapes("configs/vid_R_50_C4_1x.yaml", opts)}


def main():
    torch.set_num_threads(8)
    out = sys.argv[1] if len(sys.argv) > 1 else GOLD
    with x101_configs(), grouped_bottlenecks():
        torch.save(golden_base_x101(), os.path.join(out, "base_x101_192x320.pt"))
        torch.save(golden_mega_x101(), os.path.join(out, "mega_x101_192x320.pt"))


if __name__ == "__main__":
    main()
