"""Generate the fixtures of 3x3-strided bottlenecks (MODEL.RESNETS.STRIDE_IN_1X1 False: the first block of res3 / res4
strides its 3x3 conv2 instead of its 1x1 conv1) by running the UNMODIFIED reference with that key on seeded synthetic
weights (mega_core.b200.synth), and check the oracle with the 3x3-strided bottleneck of tests/stride3x3_oracle.py (dense
and grouped) against it on the way with the tolerances of oracle/make_golden.py:

  tests/golden/base_r101_s3x3_192x320.pt   configs/vid_R_50_C4_1x.yaml with CONV_BODY R-101-C4, one frame
  tests/golden/mega_r101_s3x3_192x320.pt   configs/MEGA/vid_R_101_C4_MEGA_1x.yaml, 4 frames (the memory fills), on the
                                           weights of tests/golden/mega_r101_192x320.pt (the MSRA layout's fixture)
  tests/golden/mega_x101_s3x3_192x320.pt   the same with NUM_GROUPS 32 / WIDTH_PER_GROUP 8 (ResNeXt-101 32x8d), 4 frames

Each fixture must exercise the layout: the oracle in the MSRA layout (STRIDE_IN_1X1 True) on the same weights gives
different class logits for the first frame, and the generator asserts it. Only outputs are stored, plus the reference
model's parameter / buffer list, which the package's module tree must equal.

Run where the reference checkout exists:   python tools/make_golden_stride3x3.py [out_dir [fixture ...]]
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
from stride3x3_oracle import strided_3x3  # noqa: E402

STRIDE_OPTS = ("MODEL.RESNETS.STRIDE_IN_1X1", False)
X101_OPTS = ("MODEL.RESNETS.NUM_GROUPS", 32, "MODEL.RESNETS.WIDTH_PER_GROUP", 8)
BASE_OPTS = ("MODEL.BACKBONE.CONV_BODY", "R-101-C4")


@contextlib.contextmanager
def extra_opts(opts):
    """every reference config built inside gets `opts` on top of its YAML"""
    saved = ref_import.build_cfg

    def build_cfg(config_file, o=()):
        return saved(config_file, tuple(o) + tuple(opts))
    ref_import.build_cfg = build_cfg
    try:
        yield
    finally:
        ref_import.build_cfg = saved


def ref_state_dict_shapes(config_file, opts=()):
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(ref_import.build_cfg(config_file, opts))
    return [(k, tuple(v.shape)) for k, v in model.state_dict().items()]


def assert_layout_matters(got, msra, what):
    """the fixture exercises the layout: the MSRA layout's result on the same weights is not the same"""
    diff = (got - msra).abs().max().item() if got.shape == msra.shape else float("inf")
    print("  %-38s MSRA layout differs by %.3e" % (what, diff))
    assert diff > 1e-3, "%s: the 3x3-strided layout gives the MSRA layout's result (%.3e)" % (what, diff)


def golden_base(arch="base_r101", seed=1, h=192, w=320, frame_index=3):
    print("  single-frame R-101, STRIDE_IN_1X1 False @%dx%d: reference vs oracle" % (h, w))
    cfg = ref_import.build_cfg("configs/vid_R_50_C4_1x.yaml", BASE_OPTS)
    assert not cfg.MODEL.RESNETS.STRIDE_IN_1X1
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(cfg).eval()
    sd = mg.synth.make_state_dict(arch, seed=seed)
    full = dict(sd)
    full["rpn.anchor_generator.cell_anchors.0"] = model.state_dict()["rpn.anchor_generator.cell_anchors.0"]
    model.load_state_dict(full, strict=True)
    img = mg.synth.synthetic_frame(frame_index, h, w)
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
    with strided_3x3():
        b, s, l = orc.forward(img)
    mg.close(orc.trace["class_logits"], hooks["class_logits"], 2e-5, "base class_logits")
    mg.close(orc.trace["box_regression"], hooks["box_regression"], 2e-5, "base box_regression")
    assert torch.equal(l, res.get_field("labels"))
    mg.close(b, res.bbox, 1e-4, "base det boxes")
    msra = mo.BaseOracle(sd, record=True)
    msra.forward(img)
    assert_layout_matters(hooks["class_logits"], msra.trace["class_logits"], "base class_logits")
    return {"arch": arch, "seed": seed, "h": h, "w": w, "frame_index": frame_index, "stride_in_1x1": False,
            "class_logits": hooks["class_logits"], "box_regression": hooks["box_regression"],
            "proposals": orc.trace["proposals"], "boxes": res.bbox.clone(),
            "scores": res.get_field("scores").clone(), "labels": res.get_field("labels").clone(),
            "state_dict_shapes": ref_state_dict_shapes("configs/vid_R_50_C4_1x.yaml", BASE_OPTS)}


def golden_mega(arch, seed, h=192, w=320, n_frames=4, total=40):
    print("  MEGA %s, STRIDE_IN_1X1 False @%dx%d: reference vs oracle, %d frames" % (arch, h, w, n_frames))
    assert not ref_import.build_cfg("configs/MEGA/vid_R_101_C4_MEGA_1x.yaml").MODEL.RESNETS.STRIDE_IN_1X1
    sd = mg.synth.make_state_dict(arch, seed=seed)
    frames = [mg.synth.synthetic_frame(i, h, w) for i in range(total)]
    gidx = mg.synth.global_frame_indices(total, seed=seed)
    globals_per_frame = [gidx[:10]] + [[gidx[(10 + t - 1) % total]] for t in range(1, n_frames)]
    ref = mg.run_reference_mega(sd, frames, globals_per_frame, n_frames)
    orc = mo.MegaOracle(sd, record=True)
    infos_of = lambda t: {"frame_category": 0 if t == 0 else 1,                                  # noqa: E731
                          "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                          "ref_g": [frames[j] for j in globals_per_frame[t]]}
    gold = []
    for t in range(n_frames):
        with strided_3x3():
            b, s, l = orc.forward(frames[t], infos_of(t))
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
    msra = mo.MegaOracle(sd, record=True)
    msra.forward(frames[0], infos_of(0))
    assert_layout_matters(gold[0]["class_logits"], msra.trace["class_logits"], "frame 0 class_logits")
    return {"arch": arch, "seed": seed, "h": h, "w": w, "total": total, "globals_per_frame": globals_per_frame,
            "stride_in_1x1": False, "frames": gold,
            "state_dict_shapes": ref_state_dict_shapes("configs/MEGA/vid_R_101_C4_MEGA_1x.yaml")}


def main():
    torch.set_num_threads(8)
    out = sys.argv[1] if len(sys.argv) > 1 else GOLD
    only = sys.argv[2:]
    want = lambda name: not only or name in only           # noqa: E731
    with extra_opts(STRIDE_OPTS):
        if want("base_r101_s3x3_192x320.pt"):
            torch.save(golden_base(), os.path.join(out, "base_r101_s3x3_192x320.pt"))
        if want("mega_r101_s3x3_192x320.pt"):
            torch.save(golden_mega("mega_r101", seed=0), os.path.join(out, "mega_r101_s3x3_192x320.pt"))
        if want("mega_x101_s3x3_192x320.pt"):
            with extra_opts(X101_OPTS), grouped_bottlenecks():
                torch.save(golden_mega("mega_x101", seed=13), os.path.join(out, "mega_x101_s3x3_192x320.pt"))


if __name__ == "__main__":
    main()
