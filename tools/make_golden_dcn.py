"""Generate the fixtures of deformable backbone stages (MODEL.RESNETS.STAGE_WITH_DCN, DCN v1 and modulated v2) by running
the UNMODIFIED reference with those keys on seeded synthetic weights (mega_core.b200.synth), and check the oracle with
the deformable bottleneck of tests/dcn_oracle.py against it on the way with the tolerances of oracle/make_golden.py:

  tests/golden/base_r101_dcn_192x320.pt        configs/vid_R_50_C4_1x.yaml with CONV_BODY R-101-C4,
                                               STAGE_WITH_DCN (False, True, True, False), v1, one frame
  tests/golden/mega_r101_mdcn_192x320.pt       configs/MEGA/vid_R_101_C4_MEGA_1x.yaml, modulated, res3 + res4,
                                               4 frames (the memory fills)
  tests/golden/base_r101_s3x3_mdcn_192x320.pt  the single-frame R-101 with STRIDE_IN_1X1 False, modulated, res3 +
                                               res4: the first res3 / res4 block samples at stride 2
  tests/golden/base_r101_dcn_g4_192x320.pt     single-frame R-101, v1 with DEFORMABLE_GROUPS 4, res3 + res4
  tests/golden/mega_r101_dcn_g2_192x320.pt     MEGA R-101, v1 with DEFORMABLE_GROUPS 2, res2 - res4, 4 frames
  tests/golden/base_r101_s3x3_dcn_g8_192x320.pt  single-frame R-101, v1 with DEFORMABLE_GROUPS 8, res2 - res4,
                                               STRIDE_IN_1X1 False: 8 channels per group in res2, stride-2 sampling

The reference's deformable functions raise on CPU tensors (layers/dcn/deform_conv_func.py:43, :174), so the run
replaces `deform_conv` / `modulated_deform_conv` where its DeformConv modules look them up with the restatement
oracle/train_ops_oracle.deform_conv2d (anchored to torchvision by tests/test_train_ops_cpu.py); no reference file is
edited. Each fixture must exercise the deformable path, and the generator asserts both:
  * the same weights run as a plain 3x3 conv2 (conv2.conv.weight, no offsets) give different class logits;
  * a non-trivial share of the samples of the first deformable block is fractional or outside the map;
  * with several deformable groups, the same weights with every group given group 0's offsets give different class
    logits (a sampling that ignores the group cannot pass).
Only outputs are stored, plus the reference model's parameter / buffer list, which the package's module tree must equal.

Run where the reference checkout exists:   python tools/make_golden_dcn.py [out_dir [fixture ...]]
"""
import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
GOLD = os.path.join(ROOT, "tests", "golden")

import dcn_oracle  # noqa: E402
import make_golden as mg  # noqa: E402
import mega_oracle as mo  # noqa: E402
import ref_import  # noqa: E402
import train_ops_oracle as to  # noqa: E402
from make_golden_stride3x3 import extra_opts, ref_state_dict_shapes  # noqa: E402

BASE_OPTS = ("MODEL.BACKBONE.CONV_BODY", "R-101-C4")


def dcn_opts(stages, modulated, stride_in_1x1=True, deformable_groups=1):
    return ("MODEL.RESNETS.STAGE_WITH_DCN", tuple(stages), "MODEL.RESNETS.WITH_MODULATED_DCN", modulated,
            "MODEL.RESNETS.DEFORMABLE_GROUPS", deformable_groups, "MODEL.RESNETS.STRIDE_IN_1X1", stride_in_1x1)


def deform_conv2_groups(x, sd, p, stride, dilation):
    """DFConv2d.forward (layers/misc.py:176-187) of a DCN v1 conv2 with any number of deformable groups: the offset conv
    has 18 rows per group, all of them the deformable conv's offsets"""
    wo, bo = sd[p + "conv2.offset.weight"], sd[p + "conv2.offset.bias"]
    if wo.shape[0] == 27:
        return dcn_oracle_deform_conv2(x, sd, p, stride, dilation)
    offset = torch.nn.functional.conv2d(x, wo, bo, stride, dilation, dilation)
    return to.deform_conv2d(x, offset, None, sd[p + "conv2.conv.weight"], None, (stride, stride),
                            (dilation, dilation), (dilation, dilation), 1, wo.shape[0] // 18)


dcn_oracle_deform_conv2 = dcn_oracle.deform_conv2


@contextlib.contextmanager
def oracle_groups():
    """inside: the oracle's deformable bottleneck (tests/dcn_oracle.py) samples every deformable group at its offsets"""
    saved = dcn_oracle.deform_conv2
    dcn_oracle.deform_conv2 = deform_conv2_groups
    try:
        yield
    finally:
        dcn_oracle.deform_conv2 = saved


def patch_reference_deform_ops():
    """the reference's DeformConv / ModulatedDeformConv call the restatement instead of the CUDA-only _C ops"""
    from torch.nn.modules.utils import _pair
    ref_import.setup()
    import mega_core.layers.dcn.deform_conv_module as dm

    def deform_conv(x, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1, im2col_step=64):
        return to.deform_conv2d(x, offset, None, weight, None, _pair(stride), _pair(padding), _pair(dilation), groups,
                                deformable_groups)

    def modulated_deform_conv(x, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                              deformable_groups=1):
        return to.deform_conv2d(x, offset, mask, weight, bias, _pair(stride), _pair(padding), _pair(dilation), groups,
                                deformable_groups)
    dm.deform_conv, dm.modulated_deform_conv = deform_conv, modulated_deform_conv


class SampleStats(object):
    """share of fractional and of outside samples over every deformable conv2 the oracle runs inside"""

    def __init__(self):
        self.first = None

    def __enter__(self):
        self.saved = dcn_oracle.deform_conv2

        def wrapped(x, sd, p, stride, dilation):
            if self.first is None:
                om = torch.nn.functional.conv2d(x, sd[p + "conv2.offset.weight"], sd[p + "conv2.offset.bias"], stride,
                                                dilation, dilation)
                off = om[:, :18].reshape(x.shape[0], 9, 2, om.shape[2], om.shape[3])
                ho, wo = om.shape[2], om.shape[3]
                ki = torch.arange(3).repeat_interleave(3).view(1, 9, 1, 1) * dilation - dilation
                kj = torch.arange(3).repeat(3).view(1, 9, 1, 1) * dilation - dilation
                hh = torch.arange(ho).view(1, 1, ho, 1) * stride + ki + off[:, :, 0]
                ww = torch.arange(wo).view(1, 1, 1, wo) * stride + kj + off[:, :, 1]
                frac = ((hh != hh.floor()) | (ww != ww.floor())).float().mean().item()
                outside = ((hh <= -1) | (ww <= -1) | (hh >= x.shape[2]) | (ww >= x.shape[3])).float().mean().item()
                partial = ((hh < 0) | (ww < 0) | (hh > x.shape[2] - 1) | (ww > x.shape[3] - 1)).float().mean().item()
                self.first = (p, frac, outside, partial)
            return self.saved(x, sd, p, stride, dilation)
        dcn_oracle.deform_conv2 = wrapped
        return self

    def __exit__(self, *a):
        dcn_oracle.deform_conv2 = self.saved
        return False

    def check(self):
        p, frac, outside, partial = self.first
        print("  %s: %.3f of the samples fractional, %.4f outside the map, %.4f with a corner outside"
              % (p, frac, outside, partial))
        assert frac > 0.5 and partial > 0.005, "the offsets hardly move the samples"


def plain_state_dict(sd):
    """the same weights with every deformable conv2 as a plain 3x3 conv (no offsets)"""
    out = {}
    for k, v in sd.items():
        if ".conv2.offset." in k:
            continue
        out[k.replace(".conv2.conv.weight", ".conv2.weight")] = v
    return out


def group0_state_dict(sd):
    """the same weights with every deformable group's offset rows replaced by group 0's"""
    out = dict(sd)
    for k, v in sd.items():
        if ".conv2.offset." in k and v.shape[0] > 18:
            out[k] = v[:18].repeat((v.shape[0] // 18,) + (1,) * (v.dim() - 1))
    return out


def assert_dcn_matters(got, plain, what, than="plain conv2"):
    diff = (got - plain).abs().max().item() if got.shape == plain.shape else float("inf")
    print("  %-38s %s differs by %.3e" % (what, than, diff))
    assert diff > 1e-3, "%s: the deformable stages give the %s result (%.3e)" % (what, than, diff)


def golden_base(name, stages, modulated, stride_in_1x1, seed=1, h=192, w=320, frame_index=3, deformable_groups=1):
    print("  %s: single-frame R-101 @%dx%d, reference vs oracle" % (name, h, w))
    opts = BASE_OPTS + dcn_opts(stages, modulated, stride_in_1x1, deformable_groups)
    cfg = ref_import.build_cfg("configs/vid_R_50_C4_1x.yaml", opts)
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(cfg).eval()
    sd = mg.synth.make_state_dict("base_r101", seed=seed, stage_with_dcn=stages, modulated_dcn=modulated,
                                  deformable_groups=deformable_groups)
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
    with dcn_oracle.deformable(stride_in_1x1), oracle_groups(), SampleStats() as st:
        b, s, l = orc.forward(img)
    st.check()
    mg.close(orc.trace["class_logits"], hooks["class_logits"], 2e-5, "base class_logits")
    mg.close(orc.trace["box_regression"], hooks["box_regression"], 2e-5, "base box_regression")
    assert torch.equal(l, res.get_field("labels"))
    mg.close(b, res.bbox, 1e-4, "base det boxes")
    plain = mo.BaseOracle(plain_state_dict(sd), record=True)
    with dcn_oracle.deformable(stride_in_1x1):
        plain.forward(img)
    assert_dcn_matters(hooks["class_logits"], plain.trace["class_logits"], "base class_logits")
    if deformable_groups > 1:
        same = mo.BaseOracle(group0_state_dict(sd), record=True)
        with dcn_oracle.deformable(stride_in_1x1), oracle_groups():
            same.forward(img)
        assert_dcn_matters(hooks["class_logits"], same.trace["class_logits"], "base class_logits",
                           "group 0's offsets in every group")
    out = {"arch": "base_r101", "seed": seed, "h": h, "w": w, "frame_index": frame_index,
           "stage_with_dcn": tuple(stages), "modulated": modulated, "stride_in_1x1": stride_in_1x1,
           "class_logits": hooks["class_logits"], "box_regression": hooks["box_regression"],
           "proposals": orc.trace["proposals"], "boxes": res.bbox.clone(),
           "scores": res.get_field("scores").clone(), "labels": res.get_field("labels").clone(),
           "state_dict_shapes": ref_state_dict_shapes("configs/vid_R_50_C4_1x.yaml", opts)}
    if deformable_groups > 1:
        out["deformable_groups"] = deformable_groups
    return out


def golden_mega(stages, modulated, seed=0, h=192, w=320, n_frames=4, total=40, deformable_groups=1):
    print("  MEGA R-101 @%dx%d, reference vs oracle, %d frames" % (h, w, n_frames))
    sd = mg.synth.make_state_dict("mega_r101", seed=seed, stage_with_dcn=stages, modulated_dcn=modulated,
                                  deformable_groups=deformable_groups)
    frames = [mg.synth.synthetic_frame(i, h, w) for i in range(total)]
    gidx = mg.synth.global_frame_indices(total, seed=seed)
    globals_per_frame = [gidx[:10]] + [[gidx[(10 + t - 1) % total]] for t in range(1, n_frames)]
    opts = dcn_opts(stages, modulated, deformable_groups=deformable_groups)
    with extra_opts(opts):
        ref = mg.run_reference_mega(sd, frames, globals_per_frame, n_frames)
        shapes = ref_state_dict_shapes("configs/MEGA/vid_R_101_C4_MEGA_1x.yaml")
    orc = mo.MegaOracle(sd, record=True)
    infos_of = lambda t: {"frame_category": 0 if t == 0 else 1,                                  # noqa: E731
                          "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                          "ref_g": [frames[j] for j in globals_per_frame[t]]}
    gold = []
    for t in range(n_frames):
        with dcn_oracle.deformable(), oracle_groups(), SampleStats() as st:
            b, s, l = orc.forward(frames[t], infos_of(t))
        if t == 0:
            st.check()
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
    plain = mo.MegaOracle(plain_state_dict(sd), record=True)
    plain.forward(frames[0], infos_of(0))
    assert_dcn_matters(gold[0]["class_logits"], plain.trace["class_logits"], "frame 0 class_logits")
    if deformable_groups > 1:
        same = mo.MegaOracle(group0_state_dict(sd), record=True)
        with dcn_oracle.deformable(), oracle_groups():
            same.forward(frames[0], infos_of(0))
        assert_dcn_matters(gold[0]["class_logits"], same.trace["class_logits"], "frame 0 class_logits",
                           "group 0's offsets in every group")
    out = {"arch": "mega_r101", "seed": seed, "h": h, "w": w, "total": total, "globals_per_frame": globals_per_frame,
           "stage_with_dcn": tuple(stages), "modulated": modulated, "stride_in_1x1": True, "frames": gold,
           "state_dict_shapes": shapes}
    if deformable_groups > 1:
        out["deformable_groups"] = deformable_groups
    return out


def main():
    torch.set_num_threads(8)
    out = sys.argv[1] if len(sys.argv) > 1 else GOLD
    only = sys.argv[2:]
    want = lambda name: not only or name in only           # noqa: E731
    patch_reference_deform_ops()
    res34 = (False, True, True, False)
    if want("base_r101_dcn_192x320.pt"):
        torch.save(golden_base("base_r101_dcn_192x320.pt", res34, False, True),
                   os.path.join(out, "base_r101_dcn_192x320.pt"))
    if want("mega_r101_mdcn_192x320.pt"):
        torch.save(golden_mega(res34, True), os.path.join(out, "mega_r101_mdcn_192x320.pt"))
    if want("base_r101_s3x3_mdcn_192x320.pt"):
        torch.save(golden_base("base_r101_s3x3_mdcn_192x320.pt", res34, True, False, seed=2),
                   os.path.join(out, "base_r101_s3x3_mdcn_192x320.pt"))
    res234 = (True, True, True, False)
    if want("base_r101_dcn_g4_192x320.pt"):
        torch.save(golden_base("base_r101_dcn_g4_192x320.pt", res34, False, True, seed=3, deformable_groups=4),
                   os.path.join(out, "base_r101_dcn_g4_192x320.pt"))
    if want("mega_r101_dcn_g2_192x320.pt"):
        torch.save(golden_mega(res234, False, seed=1, deformable_groups=2),
                   os.path.join(out, "mega_r101_dcn_g2_192x320.pt"))
    if want("base_r101_s3x3_dcn_g8_192x320.pt"):
        torch.save(golden_base("base_r101_s3x3_dcn_g8_192x320.pt", res234, False, False, seed=4, deformable_groups=8),
                   os.path.join(out, "base_r101_s3x3_dcn_g8_192x320.pt"))


if __name__ == "__main__":
    main()
