"""CPU tests of the ResNeXt C4 bodies (MODEL.RESNETS.NUM_GROUPS / WIDTH_PER_GROUP): the block-diagonal packing of a
grouped 3x3 conv, the module tree against the reference's parameter list, the config checks, and the oracle against
the X-101 32x8d fixtures that tools/make_golden_resnext.py wrote from the unmodified reference (the oracle's bottleneck
with a grouped conv2: tests/resnext_oracle.py)."""
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden")

import mega_oracle as mo  # noqa: E402
from resnext_oracle import grouped_bottlenecks  # noqa: E402


def _same_boxes(a, b, atol=2e-3):
    """same box lists, coordinates to 2e-3 px (the fixtures' convolutions ran on another host's CPU kernels)"""
    return a.shape == b.shape and torch.allclose(a, b, atol=atol, rtol=0)


def _grouped_case(gw, c=128, seed=0):
    g = torch.Generator().manual_seed(seed + gw)
    x = torch.randn(2, c, 13, 17, generator=g, dtype=torch.float64)
    w = torch.randn(c, gw, 3, 3, generator=g, dtype=torch.float64)
    return x, w, c // gw


@pytest.mark.parametrize("gw", [8, 16, 32, 64])
def test_block_diagonal_packing_equals_grouped_conv_fp64(gw):
    """each 64-channel chunk convolved densely with its [taps, 64, 64] slice == F.conv2d(groups=G), stride 2, dilation 2"""
    from mega_core.b200 import ops
    x, w, groups = _grouped_case(gw)
    packed = ops.pack_grouped_conv(w, groups, "cpu", torch.float64)
    assert packed.shape == (9, x.shape[1], 64)
    z = ops.GROUP_CHUNK
    outs = []
    for i in range(x.shape[1] // z):
        wz = packed[:, i * z:(i + 1) * z, :].reshape(3, 3, z, z).permute(2, 3, 0, 1)
        outs.append(F.conv2d(x[:, i * z:(i + 1) * z], wz, None, 2, 2, 2))
    ref = F.conv2d(x, w, None, 2, 2, 2, groups)
    assert (torch.cat(outs, 1) - ref).abs().max().item() < 1e-12
    # off-diagonal entries are exact zeros
    mask = torch.zeros(x.shape[1], z, dtype=torch.bool)
    for co in range(x.shape[1]):
        j0 = co % z // gw * gw
        mask[co, j0:j0 + gw] = True
    assert torch.all(packed[:, ~mask] == 0)


@pytest.mark.parametrize("gw", [8, 64])
def test_grouped_fields_describe_the_batched_launch(gw):
    """the batched launch that grouped_fields() describes, run by the exact-fp32 stand-in of conv_gemm (per-entry
    offsets of A, weight rows, scale / bias, output and residual), is the grouped conv with BN, residual and ReLU"""
    from fp32_shadow import _shadow_conv_gemm
    from mega_core.b200 import ops
    x, w, groups = _grouped_case(gw, seed=5)
    c = x.shape[1]
    g = torch.Generator().manual_seed(7)
    scale, bias = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g)
    res = torch.randn(2, 7, 9, c, generator=g)
    packed = ops.pack_grouped_conv(w.float(), groups, "cpu")
    a = x.float().permute(0, 2, 3, 1).contiguous()
    out = torch.zeros(2, 7, 9, c)
    _shadow_conv_gemm(a, packed, out, taps=(3, 3), dil=2, pad=2, stride=(2, 2), scale=scale, bias=bias, residual=res,
                      relu=True, **ops.grouped_fields(packed))
    ref = F.conv2d(x, w, None, 2, 2, 2, groups) * scale.double().view(1, -1, 1, 1) + bias.double().view(1, -1, 1, 1)
    ref = (ref + res.double().permute(0, 3, 1, 2)).relu().permute(0, 2, 3, 1)
    assert (out.double() - ref).abs().max().item() < 1e-4


def test_packing_rejects_unserved_group_widths():
    from mega_core.b200 import ops
    with pytest.raises(AssertionError):
        ops.pack_grouped_conv(torch.zeros(128, 4, 3, 3), 32, "cpu")       # gw 4
    with pytest.raises(AssertionError):
        ops.pack_grouped_conv(torch.zeros(96, 8, 3, 3), 12, "cpu")        # channels not a multiple of 64


@pytest.mark.parametrize("method,fixture", [("mega", "mega_x101_192x320.pt"), ("base", "base_x101_192x320.pt")])
def test_x101_module_tree_has_the_reference_parameters(method, fixture):
    """build_detection_model for a ResNeXt-101 32x8d config: every key and shape of the reference's model"""
    from mega_core.modeling.detector.detectors import build_detection_model, vid_config
    gold = torch.load(os.path.join(GOLD, fixture))
    cfg = vid_config(method, "R-101-C4", "cpu", num_groups=32, width_per_group=8)
    model = build_detection_model(cfg)
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == dict(gold["state_dict_shapes"])
    assert got["backbone.body.layer1.0.conv2.weight"] == (256, 8, 3, 3)
    assert got["roi_heads.box.feature_extractor.head.layer4.2.conv2.weight"] == (2048, 64, 3, 3)


def test_x101_state_dict_infers_groups_and_width():
    from mega_core.b200 import synth
    from mega_core.modeling.detector.detectors import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    sd = synth.make_state_dict("mega_x101", seed=0)
    model = build_detection_model_from_state_dict(sd, method="mega", device="cpu", precision="tf32")
    r = model.cfg.MODEL.RESNETS
    assert (r.NUM_GROUPS, r.WIDTH_PER_GROUP) == (32, 8)
    engine_config_from(model.cfg)          # served


@pytest.mark.parametrize("groups,wpg", [(32, 4), (1, 48), (32, 16), (16, 2)])
def test_unserved_widths_are_rejected(groups, wpg):
    from mega_core.modeling.detector.detectors import vid_config
    from mega_core.modeling.nets import engine_config_from
    with pytest.raises(NotImplementedError, match="NUM_GROUPS"):
        engine_config_from(vid_config("mega", "R-101-C4", "cpu", num_groups=groups, width_per_group=wpg))


@pytest.mark.parametrize("groups,wpg", [(32, 8), (8, 8), (64, 8), (1, 128)])
def test_served_widths_are_accepted(groups, wpg):
    from mega_core.modeling.detector.detectors import vid_config
    from mega_core.modeling.nets import engine_config_from
    engine_config_from(vid_config("mega", "R-101-C4", "cpu", num_groups=groups, width_per_group=wpg))


def test_deformable_stages_are_rejected():
    from mega_core.modeling.detector.detectors import vid_config
    from mega_core.modeling.nets import engine_config_from
    cfg = vid_config("mega", "R-101-C4", "cpu")
    cfg.MODEL.RESNETS.STAGE_WITH_DCN = (False, True, True, True)
    with pytest.raises(NotImplementedError, match="STAGE_WITH_DCN"):
        engine_config_from(cfg)


def test_shipped_configs_give_the_same_engine_config(tmp_path):
    """engine_config_from of every shipped YAML (defaults <- BASE_RCNN_1gpu.yaml <- method yaml) equals the values
    stored before ResNeXt support existed"""
    import yaml
    from mega_core.config import cfg as base
    from mega_core.modeling.nets import engine_config_from
    with open(os.path.join(GOLD, "reference_configs.json")) as fh:
        configs = json.load(fh)
    with open(os.path.join(GOLD, "shipped_engine_configs.json")) as fh:
        expected = json.load(fh)
    d = str(tmp_path)
    for name, want in expected.items():
        c = base.clone()
        for tag, data in (("base", configs["configs/BASE_RCNN_1gpu.yaml"]), ("method", configs[name])):
            p = os.path.join(d, tag + ".yaml")
            with open(p, "w") as fh:
                yaml.safe_dump(data, fh)
            c.merge_from_file(p)
        got = {k: (list(v) if isinstance(v, tuple) else v) for k, v in vars(engine_config_from(c)).items()
               if k != "precision"}
        assert got == want, name


def test_x101_tiny_backbone_engine_matches_oracle():
    """the engine's ResNet stages with grouped conv2 launches (exact-fp32 stand-ins for the kernels) against the oracle's
    grouped F.conv2d body"""
    from cpu_ops import cpu_ops
    from mega_core.b200 import engine, synth
    sd = synth.make_state_dict("mega_x101_tiny", seed=2)
    img = synth.synthetic_frame(1, 64, 96)
    with grouped_bottlenecks():
        ref = mo.resnet_c4_body(img, sd)
    with cpu_ops():
        bb = engine.Backbone(sd, "cpu")
        assert [blk.groups for blocks in bb.stages.stages for blk in blocks] == [32] * 4
        got = bb.forward(img).permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() < 1e-4 * max(ref.abs().max().item(), 1.0)


def test_oracle_matches_base_x101_reference_fixture():
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(GOLD, "base_x101_192x320.pt"))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    orc = mo.BaseOracle(sd, record=True)
    with grouped_bottlenecks():
        b, s, l = orc.forward(synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"]))
    assert torch.allclose(orc.trace["class_logits"], gold["class_logits"], atol=1e-5)
    assert torch.equal(l, gold["labels"]) and _same_boxes(b, gold["boxes"]) and torch.allclose(s, gold["scores"], atol=1e-6)


def test_oracle_matches_mega_x101_reference_fixture():
    """3 frames of the unmodified reference's GeneralizedRCNNMEGA on a ResNeXt-101 32x8d body"""
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(GOLD, "mega_x101_192x320.pt"))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    orc = mo.MegaOracle(sd, record=True)
    gpf = gold["globals_per_frame"]
    for t, ref in enumerate(gold["frames"][:3]):
        infos = {"frame_category": 0 if t == 0 else 1,
                 "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                 "ref_g": [frames[j] for j in gpf[t]]}
        with grouped_bottlenecks():
            b, s, l = orc.forward(frames[t], infos)
        assert torch.allclose(orc.trace["class_logits"], ref["class_logits"], atol=1e-5)
        assert _same_boxes(orc.trace["proposals"], ref["proposals"])
        assert torch.equal(l, ref["labels"]) and _same_boxes(b, ref["boxes"])


def test_grouped_bottleneck_with_one_group_is_the_oracles():
    """the grouped restatement of the oracle's bottleneck equals it bit for bit on a dense (NUM_GROUPS = 1) block"""
    import resnext_oracle
    from mega_core.b200 import synth
    sd = synth.make_state_dict("mega_r50_tiny", seed=4)
    x = torch.randn(1, 256, 12, 20, generator=torch.Generator().manual_seed(3))
    for p, stride, dil in (("backbone.body.layer2.0.", 2, 1), ("roi_heads.box.feature_extractor.head.layer4.0.", 1, 2)):
        xin = x if "layer2" in p else torch.randn(1, 1024, 7, 7, generator=torch.Generator().manual_seed(5))
        assert torch.equal(resnext_oracle.bottleneck(xin, sd, p, stride, dil), mo.bottleneck(xin, sd, p, stride, dil))
