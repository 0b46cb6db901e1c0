"""CPU tests of 3x3-strided bottlenecks (MODEL.RESNETS.STRIDE_IN_1X1 False, the layout of the Caffe2 / fb.torch ResNe(X)t
and torchvision weights): the config checks, the module tree against the reference's parameter lists, which conv of the
engines' first res3 / res4 block carries the stride, the oracle against the fixtures tools/make_golden_stride3x3.py wrote
from the unmodified reference, and the engines' host logic on the CPU stand-ins (tests/cpu_ops.py) against them."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden")

import mega_oracle as mo  # noqa: E402
from cpu_ops import cpu_ops  # noqa: E402
from resnext_oracle import grouped_bottlenecks  # noqa: E402
from stride3x3_oracle import strided_3x3  # noqa: E402

FIXTURES = ("base_r101_s3x3_192x320.pt", "mega_r101_s3x3_192x320.pt", "mega_x101_s3x3_192x320.pt")


def _gold(fixture):
    gold = torch.load(os.path.join(GOLD, fixture))
    assert gold["stride_in_1x1"] is False
    return gold


@pytest.mark.parametrize("method", ["base", "dff", "fgfa", "mega", "rdn"])
def test_config_is_accepted_and_passed_to_the_engine(method):
    from mega_core.modeling.detector.detectors import vid_config
    from mega_core.modeling.nets import engine_config_from
    assert engine_config_from(vid_config(method, "R-101-C4", "cpu", stride_in_1x1=False)).stride_in_1x1 is False
    assert engine_config_from(vid_config(method, "R-101-C4", "cpu")).stride_in_1x1 is True
    x101 = vid_config(method, "R-101-C4", "cpu", num_groups=32, width_per_group=8, stride_in_1x1=False)
    assert engine_config_from(x101).stride_in_1x1 is False


def test_deformable_stages_are_still_rejected_with_it():
    from mega_core.modeling.detector.detectors import vid_config
    from mega_core.modeling.nets import engine_config_from
    cfg = vid_config("mega", "R-101-C4", "cpu", num_groups=32, width_per_group=8, stride_in_1x1=False)
    cfg.MODEL.RESNETS.STAGE_WITH_DCN = (False, True, True, True)
    with pytest.raises(NotImplementedError, match="STAGE_WITH_DCN") as e:
        engine_config_from(cfg)
    assert "STRIDE_IN_1X1" not in str(e.value)


@pytest.mark.parametrize("fixture", FIXTURES)
def test_module_tree_has_the_reference_parameters(fixture):
    """build_detection_model_from_state_dict(stride_in_1x1=False): every key and shape of the reference's model, the
    stride on conv2 of the first res3 / res4 block and on its downsample, none on its conv1"""
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    gold = _gold(fixture)
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    model = build_detection_model_from_state_dict(sd, method=gold["arch"].split("_")[0], device="cpu", precision="tf32",
                                                  stride_in_1x1=False)
    assert model.cfg.MODEL.RESNETS.STRIDE_IN_1X1 is False
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == dict(gold["state_dict_shapes"])
    body = model.backbone.body
    for layer in (body.layer2, body.layer3):
        assert (layer[0].conv1.stride, layer[0].conv2.stride, layer[0].downsample[0].stride) == ((1, 1), (2, 2), (2, 2))
    msra = build_detection_model_from_state_dict(sd, method=gold["arch"].split("_")[0], device="cpu", precision="tf32")
    assert msra.cfg.MODEL.RESNETS.STRIDE_IN_1X1 is True
    b = msra.backbone.body.layer3[0]
    assert (b.conv1.stride, b.conv2.stride, b.downsample[0].stride) == ((2, 2), (1, 1), (2, 2))


def _record_body_launches(arch, stride_in_1x1, h=64, w=96):
    """(input shape, taps, stride, output shape) of every conv_gemm launch of the engine's body on the stand-ins"""
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict(arch, seed=2)
    img = synth.synthetic_frame(1, h, w)
    log = []
    with cpu_ops():
        inner = ops.conv_gemm

        def rec(a, wt, out, **kw):
            log.append((tuple(a.shape), tuple(kw.get("taps", (1, 1))), tuple(kw.get("stride", (1, 1))),
                        tuple(out.shape)))
            return inner(a, wt, out, **kw)
        ops.conv_gemm = rec
        try:
            bb = engine.Backbone(sd, "cpu", stride_in_1x1=stride_in_1x1)
            feats = bb.forward(img)
        finally:
            ops.conv_gemm = inner
    return log, feats, sd, img


@pytest.mark.parametrize("arch", ["mega_r50_tiny", "mega_x101_tiny"])
def test_engine_layout_puts_the_stride_on_conv2(arch):
    """first block of res3 / res4: conv1 at the input resolution, conv2 a 3x3 / stride-2 launch, the downsample on the
    strided view; every other launch, and the number of launches, as in the MSRA layout; the result is the oracle's"""
    s3, feats, sd, img = _record_body_launches(arch, False)
    s1, _, _, _ = _record_body_launches(arch, True)
    assert len(s3) == len(s1)
    strided = [i for i, (a, taps, stride, o) in enumerate(s3) if stride != (1, 1)]
    assert len(strided) == 3          # stem (7x1 row slabs, stride (2, 1)), then conv2 of res3 / res4's first block
    for i in strided[1:]:
        a, taps, stride, o = s3[i]
        assert taps == (3, 3) and stride == (2, 2) and o[1:3] == ((a[1] - 1) // 2 + 1, (a[2] - 1) // 2 + 1)
        conv1 = s3[i - 1]
        assert conv1[1] == (1, 1) and conv1[0][1:3] == conv1[3][1:3] == a[1:3]      # conv1 unstrided, full resolution
        down = s3[i + 1]
        assert down[0][1:3] == o[1:3] and down[3][1:3] == o[1:3]                   # downsample reads the strided view
        assert s1[i - 1][0][1:3] == o[1:3] and s1[i][2] == (1, 1)                  # MSRA: conv1 on the strided view
    assert [s3[i] for i in range(len(s3)) if i not in strided and i + 1 not in strided] == \
        [s1[i] for i in range(len(s1)) if i not in strided and i + 1 not in strided]
    with strided_3x3():
        ref = mo.resnet_c4_body(img, sd)
    if "x101" in arch:
        with grouped_bottlenecks():
            msra = mo.resnet_c4_body(img, sd)
    else:
        msra = mo.resnet_c4_body(img, sd)
    got = feats.permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() < 1e-4 * max(ref.abs().max().item(), 1.0)
    assert (msra - ref).abs().max().item() > 1e-2


def _mega_infos(gold, frames, t):
    total, gpf = gold["total"], gold["globals_per_frame"]
    return {"frame_category": 0 if t == 0 else 1,
            "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
            "ref_g": [frames[j] for j in gpf[t]]}


@pytest.mark.parametrize("fixture", FIXTURES)
def test_oracle_matches_the_reference_fixture(fixture):
    """the oracle with the 3x3-strided bottleneck (tests/stride3x3_oracle.py) against the unmodified reference (first two
    frames of the MEGA fixtures)"""
    from mega_core.b200 import synth
    gold = _gold(fixture)
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    if "frames" not in gold:
        orc = mo.BaseOracle(sd, record=True)
        with strided_3x3():
            b, s, l = orc.forward(synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"]))
        steps = [(orc.trace["class_logits"], orc.trace["proposals"], b, l, gold)]
    else:
        frames = [synth.synthetic_frame(i, gold["h"], gold["w"]) for i in range(gold["total"])]
        orc = mo.MegaOracle(sd, record=True)
        steps = []
        with strided_3x3():
            for t, ref in enumerate(gold["frames"][:2]):
                b, s, l = orc.forward(frames[t], _mega_infos(gold, frames, t))
                steps.append((orc.trace["class_logits"].clone(), orc.trace["proposals"].clone(), b, l, ref))
    for logits, props, b, l, ref in steps:
        assert torch.allclose(logits, ref["class_logits"], atol=1e-5)
        assert props.shape == ref["proposals"].shape and torch.allclose(props, ref["proposals"], atol=2e-3)
        assert torch.equal(l, ref["labels"]) and b.shape == ref["boxes"].shape
        assert torch.allclose(b, ref["boxes"], atol=2e-3)


def _match_rows(a, b, tol=0.75):
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _check(eng, det, ref, k, props, logit_tol=1e-3):
    idx = _match_rows(props, ref["proposals"])
    assert (idx >= 0).all() and k == ref["proposals"].shape[0], "proposals differ"
    assert (eng.last_pred[:k][idx, :31] - ref["class_logits"]).abs().max() < logit_tol, "class logits"
    n = int(det.count.reshape(-1)[0])
    assert n == ref["boxes"].shape[0] and torch.equal(det.labels[:n], ref["labels"]), "detections"
    assert torch.allclose(det.boxes[:n], ref["boxes"], atol=2e-2)


def test_base_engine_matches_reference_fixture():
    """BaseEngine from the model's config, exact-fp32 stand-ins for the kernels"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = _gold("base_r101_s3x3_192x320.pt")
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    img = synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"])
    with cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="base", device="cpu", precision="tf32",
                                                      stride_in_1x1=False)
        eng = engine.BaseEngine(sd, engine_config_from(model.cfg), device="cpu")
        assert eng.backbone.stages.stride_in_1x1 is False
        det = eng.forward(img, gold["w"], gold["h"])
        k = int(eng.last_cnt[0])
        _check(eng, det, gold, k, eng.last_props[:k])


def test_mega_engine_matches_reference_fixture():
    """MegaEngine from the model's config (start_video with look-ahead and global frames, then a steady frame),
    exact-fp32 stand-ins for the kernels"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = _gold("mega_r101_s3x3_192x320.pt")
    h, w, total, gpf = gold["h"], gold["w"], gold["total"], gold["globals_per_frame"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    with cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="mega", device="cpu", precision="tf32",
                                                      stride_in_1x1=False)
        eng = engine.MegaEngine(sd, engine_config_from(model.cfg), device="cpu")
        eng.use_graph = False
        for t in range(2):
            det = (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
                   eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))
            k = int(eng.cur_cnt.view(-1)[0])
            _check(eng, det, gold["frames"][t], k, eng.Bq0[:k])


def test_strided_bottleneck_of_a_dilated_or_unstrided_block_is_the_oracles():
    """the 3x3-strided restatement equals the oracle's bottleneck bit for bit where the layouts agree: a block without a
    stride (res2), and a dilated res5 block, whose stride the reference resets to 1"""
    import stride3x3_oracle
    from mega_core.b200 import synth
    sd = synth.make_state_dict("mega_r50_tiny", seed=4)
    g = torch.Generator().manual_seed(3)
    for p, cin, stride, dil in (("backbone.body.layer1.0.", 64, 1, 1), ("roi_heads.box.feature_extractor.head.layer4.0.",
                                                                        1024, 2, 2)):
        x = torch.randn(1, cin, 12, 20, generator=g)
        assert torch.equal(stride3x3_oracle.bottleneck(x, sd, p, stride, dil), mo.bottleneck(x, sd, p, stride, dil))
