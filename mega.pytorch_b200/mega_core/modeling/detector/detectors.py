"""build_detection_model(cfg) keyed by cfg.MODEL.META_ARCHITECTURE (detector/detectors.py:9-18)."""
import os

from .generalized_rcnn import (GeneralizedRCNN, GeneralizedRCNNDFF, GeneralizedRCNNFGFA, GeneralizedRCNNMEGA,
                               GeneralizedRCNNRDN)

_DETECTION_META_ARCHITECTURES = {"GeneralizedRCNN": GeneralizedRCNN, "GeneralizedRCNNMEGA": GeneralizedRCNNMEGA,
                                 "GeneralizedRCNNRDN": GeneralizedRCNNRDN, "GeneralizedRCNNFGFA": GeneralizedRCNNFGFA,
                                 "GeneralizedRCNNDFF": GeneralizedRCNNDFF}


def build_detection_model(cfg):
    return _DETECTION_META_ARCHITECTURES[cfg.MODEL.META_ARCHITECTURE](cfg)


def vid_config(method="mega", conv_body="R-101-C4", device="cuda", num_groups=1, width_per_group=64, stride_in_1x1=True):
    """the configuration tools/test_net.py ends up with for the VID configs: defaults <- BASE_RCNN_1gpu.yaml
    <- configs/MEGA/vid_R_101_C4_MEGA_1x.yaml (or configs/vid_R_50_C4_1x.yaml for method="base");
    num_groups / width_per_group: MODEL.RESNETS.NUM_GROUPS / WIDTH_PER_GROUP (32 / 8 for a ResNeXt-101 32x8d body);
    stride_in_1x1: MODEL.RESNETS.STRIDE_IN_1X1 (False for the Caffe2 / fb.torch ResNe(X)t and torchvision weights)"""
    from ...config import cfg as base
    c = base.clone()
    c.merge_from_dict({
        "MODEL": {"DEVICE": str(device), "VID": {"ENABLE": True},
                  "RPN": {"ANCHOR_SIZES": (64, 128, 256, 512), "PRE_NMS_TOP_N_TEST": 6000, "POST_NMS_TOP_N_TEST": 300},
                  "ROI_HEADS": {"SCORE_THRESH": 0.001, "NMS": 0.5, "DETECTIONS_PER_IMG": 300},
                  "ROI_BOX_HEAD": {"NUM_CLASSES": 31, "POOLER_RESOLUTION": 7, "PREDICTOR": "FPNPredictor"},
                  "RESNETS": {"RES5_DILATION": 2, "NUM_GROUPS": num_groups, "WIDTH_PER_GROUP": width_per_group,
                              "STRIDE_IN_1X1": bool(stride_in_1x1)},
                  "BACKBONE": {"CONV_BODY": conv_body}},
        "INPUT": {"MIN_SIZE_TEST": 600, "MAX_SIZE_TEST": 1000}, "TEST": {"IMS_PER_BATCH": 1, "DETECTIONS_PER_IMG": 300}})
    if method == "mega":
        c.merge_from_dict({"MODEL": {"META_ARCHITECTURE": "GeneralizedRCNNMEGA",
                                     "VID": {"METHOD": "mega", "ROI_BOX_HEAD": {"ATTENTION": {"ENABLE": True, "STAGE": 3}}},
                                     "ROI_BOX_HEAD": {"FEATURE_EXTRACTOR": "MEGAFeatureExtractor"}}})
    elif method == "rdn":     # configs/RDN/vid_R_101_C4_RDN_1x.yaml
        c.merge_from_dict({"MODEL": {"META_ARCHITECTURE": "GeneralizedRCNNRDN",
                                     "VID": {"METHOD": "rdn", "IGNORE": True,
                                             "ROI_BOX_HEAD": {"ATTENTION": {"ENABLE": True, "STAGE": 2, "ADVANCED_STAGE": 1}}},
                                     "ROI_BOX_HEAD": {"FEATURE_EXTRACTOR": "RDNFeatureExtractor"}}})
    elif method == "fgfa":    # configs/FGFA/vid_R_101_C4_FGFA_1x.yaml
        c.merge_from_dict({"MODEL": {"META_ARCHITECTURE": "GeneralizedRCNNFGFA", "VID": {"METHOD": "fgfa"},
                                     "ROI_BOX_HEAD": {"FEATURE_EXTRACTOR": "ResNetConv52MLPFeatureExtractor"}}})
    elif method == "dff":     # configs/DFF/vid_R_101_C4_DFF_1x.yaml
        c.merge_from_dict({"MODEL": {"META_ARCHITECTURE": "GeneralizedRCNNDFF", "VID": {"METHOD": "dff"},
                                     "ROI_BOX_HEAD": {"FEATURE_EXTRACTOR": "ResNetConv52MLPFeatureExtractor"}}})
    elif method == "base":
        c.merge_from_dict({"MODEL": {"META_ARCHITECTURE": "GeneralizedRCNN",
                                     "VID": {"METHOD": "base", "ROI_BOX_HEAD": {"REDUCE_CHANNEL": True}},
                                     "ROI_BOX_HEAD": {"FEATURE_EXTRACTOR": "ResNetConv52MLPFeatureExtractor"}}})
    else:
        raise ValueError(method)
    return c


def build_detection_model_from_state_dict(sd, method="mega", device="cuda", precision=None, stride_in_1x1=True):
    """convenience for benchmarks/tests: infer the conv body (depth, ResNeXt groups and width), REDUCE_CHANNEL, MEGA's
    GLOBAL.RES_STAGE and RDN's ADVANCED_STAGE from the state dict, build, load, eval. stride_in_1x1
    (MODEL.RESNETS.STRIDE_IN_1X1) is given by the caller: both stride layouts have the same keys and shapes, so the
    weights cannot tell which one they were trained with"""
    fe = "roi_heads.box.feature_extractor."
    n3 = 0
    while ("backbone.body.layer3.%d.conv1.weight" % n3) in sd:
        n3 += 1
    body = {6: "R-50-C4", 23: "R-101-C4"}.get(n3)
    l1 = "backbone.body.layer1.0.conv2."
    w2 = sd[l1 + "conv.weight"] if (l1 + "conv.weight") in sd else sd[l1 + "weight"]     # [G * width, width, 3, 3]
    cfg = vid_config(method, body or "R-101-C4", device, num_groups=w2.shape[0] // w2.shape[1],
                     width_per_group=w2.shape[1], stride_in_1x1=stride_in_1x1)
    # MODEL.RESNETS.STAGE_WITH_DCN / WITH_MODULATED_DCN / DEFORMABLE_GROUPS: a deformable conv2 keeps its weight as
    # conv2.conv.weight beside the offset conv conv2.offset.* (18 or 27 output channels per deformable group)
    offsets = [sd.get("backbone.body.layer%d.0.conv2.offset.weight" % li) for li in (1, 2, 3)]
    if any(o is not None for o in offsets):
        k = next(o for o in offsets if o is not None).shape[0]
        r = cfg.MODEL.RESNETS
        r.STAGE_WITH_DCN = tuple(o is not None for o in offsets) + (False,)
        r.WITH_MODULATED_DCN = k % 27 == 0
        r.DEFORMABLE_GROUPS = k // (27 if r.WITH_MODULATED_DCN else 18)
    if precision is not None:
        cfg.MODEL.B200.PRECISION = precision
    cfg.MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL = (fe + "conv.weight") in sd
    count = lambda name: sum(1 for k in sd if k.startswith(fe + name) and k.endswith(".weight"))     # noqa: E731
    if method == "mega":
        cfg.MODEL.VID.MEGA.GLOBAL.RES_STAGE = count("g_Wqs.") - 1
    elif method == "rdn":
        att = cfg.MODEL.VID.ROI_BOX_HEAD.ATTENTION
        att.ADVANCED_STAGE = 0 if count("Wqs.") == att.STAGE else 1
    model = build_detection_model(cfg)
    if body is None:
        model.adopt_state_dict(sd)          # non-standard depth (tests): skip the module tree, feed the engine
    else:
        missing = model.load_state_dict(sd, strict=False)
        assert not [k for k in missing.missing_keys if "cell_anchors" not in k], missing.missing_keys
        assert not missing.unexpected_keys, missing.unexpected_keys
    return model.eval()
