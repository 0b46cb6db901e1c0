"""Parameter-holding module tree with the reference's attribute / state_dict names.

The reference's checkpoints (e.g. MEGA_R_101.pth) load through `load_state_dict` because every
parameter and buffer keeps its name and shape: backbone.body.{stem,layer1..3}, rpn.head.*,
rpn.anchor_generator.cell_anchors.0, roi_heads.box.feature_extractor.{head.layer4, l_fcs, l_Wgs,
l_Wqs, l_Wks, l_Wvs, l_us, g_Wqs, g_Wks, g_Wvs, g_us}, roi_heads.box.predictor.{cls_score,bbox_pred}
(reference: modeling/backbone/resnet.py, rpn/rpn.py, roi_heads/box_head/*). The torch modules below
only HOLD the tensors; all arithmetic runs in the B200 engine (mega_core/b200/engine.py).
"""
import os
import weakref

import torch
from torch import nn

from . import registry
from ..layers import Conv2d, DFConv2d, FrozenBatchNorm2d
from ..b200 import engine as _engine

BLOCKS = {"R-50-C4": (3, 4, 6), "R-101-C4": (3, 4, 23)}


class _EngineServed(object):
    """mix-in of the sub-modules a caller of the reference may invoke on its own (model.backbone, model.rpn,
    model.roi_heads.box.feature_extractor): their forward() runs on the detector's engine. The detector registers
    itself with `_bind` (a weak reference: the parent must not become a sub-module of its child)."""

    def _bind(self, detector):
        object.__setattr__(self, "_detector_ref", weakref.ref(detector))

    @property
    def _engine(self):
        ref = getattr(self, "_detector_ref", None)
        det = ref() if ref is not None else None
        if det is None:
            raise RuntimeError("this sub-module computes through its detector's B200 engine; build it with "
                               "build_detection_model(cfg)")
        return det.engine


def _image_size(images):
    """(w, h) of the first image of an ImageList / tensor, as AnchorGenerator reads it (anchor_generator.py:112-125)"""
    if hasattr(images, "image_sizes"):
        h, w = images.image_sizes[0]
        return int(w), int(h)
    t = images.tensors if hasattr(images, "tensors") else images
    return int(t.shape[-1]), int(t.shape[-2])


class Bottleneck(nn.Module):
    def __init__(self, cin, mid, cout, stride, dilation, groups=1, stride_in_1x1=True, dcn=None):
        super().__init__()
        if cin != cout:
            self.downsample = nn.Sequential(Conv2d(cin, cout, 1, stride=(stride if dilation == 1 else 1), bias=False),
                                            FrozenBatchNorm2d(cout))
        if dilation > 1:
            stride = 1
        s1, s3 = (stride, 1) if stride_in_1x1 else (1, stride)          # resnet.py:272-275
        self.conv1 = Conv2d(cin, mid, 1, stride=s1, bias=False)
        self.bn1 = FrozenBatchNorm2d(mid)
        if dcn is not None:         # resnet.py:286-299: dcn = (with_modulated_dcn, deformable_groups)
            self.conv2 = DFConv2d(mid, mid, with_modulated_dcn=dcn[0], kernel_size=3, stride=s3, groups=groups,
                                  dilation=dilation, deformable_groups=dcn[1], bias=False)
        else:
            self.conv2 = Conv2d(mid, mid, 3, stride=s3, padding=dilation, dilation=dilation, groups=groups, bias=False)
        self.bn2 = FrozenBatchNorm2d(mid)
        self.conv3 = Conv2d(mid, cout, 1, bias=False)
        self.bn3 = FrozenBatchNorm2d(cout)


def _stage(cin, mid, cout, n, stride, dilation=1, groups=1, stride_in_1x1=True, dcn=None):
    blocks = []
    for i in range(n):
        blocks.append(Bottleneck(cin if i == 0 else cout, mid, cout, stride if i == 0 else 1, dilation, groups,
                                 stride_in_1x1, dcn))
    return nn.Sequential(*blocks)


def stage_dcn(cfg, stage):
    """(with_modulated_dcn, deformable_groups) of res`stage+1` when MODEL.RESNETS.STAGE_WITH_DCN marks it, else None
    (resnet.py:110-124)"""
    r = cfg.MODEL.RESNETS
    return (bool(r.WITH_MODULATED_DCN), r.DEFORMABLE_GROUPS) if r.STAGE_WITH_DCN[stage - 1] else None


def bottleneck_width(cfg, stage):
    """conv1 / conv2 width of res`stage+1` (resnet.py:98-108): NUM_GROUPS * WIDTH_PER_GROUP * 2^(stage-1)"""
    r = cfg.MODEL.RESNETS
    return r.NUM_GROUPS * r.WIDTH_PER_GROUP * 2 ** (stage - 1)


class Stem(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = FrozenBatchNorm2d(64)


class ResNetBody(nn.Module):
    """`backbone.body` (modeling/backbone/resnet.py:81-152)"""

    def __init__(self, cfg):
        super().__init__()
        b = BLOCKS[cfg.MODEL.BACKBONE.CONV_BODY]
        g, s1x1 = cfg.MODEL.RESNETS.NUM_GROUPS, cfg.MODEL.RESNETS.STRIDE_IN_1X1
        self.stem = Stem()
        self.layer1 = _stage(64, bottleneck_width(cfg, 1), 256, b[0], 1, groups=g, stride_in_1x1=s1x1,
                             dcn=stage_dcn(cfg, 1))
        self.layer2 = _stage(256, bottleneck_width(cfg, 2), 512, b[1], 2, groups=g, stride_in_1x1=s1x1,
                             dcn=stage_dcn(cfg, 2))
        self.layer3 = _stage(512, bottleneck_width(cfg, 3), 1024, b[2], 2, groups=g, stride_in_1x1=s1x1,
                             dcn=stage_dcn(cfg, 3))
        self.out_channels = 1024


class ResNetHead(nn.Module):
    """res5 as `feature_extractor.head` (resnet.py:155-204; stride_init=1)"""

    def __init__(self, cfg):
        super().__init__()
        self.layer4 = _stage(1024, bottleneck_width(cfg, 4), 2048, 3, 1, cfg.MODEL.RESNETS.RES5_DILATION,
                             cfg.MODEL.RESNETS.NUM_GROUPS)
        self.out_channels = 2048


class _Backbone(nn.Sequential, _EngineServed):
    """`model.backbone` = Sequential(body) (backbone/backbone.py:16-20); forward(x [n,3,H,W]) -> [feats [n,1024,H/16,W/16]]
    like ResNet.forward (resnet.py:145-152), computed by the detector's engine"""

    def forward(self, x):
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        x = x.tensors if hasattr(x, "tensors") else x
        eng = self._engine
        with torch.no_grad():
            return [eng.backbone_nchw(x.to(eng.dev).float().contiguous())]


@registry.BACKBONES.register("R-50-C4")
@registry.BACKBONES.register("R-101-C4")
def build_resnet_backbone(cfg):
    model = _Backbone()
    model.add_module("body", ResNetBody(cfg))
    model.out_channels = cfg.MODEL.RESNETS.BACKBONE_OUT_CHANNELS
    return model


class BufferList(nn.Module):
    def __init__(self, buffers):
        super().__init__()
        for i, b in enumerate(buffers):
            self.register_buffer(str(i), b)


class AnchorGenerator(nn.Module):
    def __init__(self, sizes, ratios, stride):
        super().__init__()
        self.strides = (stride,)
        self.cell_anchors = BufferList([_engine.cell_anchors(stride, sizes, ratios)])

    def num_anchors_per_location(self):
        return [self.cell_anchors._buffers["0"].shape[0]]


@registry.RPN_HEADS.register("SingleConvRPNHead")
class RPNHead(nn.Module):
    def __init__(self, cfg, in_channels, num_anchors):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, in_channels, 3, padding=1)
        self.cls_logits = nn.Conv2d(in_channels, num_anchors, 1)
        self.bbox_pred = nn.Conv2d(in_channels, num_anchors * 4, 1)


class RPNModule(nn.Module, _EngineServed):
    """`model.rpn` (rpn/rpn.py:109-243): holds head + anchors; forward() is served by the detector's engine"""

    def __init__(self, cfg, in_channels):
        super().__init__()
        r = cfg.MODEL.RPN
        self.anchor_generator = AnchorGenerator(r.ANCHOR_SIZES, r.ASPECT_RATIOS, r.ANCHOR_STRIDE[0])
        self.head = registry.RPN_HEADS[r.RPN_HEAD](cfg, in_channels, self.anchor_generator.num_anchors_per_location()[0])

    def forward(self, images, features, targets=None, version="key"):
        """RPNWithRefModule.forward in eval mode (rpn/rpn.py:213-243): `features` = (feats [n,1024,h,w],) as
        model.backbone returns them; version "key" -> POST_NMS_TOP_N_TEST proposals, "ref" -> REF_POST_NMS_TOP_N.
        Returns list[BoxList] with the field `objectness` (rpn/inference.py:118-123), one per image."""
        if self.training:
            raise NotImplementedError("the B200 build covers inference (eval mode) only")
        from ..structures.bounding_box import BoxList
        eng = self._engine
        im_w, im_h = _image_size(images)
        post = eng.cfg.post_nms_top_n if version == "key" else eng.cfg.ref_post_nms_top_n
        with torch.no_grad():
            boxes, scores, cnt = eng.rpn_nchw(features[0], im_w, im_h, post)
        out = []
        for i, k in enumerate(cnt.tolist()):
            bl = BoxList(boxes[i, :k], (im_w, im_h), mode="xyxy")
            bl.add_field("objectness", scores[i, :k])
            out.append(bl)
        return out


def _fc(i, o):
    return nn.Linear(i, o)


def _reduce_channel(extractor, cfg):
    """MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL (roi_box_feature_extractors.py:274-283, :474-483): a 1x1 conv 2048 -> 256
    (+ ReLU) between res5 and ROIAlign as `extractor.conv`; returns the channel count ROIAlign pools"""
    if cfg.MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL:
        extractor.conv = nn.Conv2d(2048, 256, 1)
        return 256
    extractor.conv = None
    return 2048


@registry.ROI_BOX_FEATURE_EXTRACTORS.register("ResNetConv52MLPFeatureExtractor")
class ResNetConv52MLPFeatureExtractor(nn.Module):
    def __init__(self, cfg, in_channels):
        super().__init__()
        self.head = ResNetHead(cfg)
        ch = _reduce_channel(self, cfg)
        res = cfg.MODEL.ROI_BOX_HEAD.POOLER_RESOLUTION
        dim = cfg.MODEL.ROI_BOX_HEAD.MLP_HEAD_DIM
        self.fc6 = _fc(ch * res * res, dim)
        self.fc7 = _fc(dim, dim)
        self.out_channels = dim


class _WindowedExtractorForward(_EngineServed):
    def forward(self, x, proposals, pre_calculate=False):
        """pre_calculate=True (extractors :885-896 / :401-410): x = feats [n,1024,h,w] (model.backbone's output or a tuple
        holding it), proposals = list[BoxList], one per image -> ROI features [sum K, 1024] after fcs[0] + ReLU.
        The aggregation call (pre_calculate=False, extractors :898-933) reads the per-video state the DETECTOR keeps in the
        engine's ring buffers; it is served through model(images) only."""
        if not pre_calculate:
            raise NotImplementedError("feature_extractor(x, proposals_list): the aggregation over window / global pool / "
                                      "memory runs inside model(images) (MegaEngine.aggregate); call the detector")
        x = x[0] if isinstance(x, (tuple, list)) else x
        boxes = torch.cat([p.bbox for p in proposals], 0).float()
        bidx = torch.cat([torch.full((len(p),), i, dtype=torch.int32) for i, p in enumerate(proposals)]).to(boxes.device)
        with torch.no_grad():
            return self._engine.roi_features(x, boxes, bidx)


@registry.ROI_BOX_FEATURE_EXTRACTORS.register("MEGAFeatureExtractor")
class MEGAFeatureExtractor(_WindowedExtractorForward, nn.Module):
    """parameters of roi_box_feature_extractors.py:457-565; forward(pre_calculate=True) / init_memory / init_global /
    update_global (:657-676) act on the detector's engine"""

    def init_memory(self):
        self._engine.init_memory()

    def init_global(self):
        self._engine.init_global()

    def update_global(self, feats):
        self._engine.update_global(feats)

    def __init__(self, cfg, in_channels):
        super().__init__()
        self.head = ResNetHead(cfg)
        ch = _reduce_channel(self, cfg)
        res = cfg.MODEL.ROI_BOX_HEAD.POOLER_RESOLUTION
        dim = cfg.MODEL.ROI_BOX_HEAD.MLP_HEAD_DIM
        att = cfg.MODEL.VID.ROI_BOX_HEAD.ATTENTION
        emb, grp, stages = att.EMBED_DIM, att.GROUP, att.STAGE
        self.l_fcs = nn.ModuleList([_fc(ch * res * res if i == 0 else dim, dim) for i in range(stages)])
        self.l_Wgs = nn.ModuleList([nn.Conv2d(emb, grp, 1) for _ in range(stages)])
        self.l_Wqs = nn.ModuleList([_fc(dim, dim) for _ in range(stages)])
        self.l_Wks = nn.ModuleList([_fc(dim, dim) for _ in range(stages)])
        self.l_Wvs = nn.ModuleList([nn.Conv2d(dim * grp, dim, 1, groups=grp) for _ in range(stages)])
        self.l_us = nn.ParameterList([nn.Parameter(torch.zeros(grp, 1, emb)) for _ in range(stages)])
        g = cfg.MODEL.VID.MEGA.GLOBAL.RES_STAGE + 1
        self.g_Wqs = nn.ModuleList([_fc(dim, dim) for _ in range(g)])
        self.g_Wks = nn.ModuleList([_fc(dim, dim) for _ in range(g)])
        self.g_Wvs = nn.ModuleList([nn.Conv2d(dim * grp, dim, 1, groups=grp) for _ in range(g)])
        self.g_us = nn.ParameterList([nn.Parameter(torch.zeros(grp, 1, emb)) for _ in range(g)])
        self.out_channels = dim


@registry.ROI_BOX_FEATURE_EXTRACTORS.register("RDNFeatureExtractor")
class RDNFeatureExtractor(_WindowedExtractorForward, nn.Module):
    """parameters of roi_box_feature_extractors.py:254-330 (fcs, Wgs, Wqs, Wks, Wvs; no `u`)"""

    def __init__(self, cfg, in_channels):
        super().__init__()
        self.head = ResNetHead(cfg)
        ch = _reduce_channel(self, cfg)
        res = cfg.MODEL.ROI_BOX_HEAD.POOLER_RESOLUTION
        dim = cfg.MODEL.ROI_BOX_HEAD.MLP_HEAD_DIM
        att = cfg.MODEL.VID.ROI_BOX_HEAD.ATTENTION
        emb, grp, base, adv = att.EMBED_DIM, att.GROUP, att.STAGE, att.ADVANCED_STAGE
        n_att = base if adv == 0 else base + adv + 1
        n_fc = base if adv == 0 else base + adv
        self.fcs = nn.ModuleList([_fc(ch * res * res if i == 0 else dim, dim) for i in range(n_fc)])
        self.Wgs = nn.ModuleList([nn.Conv2d(emb, grp, 1) for _ in range(n_att)])
        self.Wqs = nn.ModuleList([_fc(dim, dim) for _ in range(n_att)])
        self.Wks = nn.ModuleList([_fc(dim, dim) for _ in range(n_att)])
        self.Wvs = nn.ModuleList([nn.Conv2d(dim * grp, dim, 1, groups=grp) for _ in range(n_att)])
        self.out_channels = dim


@registry.ROI_BOX_PREDICTOR.register("FPNPredictor")
class FPNPredictor(nn.Module):
    def __init__(self, cfg, in_channels):
        super().__init__()
        n = cfg.MODEL.ROI_BOX_HEAD.NUM_CLASSES
        self.cls_score = nn.Linear(in_channels, n)
        self.bbox_pred = nn.Linear(in_channels, (2 if cfg.MODEL.CLS_AGNOSTIC_BBOX_REG else n) * 4)


class ROIBoxHead(nn.Module):
    """`model.roi_heads.box` (box_head/box_head.py:11-124): feature_extractor + predictor"""

    def __init__(self, cfg, in_channels):
        super().__init__()
        fe = registry.ROI_BOX_FEATURE_EXTRACTORS[cfg.MODEL.ROI_BOX_HEAD.FEATURE_EXTRACTOR]
        self.feature_extractor = fe(cfg, in_channels)
        pr = registry.ROI_BOX_PREDICTOR[cfg.MODEL.ROI_BOX_HEAD.PREDICTOR]
        self.predictor = pr(cfg, self.feature_extractor.out_channels)


class CombinedROIHeads(nn.ModuleDict):
    """`model.roi_heads` (roi_heads/roi_heads.py:9-76), box head only (MASK_ON / KEYPOINT_ON are False)"""

    def __init__(self, cfg, heads):
        super().__init__(heads)
        self.cfg = cfg.clone()


class FlowNetS(nn.Module):
    """parameters of modeling/backbone/flownet.py:14-50 (methods "fgfa" and "dff")"""

    def __init__(self, cfg):
        super().__init__()
        self.flow_conv1 = nn.Conv2d(6, 64, 7, stride=2, padding=3)
        self.conv2 = nn.Conv2d(64, 128, 5, stride=2, padding=2)
        self.conv3 = nn.Conv2d(128, 256, 5, stride=2, padding=2)
        self.conv3_1 = nn.Conv2d(256, 256, 3, padding=1)
        self.conv4 = nn.Conv2d(256, 512, 3, stride=2, padding=1)
        self.conv4_1 = nn.Conv2d(512, 512, 3, padding=1)
        self.conv5 = nn.Conv2d(512, 512, 3, stride=2, padding=1)
        self.conv5_1 = nn.Conv2d(512, 512, 3, padding=1)
        self.conv6 = nn.Conv2d(512, 1024, 3, stride=2, padding=1)
        self.conv6_1 = nn.Conv2d(1024, 1024, 3, padding=1)
        for i, cin in zip(range(1, 6), (1024, 1026, 770, 386, 194)):
            setattr(self, "Convolution%d" % i, nn.Conv2d(cin, 2, 3, padding=1))
        self.deconv5 = nn.ConvTranspose2d(1024, 512, 4, stride=2)
        self.deconv4 = nn.ConvTranspose2d(1026, 256, 4, stride=2)
        self.deconv3 = nn.ConvTranspose2d(770, 128, 4, stride=2)
        self.deconv2 = nn.ConvTranspose2d(386, 64, 4, stride=2)
        for n_ in ("6to5", "5to4", "4to3", "3to2"):
            setattr(self, "upsample_flow" + n_, nn.ConvTranspose2d(2, 2, 4, stride=2))
        if cfg.MODEL.VID.METHOD == "dff":                      # flownet.py:36-38: zero-initialised scale head
            self.Convolution5_scale = nn.Conv2d(194, 1024, 1, bias=False)
            nn.init.zeros_(self.Convolution5_scale.weight)


class EmbedNet(nn.Module):
    """parameters of modeling/backbone/embednet.py:9-17"""

    def __init__(self, cfg):
        super().__init__()
        self.embed_conv1 = nn.Conv2d(1024, 512, 1)
        self.embed_conv2 = nn.Conv2d(512, 512, 3, padding=1)
        self.embed_conv3 = nn.Conv2d(512, 2048, 1)


def build_backbone(cfg):
    return registry.BACKBONES[cfg.MODEL.BACKBONE.CONV_BODY](cfg)


def build_rpn(cfg, in_channels):
    return RPNModule(cfg, in_channels)


def build_roi_heads(cfg, in_channels):
    """roi_heads.py:58-76: under MODEL.RPN_ONLY no head at all (an empty list, falsy like the reference's), so the model's
    state_dict holds no roi_heads.* entries and the detector returns the RPN's proposals"""
    if cfg.MODEL.RPN_ONLY:
        return []
    return CombinedROIHeads(cfg, [("box", ROIBoxHead(cfg, in_channels))])


def engine_config_from(cfg):
    """reference config -> EngineConfig. Keys that change the reference's behaviour but whose non-default values the
    engines do not implement are REJECTED here instead of being ignored (a non-default YAML must not give silently
    different detections)."""
    m = cfg.MODEL
    v = m.VID
    win = {"rdn": v.RDN, "fgfa": v.FGFA}.get(v.METHOD, v.MEGA)     # window geometry of the method
    unsupported = []
    if v.METHOD in ("rdn", "mega") and v.RPN.REF_PRE_NMS_TOP_N != m.RPN.PRE_NMS_TOP_N_TEST:
        unsupported.append("MODEL.VID.RPN.REF_PRE_NMS_TOP_N != MODEL.RPN.PRE_NMS_TOP_N_TEST (the reference proposals of a frame "
                           "are taken as the prefix of its key proposals, which needs equal pre-NMS sets)")
    g, wpg = m.RESNETS.NUM_GROUPS, m.RESNETS.WIDTH_PER_GROUP
    for stage in (1, 2, 3, 4):
        width, gw = g * wpg * 2 ** (stage - 1), wpg * 2 ** (stage - 1)
        if width % 64 or (g > 1 and gw not in (8, 16, 32, 64)):
            unsupported.append("MODEL.RESNETS.NUM_GROUPS = %d / WIDTH_PER_GROUP = %d (res%d: bottleneck width %d, group "
                               "width %d; the kernels serve widths in multiples of 64 and group widths 8, 16, 32 or 64)"
                               % (g, wpg, stage + 1, width, gw))
            break
    dcn = tuple(m.RESNETS.STAGE_WITH_DCN)
    if any(dcn):
        if dcn[3]:
            unsupported.append("MODEL.RESNETS.STAGE_WITH_DCN = %s (the 4th entry, res5, must be False: in the C4 models "
                               "res5 is the box head's ResNetHead, which the reference builds without a deformable "
                               "conv, so the entry would be ignored)" % (dcn,))
        if g > 1:
            unsupported.append("MODEL.RESNETS.STAGE_WITH_DCN = %s with MODEL.RESNETS.NUM_GROUPS = %d (deformable "
                               "stages are served with dense conv2, NUM_GROUPS 1)" % (dcn, g))
        dg = m.RESNETS.DEFORMABLE_GROUPS
        widths = [bottleneck_width(cfg, stage) for stage in (1, 2, 3) if dcn[stage - 1]]
        if dg != 1 and m.RESNETS.WITH_MODULATED_DCN:
            unsupported.append("MODEL.RESNETS.DEFORMABLE_GROUPS = %d with MODEL.RESNETS.WITH_MODULATED_DCN (modulated "
                               "stages are served with one deformable group; the reference's modulated conv slices its "
                               "18 offsets and 9 masks for one group, layers/misc.py:182-184)" % dg)
        elif dg < 1 or any(c % dg or c // dg % 8 for c in widths):
            unsupported.append("MODEL.RESNETS.DEFORMABLE_GROUPS = %d (each deformable group samples a multiple of 8 "
                               "channels: the group count must divide every deformable stage's conv2 width, here %s, "
                               "into multiples of 8)" % (dg, "/".join(str(c) for c in widths)))
    att = v.ROI_BOX_HEAD.ATTENTION
    if v.METHOD == "mega":
        if not v.MEGA.GLOBAL.ENABLE:
            unsupported.append("MODEL.VID.MEGA.GLOBAL.ENABLE = False (the reference cannot run it at test time: "
                               "MEGAFeatureExtractor._forward_test reads global_res_stage, which it sets only when the "
                               "global stage is enabled, roi_box_feature_extractors.py:542-545)")
        if att.STAGE != 3:
            unsupported.append("MODEL.VID.ROI_BOX_HEAD.ATTENTION.STAGE = %d (MegaEngine runs 3 local stages)" % att.STAGE)
        if v.MEGA.GLOBAL.RES_STAGE not in (0, 1):
            unsupported.append("MODEL.VID.MEGA.GLOBAL.RES_STAGE = %d (MegaEngine runs 0 or 1 global stages after the "
                               "local ones)" % v.MEGA.GLOBAL.RES_STAGE)
    if v.METHOD == "rdn":
        if att.STAGE != 2:
            unsupported.append("MODEL.VID.ROI_BOX_HEAD.ATTENTION.STAGE = %d (RdnEngine runs 2 base stages)" % att.STAGE)
        if att.ADVANCED_STAGE not in (0, 1):
            unsupported.append("MODEL.VID.ROI_BOX_HEAD.ATTENTION.ADVANCED_STAGE = %d (RdnEngine runs 0 or 1 advanced "
                               "stages)" % att.ADVANCED_STAGE)
    if m.RPN_ONLY:
        if v.METHOD in ("mega", "rdn"):
            unsupported.append("MODEL.RPN_ONLY with MODEL.VID.METHOD '%s' (its test path reads the box head's feature "
                               "extractor, which an RPN-only model does not have; served for 'base', 'dff' and 'fgfa')"
                               % v.METHOD)
        if cfg.TEST.BBOX_AUG.ENABLED:
            unsupported.append("MODEL.RPN_ONLY with TEST.BBOX_AUG.ENABLED (test-time augmentation merges class "
                               "detections, an RPN-only model returns proposals)")
        if "B200" in m and m.B200.SEQ_NMS.ENABLED:
            unsupported.append("MODEL.RPN_ONLY with MODEL.B200.SEQ_NMS.ENABLED (Seq-NMS links and rescores class "
                               "detections by `scores` and `labels`, which proposals do not carry)")
    if unsupported:
        raise NotImplementedError("mega_core (B200 build): " + "; ".join(unsupported))
    # the reference sizes the long-range memory deques with ALL_FRAME_INTERVAL (roi_box_feature_extractors.py:660-668:
    # deque(maxlen=self.all_frame_interval)); MODEL.VID.MEGA.MEMORY.SIZE is not read at test time
    memory_size = v.MEGA.ALL_FRAME_INTERVAL if v.METHOD == "mega" else v.MEGA.MEMORY.SIZE
    return _engine.EngineConfig(
        pre_nms_top_n=m.RPN.PRE_NMS_TOP_N_TEST, post_nms_top_n=m.RPN.POST_NMS_TOP_N_TEST,
        ref_post_nms_top_n=v.RPN.REF_POST_NMS_TOP_N, rpn_nms_thresh=m.RPN.NMS_THRESH, rpn_min_size=m.RPN.MIN_SIZE,
        ratio=win.get("RATIO", 0.2), all_frame_interval=win.ALL_FRAME_INTERVAL, key_frame_location=win.KEY_FRAME_LOCATION,
        advanced_stage=v.ROI_BOX_HEAD.ATTENTION.ADVANCED_STAGE,
        memory_size=memory_size, global_size=v.MEGA.GLOBAL.SIZE, global_res_stage=v.MEGA.GLOBAL.RES_STAGE,
        stage=v.ROI_BOX_HEAD.ATTENTION.STAGE, groups=v.ROI_BOX_HEAD.ATTENTION.GROUP,
        pooler_resolution=m.ROI_BOX_HEAD.POOLER_RESOLUTION, pooler_scale=m.ROI_BOX_HEAD.POOLER_SCALES[0],
        sampling_ratio=m.ROI_BOX_HEAD.POOLER_SAMPLING_RATIO, res5_dilation=m.RESNETS.RES5_DILATION,
        score_thresh=m.ROI_HEADS.SCORE_THRESH, nms_thresh=m.ROI_HEADS.NMS, detections_per_img=m.ROI_HEADS.DETECTIONS_PER_IMG,
        bbox_reg_weights=tuple(m.ROI_HEADS.BBOX_REG_WEIGHTS), anchor_sizes=tuple(m.RPN.ANCHOR_SIZES),
        aspect_ratios=tuple(m.RPN.ASPECT_RATIOS), anchor_stride=m.RPN.ANCHOR_STRIDE[0],
        num_classes=m.ROI_BOX_HEAD.NUM_CLASSES,
        precision=os.environ.get("MEGA_B200_PRECISION", m.B200.PRECISION if "B200" in m else "f16"),
        **({"rpn_only": True} if m.RPN_ONLY else {}),
        **({"memory": False} if v.METHOD == "mega" and not v.MEGA.MEMORY.ENABLE else {}),
        **({} if m.RESNETS.STRIDE_IN_1X1 else {"stride_in_1x1": False}))
