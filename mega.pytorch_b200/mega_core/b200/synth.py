"""Synthetic video frames and a deterministic, calibration-free random initialisation.

There is no network for datasets or checkpoints, so benchmarks and parity tests use seeded
synthetic inputs. The stock initialisers of the reference give activations of O(1e2..1e3) on
0-255 inputs and NaN logits in the reference itself (SURVEY.md section 7, "hard parts"), so
this routine keeps the reference's parameter *shapes and names* but picks values analytically
so that every layer's output is O(1) -- like a trained net -- without any data-dependent
calibration (both the oracle and the CUDA path regenerate the identical state_dict from a seed;
the 690 MB of weights are never stored).
"""
import math

import numpy as np
import torch

PIXEL_MEAN = (102.9801, 115.9465, 122.7717)  # config/defaults.py:51-55 (BGR, 0-255 domain)


def synthetic_frame(index, height=600, width=1000, seed=1000, boxes=4):
    """fp32 [1,3,H,W] frame in the reference's post-transform domain (BGR*255 - mean):
    low-amplitude noise background with a few moving bright rectangles so that RPN scores are
    spread out (few exact ties) and detections move coherently."""
    g = torch.Generator().manual_seed(seed + index)
    img = torch.rand(3, height, width, generator=g) * 64.0 + 64.0
    gb = torch.Generator().manual_seed(seed)  # rectangle layout fixed per video, moves with index
    for b in range(boxes):
        bw = int(torch.randint(width // 10, width // 3, (1,), generator=gb))
        bh = int(torch.randint(height // 8, height // 2, (1,), generator=gb))
        x0 = int(torch.randint(0, width - bw, (1,), generator=gb))
        y0 = int(torch.randint(0, height - bh, (1,), generator=gb))
        vx = int(torch.randint(-6, 7, (1,), generator=gb))
        vy = int(torch.randint(-4, 5, (1,), generator=gb))
        col = torch.rand(3, 1, 1, generator=gb) * 200.0 + 30.0
        x = min(max(x0 + vx * index, 0), width - bw)
        y = min(max(y0 + vy * index, 0), height - bh)
        img[:, y:y + bh, x:x + bw] = col + torch.rand(3, bh, bw, generator=g) * 16.0
    img = img - torch.tensor(PIXEL_MEAN).view(3, 1, 1)
    return img.unsqueeze(0).contiguous()


def synthetic_image_u8(height, width, seed=5, blobs=12):
    """uint8 [H, W, 3] RGB image, as a decoder would hand it to the input transform: flat-coloured discs on a black
    background plus uniform noise in [-20, 20]. Integer arithmetic only, so every machine regenerates the same bytes."""
    g = torch.Generator().manual_seed(seed)
    yy = torch.arange(height).view(-1, 1)
    xx = torch.arange(width).view(1, -1)
    img = torch.zeros(height, width, 3, dtype=torch.int64)
    for _ in range(blobs):
        cy = int(torch.randint(0, height, (1,), generator=g))
        cx = int(torch.randint(0, width, (1,), generator=g))
        r = int(torch.randint(10, 60, (1,), generator=g))
        col = torch.randint(0, 256, (3,), generator=g)
        m = ((yy - cy) ** 2 + (xx - cx) ** 2) < r * r
        img[m] = col
    img = img + torch.randint(-20, 21, (height, width, 3), generator=g)
    return img.clamp(0, 255).to(torch.uint8)


def _kaiming(shape, gen, gain=math.sqrt(2.0)):
    fan_in = 1
    for d in shape[1:]:
        fan_in *= d
    return torch.randn(*shape, generator=gen) * (gain / math.sqrt(fan_in))


def _bn(sd, p, n, gen, out_scale=1.0, in_var=1.0):
    """FrozenBatchNorm2d buffers (layers/batch_norm.py:15-18). scale = weight * rsqrt(var)."""
    sd[p + "weight"] = (torch.rand(n, generator=gen) * 0.2 + 0.9) * out_scale
    sd[p + "bias"] = torch.randn(n, generator=gen) * 0.1
    sd[p + "running_mean"] = torch.randn(n, generator=gen) * 0.1 * math.sqrt(in_var)
    sd[p + "running_var"] = (torch.rand(n, generator=gen) * 0.2 + 0.9) * in_var


def _stage(sd, prefix, gen, cin, mid, cout, blocks, groups=1):
    for b in range(blocks):
        p = prefix + "%d." % b
        if b == 0:
            sd[p + "downsample.0.weight"] = _kaiming((cout, cin, 1, 1), gen, gain=1.0)
            _bn(sd, p + "downsample.1.", cout, gen)
        sd[p + "conv1.weight"] = _kaiming((mid, cin if b == 0 else cout, 1, 1), gen)
        _bn(sd, p + "bn1.", mid, gen)
        sd[p + "conv2.weight"] = _kaiming((mid, mid // groups, 3, 3), gen)
        _bn(sd, p + "bn2.", mid, gen)
        sd[p + "conv3.weight"] = _kaiming((cout, mid, 1, 1), gen)
        _bn(sd, p + "bn3.", cout, gen, out_scale=0.25)   # damp the residual branch
    return cout


def _linear(sd, p, nout, nin, gen, std=None, gain=1.0):
    std = std if std is not None else gain / math.sqrt(nin)
    sd[p + "weight"] = torch.randn(nout, nin, generator=gen) * std
    sd[p + "bias"] = torch.randn(nout, generator=gen) * 0.01


def make_state_dict(arch="mega_r101", seed=0, num_classes=31, reduce_channel=False, global_res_stage=1, advanced_stage=1):
    """state_dict with the reference's key names/shapes for
    arch in {"mega_r101", "mega_r50", "rdn_r101", "fgfa_r101", "dff_r101", "base_r50", "base_r101", "mega_x101", "base_x101"}
    (+ "_tiny" suffix: 1 block per stage, for fast CPU tests). x101: ResNeXt-101 32x8d (NUM_GROUPS 32, WIDTH_PER_GROUP 8:
    bottleneck widths 256 .. 2048, grouped conv2).
    MEGA / RDN options of the shipped configs (the defaults give configs/{MEGA,RDN}/vid_R_101_C4_*_1x.yaml):
      reduce_channel   MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL: the 1x1 conv 2048 -> 256 after res5, l_fcs.0 / fcs.0 read
                       256 * 49 inputs (configs/MEGA/vid_R_50_C4_MEGA_1x.yaml, configs/RDN/vid_R_50_C4_RDN_base_1x.yaml)
      global_res_stage MODEL.VID.MEGA.GLOBAL.RES_STAGE: g_* holds global_res_stage + 1 attention modules
      advanced_stage   MODEL.VID.ROI_BOX_HEAD.ATTENTION.ADVANCED_STAGE of RDN: 0 drops fcs.2 and attention modules 2, 3
                       (the RDN-base configs)
    The tensors of the defaults do not depend on these options' existence; the reduction conv is drawn last."""
    gen = torch.Generator().manual_seed(seed)
    tiny = arch.endswith("_tiny")
    base = arch.replace("_tiny", "")
    method, depth = base.split("_")
    blocks = {"r50": (3, 4, 6, 3), "r101": (3, 4, 23, 3), "x101": (3, 4, 23, 3)}[depth]
    groups, width = (32, 256) if depth == "x101" else (1, 64)      # res2 bottleneck width = NUM_GROUPS * WIDTH_PER_GROUP
    if tiny:
        blocks = (1, 1, 2, 1)
    sd = {}
    # stem: input std ~ 50 (0-255 domain); conv output variance ~ 2 * E[x^2]
    sd["backbone.body.stem.conv1.weight"] = _kaiming((64, 3, 7, 7), gen)
    _bn(sd, "backbone.body.stem.bn1.", 64, gen, in_var=2.0 * 70.0 ** 2)
    c = _stage(sd, "backbone.body.layer1.", gen, 64, width, 256, blocks[0], groups)
    c = _stage(sd, "backbone.body.layer2.", gen, c, 2 * width, 512, blocks[1], groups)
    c = _stage(sd, "backbone.body.layer3.", gen, c, 4 * width, 1024, blocks[2], groups)
    sd["rpn.anchor_generator.cell_anchors.0"] = None  # filled by the module / oracle (12 x 4)
    sd["rpn.head.conv.weight"] = _kaiming((1024, 1024, 3, 3), gen, gain=1.0)
    sd["rpn.head.conv.bias"] = torch.zeros(1024)
    sd["rpn.head.cls_logits.weight"] = torch.randn(12, 1024, 1, 1, generator=gen) * (2.0 / 32)
    sd["rpn.head.cls_logits.bias"] = torch.zeros(12)
    sd["rpn.head.bbox_pred.weight"] = torch.randn(48, 1024, 1, 1, generator=gen) * (0.25 / 32)
    sd["rpn.head.bbox_pred.bias"] = torch.zeros(48)
    fe = "roi_heads.box.feature_extractor."
    _stage(sd, fe + "head.layer4.", gen, 1024, 8 * width, 2048, blocks[3], groups)
    if method == "base":
        sd[fe + "conv.weight"] = _kaiming((256, 2048, 1, 1), gen, gain=1.0)
        sd[fe + "conv.bias"] = torch.zeros(256)
        _linear(sd, fe + "fc6.", 1024, 256 * 49, gen)
        _linear(sd, fe + "fc7.", 1024, 1024, gen)
    elif method in ("fgfa", "dff"):
        # GeneralizedRCNNFGFA / GeneralizedRCNNDFF: FlowNetS (+ EmbedNet for FGFA) next to the backbone
        # (backbone/flownet.py, embednet.py), box head = ResNetConv52MLPFeatureExtractor without the channel reduction
        # (configs/FGFA/vid_R_101_C4_FGFA_1x.yaml, configs/DFF/vid_R_101_C4_DFF_1x.yaml)
        _linear(sd, fe + "fc6.", 1024, 2048 * 49, gen)
        _linear(sd, fe + "fc7.", 1024, 1024, gen)

        def conv(name, cout, cin, k, gain=math.sqrt(2.0 / 1.01), bias=0.01):
            sd[name + ".weight"] = _kaiming((cout, cin, k, k), gen, gain=gain)
            sd[name + ".bias"] = torch.randn(cout, generator=gen) * bias

        conv("flownet.flow_conv1", 64, 6, 7)
        conv("flownet.conv2", 128, 64, 5)
        conv("flownet.conv3", 256, 128, 5)
        conv("flownet.conv3_1", 256, 256, 3)
        conv("flownet.conv4", 512, 256, 3)
        conv("flownet.conv4_1", 512, 512, 3)
        conv("flownet.conv5", 512, 512, 3)
        conv("flownet.conv5_1", 512, 512, 3)
        conv("flownet.conv6", 1024, 512, 3)
        conv("flownet.conv6_1", 1024, 1024, 3)
        for i, cin in zip(range(1, 6), (1024, 1026, 770, 386, 194)):
            conv("flownet.Convolution%d" % i, 2, cin, 3, gain=0.5)
        for name, cin, cout in (("deconv5", 1024, 512), ("deconv4", 1026, 256), ("deconv3", 770, 128), ("deconv2", 386, 64)):
            # ConvTranspose2d weight [cin, cout, 4, 4]; every output pixel sums 4 taps x cin inputs
            sd["flownet.%s.weight" % name] = torch.randn(cin, cout, 4, 4, generator=gen) * (1.4 / math.sqrt(4.0 * cin))
            sd["flownet.%s.bias" % name] = torch.randn(cout, generator=gen) * 0.01
        for name in ("upsample_flow6to5", "upsample_flow5to4", "upsample_flow4to3", "upsample_flow3to2"):
            sd["flownet.%s.weight" % name] = torch.randn(2, 2, 4, 4, generator=gen) * 0.25
            sd["flownet.%s.bias" % name] = torch.zeros(2)
        if method == "fgfa":
            conv("embednet.embed_conv1", 512, 1024, 1)
            conv("embednet.embed_conv2", 512, 512, 3)
            conv("embednet.embed_conv3", 2048, 512, 1, gain=1.0)
        else:
            # the reference zero-initialises the scale head (flownet.py:36-38: scale map == 1); a trained one is not
            # zero, so give it a spread of about +-0.3 around 1 to make the parity test see the branch
            sd["flownet.Convolution5_scale.weight"] = _kaiming((1024, 194, 1, 1), gen, gain=0.3)
    elif method == "rdn":
        # RDNFeatureExtractor with ATTENTION.STAGE = 2, ADVANCED_STAGE = 1 (configs/RDN/vid_R_101_C4_RDN_1x.yaml):
        # fcs[0..2], Wgs/Wqs/Wks/Wvs[0..3] (roi_box_feature_extractors.py:305-328)
        _linear(sd, fe + "fcs.0.", 1024, (256 if reduce_channel else 2048) * 49, gen)
        for i in (1, 2)[:1 + advanced_stage]:
            _linear(sd, fe + "fcs.%d." % i, 1024, 1024, gen)
        for i in range(4 if advanced_stage else 2):
            sd[fe + "Wgs.%d.weight" % i] = torch.randn(16, 64, 1, 1, generator=gen) * 0.2
            sd[fe + "Wgs.%d.bias" % i] = torch.rand(16, generator=gen) * 0.5
            _linear(sd, fe + "Wqs.%d." % i, 1024, 1024, gen)
            _linear(sd, fe + "Wks.%d." % i, 1024, 1024, gen)
            sd[fe + "Wvs.%d.weight" % i] = torch.randn(1024, 1024, 1, 1, generator=gen) * (0.5 / 32)
            sd[fe + "Wvs.%d.bias" % i] = torch.randn(1024, generator=gen) * 0.01
    else:
        _linear(sd, fe + "l_fcs.0.", 1024, (256 if reduce_channel else 2048) * 49, gen)
        for i in (1, 2):
            _linear(sd, fe + "l_fcs.%d." % i, 1024, 1024, gen)
        for i in range(3):
            sd[fe + "l_Wgs.%d.weight" % i] = torch.randn(16, 64, 1, 1, generator=gen) * 0.2
            sd[fe + "l_Wgs.%d.bias" % i] = torch.rand(16, generator=gen) * 0.5
            _linear(sd, fe + "l_Wqs.%d." % i, 1024, 1024, gen)
            _linear(sd, fe + "l_Wks.%d." % i, 1024, 1024, gen)
            sd[fe + "l_Wvs.%d.weight" % i] = torch.randn(1024, 1024, 1, 1, generator=gen) * (0.5 / 32)
            sd[fe + "l_Wvs.%d.bias" % i] = torch.randn(1024, generator=gen) * 0.01
        for i in range(3):
            sd[fe + "l_us.%d" % i] = torch.randn(16, 1, 64, generator=gen) * 0.1
        for i in range(global_res_stage + 1):
            _linear(sd, fe + "g_Wqs.%d." % i, 1024, 1024, gen)
            _linear(sd, fe + "g_Wks.%d." % i, 1024, 1024, gen)
            sd[fe + "g_Wvs.%d.weight" % i] = torch.randn(1024, 1024, 1, 1, generator=gen) * (0.5 / 32)
            sd[fe + "g_Wvs.%d.bias" % i] = torch.randn(1024, generator=gen) * 0.01
        for i in range(global_res_stage + 1):
            sd[fe + "g_us.%d" % i] = torch.randn(16, 1, 64, generator=gen) * 0.1
    _linear(sd, "roi_heads.box.predictor.cls_score.", num_classes, 1024, gen, std=0.03)
    _linear(sd, "roi_heads.box.predictor.bbox_pred.", num_classes * 4, 1024, gen, std=0.01)
    if reduce_channel and method in ("mega", "rdn"):
        sd[fe + "conv.weight"] = _kaiming((256, 2048, 1, 1), gen, gain=1.0)
        sd[fe + "conv.bias"] = torch.zeros(256)
    sd.pop("rpn.anchor_generator.cell_anchors.0")
    return sd


def global_frame_indices(seg_len, size=10, seed=0):
    """shuffled global-frame order per video, like datasets/vid_mega.py:112-120 (np.random there;
    a seeded torch permutation here -- only determinism matters for synthetic video)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(seg_len, generator=g).tolist()


def synthetic_proposal_dataset(seed=0, num_images=176126, max_props=300, max_gt=4, tail_images=64, tail_props=1000,
                               tail_gt=200):
    """a seeded proposal-recall workload the size of ImageNet-VID val (176,126 frames): per image 0..max_props proposals
    (objectness rounded to 3 decimals, so ties occur) and 0..max_gt GT boxes on integer pixels of a 1000 x 600 frame,
    then `tail_images` images with up to `tail_props` proposals and `tail_gt` GT boxes. Packed flat:
    (prop_boxes [P, 4] fp32, objectness [P], gt_boxes [G, 4], prop_offsets [N + 1] int64, gt_offsets [N + 1] int64)"""
    g = np.random.default_rng(seed)
    n_p = np.concatenate([g.integers(0, max_props + 1, num_images), g.integers(tail_props // 2, tail_props + 1, tail_images)])
    n_g = np.concatenate([g.integers(0, max_gt + 1, num_images), g.integers(tail_gt // 2, tail_gt + 1, tail_images)])

    def boxes(n):
        xy = g.integers(0, 900, (n, 2)).astype(np.float32)
        return np.concatenate([xy, xy + g.integers(8, 200, (n, 2)).astype(np.float32)], 1)

    po = np.concatenate([[0], np.cumsum(n_p)]).astype(np.int64)
    go = np.concatenate([[0], np.cumsum(n_g)]).astype(np.int64)
    pb = boxes(int(po[-1]))
    gb = boxes(int(go[-1]))
    # a third of the proposals sit near a GT box of their image, so the recall is not trivially 0
    img = np.repeat(np.arange(len(n_p)), n_p)
    has = n_g[img] > 0
    pick = has & (g.random(len(img)) < 1 / 3)
    gsel = go[img[pick]] + (g.random(int(pick.sum())) * n_g[img[pick]]).astype(np.int64)
    pb[pick] = gb[gsel] + g.integers(-6, 7, (int(pick.sum()), 4)).astype(np.float32)
    scores = np.round(g.random(len(img)), 3).astype(np.float32)
    return pb, scores, gb, po, go
