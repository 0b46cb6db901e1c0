"""mega_oracle -- CPU restatement of the reference's MEGA / single-frame inference path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package (`mega.pytorch_b200/`) imports this
module; it is the checker used by `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` /
`--impl reference` legs of `bench.py`.

What it is: a plain PyTorch fp32 (CPU) re-statement, function by function, of the algorithm the
reference executes for one frame, written against the reference's *state_dict key names* so the
same weights drive the reference, this oracle and the CUDA path.  Each function cites the
reference lines it follows (paths relative to the reference's `mega_core/`).  The two custom
ops (NMS, ROIAlign) are restated in plain C (`oracle/csrc/oracle_ops.c`).

Pinning (see tests/test_oracle_cpu.py, tests/golden/, oracle/make_golden.py):
  * NMS          -- the reference's golden vectors tests/test_nms.py:16-58, :65-217 and the
                    reference's nms_cpu.cpp compiled verbatim (oracle/_ref);
  * box decode   -- tests/test_box_coder.py:15-105;
  * anchors      -- the table in rpn/anchor_generator.py:199-217;
  * ROIAlign     -- the reference's ROIAlign_cpu.cpp compiled verbatim (oracle/_ref);
  * everything else (backbone, RPN selection, relation module, memory update order,
    post-processing) has NO known-answer test in the reference: it is pinned by running the
    unmodified reference Python here on identical weights/inputs (oracle/make_golden.py) and
    committing the outputs as fixtures under tests/golden/.
"""
import ctypes
import math
import os
from collections import deque

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_OPS_SO = os.path.join(_HERE, "csrc", "liboracle_ops.so")
_ops = None


def build_c_ops(force=False):
    """gcc-compile oracle/csrc/oracle_ops.c (no FMA contraction) -> liboracle_ops.so"""
    src = os.path.join(_HERE, "csrc", "oracle_ops.c")
    if force or not os.path.exists(_OPS_SO) or os.path.getmtime(_OPS_SO) < os.path.getmtime(src):
        import subprocess
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-o", _OPS_SO, src, "-lm"])
    return _OPS_SO


def _c_ops():
    global _ops
    if _ops is None:
        build_c_ops()
        _ops = ctypes.CDLL(_OPS_SO)
        _ops.oracle_nms.restype = ctypes.c_int64
        _ops.oracle_nms.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float,
                                    ctypes.c_int, ctypes.c_void_p]
        _ops.oracle_roi_align_fwd.restype = None
        _ops.oracle_roi_align_fwd.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int,
                                              ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return _ops


# --------------------------------------------------------------------------- custom ops
def nms(boxes, scores, thresh, cuda_semantics=False):
    """greedy NMS -> kept original indices, ascending (csrc/cpu/nms_cpu.cpp:6-65;
    cuda_semantics=True uses the `>` rule of csrc/cuda/nms.cu:60)."""
    boxes = boxes.detach().to(torch.float32).contiguous().cpu()
    scores = scores.detach().to(torch.float32).contiguous().cpu()
    n = boxes.shape[0]
    keep = torch.empty(max(n, 1), dtype=torch.int64)
    m = _c_ops().oracle_nms(boxes.data_ptr(), scores.data_ptr(), n, float(thresh), int(cuda_semantics),
                            keep.data_ptr())
    return keep[:m].clone()


def roi_align(feat, rois, spatial_scale, pooled_h, pooled_w, sampling_ratio):
    """ROIAlign forward, NCHW in, [K,C,ph,pw] out (csrc/cpu/ROIAlign_cpu.cpp:17-219)."""
    feat = feat.detach().to(torch.float32).contiguous().cpu()
    rois = rois.detach().to(torch.float32).contiguous().cpu()
    k = rois.shape[0]
    n, c, h, w = feat.shape
    out = torch.empty(k, c, pooled_h, pooled_w, dtype=torch.float32)
    if k:
        _c_ops().oracle_roi_align_fwd(feat.data_ptr(), c, h, w, rois.data_ptr(), k, float(spatial_scale),
                                      pooled_h, pooled_w, sampling_ratio, out.data_ptr())
    return out


# --------------------------------------------------------------------------- backbone
def frozen_bn(x, sd, p):
    """layers/batch_norm.py:26-31 -- note: no eps."""
    scale = sd[p + "weight"] * sd[p + "running_var"].rsqrt()
    bias = sd[p + "bias"] - sd[p + "running_mean"] * scale
    return x * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)


def bottleneck(x, sd, p, stride, dilation):
    """modeling/backbone/resnet.py:239-344 with STRIDE_IN_1X1=True (config/defaults.py:273)."""
    identity = x
    if dilation > 1:
        stride_eff, down_stride = 1, 1
    else:
        stride_eff, down_stride = stride, stride
    out = F.conv2d(x, sd[p + "conv1.weight"], None, stride_eff)
    out = frozen_bn(out, sd, p + "bn1.").relu()
    out = F.conv2d(out, sd[p + "conv2.weight"], None, 1, dilation, dilation)
    out = frozen_bn(out, sd, p + "bn2.").relu()
    out = F.conv2d(out, sd[p + "conv3.weight"], None, 1)
    out = frozen_bn(out, sd, p + "bn3.")
    if (p + "downsample.0.weight") in sd:
        identity = F.conv2d(x, sd[p + "downsample.0.weight"], None, down_stride)
        identity = frozen_bn(identity, sd, p + "downsample.1.")
    return (out + identity).relu()


def _count_blocks(sd, prefix):
    n = 0
    while (prefix + "%d.conv1.weight" % n) in sd:
        n += 1
    return n


def resnet_c4_body(x, sd, prefix="backbone.body."):
    """stem + res2..res4 (resnet.py:145-152, :347-366); block counts read from the state dict."""
    x = F.conv2d(x, sd[prefix + "stem.conv1.weight"], None, 2, 3)
    x = frozen_bn(x, sd, prefix + "stem.bn1.").relu()
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    for li in (1, 2, 3):
        lp = prefix + "layer%d." % li
        for b in range(_count_blocks(sd, lp)):
            x = bottleneck(x, sd, lp + "%d." % b, stride=(2 if (b == 0 and li > 1) else 1), dilation=1)
    return x


def res5_head(x, sd, prefix, dilation=2):
    """ResNetHead with stride_init=1 and RES5_DILATION (resnet.py:155-204;
    roi_box_feature_extractors.py:463-472; configs/BASE_RCNN_1gpu.yaml:18-19)."""
    lp = prefix + "layer4."
    for b in range(_count_blocks(sd, lp)):
        x = bottleneck(x, sd, lp + "%d." % b, stride=1, dilation=dilation)
    return x


# --------------------------------------------------------------------------- RPN
def cell_anchors(stride=16, sizes=(64, 128, 256, 512), ratios=(0.5, 1.0, 2.0)):
    """rpn/anchor_generator.py:220-289 (numpy float64, rounded like the reference)."""
    def whctr(a):
        w = a[2] - a[0] + 1
        h = a[3] - a[1] + 1
        return w, h, a[0] + 0.5 * (w - 1), a[1] + 0.5 * (h - 1)

    def mk(ws, hs, xc, yc):
        ws, hs = ws[:, None], hs[:, None]
        return np.hstack((xc - 0.5 * (ws - 1), yc - 0.5 * (hs - 1), xc + 0.5 * (ws - 1), yc + 0.5 * (hs - 1)))

    base = np.array([1, 1, stride, stride], dtype=np.float64) - 1
    w, h, xc, yc = whctr(base)
    size_ratios = (w * h) / np.array(ratios, dtype=np.float64)
    ws = np.round(np.sqrt(size_ratios))
    hs = np.round(ws * np.array(ratios, dtype=np.float64))
    ratio_anchors = mk(ws, hs, xc, yc)
    scales = np.array(sizes, dtype=np.float64) / stride
    out = []
    for i in range(ratio_anchors.shape[0]):
        w, h, xc, yc = whctr(ratio_anchors[i])
        out.append(mk(w * scales, h * scales, xc, yc))
    return torch.from_numpy(np.vstack(out)).float()


def grid_anchors(grid_h, grid_w, stride=16, base=None):
    """rpn/anchor_generator.py:73-95: order (h, w, a)."""
    base = cell_anchors(stride) if base is None else base
    sx = torch.arange(0, grid_w * stride, step=stride, dtype=torch.float32)
    sy = torch.arange(0, grid_h * stride, step=stride, dtype=torch.float32)
    yy, xx = torch.meshgrid(sy, sx, indexing="ij")
    shifts = torch.stack((xx.reshape(-1), yy.reshape(-1), xx.reshape(-1), yy.reshape(-1)), dim=1)
    return (shifts.view(-1, 1, 4) + base.view(1, -1, 4)).reshape(-1, 4)


BBOX_XFORM_CLIP = math.log(1000.0 / 16)


def decode_boxes(rel_codes, boxes, weights):
    """modeling/box_coder.py:52-95."""
    boxes = boxes.to(rel_codes.dtype)
    widths = boxes[:, 2] - boxes[:, 0] + 1
    heights = boxes[:, 3] - boxes[:, 1] + 1
    ctr_x = boxes[:, 0] + 0.5 * widths
    ctr_y = boxes[:, 1] + 0.5 * heights
    wx, wy, ww, wh = weights
    dx = rel_codes[:, 0::4] / wx
    dy = rel_codes[:, 1::4] / wy
    dw = torch.clamp(rel_codes[:, 2::4] / ww, max=BBOX_XFORM_CLIP)
    dh = torch.clamp(rel_codes[:, 3::4] / wh, max=BBOX_XFORM_CLIP)
    pcx = dx * widths[:, None] + ctr_x[:, None]
    pcy = dy * heights[:, None] + ctr_y[:, None]
    pw = torch.exp(dw) * widths[:, None]
    ph = torch.exp(dh) * heights[:, None]
    out = torch.zeros_like(rel_codes)
    out[:, 0::4] = pcx - 0.5 * pw
    out[:, 1::4] = pcy - 0.5 * ph
    out[:, 2::4] = pcx + 0.5 * pw - 1
    out[:, 3::4] = pcy + 0.5 * ph - 1
    return out


def clip_boxes(boxes, im_w, im_h):
    """structures/bounding_box.py:214-224 (remove_empty=False). boxes [..., 4k] xyxy."""
    b = boxes.clone()
    b[..., 0::4].clamp_(min=0, max=im_w - 1)
    b[..., 1::4].clamp_(min=0, max=im_h - 1)
    b[..., 2::4].clamp_(min=0, max=im_w - 1)
    b[..., 3::4].clamp_(min=0, max=im_h - 1)
    return b


def rpn_head(feat, sd, prefix="rpn.head."):
    """rpn/rpn.py:99-106."""
    t = F.conv2d(feat, sd[prefix + "conv.weight"], sd[prefix + "conv.bias"], 1, 1).relu()
    logits = F.conv2d(t, sd[prefix + "cls_logits.weight"], sd[prefix + "cls_logits.bias"])
    deltas = F.conv2d(t, sd[prefix + "bbox_pred.weight"], sd[prefix + "bbox_pred.bias"])
    return logits, deltas


def rpn_select(logits, deltas, im_w, im_h, pre_nms_top_n=6000, post_nms_top_n=300, nms_thresh=0.7,
               min_size=0, stride=16, cuda_semantics=False, return_aux=False):
    """rpn/inference.py:76-123 for one image: sigmoid -> top-k (sorted) -> decode -> clip ->
    remove_small_boxes -> NMS -> first post_nms_top_n. Returns (boxes [P,4], objectness [P]).

    Tie rule of the top-k: descending score, equal scores by ascending anchor index (a stable
    sort); torch.topk leaves tie order unspecified, so this is the oracle's definition."""
    _, a, h, w = logits.shape
    obj = logits[0].permute(1, 2, 0).reshape(-1).sigmoid()                 # (h, w, a) order
    reg = deltas[0].view(a, 4, h, w).permute(2, 3, 0, 1).reshape(-1, 4)
    anchors = grid_anchors(h, w, stride)
    k = min(pre_nms_top_n, obj.numel())
    order = torch.sort(obj, descending=True, stable=True)[1][:k]
    scores = obj[order]
    props = decode_boxes(reg[order], anchors[order], (1.0, 1.0, 1.0, 1.0))
    props = clip_boxes(props, im_w, im_h)
    ws = props[:, 2] - props[:, 0] + 1
    hs = props[:, 3] - props[:, 1] + 1
    keep_small = ((ws >= min_size) & (hs >= min_size)).nonzero().squeeze(1)
    props, scores, order_kept = props[keep_small], scores[keep_small], order[keep_small]
    keep = nms(props, scores, nms_thresh, cuda_semantics)
    if post_nms_top_n > 0:
        keep = keep[:post_nms_top_n]
    if return_aux:
        return props[keep], scores[keep], {"topk_idx": order, "pre_nms_boxes": props, "pre_nms_scores": scores,
                                           "keep": keep, "anchor_idx": order_kept[keep]}
    return props[keep], scores[keep]


# --------------------------------------------------------------------------- relation module
def position_matrix(bbox, ref_bbox):
    """roi_box_feature_extractors.py:146-176 -> [N, M, 4]."""
    xmin, ymin, xmax, ymax = torch.chunk(ref_bbox, 4, dim=1)
    w_ref = xmax - xmin + 1
    h_ref = ymax - ymin + 1
    cx_ref = 0.5 * (xmin + xmax)
    cy_ref = 0.5 * (ymin + ymax)
    xmin, ymin, xmax, ymax = torch.chunk(bbox, 4, dim=1)
    w = xmax - xmin + 1
    h = ymax - ymin + 1
    cx = 0.5 * (xmin + xmax)
    cy = 0.5 * (ymin + ymax)
    dx = (((cx - cx_ref.t()) / w).abs() + 1e-3).log()
    dy = (((cy - cy_ref.t()) / h).abs() + 1e-3).log()
    dw = (w / w_ref.t()).log()
    dh = (h / h_ref.t()).log()
    return torch.stack([dx, dy, dw, dh], dim=2)


def position_embedding(bbox, ref_bbox, feat_dim=64, wave_length=1000.0, dim_mat=None):
    """roi_box_feature_extractors.py:125-144 + :240-250 -> [feat_dim, N, M]
    (channel = coord*16 + {sin: k, cos: 8 + k}, k = 0..7). dim_mat: the divisors as given (e.g. the fp32 values the
    engine passes, on the boxes' device) instead of the ones computed here."""
    pm = position_matrix(bbox, ref_bbox)
    if dim_mat is None:
        feat_range = torch.arange(0, feat_dim / 8)
        dim_mat = torch.full((len(feat_range),), wave_length).pow(8.0 / feat_dim * feat_range)
    div = (pm.unsqueeze(3) * 100.0) / dim_mat.view(1, 1, 1, -1)
    emb = torch.cat([div.sin(), div.cos()], dim=3)                      # [N, M, 4, 16]
    emb = emb.reshape(emb.shape[0], emb.shape[1], -1)                   # [N, M, 64]
    return emb.permute(2, 0, 1)


def relation_attention(sd, fe_prefix, kind, index, roi_feat, ref_feat, pos_emb, group=16, u_term=True):
    """attention_module_multi_head -- MEGA variant roi_box_feature_extractors.py:567-646 (with the
    `u` bias, kind in {"l","g"}), base/RDN variant :178-238 (u_term=False, weights "Wqs" etc.).
    Written exactly in the reference's association order (softmax @ raw V, then grouped Wv)."""
    pfx = fe_prefix + (kind + "_" if kind else "")
    n, feat_dim = roi_feat.shape
    m = ref_feat.shape[0]
    dg = feat_dim // group
    q = F.linear(roi_feat, sd[pfx + "Wqs.%d.weight" % index], sd[pfx + "Wqs.%d.bias" % index])
    k = F.linear(ref_feat, sd[pfx + "Wks.%d.weight" % index], sd[pfx + "Wks.%d.bias" % index])
    qb = q.reshape(n, group, dg).permute(1, 0, 2)
    kb = k.reshape(m, group, dg).permute(1, 0, 2)
    aff = torch.bmm(qb, kb.transpose(1, 2))                              # [g, n, m]
    if u_term:
        aff = aff + torch.bmm(sd[pfx + "us.%d" % index], kb.transpose(1, 2))
    aff_scale = ((1.0 / math.sqrt(float(dg))) * aff).permute(1, 0, 2)  # [n, g, m]
    if pos_emb is not None:
        wg = sd[pfx + "Wgs.%d.weight" % index]
        bg = sd[pfx + "Wgs.%d.bias" % index]
        aff_weight = F.relu(F.conv2d(pos_emb.unsqueeze(0), wg, bg))[0].permute(1, 0, 2)   # [n, g, m]
        weighted = (aff_weight + 1e-6).log() + aff_scale
    else:
        weighted = aff_scale
    sm = F.softmax(weighted, dim=2)
    out_t = torch.matmul(sm.reshape(n * group, m), ref_feat)              # [n*g, feat_dim]
    out_t = out_t.reshape(n, group * feat_dim, 1, 1)
    out = F.conv2d(out_t, sd[pfx + "Wvs.%d.weight" % index], sd[pfx + "Wvs.%d.bias" % index], groups=group)
    return out.reshape(n, feat_dim)


# --------------------------------------------------------------------------- box head
def box_postprocess(class_logits, box_regression, proposals, im_w, im_h, score_thresh=0.001, nms_thresh=0.5,
                    detections_per_img=300, weights=(10.0, 10.0, 5.0, 5.0), cuda_semantics=False):
    """roi_heads/box_head/inference.py:45-149 for one image -> (boxes [D,4], scores [D], labels [D])."""
    prob = F.softmax(class_logits, -1)
    num_classes = prob.shape[1]
    boxes = decode_boxes(box_regression.view(proposals.shape[0], -1), proposals, weights)
    boxes = clip_boxes(boxes, im_w, im_h)
    res_b, res_s, res_l = [], [], []
    inds_all = prob > score_thresh
    for j in range(1, num_classes):
        inds = inds_all[:, j].nonzero().squeeze(1)
        sj = prob[inds, j]
        bj = boxes[inds, j * 4:(j + 1) * 4]
        keep = nms(bj, sj, nms_thresh, cuda_semantics)
        res_b.append(bj[keep])
        res_s.append(sj[keep])
        res_l.append(torch.full((keep.numel(),), j, dtype=torch.int64))
    b, s, l = torch.cat(res_b), torch.cat(res_s), torch.cat(res_l)
    if s.numel() > detections_per_img > 0:
        thresh, _ = torch.kthvalue(s, s.numel() - detections_per_img + 1)
        keep = (s >= thresh.item()).nonzero().squeeze(1)
        b, s, l = b[keep], s[keep], l[keep]
    return b, s, l


class Cfg:
    """the handful of config values the path reads (defaults: config/defaults.py:393-463,
    configs/BASE_RCNN_1gpu.yaml, configs/MEGA/vid_R_101_C4_MEGA_1x.yaml)."""
    pre_nms_top_n = 6000
    post_nms_top_n = 300          # key frame
    ref_post_nms_top_n = 75       # MODEL.VID.RPN.REF_POST_NMS_TOP_N
    rpn_nms_thresh = 0.7
    ratio = 0.2                   # MODEL.VID.MEGA.RATIO -> advanced_num = 15
    all_frame_interval = 25
    key_frame_location = 12
    memory_size = 25
    global_size = 10
    global_res_stage = 1
    stage = 3
    groups = 16
    pooler_resolution = 7
    pooler_scale = 1.0 / 16
    sampling_ratio = 0
    res5_dilation = 2
    score_thresh = 0.001
    nms_thresh = 0.5
    detections_per_img = 300
    reduce_channel = False
    cuda_nms_semantics = False

    def __init__(self, **kw):
        for k, v in kw.items():
            assert hasattr(self, k), k
            setattr(self, k, v)

    @property
    def advanced_num(self):
        return int(self.ref_post_nms_top_n * self.ratio)


FE = "roi_heads.box.feature_extractor."


class MegaOracle:
    """GeneralizedRCNNMEGA._forward_test + MEGAFeatureExtractor test path, restated.

    detector/generalized_rcnn_mega.py:137-225 (per-video state machine) and
    roi_heads/box_head/roi_box_feature_extractors.py:657-699, :754-774, :806-829, :885-933.
    Frames are fp32 [1,3,H,W] tensors already in the post-transform domain. The disk reads of
    frame 0 (generalized_rcnn_mega.py:183-193) are replaced by the caller passing the look-ahead
    frames in `infos["ref_l"]` (a list of tensors for frame_category 0)."""

    def __init__(self, state_dict, cfg=None, record=False):
        self.sd = {k: v.detach().float() for k, v in state_dict.items()}
        self.cfg = cfg or Cfg()
        self.record = record
        self.trace = {}

    # ---- per-frame feature path (update_feature: generalized_rcnn_mega.py:145-158)
    def _ref_branch(self, img):
        c = self.cfg
        feats = resnet_c4_body(img, self.sd)
        im_h, im_w = img.shape[-2:]
        logits, deltas = rpn_head(feats, self.sd)
        boxes, obj = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.ref_post_nms_top_n,
                                c.rpn_nms_thresh, cuda_semantics=c.cuda_nms_semantics)
        pfeat = self._roi_fc(feats, boxes)
        return feats, boxes, pfeat

    def _roi_fc(self, feats, boxes):
        """_forward_ref: res5 -> ROIAlign -> flatten -> l_fcs[0] + ReLU (extractors :885-896)."""
        c = self.cfg
        x = res5_head(feats, self.sd, FE + "head.", c.res5_dilation)
        rois = torch.cat([torch.zeros(boxes.shape[0], 1), boxes], dim=1)
        x = roi_align(x, rois, c.pooler_scale, c.pooler_resolution, c.pooler_resolution, c.sampling_ratio)
        x = x.flatten(start_dim=1)
        return F.relu(F.linear(x, self.sd[FE + "l_fcs.0.weight"], self.sd[FE + "l_fcs.0.bias"]))

    def _push(self, feats, boxes, pfeat):
        a = self.cfg.advanced_num
        self.q_feats.append(feats)
        self.q_boxes.append(boxes)
        self.q_boxes_dis.append(boxes[:a])
        self.q_pfeat.append(pfeat)
        self.q_pfeat_dis.append(pfeat[:a])

    def _update_lm(self, x, i=0):
        """global aggregation (extractors :690-699)."""
        g = torch.cat(list(self.global_q), dim=0)
        return x + relation_attention(self.sd, FE, "g", i, x, g, None, self.cfg.groups)

    def forward(self, img, infos):
        c = self.cfg
        a = c.advanced_num
        im_h, im_w = img.shape[-2:]
        if infos["frame_category"] == 0:
            L = c.all_frame_interval
            self.q_feats, self.q_boxes, self.q_boxes_dis = deque(maxlen=L), deque(maxlen=L), deque(maxlen=L)
            self.q_pfeat, self.q_pfeat_dis = deque(maxlen=L), deque(maxlen=L)
            self.mem_q = [{"rois": deque(maxlen=L), "feats": deque(maxlen=L)} for _ in range(c.stage)]
            self.mem = [None] * c.stage
            self.global_q = deque(maxlen=c.global_size)
            cur = self._ref_branch(img)
            while len(self.q_feats) < c.key_frame_location + 1:
                self._push(*cur)
            for im in infos["ref_l"]:
                if len(self.q_feats) >= L:
                    break
                self._push(*self._ref_branch(im))
            assert len(self.q_feats) == L, "frame 0 needs %d look-ahead frames" % (L - c.key_frame_location - 1)
        else:
            self._push(*self._ref_branch(infos["ref_l"][0]))
        for gimg in infos["ref_g"]:
            _, _, pfeat = self._ref_branch(gimg)
            self.global_q.append(pfeat)

        feats = self.q_feats[c.key_frame_location]
        logits, deltas = rpn_head(feats, self.sd)
        prop, obj = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.post_nms_top_n, c.rpn_nms_thresh,
                               cuda_semantics=c.cuda_nms_semantics)
        rois_ref = torch.cat(list(self.q_boxes), 0)
        rois_dis = torch.cat(list(self.q_boxes_dis), 0)
        x_ref = torch.cat(list(self.q_pfeat), 0)
        x_ref_dis = torch.cat(list(self.q_pfeat_dis), 0)

        # ---- MEGAFeatureExtractor._forward_test (extractors :898-933)
        x = self._roi_fc(feats, prop)
        if self.record:
            self.trace = {"proposals": prop.clone(), "objectness": obj.clone(), "x_key_fc": x.clone()}
        if len(self.global_q):
            x = self._update_lm(x)
            x_ref = self._update_lm(x_ref)
            x_ref_dis = self._update_lm(x_ref_dis)
        k = prop.shape[0]
        cache = [{"rois_cur": torch.cat([prop, rois_dis], 0), "rois_ref": rois_ref,
                  "feats_cur": torch.cat([x, x_ref_dis], 0), "feats_ref": x_ref}]
        for _ in range(c.stage - 2):
            cache.append({"rois_cur": torch.cat([prop, rois_dis], 0), "rois_ref": rois_dis})
        cache.append({"rois_cur": prop, "rois_ref": rois_dis})

        for i in range(c.stage):
            memory = self.mem[i]
            # update_memory (extractors :678-688): push BEFORE stage i runs, after `memory` was read
            npush = c.ref_post_nms_top_n if i == 0 else a
            self.mem_q[i]["rois"].append(cache[i]["rois_ref"][:npush])
            self.mem_q[i]["feats"].append(cache[i]["feats_ref"][:npush])
            self.mem[i] = {"rois": torch.cat(list(self.mem_q[i]["rois"]), 0),
                           "feats": torch.cat(list(self.mem_q[i]["feats"]), 0)}
            # _forward_test_single (extractors :806-829)
            rois_cur, rois_r = cache[i]["rois_cur"], cache[i]["rois_ref"]
            f_cur, f_ref = cache[i]["feats_cur"], cache[i]["feats_ref"]
            if memory is not None:
                rois_r = torch.cat([rois_r, memory["rois"]], 0)
                f_ref = torch.cat([f_ref, memory["feats"]], 0)
            pe = position_embedding(rois_cur, rois_r)
            f_cur = f_cur + relation_attention(self.sd, FE, "l", i, f_cur, f_ref, pe, c.groups)
            if i != c.stage - 1:
                f_cur = F.relu(F.linear(f_cur, self.sd[FE + "l_fcs.%d.weight" % (i + 1)],
                                        self.sd[FE + "l_fcs.%d.bias" % (i + 1)]))
            if i == c.stage - 1:
                x = f_cur
            elif i == c.stage - 2:
                cache[i + 1]["feats_cur"] = f_cur[:k]
                cache[i + 1]["feats_ref"] = f_cur[k:]
            else:
                cache[i + 1]["feats_cur"] = f_cur
                cache[i + 1]["feats_ref"] = f_cur[k:]
        for i in range(c.global_res_stage):
            x = self._update_lm(x, i + 1)

        # ---- predictor + post-processor (roi_box_predictors.py:50-57; box_head/inference.py:45-149)
        logits = F.linear(x, self.sd["roi_heads.box.predictor.cls_score.weight"],
                          self.sd["roi_heads.box.predictor.cls_score.bias"])
        bdelta = F.linear(x, self.sd["roi_heads.box.predictor.bbox_pred.weight"],
                          self.sd["roi_heads.box.predictor.bbox_pred.bias"])
        if self.record:
            self.trace.update({"x_final": x.clone(), "class_logits": logits.clone(), "box_regression": bdelta.clone()})
        return box_postprocess(logits, bdelta, prop, im_w, im_h, c.score_thresh, c.nms_thresh,
                               c.detections_per_img, cuda_semantics=c.cuda_nms_semantics)


class BaseOracle:
    """GeneralizedRCNN single-frame path (detector/generalized_rcnn.py:33-65) with
    ResNetConv52MLPFeatureExtractor (extractors :106-118), REDUCE_CHANNEL per config."""

    def __init__(self, state_dict, cfg=None, record=False):
        self.sd = {k: v.detach().float() for k, v in state_dict.items()}
        self.cfg = cfg or Cfg()
        self.record = record
        self.trace = {}

    def forward(self, img):
        c, sd = self.cfg, self.sd
        im_h, im_w = img.shape[-2:]
        feats = resnet_c4_body(img, sd)
        logits, deltas = rpn_head(feats, sd)
        prop, obj = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.post_nms_top_n, c.rpn_nms_thresh,
                               cuda_semantics=c.cuda_nms_semantics)
        x = res5_head(feats, sd, FE + "head.", c.res5_dilation)
        if (FE + "conv.weight") in sd:
            x = F.relu(F.conv2d(x, sd[FE + "conv.weight"], sd[FE + "conv.bias"]))
        rois = torch.cat([torch.zeros(prop.shape[0], 1), prop], dim=1)
        pooled = roi_align(x, rois, c.pooler_scale, c.pooler_resolution, c.pooler_resolution, c.sampling_ratio)
        x = pooled.flatten(start_dim=1)
        x = F.relu(F.linear(x, sd[FE + "fc6.weight"], sd[FE + "fc6.bias"]))
        x = F.relu(F.linear(x, sd[FE + "fc7.weight"], sd[FE + "fc7.bias"]))
        logits = F.linear(x, sd["roi_heads.box.predictor.cls_score.weight"], sd["roi_heads.box.predictor.cls_score.bias"])
        bdelta = F.linear(x, sd["roi_heads.box.predictor.bbox_pred.weight"], sd["roi_heads.box.predictor.bbox_pred.bias"])
        if self.record:
            self.trace = {"proposals": prop.clone(), "objectness": obj.clone(), "roi_pooled": pooled,
                          "class_logits": logits.clone(), "box_regression": bdelta.clone(), "feats": feats}
        return box_postprocess(logits, bdelta, prop, im_w, im_h, c.score_thresh, c.nms_thresh,
                               c.detections_per_img, cuda_semantics=c.cuda_nms_semantics)


class RdnOracle:
    """GeneralizedRCNNRDN._forward_test (detector/generalized_rcnn_rdn.py:108-190) + RDNFeatureExtractor test path
    (roi_heads/box_head/roi_box_feature_extractors.py:412-454, base attention module :178-238, no `u` term), restated.
    Window of cfg.all_frame_interval (37) frames, key frame at cfg.key_frame_location (18); per frame the 75 "ref"
    proposals and their fcs[0] features are cached (update_feature :116-131). Frame 0's look-ahead frames are passed
    in infos["ref"] (a list of tensors) instead of being read from disk (:154-164)."""

    def __init__(self, state_dict, cfg=None, record=False, base_stage=2, advanced_stage=1):
        self.sd = {k: v.detach().float() for k, v in state_dict.items()}
        self.cfg = cfg or Cfg(all_frame_interval=37, key_frame_location=18)
        self.base_stage, self.advanced_stage = base_stage, advanced_stage
        self.record = record
        self.trace = {}

    def _pool(self, feats, boxes):
        c = self.cfg
        x = res5_head(feats, self.sd, FE + "head.", c.res5_dilation)
        rois = torch.cat([torch.zeros(boxes.shape[0], 1), boxes], dim=1)
        x = roi_align(x, rois, c.pooler_scale, c.pooler_resolution, c.pooler_resolution, c.sampling_ratio)
        return x.flatten(start_dim=1)

    def _fc(self, i, x):
        return F.relu(F.linear(x, self.sd[FE + "fcs.%d.weight" % i], self.sd[FE + "fcs.%d.bias" % i]))

    def _ref_branch(self, img):
        c = self.cfg
        feats = resnet_c4_body(img, self.sd)
        im_h, im_w = img.shape[-2:]
        logits, deltas = rpn_head(feats, self.sd)
        boxes, _ = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.ref_post_nms_top_n, c.rpn_nms_thresh,
                              cuda_semantics=c.cuda_nms_semantics)
        return feats, boxes, self._fc(0, self._pool(feats, boxes))        # _forward_ref (:400-410)

    def forward(self, img, infos):
        c = self.cfg
        im_h, im_w = img.shape[-2:]
        L = c.all_frame_interval
        if infos["frame_category"] == 0:
            self.q_feats, self.q_boxes, self.q_pfeat = deque(maxlen=L), deque(maxlen=L), deque(maxlen=L)
            cur = self._ref_branch(img)
            while len(self.q_feats) < c.key_frame_location + 1:
                for q, v in zip((self.q_feats, self.q_boxes, self.q_pfeat), cur):
                    q.append(v)
            for im in infos["ref"]:
                if len(self.q_feats) >= L:
                    break
                for q, v in zip((self.q_feats, self.q_boxes, self.q_pfeat), self._ref_branch(im)):
                    q.append(v)
            assert len(self.q_feats) == L
        else:
            for q, v in zip((self.q_feats, self.q_boxes, self.q_pfeat), self._ref_branch(infos["ref"][0])):
                q.append(v)
        feats = self.q_feats[c.key_frame_location]
        logits, deltas = rpn_head(feats, self.sd)
        prop, obj = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.post_nms_top_n, c.rpn_nms_thresh,
                               cuda_semantics=c.cuda_nms_semantics)
        rois_ref = torch.cat(list(self.q_boxes), 0)
        x_refs = torch.cat(list(self.q_pfeat), 0)
        # ---- RDNFeatureExtractor._forward_test (:412-454)
        x = self._pool(feats, prop)
        pe = position_embedding(prop, rois_ref)
        for i in range(self.base_stage):
            x = self._fc(i, x)
            x = x + relation_attention(self.sd, FE, "", i, x, x_refs, pe, c.groups, u_term=False)
        if self.advanced_stage > 0:
            a, b = c.advanced_num, c.ref_post_nms_top_n
            x_adv = torch.cat([t[:a] for t in torch.split(x_refs, b, dim=0)], 0)
            rois_adv = torch.cat([t[:a] for t in torch.split(rois_ref, b, dim=0)], 0)
            pe_adv = torch.cat([t[..., :a] for t in torch.split(pe, b, dim=-1)], -1)
            pe2 = position_embedding(rois_adv, rois_ref)
            for i in range(self.advanced_stage):
                x_adv = x_adv + relation_attention(self.sd, FE, "", i + self.base_stage, x_adv, x_refs, pe2, c.groups,
                                                   u_term=False)
                x_adv = self._fc(i + self.base_stage, x_adv)
            x = x + relation_attention(self.sd, FE, "", self.base_stage + self.advanced_stage, x, x_adv, pe_adv,
                                       c.groups, u_term=False)
        logits = F.linear(x, self.sd["roi_heads.box.predictor.cls_score.weight"],
                          self.sd["roi_heads.box.predictor.cls_score.bias"])
        bdelta = F.linear(x, self.sd["roi_heads.box.predictor.bbox_pred.weight"],
                          self.sd["roi_heads.box.predictor.bbox_pred.bias"])
        if self.record:
            self.trace = {"proposals": prop.clone(), "x_final": x.clone(), "class_logits": logits.clone(),
                          "box_regression": bdelta.clone()}
        return box_postprocess(logits, bdelta, prop, im_w, im_h, c.score_thresh, c.nms_thresh,
                               c.detections_per_img, cuda_semantics=c.cuda_nms_semantics)


def _crop_like(x, target):
    """backbone/flownet.py:7-11"""
    if x.shape[2:] == target.shape[2:]:
        return x
    return x[:, :, 1:target.shape[2] + 1, 1:target.shape[3] + 1]


def flownet_s(x, sd, p="flownet.", with_scale=False):
    """FlowNetS.forward (backbone/flownet.py:54-118): x [B,6,H,W] (image pairs / 255) -> flow [B,2,H/16,W/16] * 2.5;
    with_scale (method "dff", :112-116): also the scale map Convolution5_scale(concat5) + 1, [B,1024,H/16,W/16]"""
    def conv(name, t, stride=1, pad=1):
        return F.conv2d(t, sd[p + name + ".weight"], sd[p + name + ".bias"], stride, pad)

    def deconv(name, t):
        return F.conv_transpose2d(t, sd[p + name + ".weight"], sd[p + name + ".bias"], stride=2)

    lrelu = lambda t: F.leaky_relu(t, 0.1)
    pool = lambda t: F.avg_pool2d(t, 2, stride=2, ceil_mode=True)
    x = pool(x)
    relu1 = lrelu(conv("flow_conv1", x, 2, 3))
    relu2 = lrelu(conv("conv2", relu1, 2, 2))
    relu3 = lrelu(conv("conv3", relu2, 2, 2))
    relu4 = lrelu(conv("conv3_1", relu3))
    relu5 = lrelu(conv("conv4", relu4, 2))
    relu6 = lrelu(conv("conv4_1", relu5))
    relu7 = lrelu(conv("conv5", relu6, 2))
    relu8 = lrelu(conv("conv5_1", relu7))
    relu9 = lrelu(conv("conv6", relu8, 2))
    relu10 = lrelu(conv("conv6_1", relu9))
    flow6 = conv("Convolution1", relu10)
    concat2 = torch.cat((relu8, lrelu(_crop_like(deconv("deconv5", relu10), relu8)),
                         _crop_like(deconv("upsample_flow6to5", flow6), relu8)), dim=1)
    flow5 = conv("Convolution2", concat2)
    concat3 = torch.cat((relu6, lrelu(_crop_like(deconv("deconv4", concat2), relu6)),
                         _crop_like(deconv("upsample_flow5to4", flow5), relu6)), dim=1)
    flow4 = conv("Convolution3", concat3)
    concat4 = torch.cat((relu4, lrelu(_crop_like(deconv("deconv3", concat3), relu4)),
                         _crop_like(deconv("upsample_flow4to3", flow4), relu4)), dim=1)
    flow3 = conv("Convolution4", concat4)
    concat5 = torch.cat((relu2, lrelu(_crop_like(deconv("deconv2", concat4), relu2)),
                         _crop_like(deconv("upsample_flow3to2", flow3), relu2)), dim=1)
    concat5 = pool(concat5)
    flow = conv("Convolution5", concat5) * 2.5
    if with_scale:
        scale = F.conv2d(concat5, sd[p + "Convolution5_scale.weight"])
        return flow, scale + torch.ones_like(scale)
    return flow


def embednet(x, sd, p="embednet."):
    """EmbedNet.forward (backbone/embednet.py:19-24)"""
    x = F.relu(F.conv2d(x, sd[p + "embed_conv1.weight"], sd[p + "embed_conv1.bias"]))
    x = F.relu(F.conv2d(x, sd[p + "embed_conv2.weight"], sd[p + "embed_conv2.bias"], 1, 1))
    return F.conv2d(x, sd[p + "embed_conv3.weight"], sd[p + "embed_conv3.bias"])


def fgfa_warp(feats, flow):
    """get_grid + resample (detector/generalized_rcnn_fgfa.py:45-62): bilinear, border padding, grid_sample's default
    align_corners (False in this container's torch, as when the reference itself runs here)"""
    m, n = flow.shape[-2:]
    sy, sx = torch.meshgrid(torch.arange(0, m, 1, dtype=torch.float32), torch.arange(0, n, 1, dtype=torch.float32),
                            indexing="ij")
    grid_dst = torch.stack((sx, sy)).unsqueeze(0)
    workspace = torch.tensor([(n - 1) / 2, (m - 1) / 2]).view(1, 2, 1, 1)
    flow_grid = ((flow + grid_dst) / workspace - 1).permute(0, 2, 3, 1)
    return F.grid_sample(feats, flow_grid, mode="bilinear", padding_mode="border")


class FgfaOracle:
    """GeneralizedRCNNFGFA._forward_test (detector/generalized_rcnn_fgfa.py:144-219), restated: window of 19 frames,
    key frame at 9; per frame backbone features + EmbedNet embedding are cached; every step FlowNetS estimates the
    flow from the key frame to all 19 window frames, the cached maps are warped, weighted per pixel by the cosine
    similarity of the warped embeddings (soft-max over frames) and summed; the single-frame box head follows.
    Frame 0's look-ahead frames come in infos["ref"] (list of tensors) instead of being read from disk (:180-190)."""

    def __init__(self, state_dict, cfg=None, record=False):
        self.sd = {k: v.detach().float() for k, v in state_dict.items()}
        self.cfg = cfg or Cfg(all_frame_interval=19, key_frame_location=9)
        self.record = record
        self.trace = {}

    def _frame(self, img):
        feats = resnet_c4_body(img, self.sd)
        return img, torch.cat([feats, embednet(feats, self.sd)], dim=1)

    def forward(self, img, infos):
        c, sd = self.cfg, self.sd
        im_h, im_w = img.shape[-2:]
        L, kl = c.all_frame_interval, c.key_frame_location
        if infos["frame_category"] == 0:
            self.images, self.features = deque(maxlen=L), deque(maxlen=L)
            cur = self._frame(img)
            while len(self.images) < kl + 1:
                self.images.append(cur[0]); self.features.append(cur[1])
            for im in infos["ref"]:
                if len(self.images) >= L:
                    break
                f = self._frame(im)
                self.images.append(f[0]); self.features.append(f[1])
            assert len(self.images) == L
        else:
            f = self._frame(infos["ref"][0])
            self.images.append(f[0]); self.features.append(f[1])
        all_images = torch.cat(list(self.images), 0)
        all_features = torch.cat(list(self.features), 0)
        cur_image = self.images[kl]
        pairs = torch.cat([cur_image.repeat(L, 1, 1, 1) / 255, all_images / 255], dim=1)
        flow = flownet_s(pairs, sd)
        warped = fgfa_warp(all_features, flow)
        wf, emb = torch.split(warped, (1024, 2048), dim=1)
        emb = emb.contiguous()
        emb_cur = emb[kl:kl + 1]
        en = emb / (torch.norm(emb, dim=1, keepdim=True) + 1e-10)
        ec = emb_cur / (torch.norm(emb_cur, dim=1, keepdim=True) + 1e-10)
        weights = F.softmax(torch.sum(en * ec, dim=1, keepdim=True), dim=0)
        feats = torch.sum(weights * wf, dim=0, keepdim=True)
        logits, deltas = rpn_head(feats, sd)
        prop, obj = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.post_nms_top_n, c.rpn_nms_thresh,
                               cuda_semantics=c.cuda_nms_semantics)
        x = res5_head(feats, sd, FE + "head.", c.res5_dilation)
        rois = torch.cat([torch.zeros(prop.shape[0], 1), prop], dim=1)
        x = roi_align(x, rois, c.pooler_scale, c.pooler_resolution, c.pooler_resolution, c.sampling_ratio).flatten(start_dim=1)
        x = F.relu(F.linear(x, sd[FE + "fc6.weight"], sd[FE + "fc6.bias"]))
        x = F.relu(F.linear(x, sd[FE + "fc7.weight"], sd[FE + "fc7.bias"]))
        cl = F.linear(x, sd["roi_heads.box.predictor.cls_score.weight"], sd["roi_heads.box.predictor.cls_score.bias"])
        bd = F.linear(x, sd["roi_heads.box.predictor.bbox_pred.weight"], sd["roi_heads.box.predictor.bbox_pred.bias"])
        if self.record:
            self.trace = {"proposals": prop.clone(), "class_logits": cl.clone(), "box_regression": bd.clone(),
                          "flow": flow.clone(), "feats": feats.clone(), "weights": weights.clone()}
        return box_postprocess(cl, bd, prop, im_w, im_h, c.score_thresh, c.nms_thresh, c.detections_per_img,
                               cuda_semantics=c.cuda_nms_semantics)


class DffOracle:
    """GeneralizedRCNNDFF._forward_test (detector/generalized_rcnn_dff.py:119-138), restated: the backbone runs on key
    frames only; every frame (key frames included) gets FlowNetS on the pair (frame, key frame) -> flow + scale map, the
    key frame's feature map is warped along the flow (get_grid / resample, :41-58 -- the same code as FGFA's) and
    multiplied by the scale map; the single-frame RPN + box head (ResNetConv52MLPFeatureExtractor, no channel
    reduction) follow."""

    def __init__(self, state_dict, cfg=None, record=False):
        self.sd = {k: v.detach().float() for k, v in state_dict.items()}
        self.cfg = cfg or Cfg()
        self.record = record
        self.trace = {}
        self.key_image = self.key_feats = None

    def forward(self, img, is_key_frame):
        c, sd = self.cfg, self.sd
        im_h, im_w = img.shape[-2:]
        if is_key_frame:
            self.key_image, self.key_feats = img, resnet_c4_body(img, sd)
        flow, scale = flownet_s(torch.cat([img / 255, self.key_image / 255], dim=1), sd, with_scale=True)
        feats = fgfa_warp(self.key_feats, flow) * scale
        logits, deltas = rpn_head(feats, sd)
        prop, obj = rpn_select(logits, deltas, im_w, im_h, c.pre_nms_top_n, c.post_nms_top_n, c.rpn_nms_thresh,
                               cuda_semantics=c.cuda_nms_semantics)
        x = res5_head(feats, sd, FE + "head.", c.res5_dilation)
        rois = torch.cat([torch.zeros(prop.shape[0], 1), prop], dim=1)
        x = roi_align(x, rois, c.pooler_scale, c.pooler_resolution, c.pooler_resolution, c.sampling_ratio).flatten(start_dim=1)
        x = F.relu(F.linear(x, sd[FE + "fc6.weight"], sd[FE + "fc6.bias"]))
        x = F.relu(F.linear(x, sd[FE + "fc7.weight"], sd[FE + "fc7.bias"]))
        cl = F.linear(x, sd["roi_heads.box.predictor.cls_score.weight"], sd["roi_heads.box.predictor.cls_score.bias"])
        bd = F.linear(x, sd["roi_heads.box.predictor.bbox_pred.weight"], sd["roi_heads.box.predictor.bbox_pred.bias"])
        if self.record:
            self.trace = {"proposals": prop.clone(), "class_logits": cl.clone(), "box_regression": bd.clone(),
                          "flow": flow.clone(), "scale": scale.clone(), "feats": feats.clone()}
        return box_postprocess(cl, bd, prop, im_w, im_h, c.score_thresh, c.nms_thresh, c.detections_per_img,
                               cuda_semantics=c.cuda_nms_semantics)


# --------------------------------------------------------------------------- ops outside the VID configs
def sigmoid_focal_loss(logits, targets, gamma, alpha):
    """layers/sigmoid_focal_loss.py:40-50 (the reference's own CPU formula for RetinaNet's focal loss)."""
    num_classes = logits.shape[1]
    class_range = torch.arange(1, num_classes + 1, dtype=targets.dtype).unsqueeze(0)
    t = targets.unsqueeze(1)
    p = torch.sigmoid(logits)
    term1 = (1 - p) ** gamma * torch.log(p)
    term2 = p ** gamma * torch.log(1 - p)
    return -(t == class_range).float() * term1 * alpha - ((t != class_range) * (t >= 0)).float() * term2 * (1 - alpha)


def deform_psroi_pool(data, rois, trans, no_trans, spatial_scale, output_dim, group_size, pooled_size, part_size,
                      sample_per_part, trans_std):
    """plain-Python restatement of DeformablePSROIPoolForwardKernel (csrc/cuda/deform_pool_kernel_cuda.cu:53-141);
    small inputs only. PARITY UNPINNED by any reference test or CPU implementation (deform_pool.h:37 has none)."""
    n_rois = rois.shape[0]
    _, channels, height, width = data.shape
    num_classes = 1 if no_trans else trans.shape[1] // 2
    cec = output_dim if no_trans else output_dim // num_classes
    out = torch.zeros(n_rois, output_dim, pooled_size, pooled_size)
    cnt = torch.zeros_like(out)
    f = np.float32
    for n in range(n_rois):
        b = int(rois[n, 0])
        sw = f(round(float(rois[n, 1]))) * f(spatial_scale) - f(0.5)
        sh = f(round(float(rois[n, 2]))) * f(spatial_scale) - f(0.5)
        ew = f(round(float(rois[n, 3])) + 1.0) * f(spatial_scale) - f(0.5)
        eh = f(round(float(rois[n, 4])) + 1.0) * f(spatial_scale) - f(0.5)
        rw, rh = max(f(ew - sw), f(0.1)), max(f(eh - sh), f(0.1))
        bh, bw = f(rh / f(pooled_size)), f(rw / f(pooled_size))
        sbh, sbw = f(bh / f(sample_per_part)), f(bw / f(sample_per_part))
        for ctop in range(output_dim):
            cls = ctop // cec
            for ph in range(pooled_size):
                for pw in range(pooled_size):
                    part_h = int(math.floor(f(ph) / pooled_size * part_size))
                    part_w = int(math.floor(f(pw) / pooled_size * part_size))
                    tx = f(0) if no_trans else f(trans[n, cls * 2, part_h, part_w]) * f(trans_std)
                    ty = f(0) if no_trans else f(trans[n, cls * 2 + 1, part_h, part_w]) * f(trans_std)
                    wstart = f(f(pw) * bw + sw) + f(tx * rw)
                    hstart = f(f(ph) * bh + sh) + f(ty * rh)
                    gw = min(max(int(math.floor(f(pw) * group_size / pooled_size)), 0), group_size - 1)
                    gh = min(max(int(math.floor(f(ph) * group_size / pooled_size)), 0), group_size - 1)
                    c = (ctop * group_size + gh) * group_size + gw
                    s, k = f(0), 0
                    for ih in range(sample_per_part):
                        for iw in range(sample_per_part):
                            w_ = f(wstart + f(iw) * sbw)
                            h_ = f(hstart + f(ih) * sbh)
                            if w_ < -0.5 or w_ > width - 0.5 or h_ < -0.5 or h_ > height - 0.5:
                                continue
                            w_ = min(max(w_, f(0)), f(width - 1))
                            h_ = min(max(h_, f(0)), f(height - 1))
                            x1, x2 = int(math.floor(w_)), int(math.ceil(w_))
                            y1, y2 = int(math.floor(h_)), int(math.ceil(h_))
                            dx, dy = f(w_ - x1), f(h_ - y1)
                            pl = data[b, c]
                            v = (1 - dx) * (1 - dy) * f(pl[y1, x1]) + (1 - dx) * dy * f(pl[y2, x1]) + \
                                dx * (1 - dy) * f(pl[y1, x2]) + dx * dy * f(pl[y2, x2])
                            s = f(s + f(v))
                            k += 1
                    out[n, ctop, ph, pw] = 0.0 if k == 0 else float(s / f(k))
                    cnt[n, ctop, ph, pw] = k
    return out, cnt
