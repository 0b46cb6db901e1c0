"""ImageNet-VID detection evaluation with the reference's function names and results
(data/datasets/evaluation/vid/vid_eval.py:14-343; SURVEY.md section 8f row 2).

Same protocol: per image and class the detections, sorted by score, are matched greedily against that class's
ground-truth boxes (IoU on integer-typed "+1" boxes, ignore flags from the motion-IoU range), the per-class match /
ignore lists are concatenated over the dataset, sorted by score, and turned into precision / recall and the
area-under-curve AP. What differs is where the time goes: the matching loops, which the reference runs in Python for every
(image, class, detection, box), are one native call per (image, class) (`mega_vid_match_host` in libmega_b200.so), and
the per-image bookkeeping is array code. Precision / recall / AP arrays equal the reference's element for element
(tests/test_vid_eval_cpu.py runs both on the same synthetic detections).

Proposal recall (box_only, the evaluation of an MODEL.RPN_ONLY run, vid_eval.py:72-119) runs on the GPU: the whole
dataset is one launch of the kernel of csrc/proposal_recall.cu, one CTA per image, instead of the reference's Python loop
of torch calls per greedy round and image."""
import os
from collections import defaultdict

import numpy as np
import torch

from ..... import _lib


def _match(pred_boxes, gt_boxes, gt_ignore, iou_thresh, empty_weight):
    p, g = pred_boxes.shape[0], gt_boxes.shape[0]
    match = np.zeros(p, dtype=np.int8)
    ignore = np.zeros(p, dtype=np.float64)
    pb = np.ascontiguousarray(pred_boxes, dtype=np.float32)
    gb = np.ascontiguousarray(gt_boxes, dtype=np.float32)
    gi = np.ascontiguousarray(gt_ignore != 0, dtype=np.uint8)
    _lib.check(_lib.lib.mega_vid_match_host(pb.ctypes.data, p, gb.ctypes.data, gi.ctypes.data, g, float(iou_thresh),
                                            float(empty_weight), match.ctypes.data, ignore.ctypes.data),
               "mega_vid_match_host")
    return match, ignore


def calc_detection_vid_prec_rec(gt_boxlists, pred_boxlists, motion_ious, iou_thresh=0.5, motion_range=(0., 1.)):
    """-> (prec, rec): lists indexed by class id (None where a class never occurs), as vid_eval.py:156-284"""
    lo, hi = motion_range
    if motion_ious is None:
        motion_ious = [None] * len(gt_boxlists)
        empty_weight = 0
    else:
        flat = np.concatenate(motion_ious, axis=0)
        empty_weight = np.count_nonzero((flat >= lo) & (flat <= hi)) / float(len(flat))
        if empty_weight == 1:
            empty_weight = 0
    n_pos = defaultdict(int)
    scores, matches, ignores = defaultdict(list), defaultdict(list), defaultdict(list)
    for gt, pred, motion in zip(gt_boxlists, pred_boxlists, motion_ious):
        pb, pl, ps = pred.bbox.numpy(), pred.get_field("labels").numpy(), pred.get_field("scores").numpy()
        gb, gl = gt.bbox.numpy(), gt.get_field("labels").numpy()
        g_ign = np.zeros(len(gb))
        if motion is not None and len(motion) > 0:
            m = np.asarray(motion, dtype=np.float64)[:len(gb)]
            g_ign[:len(m)] = ((m < lo) | (m > hi)).astype(np.float64)
        for l in np.unique(np.concatenate((pl, gl)).astype(int)):
            sel = pl == l
            order = ps[sel].argsort()[::-1]                    # the reference's (unstable) sort call: same tie order
            pb_l, ps_l = pb[sel][order], ps[sel][order]
            gsel = gl == l
            gb_l, gi_l = gb[gsel], g_ign[gsel]
            n_pos[l] += gb_l.shape[0] - gi_l.sum()
            scores[l].append(ps_l)
            if pb_l.shape[0] == 0:
                continue
            m_l, i_l = _match(pb_l, gb_l, gi_l, iou_thresh, empty_weight)
            matches[l].append(m_l)
            ignores[l].append(i_l)
    n_fg_class = max(n_pos.keys()) + 1
    prec, rec = [None] * n_fg_class, [None] * n_fg_class
    for l in n_pos.keys():
        cat = lambda parts, dt: np.concatenate(parts).astype(dt) if parts else np.zeros(0, dtype=dt)   # noqa: E731
        score_l, match_l, ign_l = cat(scores[l], np.float32), cat(matches[l], np.int8), cat(ignores[l], np.float64)
        order = score_l.argsort()[::-1]
        match_l, ign_l = match_l[order], ign_l[order]
        counted = ign_l != 1
        tps = (match_l == 1) & counted
        fps = ((match_l == 0) & counted) * np.where(ign_l == 0, 1.0, ign_l)      # fractional weight of "mixed" misses
        tp, fp = np.cumsum(tps), np.cumsum(fps)
        prec[l] = tp / (fp + tp + np.spacing(1))
        if n_pos[l] > 0:
            rec[l] = tp / n_pos[l]
    return prec, rec


def calc_detection_vid_ap(prec, rec, use_07_metric=False):
    """per-class average precision from precision / recall (vid_eval.py:287-343): area under the monotone envelope of the
    PR curve, or the 11-point VOC07 metric; NaN for classes without ground truth"""
    ap = np.full(len(prec), np.nan)
    for l, (p, r) in enumerate(zip(prec, rec)):
        if p is None or r is None:
            continue
        p = np.nan_to_num(p)
        if use_07_metric:
            ap[l] = sum((p[r >= t].max() if np.any(r >= t) else 0.0) / 11 for t in np.arange(0.0, 1.1, 0.1))
            continue
        mpre = np.concatenate(([0], p, [0]))
        mrec = np.concatenate(([0], r, [1]))
        mpre = np.maximum.accumulate(mpre[::-1])[::-1]
        step = np.where(mrec[1:] != mrec[:-1])[0]
        ap[l] = np.sum((mrec[step + 1] - mrec[step]) * mpre[step + 1])
    return ap


def eval_detection_vid(pred_boxlists, gt_boxlists, iou_thresh=0.5, motion_ranges=((0.0, 0.7), (0.7, 0.9), (0.9, 1.0)),
                       motion_specific=False, use_07_metric=False, motion_ious=None):
    """vid_eval.py:120-153; motion_specific reads the reference's vid_groundtruth_motion_iou.mat (from the working
    directory, like the reference) unless `motion_ious` is given"""
    assert len(gt_boxlists) == len(pred_boxlists), "Length of gt and pred lists need to be same."
    if motion_specific and motion_ious is None:
        import scipy.io as sio
        mat = sio.loadmat(os.path.join("mega_core", "data", "datasets", "evaluation", "vid",
                                       "vid_groundtruth_motion_iou.mat"))["motion_iou"]
        motion_ious = [[mat[i][0][j][0] if len(mat[i][0][j]) != 0 else 0 for j in range(len(mat[i][0]))]
                       for i in range(len(mat))]
    result = {}
    for index, rng in enumerate(motion_ranges):
        prec, rec = calc_detection_vid_prec_rec(gt_boxlists, pred_boxlists, motion_ious if motion_specific else None,
                                                iou_thresh, rng)
        ap = calc_detection_vid_ap(prec, rec, use_07_metric)
        result[index] = {"ap": ap, "map": np.nanmean(ap)}
    return result


def _pack(parts, out):
    """concatenate per-image fp32 tensors into `out` (a view of the pinned staging buffer)"""
    if parts:
        torch.cat([p.detach().reshape(-1).float().cpu() for p in parts], out=out.view(-1))


def _align(n, a=16):
    return (n + a - 1) // a * a


def _device():
    if not torch.cuda.is_available():
        raise _lib.MegaError("proposal recall runs on the GPU kernel of libmega_b200 only; no CUDA device is available")
    return torch.device("cuda", torch.cuda.current_device())


def proposal_recall(pred_boxlists, gt_boxlists, iou_thresh=0.5, limit=300):
    """the device half of eval_proposals_vid -> (hits, num_pos, gt_overlaps [sum G] fp32 on the host): the inputs packed
    into one pinned buffer, one host-to-device copy, one launch, one device-to-host copy of the counts and overlaps.
    gt_overlaps holds, per image and in GT order, the greedy rounds' overlaps followed by zeros; it is 0 throughout for
    images without GT or proposals, which the reference leaves out."""
    from .....b200 import ops
    assert len(gt_boxlists) == len(pred_boxlists), "Length of gt and pred lists need to be same."
    dev = _device()
    preds = [p.convert("xyxy") for p in pred_boxlists]
    gts = [g.convert("xyxy") for g in gt_boxlists]
    n = len(preds)
    p_cnt = [len(p) for p in preds]
    g_cnt = [len(g) for g in gts]
    p_tot, g_tot = sum(p_cnt), sum(g_cnt)
    sizes = [4 * 4 * p_tot, 4 * p_tot, 4 * 4 * g_tot, 8 * (n + 1), 8 * (n + 1)]
    offs = [0]
    for b in sizes:
        offs.append(offs[-1] + _align(b))
    host = torch.empty(offs[-1], dtype=torch.uint8, pin_memory=dev.type == "cuda")
    view = lambda i, dtype, shape: host[offs[i]:offs[i] + sizes[i]].view(dtype).view(*shape)   # noqa: E731
    _pack([p.bbox for p in preds], view(0, torch.float32, (p_tot, 4)))
    _pack([p.get_field("objectness") for p in preds], view(1, torch.float32, (p_tot,)))
    _pack([g.bbox for g in gts], view(2, torch.float32, (g_tot, 4)))
    view(3, torch.int64, (n + 1,)).copy_(torch.tensor([0] + p_cnt, dtype=torch.int64).cumsum(0))
    view(4, torch.int64, (n + 1,)).copy_(torch.tensor([0] + g_cnt, dtype=torch.int64).cumsum(0))
    buf = host.to(dev, non_blocking=True)
    dview = lambda i, dtype, shape: buf[offs[i]:offs[i] + sizes[i]].view(dtype).view(*shape)   # noqa: E731
    out = torch.empty(24 + _align(4 * g_tot), dtype=torch.uint8, device=dev)
    stats, overlaps = out[:24].view(torch.int64), out[24:24 + 4 * g_tot].view(torch.float32)
    ops.proposal_recall(dview(0, torch.float32, (p_tot, 4)), dview(1, torch.float32, (p_tot,)),
                        dview(3, torch.int64, (n + 1,)), dview(2, torch.float32, (g_tot, 4)),
                        dview(4, torch.int64, (n + 1,)), max(p_cnt + [0]), max(g_cnt + [0]), limit, iou_thresh,
                        overlaps, stats)
    res = out.cpu()
    hits, num_pos, rejected = res[:24].view(torch.int64).tolist()
    assert rejected == 0, "proposal_recall: %d images exceed the packed bounds" % rejected
    return hits, num_pos, res[24:24 + 4 * g_tot].view(torch.float32)


def eval_proposals_vid(pred_boxlists, gt_boxlists, iou_thresh=0.5, limit=300):
    """vid_eval.py:72-119: per image the proposals sorted by `objectness` (descending), the first `limit` of them
    matched one to one with the GT boxes, greedily by largest IoU; recall = matched overlaps >= iou_thresh over all GT.
    -> {"recall": float32 tensor}. GPU only: without a CUDA device this raises."""
    hits, num_pos, _ = proposal_recall(pred_boxlists, gt_boxlists, iou_thresh, limit)
    return {"recall": torch.tensor(float(hits), dtype=torch.float32) / float(num_pos)}


def do_vid_evaluation(dataset, predictions, output_folder, box_only, motion_specific, logger):
    """vid_eval.py:14-69; box_only (the proposals of an MODEL.RPN_ONLY run): proposal recall, logged and written to
    proposal_result.txt, returns None"""
    preds, gts = [], []
    for image_id, prediction in enumerate(predictions):
        info = dataset.get_img_info(image_id)
        preds.append(prediction.resize((info["width"], info["height"])))
        gts.append(dataset.get_groundtruth(image_id))
    if box_only:
        result = eval_proposals_vid(preds, gts, iou_thresh=0.5)
        text = "Recall: {:.4f}".format(result["recall"])
        logger.info(text)
        if output_folder:
            with open(os.path.join(output_folder, "proposal_result.txt"), "w") as fid:
                fid.write(text)
        return None
    ranges = [[0.0, 1.0], [0.0, 0.7], [0.7, 0.9], [0.9, 1.0]] if motion_specific else [[0.0, 1.0]]
    names = ["all", "fast", "medium", "slow"][:len(ranges)]
    result = eval_detection_vid(preds, gts, 0.5, ranges, motion_specific, False)
    text = "".join("AP50 | motion={:>6s} = {:0.4f}\n".format(n, result[i]["map"]) for i, n in enumerate(names))
    text += "Category AP:\n"
    for i, ap in enumerate(result[0]["ap"]):
        if i:                                          # class 0 is the background
            text += "{:<16}: {:.4f}\n".format(dataset.map_class_id_to_class_name(i), ap)
    logger.info("\n" + text)
    if output_folder:
        with open(os.path.join(output_folder, "result.txt"), "w") as fid:
            fid.write(text)
    return result
