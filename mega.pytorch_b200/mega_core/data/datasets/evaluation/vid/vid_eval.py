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
of torch calls per greedy round and image.

Detection AP can run on the GPU too (`device=True` of eval_detection_vid, `vid_eval="device"` of do_vid_evaluation,
MODEL.B200.VID_EVAL): the kernels of csrc/vid_eval.cu score every motion range of the whole dataset in one pass and hand
back the compacted precision-recall steps, whose AP the host sums with numpy as before. Ties between equal scores are
ordered by a fixed rule there (`stable_ties=True` of the host evaluator: argsort(kind="stable")[::-1]) instead of the
CPU-dependent order of numpy's default sort, so the device results equal the host evaluator with stable_ties=True bit
for bit."""
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


def _empty_weight(motion_ious, motion_range):
    """the ignore weight of detections of a class without GT in their image (vid_eval.py:171-175)"""
    if motion_ious is None:
        return 0
    lo, hi = motion_range
    flat = np.concatenate(motion_ious, axis=0)
    empty_weight = np.count_nonzero((flat >= lo) & (flat <= hi)) / float(len(flat))
    return 0 if empty_weight == 1 else empty_weight


def _argsort_desc(a, stable_ties):
    """the reference's a.argsort()[::-1] (numpy's default sort: the order of tied scores depends on the CPU's SIMD
    dispatch), or with stable_ties the same order with ties defined: later position first"""
    return (np.argsort(a, kind="stable") if stable_ties else a.argsort())[::-1]


def calc_detection_vid_prec_rec(gt_boxlists, pred_boxlists, motion_ious, iou_thresh=0.5, motion_range=(0., 1.),
                                stable_ties=False, return_n_pos=False):
    """-> (prec, rec): lists indexed by class id (None where a class never occurs), as vid_eval.py:156-284.
    stable_ties: both score sorts order ties by argsort(kind="stable")[::-1], the order of the device evaluator.
    return_n_pos: -> (prec, rec, {class: n_pos})"""
    lo, hi = motion_range
    empty_weight = _empty_weight(motion_ious, motion_range)
    if motion_ious is None:
        motion_ious = [None] * len(gt_boxlists)
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
            order = _argsort_desc(ps[sel], stable_ties)
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
        order = _argsort_desc(score_l, stable_ties)
        match_l, ign_l = match_l[order], ign_l[order]
        counted = ign_l != 1
        tps = (match_l == 1) & counted
        fps = ((match_l == 0) & counted) * np.where(ign_l == 0, 1.0, ign_l)      # fractional weight of "mixed" misses
        tp, fp = np.cumsum(tps), np.cumsum(fps)
        prec[l] = tp / (fp + tp + np.spacing(1))
        if n_pos[l] > 0:
            rec[l] = tp / n_pos[l]
    if return_n_pos:
        return prec, rec, dict(n_pos)
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
                       motion_specific=False, use_07_metric=False, motion_ious=None, stable_ties=False, device=False,
                       return_curves=False, image_sizes=None):
    """vid_eval.py:120-153; motion_specific reads the reference's vid_groundtruth_motion_iou.mat (from the working
    directory, like the reference) unless `motion_ious` is given.
    device: all ranges in one pass of the kernels of csrc/vid_eval.cu (ties ordered as with stable_ties=True; GPU only,
    without a CUDA device this raises); image_sizes (device only): per image the (width, height) the predictions are
    resized to first, BoxList.resize applied in the kernel. return_curves: each result also holds "prec", "rec" (lists
    by class) and "n_pos" ({class: count})."""
    assert len(gt_boxlists) == len(pred_boxlists), "Length of gt and pred lists need to be same."
    if motion_specific and motion_ious is None:
        import scipy.io as sio
        mat = sio.loadmat(os.path.join("mega_core", "data", "datasets", "evaluation", "vid",
                                       "vid_groundtruth_motion_iou.mat"))["motion_iou"]
        motion_ious = [[mat[i][0][j][0] if len(mat[i][0][j]) != 0 else 0 for j in range(len(mat[i][0]))]
                       for i in range(len(mat))]
    motion = motion_ious if motion_specific else None
    if device:
        return vid_eval_device(pred_boxlists, gt_boxlists, motion, iou_thresh, motion_ranges, use_07_metric,
                               return_curves, image_sizes)
    assert image_sizes is None, "image_sizes: device evaluation only"
    result = {}
    for index, rng in enumerate(motion_ranges):
        prec, rec, n_pos = calc_detection_vid_prec_rec(gt_boxlists, pred_boxlists, motion, iou_thresh, rng,
                                                       stable_ties, return_n_pos=True)
        ap = calc_detection_vid_ap(prec, rec, use_07_metric)
        result[index] = {"ap": ap, "map": np.nanmean(ap)}
        if return_curves:
            result[index].update({"prec": prec, "rec": rec, "n_pos": n_pos})
    return result


def _ap_from_steps(dr, mp, rr, use_07_metric):
    """calc_detection_vid_ap of one class from its compacted recall steps (mega_vid_eval): the products and np.sum of
    :98-102 over the same values; the VOC07 maximum over r >= t is the envelope at the first step reaching t"""
    if use_07_metric:
        return sum((mp[rr >= t].max() if np.any(rr >= t) else 0.0) / 11 for t in np.arange(0.0, 1.1, 0.1))
    return np.sum(dr * mp)


class _VidEvalInputs(object):
    """the packed inputs of mega_vid_eval in one (pinned) host buffer: section i of `buf` is view(buf, i), in the order
    of the C ABI's arguments (det boxes, scores, labels, offsets, scales, GT boxes, labels, motion, offsets, step
    offsets); the sizes and ranges ride along"""

    def __init__(self, pred_boxlists, gt_boxlists, motion_ious, motion_ranges, image_sizes, pin):
        n = len(pred_boxlists)
        preds, scale = [], torch.ones(n, 2, dtype=torch.float32)
        if image_sizes is not None:
            assert len(image_sizes) == n
            for i, (p, (w, h)) in enumerate(zip(pred_boxlists, image_sizes)):
                if p.mode == "xyxy":             # BoxList.resize: bbox * tensor([rw, rh, rw, rh]) (fp32), in the kernel
                    scale[i] = torch.tensor([float(w) / p.size[0], float(h) / p.size[1]])
                    preds.append(p)
                else:
                    preds.append(p.resize((w, h)))
        else:
            preds = list(pred_boxlists)
        p_cnt = [len(p) for p in preds]
        g_cnt = [len(g) for g in gt_boxlists]
        p_tot, g_tot = sum(p_cnt), sum(g_cnt)
        det_labels = torch.cat([p.get_field("labels").reshape(-1).to(torch.int32) for p in preds] +
                               [torch.zeros(0, dtype=torch.int32)])
        gt_labels = torch.cat([g.get_field("labels").reshape(-1).to(torch.int32) for g in gt_boxlists] +
                              [torch.zeros(0, dtype=torch.int32)])
        both = torch.cat([det_labels, gt_labels])
        assert both.numel() > 0, "VID evaluation: no detections and no ground truth"
        assert int(both.min()) >= 0, "VID evaluation: negative class labels"
        num_classes = int(both.max()) + 1
        # capacity of a class's recall steps: its GT count + 2 (n_pos + 1 at most, see ve_steps)
        step_off = np.concatenate([[0], np.cumsum(np.bincount(gt_labels.numpy(), minlength=num_classes) + 2)])
        gt_motion = np.full(g_tot, np.nan)
        if motion_ious is not None:
            assert len(motion_ious) == n
            if all(m is not None and np.ndim(m) == 1 and len(m) == c for m, c in zip(motion_ious, g_cnt)):
                if g_tot:
                    gt_motion[:] = np.concatenate([np.asarray(m, dtype=np.float64) for m in motion_ious])
            else:                                # vid_eval.py:193-197: motion[:len(gb)], the rest not ignored
                off = 0
                for m, c in zip(motion_ious, g_cnt):
                    if m is not None and len(m) > 0:
                        m = np.asarray(m, dtype=np.float64)[:c]
                        gt_motion[off:off + len(m)] = m
                    off += c
        self.n, self.p_tot, self.g_tot, self.num_classes = n, p_tot, g_tot, num_classes
        self.ranges = [(float(lo), float(hi), float(_empty_weight(motion_ious, (lo, hi)))) for lo, hi in motion_ranges]
        self.step_off = step_off.astype(np.int64)
        self.num_steps = int(step_off[-1])
        self.sizes = [16 * p_tot, 4 * p_tot, 4 * p_tot, 8 * (n + 1), 8 * n, 16 * g_tot, 4 * g_tot, 8 * g_tot,
                      8 * (n + 1), 8 * (num_classes + 1)]
        self.offs = [0]
        for b in self.sizes:
            self.offs.append(self.offs[-1] + _align(b))
        self.host = torch.empty(self.offs[-1], dtype=torch.uint8, pin_memory=pin)
        _pack([p.bbox for p in preds], self.view(self.host, 0))
        _pack([p.get_field("scores") for p in preds], self.view(self.host, 1))
        self.view(self.host, 2).copy_(det_labels)
        self.view(self.host, 3).copy_(torch.tensor([0] + p_cnt, dtype=torch.int64).cumsum(0))
        self.view(self.host, 4).copy_(scale)
        _pack([g.bbox for g in gt_boxlists], self.view(self.host, 5))
        self.view(self.host, 6).copy_(gt_labels)
        self.view(self.host, 7).copy_(torch.from_numpy(gt_motion))
        self.view(self.host, 8).copy_(torch.tensor([0] + g_cnt, dtype=torch.int64).cumsum(0))
        self.view(self.host, 9).copy_(torch.from_numpy(self.step_off))

    def view(self, buf, i):
        p, g, n, c = self.p_tot, self.g_tot, self.n, self.num_classes
        dtype, shape = [(torch.float32, (p, 4)), (torch.float32, (p,)), (torch.int32, (p,)), (torch.int64, (n + 1,)),
                        (torch.float32, (n, 2)), (torch.float32, (g, 4)), (torch.int32, (g,)), (torch.float64, (g,)),
                        (torch.int64, (n + 1,)), (torch.int64, (c + 1,))][i]
        return buf[self.offs[i]:self.offs[i] + self.sizes[i]].view(dtype).view(*shape)

    def stats_count(self):
        return 3 * self.num_classes + 2 * len(self.ranges) * self.num_classes + 1

    def results(self, stats, steps, curves, use_07_metric=False, return_curves=False):
        """stats [stats_count()] int64, steps [R, 3, num_steps] fp64, curves [2, R, P] fp64 or None (numpy, host) ->
        {range index: {"ap", "map"} (+ "prec", "rec", "n_pos" with return_curves)}"""
        C, nr = self.num_classes, len(self.ranges)
        present, begin, end = stats[:C], stats[C:2 * C], stats[2 * C:3 * C]
        n_pos = stats[3 * C:3 * C + nr * C].reshape(nr, C)
        n_steps = stats[3 * C + nr * C:3 * C + 2 * nr * C].reshape(nr, C)
        assert stats[-1] == 0, "vid_eval: %d labels out of range or step lists over capacity" % stats[-1]
        n_fg = int(np.nonzero(present)[0].max()) + 1
        result = {}
        for r in range(nr):
            ap = np.full(n_fg, np.nan)
            for c in range(n_fg):
                k = int(n_steps[r, c])
                if present[c] and k >= 0:
                    o = int(self.step_off[c])
                    ap[c] = _ap_from_steps(steps[r, 0, o:o + k], steps[r, 1, o:o + k], steps[r, 2, o:o + k],
                                           use_07_metric)
            result[r] = {"ap": ap, "map": np.nanmean(ap)}
            if return_curves:
                result[r]["prec"] = [curves[0, r, begin[c]:end[c]] if present[c] else None for c in range(n_fg)]
                result[r]["rec"] = [curves[1, r, begin[c]:end[c]] if present[c] and n_pos[r, c] > 0 else None
                                    for c in range(n_fg)]
                result[r]["n_pos"] = {c: int(n_pos[r, c]) for c in range(n_fg) if present[c]}
        return result


def vid_eval_device(pred_boxlists, gt_boxlists, motion_ious, iou_thresh, motion_ranges, use_07_metric=False,
                    return_curves=False, image_sizes=None):
    """the device half of eval_detection_vid: inputs packed into one pinned buffer, one host-to-device copy, one launch
    sequence of mega_vid_eval for all ranges, one device-to-host copy of the counts and recall steps (plus prec / rec
    per detection with return_curves). -> {range index: {"ap", "map"}}"""
    from .....b200 import ops
    dev = _device("VID evaluation (MODEL.B200.VID_EVAL = \"device\")")
    x = _VidEvalInputs(pred_boxlists, gt_boxlists, motion_ious, motion_ranges, image_sizes, pin=True)
    nr, n_stats = len(x.ranges), x.stats_count()
    buf = x.host.to(dev, non_blocking=True)
    out = torch.empty(8 * n_stats + 8 * nr * 3 * x.num_steps, dtype=torch.uint8, device=dev)
    stats, steps = out[:8 * n_stats].view(torch.int64), out[8 * n_stats:].view(torch.float64)
    curves = torch.empty(2, nr, x.p_tot, dtype=torch.float64, device=dev)
    ops.vid_eval(*[x.view(buf, i) for i in range(9)], x.num_classes, x.ranges, iou_thresh, x.view(buf, 9),
                 x.num_steps, curves[0], curves[1], stats, steps)
    res = out.cpu()
    return x.results(res[:8 * n_stats].view(torch.int64).numpy(),
                     res[8 * n_stats:].view(torch.float64).numpy().reshape(nr, 3, x.num_steps),
                     curves.cpu().numpy() if return_curves else None, use_07_metric, return_curves)


def _pack(parts, out):
    """concatenate per-image fp32 tensors into `out` (a view of the pinned staging buffer)"""
    if parts:
        torch.cat([p.detach().reshape(-1).float().cpu() for p in parts], out=out.view(-1))


def _align(n, a=16):
    return (n + a - 1) // a * a


def _device(what="proposal recall"):
    if not torch.cuda.is_available():
        raise _lib.MegaError("%s runs on the GPU kernels of libmega_b200 only; no CUDA device is available" % what)
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


def do_vid_evaluation(dataset, predictions, output_folder, box_only, motion_specific, logger, vid_eval="host"):
    """vid_eval.py:14-69; box_only (the proposals of an MODEL.RPN_ONLY run): proposal recall, logged and written to
    proposal_result.txt, returns None. vid_eval (MODEL.B200.VID_EVAL): "host" -- the host evaluator, the reference's
    tie order; "device" -- all motion ranges in one pass of the GPU kernels, ties ordered as with stable_ties=True,
    the predictions resized to the images' sizes in the kernel"""
    if vid_eval not in ("host", "device"):
        raise ValueError("MODEL.B200.VID_EVAL must be \"host\" or \"device\", got %r" % (vid_eval,))
    device = vid_eval == "device" and not box_only
    preds, gts, sizes = [], [], []
    for image_id, prediction in enumerate(predictions):
        info = dataset.get_img_info(image_id)
        if device:
            preds.append(prediction)
            sizes.append((info["width"], info["height"]))
        else:
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
    result = eval_detection_vid(preds, gts, 0.5, ranges, motion_specific, False, device=device,
                                image_sizes=sizes if device else None)
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
