"""Seq-NMS (Han et al., "Seq-NMS for Video Object Detection", arXiv:1602.08465): sequence-level post-processing of the
detections of whole videos, run after the per-frame detector and before VID evaluation. The FGFA / MEGA papers report
results with and without it; the reference ships no implementation.

Per video and class: link boxes of consecutive frames whose IoU exceeds `link_iou`, pick the chain with the highest
score sum, give its boxes the chain's average (`rescore="avg"`) or maximum (`"max"`) score, suppress the boxes of each of
its frames that overlap its box there by more than `nms_iou`, and repeat until no box of the class is left. The exact
rule is the contract of `mega_seq_nms` (include/mega_b200.h); the work runs in the CUDA kernels of csrc/seq_nms.cu, many
videos per launch. GPU only, like every op of this package: without a CUDA device the calls raise."""
import torch

from .. import _lib
from ..b200 import ops
from ..structures.bounding_box import BoxList

DEFAULTS = {"link_iou": 0.5, "nms_iou": 0.3, "rescore": "avg"}
# frames per launch: bounds the workspace (about 0.2 GB at 300 detections per frame and 31 classes)
FRAMES_PER_LAUNCH = 16384


def _device():
    if not torch.cuda.is_available():
        raise _lib.MegaError("seq_nms runs on the GPU kernels of libmega_b200 only; no CUDA device is available")
    return torch.device("cuda", torch.cuda.current_device())


def _run(videos, link_iou, nms_iou, rescore):
    """videos: list of lists of BoxLists -> the same nesting, Seq-NMS applied per video; one launch per chunk of
    FRAMES_PER_LAUNCH frames (whole videos)."""
    frames = [b.convert("xyxy") for v in videos for b in v]
    if not frames:
        return [[] for _ in videos]
    dev = _device()
    counts = [len(b) for b in frames]
    d = max(max(counts), 1)
    labels_all = [b.get_field("labels").reshape(-1).long().cpu() for b in frames]
    num_classes = max([int(l.max()) + 1 for l in labels_all if l.numel()] + [1])
    if any(int(l.min()) < 0 for l in labels_all if l.numel()):
        raise ValueError("seq_nms: labels must be non-negative class ids")
    # the kernels take each frame's detections class-major (labels ascending); a stable sort keeps the input order
    # inside a class, which is the order the rules' "smallest index" ties refer to
    orders = [torch.argsort(l, stable=True) for l in labels_all]
    f_total = len(frames)
    boxes = torch.zeros(f_total, d, 4, dtype=torch.float32)
    scores = torch.zeros(f_total, d, dtype=torch.float32)
    labels = torch.zeros(f_total, d, dtype=torch.int32)
    for i, (b, l, o) in enumerate(zip(frames, labels_all, orders)):
        n = counts[i]
        boxes[i, :n] = b.bbox.float().cpu()[o]
        scores[i, :n] = b.get_field("scores").reshape(-1).float().cpu()[o]
        labels[i, :n] = l[o].int()
    new_scores = torch.zeros(f_total, d, dtype=torch.float32)
    keep = torch.zeros(f_total, d, dtype=torch.uint8)
    lengths = [len(v) for v in videos]
    start = v0 = 0
    while v0 < len(videos):
        v1, n_frames = v0, 0
        while v1 < len(videos) and (v1 == v0 or n_frames + lengths[v1] <= FRAMES_PER_LAUNCH):
            n_frames += lengths[v1]
            v1 += 1
        offsets = torch.tensor([0] + lengths[v0:v1], dtype=torch.int32).cumsum(0).int()
        sl = slice(start, start + n_frames)
        if n_frames:
            ns, kp = ops.seq_nms(boxes[sl].to(dev), scores[sl].to(dev), labels[sl].to(dev),
                                 torch.tensor(counts[sl], dtype=torch.int32).to(dev), offsets.to(dev), num_classes,
                                 link_iou=link_iou, nms_iou=nms_iou, rescore=rescore)
            new_scores[sl], keep[sl] = ns.cpu(), kp.cpu()
        start, v0 = start + n_frames, v1
    out, i = [], 0
    for v in videos:
        res = []
        for b in v:
            n, o = counts[i], orders[i]
            k = torch.zeros(n, dtype=torch.bool)
            s = torch.zeros(n, dtype=torch.float32)
            k[o] = keep[i, :n].bool()
            s[o] = new_scores[i, :n]
            idx = torch.nonzero(k).reshape(-1)
            r = b[idx.to(b.bbox.device)]
            r.add_field("scores", s[idx].to(b.bbox.device))
            res.append(r)
            i += 1
        out.append(res)
    return out


def seq_nms(boxlists, link_iou=0.5, nms_iou=0.3, rescore="avg"):
    """Seq-NMS of ONE video: `boxlists` = its frames in frame order (BoxLists with `scores` and `labels`, as the
    detector returns them). Returns one BoxList per frame: the selected boxes with their new scores and unchanged labels
    and other fields, in the input order; suppressed boxes are gone."""
    return _run([list(boxlists)], link_iou, nms_iou, rescore)[0]


def seq_nms_predictions(predictions, dataset, link_iou=0.5, nms_iou=0.3, rescore="avg"):
    """{image_id: BoxList} of a VID dataset -> {image_id: BoxList} after Seq-NMS. Frames are grouped into videos by the
    dataset's `pattern` (the video) and `frame_seg_id` (the frame's position in it); a missing frame ends a chain like
    an empty one. All videos go through the kernels together, many per launch."""
    ids = sorted(predictions.keys(), key=lambda i: (dataset.pattern[i], dataset.frame_seg_id[i]))
    videos, video_ids, prev = [], [], None
    for i in ids:
        key = (dataset.pattern[i], dataset.frame_seg_id[i])
        if prev is None or key[0] != prev[0] or key[1] != prev[1] + 1:
            videos.append([])
            video_ids.append([])
        videos[-1].append(predictions[i])
        video_ids[-1].append(i)
        prev = key
    out = {}
    for vid, res in zip(video_ids, _run(videos, link_iou, nms_iou, rescore)):
        out.update(zip(vid, res))
    return out
