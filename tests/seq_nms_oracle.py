"""Plain NumPy restatement of Seq-NMS as include/mega_b200.h (mega_seq_nms) specifies it -- the oracle the kernels of
csrc/seq_nms.cu and their host build must equal bit for bit. It recomputes the whole DP every iteration (the kernels
update it incrementally) and keeps every value in a plain array.

A video is a list of frames (boxes [n, 4] xyxy, scores [n], labels [n]); the result is, per frame, (keep bool [n],
new_scores float32 [n]) in the input order. Also: a seeded generator of synthetic videos, and the packing of videos into
the [F, D] tensors of the C ABI."""
import numpy as np

f32 = np.float32


def iou_gt(a, b, thresh):
    """bool [n, m]: RN(inter / union) > thresh, "+1" pixel convention, every operation rounded to fp32"""
    a = np.asarray(a, f32).reshape(-1, 4)
    b = np.asarray(b, f32).reshape(-1, 4)
    one = f32(1)
    sa = ((a[:, 2] - a[:, 0]) + one) * ((a[:, 3] - a[:, 1]) + one)
    sb = ((b[:, 2] - b[:, 0]) + one) * ((b[:, 3] - b[:, 1]) + one)
    w = np.maximum((np.minimum(a[:, None, 2], b[None, :, 2]) - np.maximum(a[:, None, 0], b[None, :, 0])) + one, f32(0))
    h = np.maximum((np.minimum(a[:, None, 3], b[None, :, 3]) - np.maximum(a[:, None, 1], b[None, :, 1])) + one, f32(0))
    inter = w * h
    union = (sa[:, None] + sb[None, :]) - inter
    with np.errstate(all="ignore"):
        return (inter / union) > f32(thresh)


def seq_nms_video(frames, link_iou=0.5, nms_iou=0.3, rescore="avg"):
    assert rescore in ("avg", "max")
    frames = [(np.asarray(b, f32).reshape(-1, 4), np.asarray(s, f32).reshape(-1), np.asarray(l).reshape(-1))
              for b, s, l in frames]
    T = len(frames)
    keep = [np.zeros(len(s), bool) for _, s, _ in frames]
    new_scores = [np.zeros(len(s), f32) for _, s, _ in frames]
    classes = sorted(set(int(c) for _, _, l in frames for c in l))
    for c in classes:
        idx = [np.nonzero(l == c)[0] for _, _, l in frames]              # class-c boxes, input order
        B = [frames[t][0][idx[t]] for t in range(T)]
        S = [frames[t][1][idx[t]] for t in range(T)]
        links = [iou_gt(B[t], B[t + 1], link_iou) for t in range(T - 1)]
        alive = [np.ones(len(i), bool) for i in idx]
        while any(a.any() for a in alive):
            best, succ = [None] * T, [None] * T
            for t in range(T - 1, -1, -1):
                n = len(B[t])
                m, arg = np.zeros(n), np.full(n, -1)
                if t + 1 < T and n and len(B[t + 1]):
                    cand = np.where(links[t] & alive[t + 1][None, :], best[t + 1][None, :], -np.inf)
                    has = cand.max(1) > -np.inf
                    m = np.where(has, cand.max(1), 0.0)
                    arg = np.where(has, cand.argmax(1), -1)               # argmax: first maximum = smallest j
                best[t] = np.where(alive[t], S[t].astype(np.float64) + m, -np.inf)
                succ[t] = arg
            root_v, root = -np.inf, None
            for t in range(T):                                           # strict >: smallest t, then smallest i
                if len(best[t]) and best[t].max() > root_v:
                    root_v, root = best[t].max(), (t, int(best[t].argmax()))
            chain = [root]
            while chain[-1][0] + 1 < T and succ[chain[-1][0]][chain[-1][1]] >= 0:
                t, i = chain[-1]
                chain.append((t + 1, int(succ[t][i])))
            if rescore == "avg":
                score = f32(root_v / len(chain))
            else:
                score = max(S[t][i] for t, i in chain)
            for t, i in chain:
                alive[t][i] = False
                keep[t][idx[t][i]] = True
                new_scores[t][idx[t][i]] = score
            for t, i in chain:
                alive[t] &= ~iou_gt(B[t], B[t][i], nms_iou)[:, 0]
    return list(zip(keep, new_scores))


def make_video(rng, n_frames, n_det, num_classes, dense_class=None, junk=0.8, size=(1000, 600)):
    """Seeded synthetic detections shaped like a detector's output on one video: a few objects drifting through the
    frames (several noisy boxes each, scores that wander), the rest junk boxes with scores just above the 0.001 test
    threshold. dense_class: a class that gets at least 100 boxes per frame. Labels ascending per frame (class-major)."""
    W, H = size
    n_obj = max(1, int(n_det * (1 - junk) / 6))
    obj_cls = rng.integers(1, num_classes, n_obj)
    pos = rng.uniform([0, 0], [W * 0.7, H * 0.7], (n_obj, 2))
    wh = rng.uniform(30, 300, (n_obj, 2))
    vel = rng.normal(0, 6, (n_obj, 2))
    frames = []
    for t in range(n_frames):
        pos = pos + vel
        boxes, scores, labels = [], [], []
        for o in range(n_obj):
            k = rng.integers(3, 9)
            jitter = rng.normal(0, 0.06, (k, 4)) * np.r_[wh[o], wh[o]]
            b = np.r_[pos[o], pos[o] + wh[o]] + jitter
            boxes.append(b)
            scores.append(np.clip(rng.beta(5, 2, k) * rng.uniform(0.3, 1.0), 1e-3, 1))
            labels.append(np.full(k, obj_cls[o]))
        n_fill = max(0, n_det - sum(len(s) for s in scores))
        n_dense = min(n_fill, 100) if dense_class is not None else 0
        xy = rng.uniform([0, 0], [W, H], (n_fill, 2))
        bw = rng.uniform(8, 400, (n_fill, 2))
        boxes.append(np.c_[xy, xy + bw])
        scores.append(1e-3 + rng.exponential(0.01, n_fill))
        lab = rng.integers(1, num_classes, n_fill)
        lab[:n_dense] = dense_class if dense_class is not None else 0
        labels.append(lab)
        b = np.concatenate(boxes).astype(f32)
        b = np.round(b * 4) / 4                      # quarter-pixel grid: exact IoU ties occur
        b[:, 2:] = np.maximum(b[:, 2:], b[:, :2])
        s = np.concatenate(scores).astype(f32)
        l = np.concatenate(labels).astype(np.int64)
        o = np.arange(min(len(l), n_det))
        o = o[np.argsort(l[o], kind="stable")]
        frames.append((b[o], s[o], l[o]))
    return frames


def pack(videos):
    """videos -> boxes [F, D, 4], scores [F, D], labels [F, D] int32, counts [F] int32, video_offsets [V+1] int32,
    num_classes (numpy arrays, the layout mega_seq_nms takes)"""
    frames = [f for v in videos for f in v]
    d = max([len(s) for _, s, _ in frames] + [1])
    F = len(frames)
    boxes, scores = np.zeros((F, d, 4), f32), np.zeros((F, d), f32)
    labels, counts = np.zeros((F, d), np.int32), np.zeros(F, np.int32)
    for i, (b, s, l) in enumerate(frames):
        n = len(s)
        boxes[i, :n], scores[i, :n], labels[i, :n], counts[i] = b, s, l, n
    offsets = np.cumsum([0] + [len(v) for v in videos]).astype(np.int32)
    num_classes = int(max([int(l.max()) + 1 for _, _, l in frames if len(l)] + [1]))
    return boxes, scores, labels, counts, offsets, num_classes


def unpack(videos, keep, new_scores):
    """[F, D] outputs -> per video, per frame (keep bool [n], new_scores float32 [n]); scores 0 where not kept"""
    out, f = [], 0
    for v in videos:
        res = []
        for _, s, _ in v:
            n = len(s)
            k = np.asarray(keep[f, :n]).astype(bool)
            res.append((k, np.where(k, np.asarray(new_scores[f, :n]), f32(0)).astype(f32)))
            f += 1
        out.append(res)
    return out
