"""Shared pieces of the proposal / NMS / box-head post-processing conformance suite
(test_proposals_conformance_cpu.py / _gpu.py).

Kernels covered: csrc/proposals.cu (mega_nms: nms_sort_kernel, nms_mask_kernel, nms_sweep_kernel, nms_finalize_kernel;
mega_rpn_select: rpn_topk_decode_kernel, then rpn_nms_greedy_kernel or nms_mask_kernel + nms_sweep_kernel +
rpn_write_kernel) and csrc/postprocess.cu (mega_box_postprocess: box_class_nms_kernel, box_final_kernel).

Continuous values (RPN scores, decoded and clipped boxes, class probabilities). An exact-order fp32 restatement of
decode_box / clip_box (proposals.cu) and class_softmax_prob / decode_clip_box (box_head.cuh), with every expf result
replaced by the two floats 2 ulp below and 2 ulp above RN(exp(x)) (the CUDA Programming Guide's bound for expf; the
library is built without -use_fast_math). Sigmoid, decode and clip are monotone in each expf result, so the chain
evaluated at the two ends of the bracket gives a sound interval with no fitted constant. The soft-max bounds the
numerator and the in-order fp32 sum separately: lo = RN(e_j,lo / sum_hi), hi = RN(e_j,hi / sum_lo).

Decisions (top-k set and order, min_size validity, NMS keep lists, score cut, detections_per_img cut, output order, zero
fill) must be exact, given the device's own continuous values. A "transparency" call of the same kernels returns those
values: RPN with nms_thresh = 1, min_size = 0, post = k (every pre-NMS box, score and anchor, in the kernel's order: for
boxes with non-negative +1 widths inter <= min(sa, sb) in fp32, so RN(inter / u) <= 1 and no IoU exceeds 1); the box
head with score_thresh = -1, nms_thresh = 1, max_det = 0 and out_cap = (C - 1) R (every (class, proposal) probability and
box, class-major). expected_rpn / expected_box compute the real call's result on the host from them.

restated_rpn / restated_nms / restated_box run the whole contract on the host (top-k radix tie quota, the greedy
64-chunk sweep or the mask + sweep path, the class-major compaction); `bugs` plants a named mistake in them, and the
CPU file checks that the GPU file's checks reject each one.
"""
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mega_oracle  # noqa: E402

F32 = np.float32
CSRC = os.path.join(ROOT, "mega.pytorch_b200", "csrc")
EXP_ULP = 2                                  # expf error bound (CUDA Programming Guide, single-precision functions)
CLIP = F32(4.135166556742356)                # log(1000 / 16), the dw / dh clamp of both decoders
BOX_W = (10.0, 10.0, 5.0, 5.0)               # MODEL.ROI_HEADS.BBOX_REG_WEIGHTS

# constants of the kernels (test_proposals_conformance_cpu.py reads them back from the source)
K_NMS_MAX_BOXES = 8192
K_GREEDY_MAX_KEEP = 1024
K_MAX_ROIS = 512


def source_constant(fname, name):
    src = open(os.path.join(CSRC, fname)).read()
    return int(re.search(r"constexpr int %s = (\d+);" % name, src).group(1))


# ------------------------------------------------------------------------------------------------ dispatch
SORT, MASK, SWEEP, FINAL = "nms_sort_kernel", "nms_mask_kernel", "nms_sweep_kernel", "nms_finalize_kernel"
TOPK, GREEDY, WRITE = "rpn_topk_decode_kernel", "rpn_nms_greedy_kernel", "rpn_write_kernel"
CLS_NMS, BOX_FINAL = "box_class_nms_kernel", "box_final_kernel"
ALL_KERNELS = (SORT, MASK, SWEEP, FINAL, TOPK, GREEDY, WRITE, CLS_NMS, BOX_FINAL)


def nms_kernels(n):
    """mega_nms: nothing for n = 0 (count set by a memset), else sort, mask, sweep, finalize"""
    return [] if n == 0 else [SORT, MASK, SWEEP, FINAL]


def rpn_path(post):
    return "greedy" if post <= K_GREEDY_MAX_KEEP else "mask"


def rpn_kernels(n_anchors, pre, post):
    """mega_rpn_select: top-k + decode, then the one-CTA greedy NMS (post <= kGreedyMaxKeep) or mask + sweep + write;
    an empty map (k = 0) on the mask path launches only the write kernel"""
    k = min(pre, n_anchors)
    if rpn_path(post) == "greedy":
        return [TOPK, GREEDY]
    return [TOPK, MASK, SWEEP, WRITE] if k > 0 else [TOPK, WRITE]


def box_kernels():
    return [CLS_NMS, BOX_FINAL]


# ------------------------------------------------------------------------------------------------ fp32 helpers
def f32(x):
    return np.asarray(x, dtype=F32)


def exp_rn(x):
    """RN(exp(x)) of fp32 x, the centre of the expf bracket"""
    with np.errstate(over="ignore"):
        return np.exp(np.asarray(x, dtype=np.float64)).astype(F32)


def _step(v, n, up):
    v = np.array(v, dtype=F32, copy=True)
    to = F32(np.inf) if up else F32(0)
    for _ in range(n):
        v = np.where(np.isnan(v), v, np.nextafter(v, to))
    return v


def exp_bracket(x):
    """(lo, hi): the floats EXP_ULP ulp below and above RN(exp(x)); exp is positive, so lo >= 0"""
    x = f32(x)
    c = exp_rn(x)
    lo, hi = _step(c, EXP_ULP, False), _step(c, EXP_ULP, True)
    over, under = x >= F32(89), x <= F32(-110)     # far past overflow / below half the smallest subnormal: exact
    return np.where(over, F32(np.inf), np.where(under, F32(0), lo)), np.where(over, F32(np.inf), np.where(under, F32(0), hi))


def ord_key(s):
    """the kernels' ascending sort key of a score: ~f2ord(s) (descending score, a positive NaN first)"""
    b = np.asarray(s, dtype=F32).view(np.uint32)
    o = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return (~o).astype(np.uint32)


def ulp_dist(a, b):
    """distance in units in the last place between fp32 arrays (same sign assumed; 0 where equal)"""
    ia = np.asarray(a, dtype=F32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, dtype=F32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


# ------------------------------------------------------------------------------------------------ continuous values
def sigmoid32(e):
    """1 / (1 + expf(-logit)) in fp32, e = expf(-logit)"""
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        return F32(1) / (F32(1) + f32(e))


def score_interval(logits):
    """(lo, centre, hi) of the RPN score of each logit"""
    lo_e, hi_e = exp_bracket(-f32(logits))
    return sigmoid32(hi_e), sigmoid32(exp_rn(-f32(logits))), sigmoid32(lo_e)


def decode_args(d, w):
    """dw, dh: the expf arguments of decode_box / decode_clip_box (d [..., 4])"""
    d = f32(d)
    return np.minimum(d[..., 2] / F32(w[2]), CLIP), np.minimum(d[..., 3] / F32(w[3]), CLIP)


def decode_clip32(d, box, ew, eh, w, im_w, im_h):
    """decode_box + clip_box (proposals.cu) == decode_clip_box (box_head.cuh), fp32 in the kernels' order, with the
    expf results ew, eh given"""
    d, box = f32(d), f32(box)
    with np.errstate(over="ignore", invalid="ignore"):
        widths = (box[..., 2] - box[..., 0]) + F32(1)
        heights = (box[..., 3] - box[..., 1]) + F32(1)
        ctr_x = box[..., 0] + F32(0.5) * widths
        ctr_y = box[..., 1] + F32(0.5) * heights
        dx, dy = d[..., 0] / F32(w[0]), d[..., 1] / F32(w[1])
        pcx, pcy = dx * widths + ctr_x, dy * heights + ctr_y
        pw, ph = f32(ew) * widths, f32(eh) * heights
        o = np.stack([pcx - F32(0.5) * pw, pcy - F32(0.5) * ph, (pcx + F32(0.5) * pw) - F32(1),
                      (pcy + F32(0.5) * ph) - F32(1)], -1)
    lim = f32([F32(im_w) - F32(1), F32(im_h) - F32(1)] * 2)
    return np.minimum(np.maximum(o, F32(0)), lim)        # fminf(fmaxf(v, 0), lim): NaN-free inputs here


def box_interval(d, box, w, im_w, im_h):
    """(lo, centre, hi) of every decoded, clipped coordinate"""
    dw, dh = decode_args(d, w)
    (wl, wh), (hl, hh) = exp_bracket(dw), exp_bracket(dh)
    a = decode_clip32(d, box, wl, hl, w, im_w, im_h)
    b = decode_clip32(d, box, wh, hh, w, im_w, im_h)
    return np.minimum(a, b), decode_clip32(d, box, exp_rn(dw), exp_rn(dh), w, im_w, im_h), np.maximum(a, b)


def softmax32(l, exp=exp_rn):
    """class_softmax_prob for every class of rows l [R, C]: max, in-order fp32 sum of expf(l - max), one division"""
    l = f32(l)
    x = l - l.max(1, keepdims=True)
    e = f32(exp(x))
    s = np.zeros(l.shape[0], dtype=F32)
    for c in range(l.shape[1]):
        s = s + e[:, c]
    return e / s[:, None]


def prob_interval(l):
    """(lo, centre, hi) of every class probability"""
    l = f32(l)
    x = l - l.max(1, keepdims=True)
    lo, hi = exp_bracket(x)
    s_lo = np.zeros(l.shape[0], dtype=F32)
    s_hi = np.zeros(l.shape[0], dtype=F32)
    for c in range(l.shape[1]):
        s_lo, s_hi = s_lo + lo[:, c], s_hi + hi[:, c]
    return lo / s_hi[:, None], softmax32(l), hi / s_lo[:, None]


def exact_interval(v, lo, hi):
    """every element of v lies in [lo, hi] (NaN only where both ends are NaN)"""
    v, lo, hi = f32(v), f32(lo), f32(hi)
    nan = np.isnan(lo) | np.isnan(hi)
    return np.where(nan, np.isnan(v), (v >= lo) & (v <= hi))


# ------------------------------------------------------------------------------------------------ IoU decisions
def iou32(a, b):
    """iou_plus1 (proposals.cu) in fp32: RN(inter / RN(RN(sa + sb) - inter))"""
    a, b = f32(a), f32(b)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        wdt = np.maximum(np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]) + F32(1), F32(0))
        hgt = np.maximum(np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]) + F32(1), F32(0))
        inter = wdt * hgt
        sa = ((a[..., 2] - a[..., 0]) + F32(1)) * ((a[..., 3] - a[..., 1]) + F32(1))
        sb = ((b[..., 2] - b[..., 0]) + F32(1)) * ((b[..., 3] - b[..., 1]) + F32(1))
        return inter / ((sa + sb) - inter)


def iou_gt(a, b, thresh, bugs=()):
    q = iou32(a, b)
    return q >= F32(thresh) if "iou_ge" in bugs else q > F32(thresh)


def greedy_keep(boxes, order_valid, thresh, max_keep, chunk=None, bugs=()):
    """positions kept by the greedy sweep over boxes [n, 4] in the given order; a position whose order_valid is False
    is skipped (remove_small_boxes). chunk=64 resolves candidates 64 at a time as rpn_nms_greedy_kernel does."""
    n = boxes.shape[0]
    kept = []
    chunks = range(0, n, chunk) if chunk else [0]
    csz = chunk or n
    for ci, base in enumerate(chunks):
        if "drop_last_chunk" in bugs and chunk and base + chunk > n and n % chunk:
            break
        for i in range(base, min(base + csz, n)):
            if len(kept) >= max_keep:
                break
            if not order_valid[i]:
                continue
            if kept and bool(iou_gt(boxes[kept], boxes[i][None], thresh, bugs).any()):
                continue
            kept.append(i)
        if len(kept) >= max_keep:
            break
    return kept


# ------------------------------------------------------------------------------------------------ restated RPN
def anchor_grid(h, w, base, stride, bugs=()):
    """anchor of index (y * w + x) * A + a: (x * stride + base[a, 0], y * stride + base[a, 1], ...) in fp32"""
    base = f32(base)
    a = base.shape[0]
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    if "grid_wh" in bugs:       # the cell index read as x * h + y
        xs, ys = np.divmod(np.arange(h * w).reshape(h, w), h)
    sx = (xs.reshape(-1) * stride).astype(F32)
    sy = (ys.reshape(-1) * stride).astype(F32)
    shift = np.stack([sx, sy, sx, sy], -1)
    return (shift[:, None, :] + base[None, :, :]).reshape(-1, 4)


def restated_rpn(head, base, im_w, im_h, pre, post, thresh, min_size, stride=16, exp=exp_rn, bugs=()):
    """one image of mega_rpn_select on the host. head [h, w, ld] fp32 -> (boxes [post, 4], scores [post], anchor [post],
    count), rows past count zero (anchor -1)"""
    head = f32(head)
    h, w, ld = head.shape
    a = f32(base).shape[0]
    n = h * w * a
    k = min(pre, n)
    logits = head[..., :a].reshape(-1)
    with np.errstate(over="ignore"):
        scores = sigmoid32(exp(-logits)) if n else np.zeros(0, F32)
    keys = ord_key(scores).astype(np.int64)
    idx = np.arange(n)
    order = np.lexsort((-idx if "tie_high" in bugs else idx, keys))[:k]     # ties: lowest index first
    order = order[np.lexsort((order, keys[order]))]                            # sorted (key, index)
    deltas = head[..., a:5 * a].reshape(-1, a, 4)
    cells = order // a
    if "wrong_deltas" in bugs:
        cells = np.minimum(cells + 1, h * w - 1)
    d = deltas[cells, order % a]
    anchors = anchor_grid(h, w, base, stride, bugs)[order]
    dw, dh = decode_args(d, (1, 1, 1, 1))
    boxes = decode_clip32(d, anchors, exp(dw), exp(dh), (1, 1, 1, 1), im_w, im_h)
    ws = (boxes[:, 2] - boxes[:, 0]) + F32(1)
    hs = (boxes[:, 3] - boxes[:, 1]) + F32(1)
    m = F32(min_size)
    valid = (ws > m) & (hs > m) if "min_size_gt" in bugs else (ws >= m) & (hs >= m)
    if rpn_path(post) == "greedy":
        kept = greedy_keep(boxes, valid, thresh, post, chunk=64, bugs=bugs)
    else:
        v = np.ones(k, bool) if "valid_ignored" in bugs else valid
        kept = greedy_keep(boxes, v, thresh, post, bugs=bugs)
    cnt = min(len(kept), post)
    ob = np.zeros((post, 4), F32)
    os_ = np.zeros(post, F32)
    oa = np.full(post, -1, np.int32)
    ob[:cnt], os_[:cnt], oa[:cnt] = boxes[kept[:cnt]], scores[order[kept[:cnt]]], order[kept[:cnt]]
    return ob, os_, oa, cnt


def transparency_rpn(pre, n):
    """parameters of the transparency call: every pre-NMS box in the kernel's order"""
    return dict(post=min(pre, n), thresh=1.0, min_size=0.0)


def check_topk(logits, t_anchor, t_score, exact):
    """the transparency call's selection and order: device scores in their intervals, sorted by (score desc, anchor
    asc) on the device's own values, and no anchor left out that must have beaten the last one taken. exact=False
    (Gaussian logits) tolerates a left-out anchor whose score interval overlaps the last taken score's interval."""
    logits = f32(logits)
    n = logits.size
    k = t_anchor.size
    lo, _, hi = score_interval(logits)
    errs = []
    if k != min(n, k) or len(set(t_anchor.tolist())) != k or (k and (t_anchor.min() < 0 or t_anchor.max() >= n)):
        return ["selection is not k distinct anchors"]
    ok = exact_interval(t_score, lo[t_anchor], hi[t_anchor])
    if not ok.all():
        errs.append("%d scores outside their interval" % int((~ok).sum()))
    keys = ord_key(t_score).astype(np.int64)
    order_ok = np.all((keys[:-1] < keys[1:]) | ((keys[:-1] == keys[1:]) & (t_anchor[:-1] < t_anchor[1:])))
    if not order_ok:
        errs.append("not sorted by (score desc, anchor asc)")
    if 0 < k < n:
        last, s_last = int(t_anchor[-1]), F32(t_score[-1])
        rest = np.setdiff1d(np.arange(n), t_anchor)
        same = logits[rest].view(np.uint32) == logits[last].view(np.uint32)
        same |= (lo[rest] == s_last) & (hi[rest] == s_last)           # a saturated score: certainly equal
        bad = same & (rest < last)                                    # an equal logit gives the same device score
        kl, kh = ord_key(hi[rest]).astype(np.int64), ord_key(lo[rest]).astype(np.int64)
        k_last = int(ord_key(s_last))
        if np.isnan(lo[last]):
            definite = np.zeros(rest.size, bool)
        else:
            definite = ~same & (kh < k_last)                          # certainly a higher score than the last taken
        amb = ~same & ~definite & (kl <= k_last)
        bad |= definite
        if exact:
            bad |= amb
        if bad.any():
            errs.append("%d anchors left out that rank before the last one taken (first %d)" % (
                int(bad.sum()), int(rest[bad][0])))
    return errs


def check_decode(head, base, stride, im_w, im_h, t_anchor, t_box):
    """the transparency call's boxes lie in the decode interval of their anchors"""
    head = f32(head)
    h, w, _ = head.shape
    a = f32(base).shape[0]
    d = head[..., a:5 * a].reshape(-1, a, 4)[t_anchor // a, t_anchor % a]
    anc = anchor_grid(h, w, base, stride)[t_anchor]
    lo, _, hi = box_interval(d, anc, (1, 1, 1, 1), im_w, im_h)
    ok = exact_interval(t_box, lo, hi)
    return [] if ok.all() else ["%d box coordinates outside their interval (first anchor %d)" % (
        int((~ok).sum()), int(t_anchor[np.nonzero(~ok.all(1))[0][0]]))]


def expected_rpn(t_box, t_score, t_anchor, post, thresh, min_size):
    """the real call's result, from the transparency call's values: validity in fp32, greedy NMS (oracle, CUDA `>`
    rule) over the valid boxes in the kernel's order, the first `post`"""
    ws = (t_box[:, 2] - t_box[:, 0]) + F32(1)
    hs = (t_box[:, 3] - t_box[:, 1]) + F32(1)
    pos = np.nonzero((ws >= F32(min_size)) & (hs >= F32(min_size)))[0]
    keep = mega_oracle.nms(torch.from_numpy(t_box[pos].copy()), torch.from_numpy(t_score[pos].copy()), thresh,
                           cuda_semantics=True).numpy()
    kept = pos[keep][:post]
    cnt = kept.size
    ob = np.zeros((post, 4), F32)
    os_ = np.zeros(post, F32)
    oa = np.full(post, -1, np.int32)
    ob[:cnt], os_[:cnt], oa[:cnt] = t_box[kept], t_score[kept], t_anchor[kept]
    return ob, os_, oa, cnt


def compare_exact(got, want, what):
    """bit-for-bit equality of (boxes, scores, anchors|labels, count) tuples"""
    errs = []
    if int(got[3]) != int(want[3]):
        errs.append("%s: count %d, expected %d" % (what, int(got[3]), int(want[3])))
    for name, g, w_ in zip(("boxes", "scores", "index"), got[:3], want[:3]):
        g, w_ = np.asarray(g), np.asarray(w_)
        if g.shape != w_.shape:
            errs.append("%s: %s shape %s, expected %s" % (what, name, g.shape, w_.shape))
            continue
        gb = g.view(np.uint32) if g.dtype == F32 else g
        wb = w_.view(np.uint32) if w_.dtype == F32 else w_
        if not np.array_equal(gb, wb):
            bad = np.nonzero((gb != wb).reshape(gb.shape[0], -1).any(1))[0]
            errs.append("%s: %s differ in %d rows (first %d)" % (what, name, bad.size, bad[0]))
    return errs


def check_rpn(head, base, stride, im_w, im_h, pre, post, thresh, min_size, trans, real, exact=True):
    """every check of one image: the transparency call's selection and continuous values, and the real call against
    the host's decisions on the transparency values. -> list of failures"""
    a = f32(base).shape[0]
    logits = f32(head)[..., :a].reshape(-1)
    tb, ts, ta, tc = trans
    n = logits.size
    k = min(pre, n)
    errs = []
    if int(tc) != k:
        return ["transparency call kept %d of %d pre-NMS boxes" % (int(tc), k)]
    tb, ts, ta = f32(tb)[:k], f32(ts)[:k], np.asarray(ta)[:k].astype(np.int64)
    errs += check_topk(logits, ta, ts, exact)
    if errs:
        return errs
    errs += check_decode(head, base, stride, im_w, im_h, ta, tb)
    want = expected_rpn(tb, ts, ta.astype(np.int32), post, thresh, min_size)
    errs += compare_exact(real, want, "rpn")
    return errs


# ------------------------------------------------------------------------------------------------ restated generic NMS
def restated_nms(boxes, scores, thresh, bugs=()):
    """mega_nms on the host: sort (score desc, NaN first, index asc), greedy sweep, kept indices ascending"""
    boxes, scores = f32(boxes), f32(scores)
    order = np.lexsort((np.arange(scores.size), ord_key(scores).astype(np.int64)))
    kept = greedy_keep(boxes[order], np.ones(scores.size, bool), thresh, scores.size, bugs=bugs)
    return np.sort(order[kept])


# ------------------------------------------------------------------------------------------------ restated box head
def restated_box(logits, deltas, props, count, num_classes, im_w, im_h, score_thresh, nms_thresh, max_det, out_cap,
                 exp=exp_rn, bugs=()):
    """mega_box_postprocess on the host -> (boxes [m, 4], scores [m], labels [m], count), m = count rows written"""
    r = min(int(count), props.shape[0])
    c = num_classes
    prob = softmax32(f32(logits)[:r, :c], exp) if r else np.zeros((0, c), F32)
    d = f32(deltas)[:r, :4 * c].reshape(r, c, 4)
    dw, dh = decode_args(d, BOX_W)
    boxes = decode_clip32(d, f32(props)[:r, None, :], exp(dw), exp(dh), BOX_W, im_w, im_h)
    kept = []                                   # (class, proposal) in class-major order
    for j in range(1, c):
        cand = np.nonzero(prob[:, j] > F32(score_thresh))[0]
        o = cand[np.lexsort((cand, ord_key(prob[cand, j]).astype(np.int64)))]
        keep = greedy_keep(boxes[o, j], np.ones(o.size, bool), nms_thresh, o.size, bugs=bugs)
        rs = np.sort(o[keep])
        if "proposals_desc" in bugs:
            rs = rs[::-1]
        kept += [(j, int(x)) for x in rs]
    sc = np.array([prob[x, j] for j, x in kept], F32)
    if len(kept) > max_det > 0:
        thr = np.sort(ord_key(sc))[max_det - 1]
        sel = ord_key(sc) < thr if "cut_drops_ties" in bugs else ord_key(sc) <= thr
        kept = [kv for kv, s in zip(kept, sel) if s]
    kept = kept[:out_cap]
    lab_off = 1 if "label_off" in bugs else 0
    ob = np.array([boxes[x, j] for j, x in kept], F32).reshape(-1, 4)
    os_ = np.array([prob[x, j] for j, x in kept], F32)
    ol = np.array([j + lab_off for j, x in kept], np.int64)
    return ob, os_, ol, len(kept)


def resolve_run(run, t_score):
    """(score_thresh, nms_thresh, max_det, out_cap) of a box run; score_thresh "at": the median of the transparency
    call's probabilities, so that some scores equal the threshold exactly"""
    st, nt, md, cap = run
    if st == "at":
        st = float(np.sort(f32(t_score))[len(t_score) // 2])
    return st, nt, md, cap


def transparency_box(num_classes, r):
    return dict(score_thresh=-1.0, nms_thresh=1.0, max_det=0, out_cap=(num_classes - 1) * r)


def expected_box(t_box, t_score, r, num_classes, score_thresh, nms_thresh, max_det, out_cap):
    """the real call's result from the transparency values t_box [(C-1) * r, 4] / t_score (class-major)"""
    c = num_classes
    tb, ts = f32(t_box).reshape(c - 1, r, 4), f32(t_score).reshape(c - 1, r)
    kb, ks, kl = [], [], []
    for j in range(1, c):
        cand = np.nonzero(ts[j - 1] > F32(score_thresh))[0]
        keep = mega_oracle.nms(torch.from_numpy(tb[j - 1, cand].copy()), torch.from_numpy(ts[j - 1, cand].copy()),
                               nms_thresh, cuda_semantics=True).numpy()
        rs = cand[keep]                      # ascending proposal index
        kb.append(tb[j - 1, rs])
        ks.append(ts[j - 1, rs])
        kl.append(np.full(rs.size, j, np.int64))
    b, s, lab = np.concatenate(kb), np.concatenate(ks), np.concatenate(kl)
    if s.size > max_det > 0:
        thr = torch.kthvalue(torch.from_numpy(s.copy()), s.size - max_det + 1)[0].item()
        sel = s >= F32(thr)
        b, s, lab = b[sel], s[sel], lab[sel]
    m = min(s.size, out_cap)
    return b[:m], s[:m], lab[:m], m


def check_box(logits, deltas, props, count, num_classes, im_w, im_h, trans, real, score_thresh, nms_thresh, max_det,
              out_cap):
    r = min(int(count), props.shape[0])
    c = num_classes
    tb, ts, tl, tc = trans
    errs = []
    if int(tc) != (c - 1) * r:
        return ["transparency call returned %d of %d (class, proposal) pairs" % (int(tc), (c - 1) * r)]
    if r:
        if not np.array_equal(np.asarray(tl)[:(c - 1) * r], np.repeat(np.arange(1, c), r)):
            errs.append("transparency labels are not class-major")
        plo, _, phi = prob_interval(f32(logits)[:r, :c])
        ok = exact_interval(f32(ts)[:(c - 1) * r], plo[:, 1:].T.reshape(-1), phi[:, 1:].T.reshape(-1))
        if not ok.all():
            errs.append("%d class probabilities outside their interval" % int((~ok).sum()))
        d = f32(deltas)[:r, :4 * c].reshape(r, c, 4)
        blo, _, bhi = box_interval(d, f32(props)[:r, None, :], BOX_W, im_w, im_h)
        ok = exact_interval(f32(tb)[:(c - 1) * r], blo[:, 1:].transpose(1, 0, 2).reshape(-1, 4),
                            bhi[:, 1:].transpose(1, 0, 2).reshape(-1, 4))
        if not ok.all():
            errs.append("%d box coordinates outside their interval" % int((~ok).sum()))
    want = expected_box(f32(tb)[:(c - 1) * r], f32(ts)[:(c - 1) * r], r, c, score_thresh, nms_thresh, max_det, out_cap)
    m = int(real[3])
    errs += compare_exact((f32(real[0])[:m], f32(real[1])[:m], np.asarray(real[2])[:m], m), want, "box")
    return errs


# ------------------------------------------------------------------------------------------------ case table
def cell_anchors():
    return mega_oracle.cell_anchors(16).numpy()


# score levels whose expf brackets are far apart: logit -> score is strictly ordered even at 2 ulp
LEVELS = np.array([-30.0, -12.0, -8.0, -6.0, -4.5, -3.0, -2.0, -1.25, -0.5, 0.0, 0.5, 1.25, 2.0, 3.0, 4.5, 6.0, 8.0,
                   12.0], dtype=F32)


def _rpn_head(seed, n_img, h, w, a, ld, scores, deltas, extra=None):
    """[n_img, h, w, ld] fp32 head: logits by `scores`, deltas by `deltas`, different content per image"""
    head = np.zeros((n_img, h, w, ld), F32)
    for i in range(n_img):
        g = np.random.default_rng(seed * 131 + i)
        n = h * w * a
        if scores == "levels":
            lg = g.choice(LEVELS, n)
        elif scores == "gauss":
            lg = g.standard_normal(n).astype(F32) * F32(1.5)
        elif scores == "equal":
            lg = np.full(n, 0.75, F32)
        elif scores == "tie_boundary":       # 300 logits above 700 equal ones, the rest below: k = 640 or 900 takes
            #                                  part of the equal block (quota_eq in (1, #equal))
            lg = g.choice(LEVELS[:8], n)
            lg[g.choice(n, 700, replace=False)] = F32(1.25)
            lg[g.choice(np.nonzero(lg != F32(1.25))[0], 300, replace=False)] = F32(3.0)
        elif scores == "saturated":          # exactly 1.0 and exactly 0.0 scores, +-inf and one NaN
            lg = g.choice(LEVELS, n)
            lg[g.choice(n, n // 4, replace=False)] = g.choice(np.array([20.0, 25.0, 40.0, np.inf], F32), n // 4)
            lg[g.choice(n, n // 4, replace=False)] = g.choice(np.array([-104.0, -120.0, -np.inf], F32), n // 4)
            lg[g.integers(n)] = F32(np.nan)
        else:
            raise ValueError(scores)
        head[i, :, :, :a] = lg.reshape(h, w, a)
        if deltas == "normal":
            dl = g.standard_normal((h, w, 4 * a)).astype(F32) * F32(0.3)
        else:                                # clamp edges, clipping on every border
            dl = g.standard_normal((h, w, 4 * a)).astype(F32) * F32(1.5)
            dl.reshape(-1, 4)[g.choice(h * w * a, h * w * a // 8, replace=False), 2:] = F32(4.135166556742356)
            dl.reshape(-1, 4)[g.choice(h * w * a, h * w * a // 8, replace=False), 2:] = F32(6.0)
        head[i, :, :, a:5 * a] = dl
        head[i, :, :, 5 * a:] = F32(np.nan)  # padding columns past 5A are never read
    return head


def make_rpn_cases():
    """RPN cases. Each names its head, the (pre, post) pairs it runs, nms_thresh and min_size ("ws": read from the
    transparency call, see min_size_at). exact: the top-k is fully determined."""
    C = []

    def add(id_, h, w, n_img, scores, deltas, runs, im=None, thresh=0.7, min_size=(0.0,), seed=None, slice_of=0,
            ld=64):
        C.append(dict(id=id_, h=h, w=w, n_img=n_img, scores=scores, deltas=deltas, runs=runs,
                      im=im or (w * 16.0, h * 16.0), thresh=thresh, min_size=min_size, seed=seed or len(C) + 1,
                      slice_of=slice_of, ld=ld, exact=scores != "gauss"))

    # engine geometries: the key frame and the MEGA reference frames of a 600 x 1000 image
    add("engine_38x63", 38, 63, 1, "levels", "normal", [(6000, 300), (6000, 75)], im=(1000.0, 600.0),
        min_size=(0.0, "ws"))
    add("engine_38x63_gauss", 38, 63, 1, "gauss", "normal", [(6000, 300), (6000, 2000)], im=(1000.0, 600.0))
    add("fixture_12x20", 12, 20, 1, "levels", "edge", [(6000, 300), (2880, 2000), (1024, 1024), (1024, 1025)],
        im=(313.0, 187.0), min_size=(0.0, 16.0, "ws"))
    add("large_75x125", 75, 125, 1, "levels", "normal", [(8192, 300), (8192, 8192)], im=(1995.0, 1190.0),
        min_size=(0.0, 16.0))
    # batches, different content per image; one batch is a slice of a larger head buffer
    add("batch2", 20, 31, 2, "levels", "normal", [(2000, 300), (2000, 1025)], im=(490.0, 313.0))
    add("batch3_slice", 17, 23, 3, "levels", "edge", [(1500, 75), (1500, 2000)], im=(361.0, 270.0), slice_of=5,
        min_size=(0.0, "ws"))
    add("batch8", 9, 14, 8, "levels", "normal", [(600, 300), (600, 1025)], im=(221.0, 140.0))
    # k and post edges
    add("k_small", 4, 5, 1, "levels", "normal", [(1, 1), (2, 75), (63, 300), (64, 300), (65, 300), (65, 1025),
                                                 (240, 2000), (8192, 8192)], im=(70.0, 77.0))
    add("k_1024", 10, 12, 1, "levels", "normal", [(1024, 75), (1025, 1024), (1025, 1025), (1440, 8192)],
        im=(190.0, 155.0), min_size=(0.0, 16.0))
    add("k_8192", 30, 40, 1, "levels", "edge", [(8192, 2000), (8192, 1024), (8192, 1025)], im=(640.0, 480.0))
    add("cap_in_chunk", 12, 20, 1, "levels", "normal", [(2880, 100), (2880, 1)], im=(320.0, 192.0), thresh=0.3)
    # score edges
    add("tie_boundary", 12, 20, 1, "tie_boundary", "normal", [(640, 300), (640, 1025), (900, 1024)],
        im=(320.0, 192.0))
    add("all_equal", 8, 10, 1, "equal", "normal", [(200, 75), (200, 1025), (960, 1024)], im=(160.0, 128.0))
    add("saturated", 12, 20, 2, "saturated", "edge", [(2000, 300), (2000, 1025)], im=(320.0, 192.0),
        min_size=(0.0, "ws"))
    return C


def min_size_at(t_box):
    """min_size "ws": min(ws, hs) of the top-scoring pre-NMS box, which then sits exactly on the min_size edge"""
    b = f32(t_box)[0]
    return float(min((b[2] - b[0]) + F32(1), (b[3] - b[1]) + F32(1)))


def rpn_inputs(c):
    """(head [n_img, h, w, ld] as laid out in memory, base anchors [A, 4])"""
    base = cell_anchors()
    n = max(c["n_img"], c["slice_of"])
    head = _rpn_head(c["seed"], n, c["h"], c["w"], base.shape[0], c["ld"], c["scores"], c["deltas"])
    return head, base


# generic NMS: (id, boxes, scores, thresholds)
def _rand_boxes(g, n, w=1000.0, h=600.0, lo=4.0, hi=260.0):
    xy = g.random((n, 2)) * np.array([w * 0.9, h * 0.9])
    wh = g.random((n, 2)) * (hi - lo) + lo
    return np.concatenate([xy, xy + wh], 1).astype(F32)


def threshold_pairs():
    """box pairs whose fp32 IoU is exactly the threshold, and one ulp of the box either side"""
    base = f32([0, 0, 9, 9])
    out = []
    for t, other in ((0.7, [0, 0, 9, 6]), (0.5, [0, 0, 9, 4]), (0.3, [0, 0, 2, 9])):
        o = f32(other)
        for dy in (0, 1, -1):
            b = o.copy()
            if dy:
                b[3] = np.nextafter(b[3], F32(np.inf) if dy > 0 else F32(-np.inf))
            out.append((t, base, b))
    return out


def make_nms_cases():
    C = []
    g = np.random.default_rng(7)
    for n in (0, 1, 63, 64, 65, 4096, 8191, 8192):
        b = _rand_boxes(g, n)
        s = g.random(n).astype(F32)
        if n >= 64:
            s[10] = s[3]
            b[20] = b[7]
        C.append(dict(id="rand_%d" % n, boxes=b, scores=s, threshs=(0.0, 1e-6, 0.3, 0.5, 0.7, 1.0)))
    # exact-threshold pairs, each pair repeated in a block of 64 boxes: pair i at positions (2i, 2i + 1)
    pairs = threshold_pairs()
    b = np.concatenate([np.stack([p[1], p[2]]) + F32(40 * i) for i, p in enumerate(pairs)])
    s = np.tile(f32([0.9, 0.8]), len(pairs))
    for t in (0.3, 0.5, 0.7):
        C.append(dict(id="iou_at_thresh_%g" % t, boxes=b, scores=s, threshs=(t,)))
    # duplicates, all-equal scores, degenerate and inf boxes, NaN and inf scores
    d = _rand_boxes(g, 200, 300.0, 300.0)
    d[50:80] = d[10]
    d[100:110, 2] = d[100:110, 0] - F32(1)                     # zero +1 width
    d[110:120, 2] = d[110:120, 0] - F32(3)                     # negative +1 width (union <= 0 against itself)
    d[120:125, 3] = d[120:125, 1] - F32(5)
    d[130, 2] = F32(np.inf)
    d[131, 0] = F32(-np.inf)
    C.append(dict(id="degenerate", boxes=d, scores=np.full(200, 0.5, F32), threshs=(0.0, 0.5, 0.7, 1.0)))
    s = g.random(200).astype(F32)
    s[[5, 17, 150]] = F32(np.nan)
    s[[6, 40]] = F32(np.inf)
    s[[7, 41]] = F32(-np.inf)
    C.append(dict(id="nan_inf_scores", boxes=_rand_boxes(g, 200, 300.0, 300.0), scores=s, threshs=(0.3, 0.7)))
    return C


def make_box_cases():
    """box-head cases: logits / deltas / proposals, the `count` device scalar, and (score_thresh, nms_thresh, max_det,
    out_cap) of each run"""
    C = []

    def add(id_, c, r, count, logits, deltas, props, runs, im=(1000.0, 600.0)):
        C.append(dict(id=id_, c=c, r=r, count=count, logits=f32(logits), deltas=f32(deltas), props=f32(props),
                      runs=runs, im=im))

    g = np.random.default_rng(11)
    std = lambda c, r: (0.001, 0.5, 300, (c - 1) * r)
    for c, r, count in ((31, 300, 300), (31, 300, 137), (2, 300, 300), (31, 1, 1), (2, 512, 512), (31, 512, 600),
                        (31, 300, 0)):
        lg = g.standard_normal((r, c)).astype(F32) * F32(2.5)
        dl = g.standard_normal((r, 4 * c)).astype(F32) * F32(0.5)
        pr = _rand_boxes(g, r)
        add("c%d_r%d_n%d" % (c, r, count), c, r, count, lg, dl, pr,
            [std(c, r), (0.05, 0.5, 100, (c - 1) * r), (0.001, 0.5, 0, (c - 1) * r), (0.001, 0.5, 300, 57)])
    # scores exactly at score_thresh: a thresh equal to a computed probability is set by the runner ("at")
    lg = g.standard_normal((300, 31)).astype(F32)
    add("thresh_exact", 31, 300, 300, lg, g.standard_normal((300, 124)).astype(F32) * F32(0.3), _rand_boxes(g, 300),
        [("at", 0.5, 300, 30 * 300), ("at", 0.5, 40, 30 * 300)])
    # ties at the detections_per_img cut, inside one class (repeated rows) and across classes (equal logits in a row)
    lg = np.tile(g.choice(f32([-2.0, -1.0, 0.0, 1.0, 2.0]), (60, 31)), (5, 1)).astype(F32)
    lg[:, 2] = lg[:, 1]
    pr = _rand_boxes(g, 300, 1000.0, 600.0, 40.0, 80.0)
    add("ties_at_cut", 31, 300, 300, lg, g.standard_normal((300, 124)).astype(F32) * F32(0.3), pr,
        [(0.001, 0.5, 300, 9000), (0.001, 0.5, 77, 9000), (0.001, 0.5, 1, 9000), (0.001, 0.5, 10 ** 6, 9000),
         (0.001, 0.5, 300, 120)])
    # one class holds all 512 candidates (well-separated boxes, so NMS keeps them all)
    lg = np.full((512, 2), -8.0, F32)
    lg[:, 1] = f32(np.linspace(0.0, 8.0, 512))
    xy = np.stack(np.meshgrid(np.arange(32), np.arange(16), indexing="xy"), -1).reshape(-1, 2).astype(F32) * F32(30)
    pr = np.concatenate([xy, xy + F32(20)], 1)
    add("one_class_512", 2, 512, 512, lg, np.zeros((512, 8), F32), pr,
        [(0.001, 0.5, 300, 512), (0.001, 0.5, 0, 512), (0.001, 0.5, 0, 200)], im=(1000.0, 600.0))
    return C


# properties the table must cover (test_proposals_conformance_cpu.py)
def rpn_coverage():
    """the (property, value) pairs the RPN table exercises"""
    got = set()
    for c in make_rpn_cases():
        n = c["h"] * c["w"] * 12
        for pre, post in c["runs"]:
            k = min(pre, n)
            got |= {("k", k), ("post", post), ("path", rpn_path(post)), ("n_img", c["n_img"]), ("scores", c["scores"])}
            if pre >= n:
                got.add(("pre>=n", True))
            if post > k:
                got.add(("post>k", True))
            for m in c["min_size"]:
                got.add(("min_size", (m, rpn_path(post))))
        if c["slice_of"]:
            got.add(("slice", True))
        if c["im"][0] % 16 or c["im"][1] % 16:
            got.add(("im_not_multiple", True))
        if c["deltas"] == "edge":
            got.add(("clamp", True))
    return got
