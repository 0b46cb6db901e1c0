"""CPU side of the proposal / NMS / box-head conformance suite (proposals_ref.py):

  * the exact-order fp32 restatement equals mega_oracle.rpn_select / box_postprocess where both use the same exp, and
    the g++ builds of box_head.cuh / iou.cuh (tests/native/proposals_host.cpp) on decode, clip, soft-max and IoU
    decisions;
  * the expf-bracket intervals contain the fp64 values; no IoU of boxes with non-negative +1 widths exceeds 1, so the
    transparency calls (nms_thresh = 1) suppress nothing;
  * oracle_nms ranks NaN scores first, ties by index;
  * every planted bug in the restatement is rejected by the checks the GPU file applies;
  * the case table covers every dispatch path and edge it promises; the restated constants match the kernel source.
"""
import ctypes
import hashlib
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import proposals_ref as R

ROOT = R.ROOT
F32 = np.float32
_host = None


def host_lib():
    """g++ build of box_head.cuh / iou.cuh, cached in the temp directory under the digest of its sources"""
    global _host
    if _host is None:
        src = os.path.join(ROOT, "tests", "native", "proposals_host.cpp")
        deps = [src] + [os.path.join(R.CSRC, n) for n in ("box_head.cuh", "iou.cuh")]
        digest = hashlib.sha256(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
        so_path = os.path.join(tempfile.gettempdir(), "mega_proposals_host_%s_%d.so" % (digest, os.getuid()))
        if not os.path.exists(so_path):
            tmp = so_path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-I", R.CSRC,
                                   "-o", tmp, src])
            os.replace(tmp, so_path)
        _host = ctypes.CDLL(so_path)
        _vp, _i, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
        _host.proposals_decode_clip.argtypes = [_vp, _vp, _i, _vp, _f, _f, _vp]
        _host.proposals_softmax.argtypes = [_vp, _i, _i, _vp]
        _host.proposals_iou_gt.argtypes = [_vp, _vp, _i, _f, _vp]
    return _host


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


_libm = ctypes.CDLL("libm.so.6")
_libm.expf.argtypes = [ctypes.c_float]
_libm.expf.restype = ctypes.c_float


def libm_exp(x):
    """the host build's expf, element by element"""
    x = R.f32(x)
    return np.array([_libm.expf(float(v)) for v in x.reshape(-1)], F32).reshape(x.shape)


def torch_exp(x):
    return torch.exp(torch.from_numpy(np.ascontiguousarray(R.f32(x)))).numpy()


def _bits(a):
    return np.ascontiguousarray(R.f32(a)).view(np.uint32)


# ------------------------------------------------------------------------------------------------ restatement vs oracle
def _oracle_layout(head, a):
    h, w, _ = head.shape
    logits = torch.from_numpy(np.ascontiguousarray(head[..., :a].transpose(2, 0, 1)))[None]
    deltas = torch.from_numpy(np.ascontiguousarray(head[..., a:5 * a].transpose(2, 0, 1)))[None]
    return logits, deltas


@pytest.mark.parametrize("pre,post,min_size", [(2000, 300, 0.0), (2000, 1025, 16.0), (63, 300, 0.0)])
def test_restated_rpn_matches_oracle(pre, post, min_size):
    """same anchors in the same order and the same boxes bit for bit (both decode with torch.exp); the oracle's scores
    (torch.sigmoid) lie in the restatement's interval"""
    import mega_oracle as mo
    c = next(x for x in R.make_rpn_cases() if x["id"] == "fixture_12x20")
    head, base = R.rpn_inputs(c)
    head = head[0]
    im_w, im_h = c["im"]
    ob, os_, oa, cnt = R.restated_rpn(head, base, im_w, im_h, pre, post, 0.7, min_size, exp=torch_exp)
    logits, deltas = _oracle_layout(head, base.shape[0])
    rb, rs, aux = mo.rpn_select(logits, deltas, im_w, im_h, pre, post, 0.7, min_size, cuda_semantics=True,
                                return_aux=True)
    assert cnt == rb.shape[0]
    assert np.array_equal(oa[:cnt], aux["anchor_idx"].numpy())
    assert np.array_equal(_bits(ob[:cnt]), _bits(rb.numpy()))
    lo, _, hi = R.score_interval(head[..., :base.shape[0]].reshape(-1)[oa[:cnt]])
    assert R.exact_interval(rs.numpy(), lo, hi).all()
    assert (ob[cnt:] == 0).all() and (os_[cnt:] == 0).all() and (oa[cnt:] == -1).all()


def test_restated_box_matches_oracle():
    """labels and boxes bit for bit (both decode with torch.exp); the oracle's F.softmax sums in another order, so its
    scores agree to a few ulps"""
    import mega_oracle as mo
    c = next(x for x in R.make_box_cases() if x["id"] == "c31_r300_n137")
    r = 137
    ob, os_, ol, m = R.restated_box(c["logits"], c["deltas"], c["props"], r, 31, *c["im"], 0.001, 0.5, 300, 9000,
                                    exp=torch_exp)
    rb, rs, rl = mo.box_postprocess(torch.from_numpy(c["logits"][:r]), torch.from_numpy(c["deltas"][:r]),
                                    torch.from_numpy(c["props"][:r]), *c["im"], cuda_semantics=True)
    assert m == rl.numel()
    assert np.array_equal(ol, rl.numpy())
    assert np.array_equal(_bits(ob), _bits(rb.numpy()))
    assert R.exact_interval(rs.numpy(), os_ - np.abs(os_) * F32(2 ** -20), os_ + np.abs(os_) * F32(2 ** -20)).all()


def test_restatement_matches_host_build():
    """decode + clip, soft-max and the IoU decision: the restatement with the host's expf equals the g++ build of
    box_head.cuh / iou.cuh bit for bit"""
    lib = host_lib()
    g = np.random.default_rng(3)
    n = 4000
    d = (g.standard_normal((n, 4)) * 2.0).astype(F32)
    d[::7, 2:] = R.CLIP * F32(5)
    box = R._rand_boxes(g, n, 1200.0, 800.0, 0.5, 900.0)
    box[::11] -= F32(300)
    w = R.f32(R.BOX_W)
    out = np.zeros((n, 4), F32)
    lib.proposals_decode_clip(_p(d), _p(box), n, _p(w), 1000.0, 600.0, _p(out))
    dw, dh = R.decode_args(d, R.BOX_W)
    mine = R.decode_clip32(d, box, libm_exp(dw), libm_exp(dh), R.BOX_W, 1000.0, 600.0)
    assert np.array_equal(_bits(out), _bits(mine))
    for nc in (2, 31):
        lg = (g.standard_normal((300, nc)) * 4).astype(F32)
        lg[::5, 1] = lg[::5, 0]
        outp = np.zeros((300, nc), F32)
        lib.proposals_softmax(_p(lg), 300, nc, _p(outp))
        assert np.array_equal(_bits(outp), _bits(R.softmax32(lg, libm_exp)))
    a = np.repeat(f32_pairs()[0], 1, 0)
    b = f32_pairs()[1]
    for t in (0.0, 1e-6, 0.3, 0.5, 0.7, 1.0):
        got = np.zeros(a.shape[0], np.uint8)
        lib.proposals_iou_gt(_p(a), _p(b), a.shape[0], t, _p(got))
        assert np.array_equal(got.astype(bool), R.iou_gt(a, b, t)), t


def f32_pairs():
    """random, exact-threshold, duplicate, degenerate and inf box pairs"""
    g = np.random.default_rng(5)
    a = R._rand_boxes(g, 3000, 200.0, 200.0, 0.0, 120.0)
    b = R._rand_boxes(g, 3000, 200.0, 200.0, 0.0, 120.0)
    b[:300] = a[:300]
    a[300:400, 2] = a[300:400, 0] - F32(1)
    b[400:500, 3] = b[400:500, 1] - F32(4)
    a[500:510, 2] = F32(np.inf)
    pa = np.stack([p[1] for p in R.threshold_pairs()])
    pb = np.stack([p[2] for p in R.threshold_pairs()])
    return np.concatenate([a, pa]).astype(F32), np.concatenate([b, pb]).astype(F32)


# ------------------------------------------------------------------------------------------------ intervals, IoU <= 1
def test_intervals_contain_fp64():
    g = np.random.default_rng(9)
    lg = np.concatenate([(g.standard_normal(20000) * 6), [20.0, 40.0, -104.0, 0.0, 88.0, -88.0]]).astype(F32)
    lo, cen, hi = R.score_interval(lg)
    ref = 1.0 / (1.0 + np.exp(-lg.astype(np.float64)))
    tol = ref * 2.0 ** -23 + 2.0 ** -149            # the roundings of 1 + e and of the quotient (subnormal floor)
    assert ((lo <= ref + tol) & (hi >= ref - tol)).all()
    assert ((lo <= cen) & (cen <= hi)).all()
    l = (g.standard_normal((500, 31)) * 3).astype(F32)
    lo, cen, hi = R.prob_interval(l)
    x = l.astype(np.float64)
    e = np.exp(x - x.max(1, keepdims=True))
    ref = e / e.sum(1, keepdims=True)
    assert ((lo <= ref * (1 + 2 ** -20)) & (hi >= ref * (1 - 2 ** -20))).all()      # + 31 in-order fp32 additions
    assert ((lo <= cen) & (cen <= hi)).all()
    d = (g.standard_normal((5000, 4)) * 1.5).astype(F32)
    box = R._rand_boxes(g, 5000)
    lo, cen, hi = R.box_interval(d, box, (1, 1, 1, 1), 1000.0, 600.0)
    dd, bb = d.astype(np.float64), box.astype(np.float64)
    wd, ht = bb[:, 2] - bb[:, 0] + 1, bb[:, 3] - bb[:, 1] + 1
    cx, cy = bb[:, 0] + 0.5 * wd + dd[:, 0] * wd, bb[:, 1] + 0.5 * ht + dd[:, 1] * ht
    pw, ph = np.exp(np.minimum(dd[:, 2], float(R.CLIP))) * wd, np.exp(np.minimum(dd[:, 3], float(R.CLIP))) * ht
    ref = np.stack([cx - 0.5 * pw, cy - 0.5 * ph, cx + 0.5 * pw - 1, cy + 0.5 * ph - 1], 1)
    ref = np.minimum(np.maximum(ref, 0), [999.0, 599.0, 999.0, 599.0])
    mag = np.abs(np.stack([cx, cy, cx, cy], 1)) + np.abs(np.stack([pw, ph, pw, ph], 1)) + np.abs(bb) + 1
    slack = 8 * 2.0 ** -24 * mag                     # the roundings of the fp32 chain besides expf
    assert ((lo <= ref + slack) & (hi >= ref - slack)).all()
    assert ((lo <= cen) & (cen <= hi)).all()


def test_iou_never_exceeds_one():
    """boxes with non-negative +1 widths: inter <= min(sa, sb) in fp32, so RN(inter / u) <= 1 and nms_thresh = 1
    suppresses nothing (the transparency calls rely on it)"""
    g = np.random.default_rng(13)
    a = R._rand_boxes(g, 200000, 2000.0, 2000.0, 0.0, 1500.0)
    b = R._rand_boxes(g, 200000, 2000.0, 2000.0, 0.0, 1500.0)
    b[:50000] = a[:50000]                                              # identical boxes: IoU exactly 1
    b[50000:60000] = a[50000:60000] + F32(2 ** -10)
    a[60000:70000, 2] = a[60000:70000, 0] - F32(1)                     # +1 width exactly 0
    a[70000:80000] *= F32(1e6)
    b[70000:80000] = a[70000:80000] + F32(1)
    v = R.iou32(a, b)
    assert not (v > 1).any()
    assert (v[:50000] == 1).all()


# ------------------------------------------------------------------------------------------------ oracle NaN order
def test_oracle_nms_ranks_nan_first():
    import mega_oracle as mo
    boxes = np.tile(R.f32([[0, 0, 10, 10]]), (6, 1))
    for scores, first in (([0.5, np.nan, 0.9, np.nan, np.inf, 0.1], 1), ([np.inf, 0.2, 0.3, 0.4, 0.5, np.nan], 5),
                          ([0.3, 0.3, 0.3, 0.3, 0.3, 0.3], 0)):
        keep = mo.nms(torch.from_numpy(boxes), torch.tensor(scores, dtype=torch.float32), 0.5, cuda_semantics=True)
        assert keep.tolist() == [first]
    g = np.random.default_rng(17)
    b = R._rand_boxes(g, 400, 200.0, 200.0)
    s = g.random(400).astype(F32)
    s[g.choice(400, 40, replace=False)] = F32(np.nan)
    s[g.choice(400, 10, replace=False)] = F32(np.inf)
    for t in (0.3, 0.7):
        want = R.restated_nms(b, s, t)
        got = mo.nms(torch.from_numpy(b), torch.from_numpy(s), t, cuda_semantics=True).numpy()
        assert np.array_equal(got, want)
        order = torch.sort(torch.from_numpy(s), descending=True, stable=True)[1].numpy()
        assert np.array_equal(order, np.lexsort((np.arange(400), R.ord_key(s).astype(np.int64))))


@pytest.mark.parametrize("case", R.make_nms_cases(), ids=lambda c: c["id"])
def test_restated_nms_matches_oracle(case):
    import mega_oracle as mo
    if case["boxes"].shape[0] > 1000:
        pytest.skip("the oracle alone covers the large cases (on the GPU)")
    for t in case["threshs"]:
        want = mo.nms(torch.from_numpy(case["boxes"]), torch.from_numpy(case["scores"]), t, cuda_semantics=True).numpy()
        assert np.array_equal(R.restated_nms(case["boxes"], case["scores"], t), want), t


# ------------------------------------------------------------------------------------------------ mutations
def _rpn_check(case_id, pre, post, thresh, min_size, bugs, img=0):
    c = next(x for x in R.make_rpn_cases() if x["id"] == case_id)
    head, base = R.rpn_inputs(c)
    head = head[img]
    n = head.shape[0] * head.shape[1] * base.shape[0]
    k = min(pre, n)
    im_w, im_h = c["im"]
    trans = R.restated_rpn(head, base, im_w, im_h, pre, k, 1.0, 0.0, bugs=bugs)
    if min_size == "ws":
        good = R.restated_rpn(head, base, im_w, im_h, pre, k, 1.0, 0.0)
        min_size = R.min_size_at(good[0])
    real = R.restated_rpn(head, base, im_w, im_h, pre, post, thresh, min_size, bugs=bugs)
    return R.check_rpn(head, base, 16, im_w, im_h, pre, post, thresh, min_size, trans, real, exact=c["exact"])


RPN_MUTANTS = [("tie_high", "tie_boundary", 640, 300, 0.7, 0.0), ("tie_high", "tie_boundary", 900, 1024, 0.7, 0.0),
               ("min_size_gt", "fixture_12x20", 6000, 300, 0.7, "ws"),
               ("min_size_gt", "fixture_12x20", 6000, 2000, 0.7, "ws"),
               ("valid_ignored", "fixture_12x20", 6000, 2000, 0.7, 16.0),
               ("drop_last_chunk", "k_1024", 1000, 1024, 0.7, 0.0),
               ("grid_wh", "batch2", 2000, 300, 0.7, 0.0),
               ("wrong_deltas", "batch2", 2000, 300, 0.7, 0.0)]


@pytest.mark.parametrize("bug,case,pre,post,thresh,min_size", RPN_MUTANTS, ids=["%s-%s-%d" % (m[0], m[1], m[3])
                                                                                  for m in RPN_MUTANTS])
def test_rpn_checks_reject_planted_bug(bug, case, pre, post, thresh, min_size):
    assert _rpn_check(case, pre, post, thresh, min_size, ()) == []
    assert _rpn_check(case, pre, post, thresh, min_size, (bug,)) != []


def test_nms_checks_reject_iou_ge():
    """`>=` instead of `>`: the exact-threshold pairs change the keep list"""
    import mega_oracle as mo
    for c in R.make_nms_cases():
        if c["id"].startswith("iou_at_thresh"):
            t = c["threshs"][0]
            want = mo.nms(torch.from_numpy(c["boxes"]), torch.from_numpy(c["scores"]), t, cuda_semantics=True).numpy()
            assert np.array_equal(R.restated_nms(c["boxes"], c["scores"], t), want)
            assert not np.array_equal(R.restated_nms(c["boxes"], c["scores"], t, bugs=("iou_ge",)), want), c["id"]


def _box_check(case_id, run_i, bugs):
    c = next(x for x in R.make_box_cases() if x["id"] == case_id)
    C, r = c["c"], c["r"]
    tr = R.transparency_box(C, r)
    trans = R.restated_box(c["logits"], c["deltas"], c["props"], c["count"], C, *c["im"], tr["score_thresh"],
                           tr["nms_thresh"], tr["max_det"], tr["out_cap"], bugs=bugs)
    run = R.resolve_run(c["runs"][run_i], trans[1])
    real = R.restated_box(c["logits"], c["deltas"], c["props"], c["count"], C, *c["im"], *run, bugs=bugs)
    return R.check_box(c["logits"], c["deltas"], c["props"], c["count"], C, *c["im"], trans, real, *run)


BOX_MUTANTS = [("cut_drops_ties", "ties_at_cut", 1), ("label_off", "c2_r300_n300", 0),
               ("proposals_desc", "c31_r300_n137", 0), ("iou_ge", "one_class_512", 0)]


@pytest.mark.parametrize("bug,case,run", BOX_MUTANTS, ids=[m[0] for m in BOX_MUTANTS])
def test_box_checks_reject_planted_bug(bug, case, run):
    assert _box_check(case, run, ()) == []
    errs = _box_check(case, run, (bug,))
    if bug == "iou_ge":                  # no exact-threshold pair in this case: the bug is invisible, as it should be
        assert errs == []
    else:
        assert errs != []


def test_box_cut_has_ties_at_the_cut():
    """the detections_per_img runs of ties_at_cut put equal scores on both sides of the cut, inside one class and
    across classes"""
    c = next(x for x in R.make_box_cases() if x["id"] == "ties_at_cut")
    everything = R.restated_box(c["logits"], c["deltas"], c["props"], c["count"], 31, *c["im"], 0.001, 0.5, 0, 9000)
    s, lab = everything[1], everything[2]
    for md in (77, 300):
        thr = np.sort(s)[::-1][md - 1]
        assert (s == thr).sum() > 1 and (s > thr).sum() < md < (s >= thr).sum(), md
    for md in (77,):
        thr = np.sort(s)[::-1][md - 1]
        assert len(set(lab[s == thr].tolist())) > 1
    # and the real cut keeps them all
    got = R.restated_box(c["logits"], c["deltas"], c["props"], c["count"], 31, *c["im"], 0.001, 0.5, 77, 9000)
    assert got[3] > 77


# ------------------------------------------------------------------------------------------------ table and rule
def test_constants_match_source():
    assert R.source_constant("proposals.cu", "kNmsMaxBoxes") == R.K_NMS_MAX_BOXES
    assert R.source_constant("proposals.cu", "kGreedyMaxKeep") == R.K_GREEDY_MAX_KEEP
    assert R.source_constant("postprocess.cu", "kMaxRois") == R.K_MAX_ROIS
    src = open(os.path.join(R.CSRC, "proposals.cu")).read()
    assert "if (post_nms <= kGreedyMaxKeep)" in src
    launched = set(re.findall(r"(\w+_kernel)<<<", src + open(os.path.join(R.CSRC, "postprocess.cu")).read()))
    launched |= {"box_final_kernel"} if "box_final_kernel<<<" in open(os.path.join(R.CSRC, "postprocess.cu")).read() \
        else set()
    assert launched == set(R.ALL_KERNELS), launched
    body = src[src.index('extern "C" int mega_nms('):src.index("extern \"C\" long long mega_rpn_select_workspace")]
    assert re.findall(r"(\w+_kernel)<<<", body) == R.nms_kernels(5)
    body = src[src.index('extern "C" int mega_rpn_select('):]
    assert re.findall(r"(\w+_kernel)<<<", body) == [R.TOPK, R.GREEDY, R.MASK, R.SWEEP, R.WRITE]


def test_case_table_covers_every_path_and_edge():
    got = R.rpn_coverage()
    for k in (1, 2, 63, 64, 65, 1024, 1025, 8192):
        assert ("k", k) in got, k
    for p in (1, 75, 300, 1024, 1025, 2000, 8192):
        assert ("post", p) in got, p
    for n in (1, 2, 3, 8):
        assert ("n_img", n) in got, n
    for s in ("levels", "gauss", "equal", "tie_boundary", "saturated"):
        assert ("scores", s) in got
    for m in (0.0, 16.0, "ws"):
        for path in ("greedy", "mask"):
            assert ("min_size", (m, path)) in got, (m, path)
    for prop in ("pre>=n", "post>k", "slice", "im_not_multiple", "clamp"):
        assert (prop, True) in got, prop
    ids = {c["id"] for c in R.make_rpn_cases()}
    assert {"engine_38x63", "large_75x125", "fixture_12x20", "cap_in_chunk"} <= ids
    geo = {(c["h"], c["w"]) for c in R.make_rpn_cases()}
    assert {(38, 63), (12, 20), (75, 125)} <= geo
    nms = {c["boxes"].shape[0] for c in R.make_nms_cases()}
    assert {0, 1, 63, 64, 65, 4096, 8191, 8192} <= nms
    ths = set().union(*[set(c["threshs"]) for c in R.make_nms_cases()])
    assert {0.0, 1e-6, 0.3, 0.5, 0.7, 1.0} <= ths
    box = R.make_box_cases()
    assert {c["c"] for c in box} == {2, 31}
    assert {1, 300, 512} <= {c["r"] for c in box}
    rel = {("0" if c["count"] == 0 else "<" if c["count"] < c["r"] else "=" if c["count"] == c["r"] else ">")
           for c in box}
    assert rel == {"0", "<", "=", ">"}
    runs = [(c, run) for c in box for run in c["runs"]]
    assert any(run[0] == "at" for _, run in runs)
    assert any(run[2] == 0 for _, run in runs) and any(run[2] >= 10 ** 6 for _, run in runs)
    assert any(run[3] < (c["c"] - 1) * c["r"] for c, run in runs)


def test_rpn_levels_are_separated():
    """the exact-selection score levels have disjoint expf-bracket intervals"""
    lo, _, hi = R.score_interval(R.LEVELS)
    assert (hi[:-1] < lo[1:]).all()


def test_saturated_scores_are_exact():
    lo, _, hi = R.score_interval(R.f32([20.0, 25.0, np.inf, -np.inf]))
    assert (lo[:3] == 1).all() and (hi[:3] == 1).all() and lo[3] == 0 and hi[3] == 0
    lo, _, hi = R.score_interval(R.f32([-104.0]))
    assert lo[0] == 0
