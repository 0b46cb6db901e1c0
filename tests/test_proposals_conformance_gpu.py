"""Conformance of the RPN proposal selection, generic NMS and box-head post-processing kernels (csrc/proposals.cu,
csrc/postprocess.cu) against the exact references of proposals_ref.py, decision by decision.

For every case and path of the table:
  * continuous values (RPN scores, decoded boxes, class probabilities, read back through a transparency call) lie in
    their expf-bracket intervals;
  * every decision (top-k set and order, min_size, NMS keep lists, score and detections_per_img cuts, output order) is
    exactly the host's, given the device's own continuous values; generic NMS is exactly the C oracle's;
  * both RPN paths agree where both are legal (post 1024 against 1025 over the first 1024 rows);
  * each image of a batch equals the same image run alone; two launches are bit-identical;
  * outputs go into views of sentinel-filled larger buffers: rows past count are zero up to post (RPN), the sentinel
    survives past count (NMS, box head), before and after the views;
  * inputs are bit-unchanged.
A child process profiles one call per dispatch path; the last test asserts that all nine kernels ran, in the paths the
dispatch rule predicts, in cases that passed.

The intervals assume expf within 2 ulp of RN(exp) (the CUDA Programming Guide's bound). Largest distance of a device
value from the exact-order fp32 restatement evaluated with RN(exp), over the whole table, measured on an NVIDIA H100
80GB HBM3 (SXM, 700 W power limit):
    RPN scores                          2 ulp
    class probabilities                 5 ulp   (31 bracketed terms in the in-order sum)
    box coordinates (>= 1 pixel)        256 ulp (a coordinate just above 1 that the chain computes near 1000: the
                                                 cancellation in pcx -+ 0.5 pw, inside the interval)
test_zz_every_kernel_ran prints these figures (PROPOSALS_CONFORMANCE_REPORT=path also writes them as JSON).

Sensitivity: each of these decision bugs, built into a copy of the kernels, fails tests of this file (failure counts on
the H100 above): the tie quota taken from the highest index in rpn_topk_decode_kernel (12), `>=` in nms_mask_kernel's
IoU test (17), `valid` ignored in nms_sweep_kernel (5), chunks of rpn_nms_greedy_kernel not tested against the boxes
kept before them (15), box_final_kernel's detections_per_img cut dropping ties (8), and rpn_write_kernel reading every
image's sorted boxes from image 0 (4).
"""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import proposals_ref as R

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
SENT = 0x7FA5A5A5               # a NaN payload no kernel produces
SENT64 = -0x5A5A5A5A5A5A5A5B
GUARD = 16                      # guard rows before and after each output view (keeps float4 rows 16-byte aligned)
RPN_CASES = R.make_rpn_cases()
NMS_CASES = R.make_nms_cases()
BOX_CASES = R.make_box_cases()
PASSED = set()                  # dispatch paths exercised by cases that passed
ULPS = {"score": 0, "box": 0, "prob": 0}


def _bits(t):
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int64)


def _guarded(shape, dtype, dev):
    """(buffer, contiguous view of `shape`) with GUARD sentinel rows of shape[1:] before and after"""
    row = int(np.prod(shape[1:])) if len(shape) > 1 else 1
    buf = torch.empty((shape[0] + 2 * GUARD) * row, dtype=dtype, device=dev)
    _bits(buf).fill_(SENT64 if dtype == torch.int64 else SENT)
    return buf, buf[GUARD * row:(GUARD + shape[0]) * row].view(*shape)


def _guards_ok(buf, n_rows, row, from_row=None):
    """sentinel intact before the view, after it, and (from_row) in the view's rows from that row on"""
    b = _bits(buf)
    sent = SENT64 if buf.dtype == torch.int64 else SENT
    lo = GUARD * row + (n_rows if from_row is None else from_row) * row
    return bool((b[:GUARD * row] == sent).all()) and bool((b[lo:] == sent).all())


def _np(t):
    return t.detach().cpu().numpy()


def _ulps(kind, got, centre):
    """largest distance in ulps from the RN(exp) centre; box coordinates below one pixel (where an ulp is far below
    the rounding of the chain's larger intermediates) are left out"""
    g, c = R.f32(got), R.f32(centre)
    fin = np.isfinite(g) & np.isfinite(c) & ((np.abs(c) >= 1) if kind == "box" else True)
    if fin.any():
        ULPS[kind] = max(ULPS[kind], int(R.ulp_dist(g[fin], c[fin]).max()))


# ------------------------------------------------------------------------------------------------ RPN
def _rpn_call(ops, head, n_img, c, base, pre, post, thresh, min_size, dev):
    out_b, ob = _guarded((n_img, post, 4), torch.float32, dev)
    out_s, os_ = _guarded((n_img, post), torch.float32, dev)
    out_a, oa = _guarded((n_img, post), torch.int32, dev)
    out_c, oc = _guarded((n_img,), torch.int32, dev)
    ops.rpn_select(head, n_img, c["h"], c["w"], base, c["im"][0], c["im"][1], pre, post, thresh, min_size, 16,
                   out=(ob, os_, oa, oc))
    torch.cuda.synchronize()
    for buf, row in ((out_b, post * 4), (out_s, post), (out_a, post), (out_c, 1)):
        assert _guards_ok(buf, n_img, row), "%s: wrote outside its output views" % c["id"]
    return _np(ob), _np(os_), _np(oa), _np(oc)


def run_rpn_case(c, dev):
    from mega_core.b200 import ops
    head_np, base_np = R.rpn_inputs(c)
    n_img, h, w = c["n_img"], c["h"], c["w"]
    a = base_np.shape[0]
    n = h * w * a
    full = torch.from_numpy(head_np).to(dev)
    head = full[1:1 + n_img] if c["slice_of"] else full
    base = torch.from_numpy(base_np).to(dev)
    keep = [(full, full.clone()), (base, base.clone())]
    img_np = head_np[1:1 + n_img] if c["slice_of"] else head_np
    paths = set()
    for pre, post in c["runs"]:
        k = min(pre, n)
        tb, ts, ta, tc = _rpn_call(ops, head, n_img, c, base, pre, k, 1.0, 0.0, dev)
        for i in range(n_img):
            lo, cen, hi = R.score_interval(img_np[i, ..., :a].reshape(-1)[ta[i, :k]])
            _ulps("score", ts[i, :k], cen)
            d = img_np[i, ..., a:5 * a].reshape(-1, a, 4)[ta[i, :k] // a, ta[i, :k] % a]
            anc = R.anchor_grid(h, w, base_np, 16)[ta[i, :k]]
            _ulps("box", tb[i, :k], R.box_interval(d, anc, (1, 1, 1, 1), c["im"][0], c["im"][1])[1])
        for m in c["min_size"]:
            if m == "ws":
                m = R.min_size_at(tb[0])
            real = _rpn_call(ops, head, n_img, c, base, pre, post, c["thresh"], m, dev)
            again = _rpn_call(ops, head, n_img, c, base, pre, post, c["thresh"], m, dev)
            for x, y in zip(real, again):
                assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                      y.view(np.uint32) if y.dtype == np.float32 else y), \
                    "%s pre %d post %d: two launches differ" % (c["id"], pre, post)
            for i in range(n_img):
                errs = R.check_rpn(img_np[i], base_np, 16, c["im"][0], c["im"][1], pre, post, c["thresh"], m,
                                   (tb[i], ts[i], ta[i], tc[i]), (real[0][i], real[1][i], real[2][i], real[3][i]),
                                   exact=c["exact"])
                assert not errs, "%s img %d pre %d post %d min_size %r: %s" % (c["id"], i, pre, post, m, errs)
                if n_img > 1:
                    alone = _rpn_call(ops, head[i:i + 1], 1, c, base, pre, post, c["thresh"], m, dev)
                    assert R.compare_exact([x[0] for x in alone], [x[i] for x in real], "alone") == [], \
                        "%s img %d: differs from the image run alone" % (c["id"], i)
            paths.add("rpn_" + R.rpn_path(post))
        for t, before in keep:
            assert torch.equal(_bits(t), _bits(before)), "%s: an input changed" % c["id"]
    # both NMS paths on the same selection: post 1024 (greedy) against 1025 (mask), over the first 1024 rows
    pre = c["runs"][0][0]
    g = _rpn_call(ops, head, n_img, c, base, pre, 1024, c["thresh"], 0.0, dev)
    m_ = _rpn_call(ops, head, n_img, c, base, pre, 1025, c["thresh"], 0.0, dev)
    for i in range(n_img):
        mine = (m_[0][i][:1024], m_[1][i][:1024], m_[2][i][:1024], min(int(m_[3][i]), 1024))
        assert R.compare_exact((g[0][i], g[1][i], g[2][i], g[3][i]), mine, "paths") == [], \
            "%s img %d: greedy and mask paths differ" % (c["id"], i)
    PASSED.update(paths)


@pytest.mark.parametrize("case", RPN_CASES, ids=[c["id"] for c in RPN_CASES])
def test_rpn_select_conforms(cuda_dev, case):
    run_rpn_case(case, cuda_dev)


@pytest.mark.parametrize("post", [300, 1025])
def test_rpn_select_empty_map(cuda_dev, post):
    """a map without cells: count 0, boxes and scores zero, anchors -1, on both paths"""
    from mega_core.b200 import ops
    c = dict(id="empty", h=0, w=5, im=(80.0, 64.0))
    head = torch.zeros(2, 0, 5, 64, device=cuda_dev)
    base = torch.from_numpy(R.cell_anchors()).to(cuda_dev)
    b, s, a, n = _rpn_call(ops, head, 2, c, base, 6000, post, 0.7, 0.0, cuda_dev)
    assert (n == 0).all() and (b == 0).all() and (s == 0).all() and (a == -1).all()
    PASSED.add("rpn_empty_" + R.rpn_path(post))


# ------------------------------------------------------------------------------------------------ generic NMS
def run_nms_case(c, dev):
    import mega_oracle as mo
    from mega_core.b200 import ops
    n = c["boxes"].shape[0]
    boxes = torch.from_numpy(c["boxes"]).to(dev)
    scores = torch.from_numpy(c["scores"]).to(dev)
    keep_in = [(boxes, boxes.clone()), (scores, scores.clone())]
    for t in c["threshs"]:
        want = mo.nms(torch.from_numpy(c["boxes"]), torch.from_numpy(c["scores"]), t, cuda_semantics=True).numpy()
        res = []
        for _ in range(2):
            kb, keep = _guarded((max(n, 1),), torch.int64, dev)
            cb, cnt = _guarded((1,), torch.int32, dev)
            ops.nms_device(boxes, scores, t, keep=keep, count=cnt)
            torch.cuda.synchronize()
            m = int(cnt.item())
            assert _guards_ok(kb, max(n, 1), 1, from_row=m) and _guards_ok(cb, 1, 1), "%s: wrote past count" % c["id"]
            res.append(_np(keep[:m]))
        assert np.array_equal(res[0], res[1]), "%s %g: two launches differ" % (c["id"], t)
        assert np.array_equal(res[0], want), "%s thresh %g: keep %s, oracle %s" % (c["id"], t, res[0][:20], want[:20])
    for t_, before in keep_in:
        assert torch.equal(_bits(t_), _bits(before)), "%s: an input changed" % c["id"]
    if n:
        PASSED.add("nms")


@pytest.mark.parametrize("case", NMS_CASES, ids=[c["id"] for c in NMS_CASES])
def test_nms_conforms(cuda_dev, case):
    run_nms_case(case, cuda_dev)


# ------------------------------------------------------------------------------------------------ box head
def _box_call(ops, pred, c, props, cnt, run, dev):
    st, nt, md, cap = run
    C = c["c"]
    bb, ob = _guarded((cap, 4), torch.float32, dev)
    sb, os_ = _guarded((cap,), torch.float32, dev)
    lb, ol = _guarded((cap,), torch.int64, dev)
    cb, oc = _guarded((1,), torch.int32, dev)
    ops.box_postprocess(pred[:, :C], pred[:, C:], props, cnt, C, c["im"][0], c["im"][1], st, nt, md, R.BOX_W,
                        (ob, os_, ol, oc))
    torch.cuda.synchronize()
    m = int(oc.item())
    for buf, row in ((bb, 4), (sb, 1), (lb, 1)):
        assert _guards_ok(buf, cap, row, from_row=m), "%s: wrote past count or outside the view" % c["id"]
    assert _guards_ok(cb, 1, 1)
    return _np(ob), _np(os_), _np(ol), m


def run_box_case(c, dev):
    from mega_core.b200 import ops
    C, r = c["c"], c["r"]
    ld = 5 * C + 3
    pred_np = np.full((r, ld), np.nan, np.float32)
    pred_np[:, :C] = c["logits"]
    pred_np[:, C:5 * C] = c["deltas"]
    pred = torch.from_numpy(pred_np).to(dev)
    props = torch.from_numpy(c["props"]).to(dev)
    cnt = torch.tensor([c["count"]], dtype=torch.int32, device=dev)
    keep = [(pred, pred.clone()), (props, props.clone()), (cnt, cnt.clone())]
    tr = R.transparency_box(C, r)
    trans = _box_call(ops, pred, c, props, cnt, (tr["score_thresh"], tr["nms_thresh"], tr["max_det"], tr["out_cap"]),
                      dev)
    rr = min(c["count"], r)
    if rr:
        _ulps("prob", trans[1][:(C - 1) * rr], R.prob_interval(c["logits"][:rr])[1][:, 1:].T.reshape(-1))
        d = c["deltas"][:rr].reshape(rr, C, 4)
        _ulps("box", trans[0][:(C - 1) * rr], R.box_interval(d, c["props"][:rr, None, :], R.BOX_W, c["im"][0], c["im"][1])[1][:, 1:]
              .transpose(1, 0, 2).reshape(-1, 4))
    for run in c["runs"]:
        run = R.resolve_run(run, trans[1])
        real = _box_call(ops, pred, c, props, cnt, run, dev)
        again = _box_call(ops, pred, c, props, cnt, run, dev)
        assert R.compare_exact(real, again, "again") == [], "%s %s: two launches differ" % (c["id"], run)
        errs = R.check_box(c["logits"], c["deltas"], c["props"], c["count"], C, c["im"][0], c["im"][1], trans, real,
                           *run)
        assert not errs, "%s run %s: %s" % (c["id"], run, errs)
    for t, before in keep:
        assert torch.equal(_bits(t), _bits(before)), "%s: an input changed" % c["id"]
    PASSED.add("box")


@pytest.mark.parametrize("case", BOX_CASES, ids=[c["id"] for c in BOX_CASES])
def test_box_postprocess_conforms(cuda_dev, case):
    run_box_case(case, cuda_dev)


# ------------------------------------------------------------------------------------------------ host-side rejections
def test_nms_rejects_8193(cuda_dev):
    from mega_core._lib import MegaError
    from mega_core.b200 import ops
    with pytest.raises(MegaError):
        ops.nms_device(torch.zeros(8193, 4, device=cuda_dev), torch.zeros(8193, device=cuda_dev), 0.5)


REJECT = ["rpn_head_f16", "rpn_head_channel_slice", "rpn_head_hw_mismatch", "rpn_base_f64", "rpn_base_strided",
          "rpn_out_boxes_misaligned", "rpn_out_scores_short", "rpn_out_anchor_int64", "rpn_out_count_short",
          "rpn_n_img_0", "rpn_h_negative", "rpn_no_anchors", "box_props_misaligned", "box_logits_inner_stride",
          "box_logits_narrow", "box_deltas_narrow", "box_count_int64", "box_scores_short", "box_labels_int32",
          "nms_keep_short", "nms_keep_int32", "nms_boxes_not_n4"]


@pytest.mark.parametrize("what", REJECT)
def test_rejects_layouts_before_launch(cuda_dev, what):
    from mega_core import _lib
    from mega_core._lib import MegaError
    from mega_core.b200 import ops
    dev = cuda_dev
    sentinel_bufs = []

    def guarded(shape, dtype=torch.float32):
        buf, v = _guarded(shape, dtype, dev)
        sentinel_bufs.append((buf, _bits(buf).clone()))
        return v

    if what.startswith("rpn"):
        h, w, n_img, post = 6, 7, 2, 40
        head = torch.zeros(n_img, h, w, 64, device=dev)
        base = torch.from_numpy(R.cell_anchors()).to(dev)
        ob, os_, oa, oc = guarded((n_img, post, 4)), guarded((n_img, post)), guarded((n_img, post), torch.int32), \
            guarded((n_img,), torch.int32)
        args = dict(h=h, w=w, n_img=n_img)
        if what == "rpn_head_f16":
            head = head.half()
        elif what == "rpn_head_channel_slice":
            head = torch.zeros(n_img, h, w, 128, device=dev)[..., :64]
        elif what == "rpn_head_hw_mismatch":
            args["w"] = 6
        elif what == "rpn_base_f64":
            base = base.double()
        elif what == "rpn_base_strided":
            base = torch.zeros(12, 8, device=dev)[:, :4]
        elif what == "rpn_out_boxes_misaligned":
            ob = guarded((n_img * post * 4 + 1,))[1:].view(n_img, post, 4)
        elif what == "rpn_out_scores_short":
            os_ = os_[:, :post - 1]
        elif what == "rpn_out_anchor_int64":
            oa = guarded((n_img, post), torch.int64)
        elif what == "rpn_out_count_short":
            oc = oc[:1]
        elif what == "rpn_n_img_0":
            args["n_img"] = 0
        elif what == "rpn_h_negative":
            args["h"] = -1
        else:
            base = base[:0]
        call = lambda: ops.rpn_select(head, args["n_img"], args["h"], args["w"], base, 100.0, 90.0, 600, post, 0.7,
                                      0.0, 16, out=(ob, os_, oa, oc))
    elif what.startswith("box"):
        C, r = 3, 20
        pred = torch.zeros(r, 5 * C, device=dev)
        logits, deltas = pred[:, :C], pred[:, C:]
        props = torch.zeros(r, 4, device=dev)
        cnt = torch.tensor([r], dtype=torch.int32, device=dev)
        cap = (C - 1) * r
        ob, os_, ol, oc = guarded((cap, 4)), guarded((cap,)), guarded((cap,), torch.int64), guarded((1,), torch.int32)
        if what == "box_props_misaligned":
            props = torch.zeros(r * 4 + 1, device=dev)[1:].view(r, 4)
        elif what == "box_logits_inner_stride":
            logits = torch.zeros(C, r, device=dev).t()
        elif what == "box_logits_narrow":
            logits = pred[:, :C - 1]
        elif what == "box_deltas_narrow":
            deltas = pred[:, C:4 * C]
        elif what == "box_count_int64":
            cnt = cnt.long()
        elif what == "box_scores_short":
            os_ = os_[:cap - 1]
        else:
            ol = guarded((cap,), torch.int32)
        call = lambda: ops.box_postprocess(logits, deltas, props, cnt, C, 100.0, 90.0, 0.001, 0.5, 10, R.BOX_W,
                                           (ob, os_, ol, oc))
    else:
        n = 50
        boxes = torch.zeros(n, 4, device=dev)
        scores = torch.zeros(n, device=dev)
        keep = guarded((n,), torch.int64)
        cnt = guarded((1,), torch.int32)
        if what == "nms_keep_short":
            keep = keep[:n - 1]
        elif what == "nms_keep_int32":
            keep = guarded((n,), torch.int32)
        else:
            boxes = torch.zeros(n, 5, device=dev)
        call = lambda: ops.nms_device(boxes, scores, 0.5, keep=keep, count=cnt)
    with pytest.raises(MegaError):
        call()
    torch.cuda.synchronize()
    for buf, before in sentinel_bufs:
        assert torch.equal(_bits(buf), before), "%s: an output was written" % what
    assert _lib.lib.mega_device_ok() == 1


# ------------------------------------------------------------------------------------------------ dispatch gate
def _kernel_names(prof):
    names = []
    for e in prof.events():
        m = re.search(r"mega::(\w+_kernel)\(", e.name)
        if m and m.group(1) in R.ALL_KERNELS and m.group(1) not in names:
            names.append(m.group(1))
    return sorted(names)


def profile_child(out_path):
    """runs one call per dispatch path under the profiler in this (child) process; writes the kernels each launched"""
    from torch.profiler import ProfilerActivity, profile
    from mega_core.b200 import ops
    dev = torch.device("cuda:0")
    c = next(x for x in RPN_CASES if x["id"] == "fixture_12x20")
    head = torch.from_numpy(R.rpn_inputs(c)[0]).to(dev)
    base = torch.from_numpy(R.cell_anchors()).to(dev)
    empty = torch.zeros(1, 0, 5, 64, device=dev)
    bc = next(x for x in BOX_CASES if x["id"] == "c31_r300_n300")
    pred = torch.from_numpy(np.concatenate([bc["logits"], bc["deltas"]], 1)).to(dev)
    props = torch.from_numpy(bc["props"]).to(dev)
    cnt = torch.tensor([300], dtype=torch.int32, device=dev)
    out = (torch.zeros(9000, 4, device=dev), torch.zeros(9000, device=dev),
           torch.zeros(9000, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
    nb = torch.from_numpy(NMS_CASES[4]["boxes"]).to(dev)
    ns = torch.from_numpy(NMS_CASES[4]["scores"]).to(dev)
    calls = {
        "nms": (lambda: ops.nms_device(nb, ns, 0.5), R.nms_kernels(nb.shape[0])),
        "rpn_greedy": (lambda: ops.rpn_select(head, 1, 12, 20, base, 313.0, 187.0, 6000, 300, 0.7),
                       R.rpn_kernels(2880, 6000, 300)),
        "rpn_mask": (lambda: ops.rpn_select(head, 1, 12, 20, base, 313.0, 187.0, 6000, 2000, 0.7),
                     R.rpn_kernels(2880, 6000, 2000)),
        "rpn_empty_mask": (lambda: ops.rpn_select(empty, 1, 0, 5, base, 80.0, 64.0, 6000, 2000, 0.7),
                           R.rpn_kernels(0, 6000, 2000)),
        "box": (lambda: ops.box_postprocess(pred[:, :31], pred[:, 31:], props, cnt, 31, 1000.0, 600.0, 0.001, 0.5, 300,
                                            R.BOX_W, out), R.box_kernels()),
    }
    seen = {}
    for name, (fn, want) in calls.items():
        fn()
        torch.cuda.synchronize()
        names = []
        for attempt in range(8):       # a session now and then delivers no kernel record: retry after a growing pause
            if attempt:
                time.sleep(0.05 * 2 ** attempt)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            names = _kernel_names(prof)
            if names:
                break
        seen[name] = dict(names=names, want=sorted(want))
    with open(out_path, "w") as fh:
        json.dump(seen, fh)


def test_zz_every_kernel_ran(cuda_dev, tmp_path):
    """runs last in this file: the profiler, in a process of its own, sees each dispatch path launch exactly the kernels
    the restated rule predicts; each of those paths ran in cases of this file that passed; together they launch all
    nine kernels. It reads the session-wide record, so it fails when the file runs in part."""
    out = tmp_path / "kernels.json"
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(
        [TESTS, ROOT, os.path.join(ROOT, "mega.pytorch_b200"), os.path.join(ROOT, "oracle")]
        + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    code = "import sys, test_proposals_conformance_gpu as t; t.profile_child(sys.argv[1])"
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, str(out)]
    res = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    seen = json.loads(out.read_text())
    report = dict(seen=seen, passed=sorted(PASSED), max_ulps=ULPS)
    print("proposals conformance:", json.dumps(report))
    path = os.environ.get("PROPOSALS_CONFORMANCE_REPORT")
    if path:
        with open(path, "w") as fh:
            json.dump(report, fh, indent=1)
    for name, rec in seen.items():
        assert rec["names"] == rec["want"], "%s launched %s, the dispatch rule says %s" % (name, rec["names"], rec["want"])
    need = {"nms", "rpn_greedy", "rpn_mask", "rpn_empty_mask", "box"}
    assert need <= PASSED, "paths without a passing case: %s" % sorted(need - PASSED)
    ran = set().union(*[set(rec["names"]) for rec in seen.values()])
    assert ran == set(R.ALL_KERNELS), sorted(set(R.ALL_KERNELS) - ran)
