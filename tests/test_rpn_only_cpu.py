"""MODEL.RPN_ONLY and proposal-recall evaluation without a GPU:
  1. the kernel's per-image body (csrc/proposal_recall.cuh, built by g++ through tests/native/proposal_recall_host.cpp
     with the C ABI's names) equals the reference's eval_proposals_vid on the cases of tests/golden/rpn_only.pt
     (oracle/make_golden_rpn_only.py): recall bit for bit and every greedy-round overlap;
  2. the RPN-only module tree has the reference's state_dict layout for the single-frame, DFF and FGFA configs, and a
     full checkpoint loads into it;
  3. the configurations the engines do not serve are refused naming MODEL.RPN_ONLY;
  4. the Python layer (gather_predictions, do_vid_evaluation(box_only=True), inference / inference_no_model) driven
     end to end with the host build patched over the library's entry points -- the patching exists in this test only,
     the product has no CPU path."""
import ctypes
import hashlib
import logging
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "rpn_only.pt"), weights_only=False)
_host = None


def host_lib():
    """g++ build of csrc/proposal_recall.cuh, cached in the temp directory under the digest of its sources"""
    global _host
    if _host is None:
        src = os.path.join(ROOT, "tests", "native", "proposal_recall_host.cpp")
        deps = [src] + [os.path.join(ROOT, "mega.pytorch_b200", "csrc", n) for n in ("proposal_recall.cuh", "iou.cuh")] + [
            os.path.join(ROOT, "include", "mega_b200.h")]
        digest = hashlib.sha256(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
        so_path = os.path.join(tempfile.gettempdir(), "mega_proposal_recall_host_%s_%d.so" % (digest, os.getuid()))
        if not os.path.exists(so_path):
            tmp = so_path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-I",
                                   os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                                   "-o", tmp, src])
            os.replace(tmp, so_path)
        _host = ctypes.CDLL(so_path)
        from mega_core import _lib
        for name in ("mega_proposal_recall", "mega_proposal_recall_workspace_bytes"):
            fn, real = getattr(_host, name), getattr(_lib.lib, name)
            fn.argtypes, fn.restype = real.argtypes, real.restype
    return _host


def host_run(images, iou_thresh, limit):
    """images: list of (boxes [P, 4], objectness [P], gt [G, 4]) -> (hits, num_pos, rejected, gt_overlaps [sum G])"""
    lib = host_lib()
    f = lambda a: np.ascontiguousarray(np.asarray(a, np.float32))            # noqa: E731
    pb = f(np.concatenate([np.asarray(i[0]).reshape(-1, 4) for i in images] + [np.zeros((0, 4))]))
    ps = f(np.concatenate([np.asarray(i[1]).reshape(-1) for i in images] + [np.zeros(0)]))
    gb = f(np.concatenate([np.asarray(i[2]).reshape(-1, 4) for i in images] + [np.zeros((0, 4))]))
    pc = [len(i[1]) for i in images]
    gc = [len(i[2]) for i in images]
    po = np.concatenate([[0], np.cumsum(pc)]).astype(np.int64)
    go = np.concatenate([[0], np.cumsum(gc)]).astype(np.int64)
    mp, mg = max(pc + [0]), max(gc + [0])
    nbytes = lib.mega_proposal_recall_workspace_bytes(len(images), mp, mg, limit)
    assert nbytes >= 0
    ws = np.zeros(nbytes // 4 + 1, np.float32)
    ov = np.full(len(gb), np.nan, np.float32)
    stats = np.zeros(3, np.uint64)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)                            # noqa: E731
    assert lib.mega_proposal_recall(p(pb), p(ps), p(po), p(gb), p(go), len(images), mp, mg, limit, iou_thresh, p(ws),
                                    nbytes, p(ov), p(stats), None) == 0
    return int(stats[0]), int(stats[1]), int(stats[2]), ov


def contributing(images, limit, ov):
    """the per-image overlap lists the reference concatenates: images with proposals (after the limit) and GT"""
    out, off = [], 0
    for b, s, g in images:
        n = len(g)
        if n and min(len(s), limit):
            out.append(ov[off:off + n])
        off += n
    return out


@pytest.mark.parametrize("case", GOLD["recall_cases"], ids=[c["name"] for c in GOLD["recall_cases"]])
def test_host_build_equals_the_reference_evaluator(case):
    images = [(im["boxes"].numpy(), im["objectness"].numpy(), im["gt"].numpy()) for im in case["images"]]
    hits, num_pos, rejected, ov = host_run(images, case["iou_thresh"], case["limit"])
    assert rejected == 0
    got = contributing(images, case["limit"], ov)
    want = [t.numpy() for t in case["gt_overlaps"]]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert np.array_equal(g.view(np.uint32), w.astype(np.float32).view(np.uint32)), (g, w)
    assert not np.isnan(ov).any()
    recall = torch.tensor(float(hits), dtype=torch.float32) / float(num_pos)
    assert recall.dtype == case["recall"].dtype and torch.equal(recall, case["recall"])


def reference_loop(images, iou_thresh=0.5, limit=300):
    """eval_proposals_vid (vid_eval.py:72-119) restated with the same torch calls, per image and greedy round ->
    (recall, the concatenated per-image overlaps)"""
    def boxlist_iou(box1, box2):                               # structures/boxlist_ops.py:53-90
        area1 = (box1[:, 2] - box1[:, 0] + 1) * (box1[:, 3] - box1[:, 1] + 1)
        area2 = (box2[:, 2] - box2[:, 0] + 1) * (box2[:, 3] - box2[:, 1] + 1)
        lt = torch.max(box1[:, None, :2], box2[:, :2])
        rb = torch.min(box1[:, None, 2:], box2[:, 2:])
        wh = (rb - lt + 1).clamp(min=0)
        inter = wh[:, :, 0] * wh[:, :, 1]
        return inter / (area1[:, None] + area2 - inter)

    gt_overlaps, num_pos = [], 0
    for b, s, g in images:
        b, s, g = (torch.as_tensor(np.asarray(x, np.float32)) for x in (b, s, g))
        inds = s.sort(descending=True)[1]
        b = b.reshape(-1, 4)[inds][:limit]
        num_pos += len(g)
        if len(g) == 0 or len(b) == 0:
            continue
        overlaps = boxlist_iou(b, g.reshape(-1, 4))
        o = torch.zeros(len(g))
        for j in range(min(len(b), len(g))):
            max_overlaps, argmax_overlaps = overlaps.max(dim=0)
            gt_ovr, gt_ind = max_overlaps.max(dim=0)
            box_ind = argmax_overlaps[gt_ind]
            o[j] = overlaps[box_ind, gt_ind]
            overlaps[box_ind, :] = -1
            overlaps[:, gt_ind] = -1
        gt_overlaps.append(o)
    cat = torch.cat(gt_overlaps) if gt_overlaps else torch.zeros(0)
    return (cat >= iou_thresh).float().sum() / float(num_pos), cat


def test_host_build_equals_a_torch_restatement_on_tie_heavy_random_images():
    """objectness with 0-2 decimals (many ties, so the sort's tie order decides which proposals pass the limit), integer
    boxes (IoU ties), 1-700 proposals per image"""
    rng = np.random.default_rng(21)
    images = []
    for _ in range(60):
        p, g = int(rng.integers(1, 700)), int(rng.integers(1, 15))
        x = rng.integers(0, 800, (p, 2))
        b = np.concatenate([x, x + rng.integers(4, 80, (p, 2))], 1)
        gx = rng.integers(0, 800, (g, 2))
        gt = np.concatenate([gx, gx + rng.integers(4, 80, (g, 2))], 1)
        images.append((b, np.round(rng.uniform(0, 1, p), int(rng.integers(0, 3))), gt))
    for limit in (300, 20):
        hits, num_pos, _, ov = host_run(images, 0.5, limit)
        recall, want = reference_loop(images, 0.5, limit)
        got = np.concatenate(contributing(images, limit, ov))
        assert np.array_equal(got.view(np.uint32), want.numpy().view(np.uint32))
        assert torch.equal(torch.tensor(float(hits), dtype=torch.float32) / float(num_pos), recall)


def test_the_fixture_covers_the_cases_the_rules_distinguish():
    by = {c["name"]: c for c in GOLD["recall_cases"]}
    ties = by["ties"]["images"]
    assert any(len(torch.unique(im["objectness"])) < len(im["objectness"]) for im in ties)
    assert all(len(im["objectness"]) > 300 for im in by["limit_bites"]["images"])
    assert all(len(im["objectness"]) < len(im["gt"]) for im in by["fewer_proposals_than_gt"]["images"])
    empty = by["empty_images"]["images"]
    assert any(len(im["gt"]) == 0 for im in empty) and any(len(im["objectness"]) == 0 for im in empty)


def test_iou_ties_between_proposals_resolve_to_the_lowest_sorted_index():
    """two proposals with the same IoU to the one GT box; the first in objectness order wins, ties in objectness go to
    the lower input index. A second GT box then takes the other proposal."""
    gt = [[10, 10, 29, 29], [100, 100, 119, 119]]
    boxes = [[12, 10, 31, 29], [8, 10, 27, 29], [100, 100, 119, 119]]
    for scores, first in (([0.5, 0.9, 0.1], 1), ([0.9, 0.5, 0.1], 0), ([0.7, 0.7, 0.1], 0)):
        hits, num_pos, _, ov = host_run([(boxes, scores, gt)], 0.5, 300)
        assert (hits, num_pos) == (2, 2)
        assert ov[0] == 1.0                          # the exact match of GT 1 is the largest entry
        # round 2: GT 0 against the two shifted boxes (IoU 18*20 / (2*400 - 360) = 360 / 440)
        assert ov[1] == np.float32(360.0) / np.float32(440.0)
    hits, _, _, ov = host_run([(boxes[:2], [0.5, 0.5], gt[:1])], 0.5, 1)     # limit 1: only index 0 is kept
    assert hits == 1 and ov[0] == np.float32(360.0) / np.float32(440.0)


def test_more_proposals_than_the_cap_is_an_argument_error():
    lib = host_lib()
    assert lib.mega_proposal_recall_workspace_bytes(4, 8192, 10, 300) == 0
    assert lib.mega_proposal_recall_workspace_bytes(4, 8193, 10, 300) == -1
    from mega_core.b200 import ops
    with pytest.raises(Exception, match="8192"):
        ops.proposal_recall_workspace_bytes(4, 9000, 10, 300)


def test_large_matrices_use_the_workspace_and_give_the_same_result():
    rng = np.random.default_rng(3)
    images = []
    for _ in range(5):
        p, g = int(rng.integers(400, 900)), int(rng.integers(120, 200))
        x = rng.uniform(0, 900, (p, 2)).astype(np.float32)
        b = np.concatenate([x, x + rng.uniform(5, 120, (p, 2)).astype(np.float32)], 1)
        gx = rng.uniform(0, 900, (g, 2)).astype(np.float32)
        gt = np.concatenate([gx, gx + rng.uniform(5, 120, (g, 2)).astype(np.float32)], 1)
        images.append((b, np.round(rng.uniform(0, 1, p), 2).astype(np.float32), gt))
    assert host_lib().mega_proposal_recall_workspace_bytes(5, 900, 200, 300) > 0
    big = host_run(images, 0.5, 300)
    # one image per call, where the bounds are that image's: same overlaps (the matrix may fit shared memory now)
    ov = np.concatenate([host_run([im], 0.5, 300)[3] for im in images])
    assert np.array_equal(big[3], ov) and big[2] == 0


# ------------------------------------------------------------------ model and config layer
def _cfg(method, rpn_only=True, **extra):
    from mega_core.modeling.detector.detectors import vid_config
    body = "R-50-C4" if method == "base" else "R-101-C4"
    c = vid_config(method, body, device="cpu")
    c.MODEL.RPN_ONLY = rpn_only
    for k, v in extra.items():
        node = c
        *path, last = k.split(".")
        for p in path:
            node = getattr(node, p)
        setattr(node, last, v)
    return c


@pytest.mark.parametrize("method,name", [("base", "base_r50"), ("dff", "dff_r101"), ("fgfa", "fgfa_r101")])
def test_state_dict_layout_equals_the_reference(method, name):
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(_cfg(method))
    assert model.roi_heads == [] and not model.roi_heads
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == GOLD["state_dicts"][name]


def test_full_checkpoint_loads_into_the_rpn_only_model(tmp_path):
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model
    from mega_core.utils.checkpoint import DetectronCheckpointer
    sd = synth.make_state_dict("base_r50", seed=1)
    assert any(k.startswith("roi_heads.") for k in sd)
    path = os.path.join(tmp_path, "model_final.pth")
    torch.save({"model": sd}, path)
    cfg = _cfg("base")
    model = build_detection_model(cfg)
    DetectronCheckpointer(cfg, model).load(path, use_latest=False)
    own = model.state_dict()
    assert not any(k.startswith("roi_heads.") for k in own)
    for k, v in own.items():
        if k in sd:
            assert torch.equal(v, sd[k]), k
    assert sum(k in sd for k in own) == len(own) - 1            # everything but the anchors (a buffer, not saved)


def test_engine_config_carries_rpn_only():
    from mega_core.modeling.nets import engine_config_from
    assert engine_config_from(_cfg("fgfa")).rpn_only is True
    assert engine_config_from(_cfg("fgfa", rpn_only=False)).rpn_only is False


@pytest.mark.parametrize("method,extra", [("mega", {}), ("rdn", {}), ("base", {"TEST.BBOX_AUG.ENABLED": True}),
                                          ("base", {"MODEL.B200.SEQ_NMS.ENABLED": True}),
                                          ("dff", {"MODEL.B200.SEQ_NMS.ENABLED": True})])
def test_unserved_combinations_are_refused(method, extra):
    from mega_core.modeling.nets import engine_config_from
    with pytest.raises(NotImplementedError, match="MODEL.RPN_ONLY"):
        engine_config_from(_cfg(method, **extra))


def test_windowed_engines_refuse_rpn_only():
    from mega_core.b200 import engine
    with pytest.raises(NotImplementedError, match="MODEL.RPN_ONLY"):
        engine.MegaEngine({}, engine.EngineConfig(rpn_only=True), device="cpu")


# ------------------------------------------------------------------ plumbing
def _proposals(rng, n, size=(1000, 600)):
    from mega_core.structures.bounding_box import BoxList
    x = rng.uniform(0, 800, (n, 2)).astype(np.float32)
    b = BoxList(torch.from_numpy(np.concatenate([x, x + rng.uniform(5, 150, (n, 2)).astype(np.float32)], 1)), size)
    b.add_field("objectness", torch.from_numpy(np.sort(rng.uniform(0, 1, n).astype(np.float32))[::-1].copy()))
    return b


def test_gather_predictions_round_trips_proposals():
    from mega_core.utils.comm import gather_predictions
    rng = np.random.default_rng(1)
    preds = {i: _proposals(rng, n) for i, n in zip([2, 0, 1], [5, 0, 300])}
    out = gather_predictions(preds)
    assert len(out) == 3
    for i, b in enumerate(out):
        assert b.fields() == ["objectness"] and b.size == preds[i].size
        assert torch.equal(b.bbox, preds[i].bbox) and torch.equal(b.get_field("objectness"), preds[i].get_field("objectness"))


@pytest.fixture
def host_recall(monkeypatch):
    """mega_proposal_recall served by the host build, the evaluator's device set to the CPU"""
    from mega_core import _lib
    from mega_core.b200 import ops
    from mega_core.data.datasets.evaluation.vid import vid_eval
    host = host_lib()
    for name in ("mega_proposal_recall", "mega_proposal_recall_workspace_bytes"):
        monkeypatch.setattr(_lib.lib, name, getattr(host, name))
    monkeypatch.setattr(ops, "require_cuda", lambda *t: None)
    monkeypatch.setattr(ops, "stream_ptr", lambda: None)
    monkeypatch.setattr(vid_eval, "_device", lambda: torch.device("cpu"))
    return vid_eval


class _Dataset(object):
    """images of 1000 x 600 whose GT are the first boxes of seeded proposal sets"""

    def __init__(self, n=12):
        rng = np.random.default_rng(7)
        self.props = [_proposals(rng, int(rng.integers(0, 40))) for _ in range(n)]
        self.gt = []
        for i, p in enumerate(self.props):
            g = p.bbox[: i % 4].clone() + 3.0
            from mega_core.structures.bounding_box import BoxList
            self.gt.append(BoxList(g.reshape(-1, 4), (1000, 600)))

    def __len__(self):
        return len(self.props)

    def get_img_info(self, i):
        return {"width": 1000, "height": 600}

    def get_groundtruth(self, i):
        return self.gt[i]


def _want_recall(ds):
    images = [(p.bbox.numpy(), p.get_field("objectness").numpy(), g.bbox.numpy()) for p, g in zip(ds.props, ds.gt)]
    hits, num_pos, _, _ = host_run(images, 0.5, 300)
    return torch.tensor(float(hits), dtype=torch.float32) / float(num_pos)


def test_box_only_evaluation_writes_the_reference_report(tmp_path, host_recall):
    ds = _Dataset()
    logger = logging.getLogger("test_rpn_only")
    res = host_recall.do_vid_evaluation(ds, ds.props, str(tmp_path), True, False, logger)
    assert res is None
    text = open(os.path.join(tmp_path, "proposal_result.txt")).read()
    want = _want_recall(ds)
    assert 0 < want.item() < 1
    assert text == "Recall: {:.4f}".format(want)
    assert torch.equal(host_recall.eval_proposals_vid(ds.props, ds.gt)["recall"], want)


def test_inference_and_saved_predictions_evaluate_recall(tmp_path, host_recall):
    from mega_core.config import cfg as base
    from mega_core.engine.inference import inference, inference_no_model
    ds = _Dataset()

    class Loader(object):
        dataset = ds

        def __iter__(self):
            for i in range(len(ds)):
                yield torch.zeros(1, 3, 4, 4), None, [i]

    class Model(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.i = 0

        def forward(self, images):
            self.i += 1
            return [ds.props[self.i - 1]]

    c = base.clone()
    c.MODEL.VID.METHOD = "base"
    c.MODEL.RPN_ONLY = True
    logging.getLogger("mega_core.inference").setLevel(logging.ERROR)
    assert inference(c, Model(), Loader(), "VID_val_synthetic", box_only=True, device="cpu",
                     output_folder=str(tmp_path)) is None
    text = open(os.path.join(tmp_path, "proposal_result.txt")).read()
    assert text == "Recall: {:.4f}".format(_want_recall(ds))
    saved = torch.load(os.path.join(tmp_path, "predictions.pth"), weights_only=False)
    assert all(p.fields() == ["objectness"] for p in saved)
    os.remove(os.path.join(tmp_path, "proposal_result.txt"))
    assert inference_no_model(Loader(), box_only=True, output_folder=str(tmp_path)) is None
    assert open(os.path.join(tmp_path, "proposal_result.txt")).read() == text


def test_evaluator_raises_without_a_device(monkeypatch):
    from mega_core import _lib
    from mega_core.data.datasets.evaluation.vid import eval_proposals_vid
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    ds = _Dataset(2)
    with pytest.raises(_lib.MegaError, match="GPU"):
        eval_proposals_vid(ds.props, ds.gt)
