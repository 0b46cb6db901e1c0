"""The device VID evaluator (MODEL.B200.VID_EVAL = "device") without a GPU:
  1. the bodies of csrc/vid_eval.cuh, driven in the kernels' order by a g++ build (tests/native/vid_eval_host.cpp, the
     C ABI's names) and fed by the device path's own packing and AP code (_VidEvalInputs), equal the host evaluator
     with stable_ties=True bit for bit -- n_pos, prec, rec and AP -- on both cases of tests/golden/vid_eval.pt (plain
     protocol and the four motion ranges in one call) and on a tie-heavy synthetic set with the edge cases;
  2. the resize of the predictions to the images' sizes, applied from per-image ratios, equals BoxList.resize;
  3. stable_ties=True changes nothing where no scores tie; the switch defaults to "host"; "device" without a GPU
     raises."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RANGES4 = [[0.0, 1.0], [0.0, 0.7], [0.7, 0.9], [0.9, 1.0]]
_host = None


def host_lib():
    """g++ build of csrc/vid_eval.cuh, cached in the temp directory under the digest of its sources"""
    global _host
    if _host is None:
        src = os.path.join(ROOT, "tests", "native", "vid_eval_host.cpp")
        deps = [src] + [os.path.join(ROOT, "mega.pytorch_b200", "csrc", n) for n in ("vid_eval.cuh", "iou.cuh")] + [
            os.path.join(ROOT, "include", "mega_b200.h")]
        digest = hashlib.sha256(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
        so_path = os.path.join(tempfile.gettempdir(), "mega_vid_eval_host_%s_%d.so" % (digest, os.getuid()))
        if not os.path.exists(so_path):
            tmp = so_path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-I",
                                   os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                                   "-o", tmp, src])
            os.replace(tmp, so_path)
        _host = ctypes.CDLL(so_path)
        from mega_core import _lib
        for name in ("mega_vid_eval", "mega_vid_eval_workspace_bytes"):
            fn, real = getattr(_host, name), getattr(_lib.lib, name)
            fn.argtypes, fn.restype = real.argtypes, real.restype
    return _host


def host_device_eval(preds, gts, motion, ranges, iou_thresh=0.5, image_sizes=None, use_07_metric=False):
    """the device path of eval_detection_vid with the g++ build in place of the kernels"""
    from mega_core.data.datasets.evaluation.vid.vid_eval import _VidEvalInputs
    x = _VidEvalInputs(preds, gts, motion, ranges, image_sizes, pin=False)
    nr = len(x.ranges)
    stats = np.zeros(x.stats_count(), np.int64)
    steps = np.zeros((nr, 3, x.num_steps), np.float64)
    curves = np.zeros((2, nr, x.p_tot), np.float64)
    rng = np.ascontiguousarray(np.asarray(x.ranges, np.float64).reshape(-1))
    p = lambda a: ctypes.c_void_p(a.ctypes.data)                                  # noqa: E731
    t = lambda i: ctypes.c_void_p(x.view(x.host, i).data_ptr())                    # noqa: E731
    lib = host_lib()
    assert lib.mega_vid_eval_workspace_bytes(x.p_tot, x.g_tot, x.n, x.num_classes, nr) == 0
    assert lib.mega_vid_eval(t(0), t(1), t(2), t(3), t(4), x.p_tot, t(5), t(6), t(7), t(8), x.g_tot, x.n,
                             x.num_classes, p(rng), nr, iou_thresh, t(9), x.num_steps, None, 0,
                             p(curves[0]), p(curves[1]), p(stats), p(steps), None) == 0
    return x.results(stats, steps, curves, use_07_metric, return_curves=True)


def _boxlists(images):
    from mega_core.structures.bounding_box import BoxList
    gts, preds = [], []
    for im in images:
        gt = BoxList(im["gt"], im["size"], mode="xyxy")
        gt.add_field("labels", im["gt_labels"])
        pr = BoxList(im["boxes"], im["pred_size"] if "pred_size" in im else im["size"], mode="xyxy")
        pr.add_field("labels", im["labels"])
        pr.add_field("scores", im["scores"])
        gts.append(gt)
        preds.append(pr)
    return gts, preds


def synthetic(seed, n_images=160, n_classes=7, decimals=1, edge_cases=True):
    """detections around the GT boxes (jittered copies and clutter) with scores rounded to `decimals` (ties), motion
    IoUs over the three ranges; with edge_cases: images without detections, without GT, a class present only in GT,
    motion lists shorter than the GT list, single-detection classes"""
    g = np.random.default_rng(seed)
    images = []
    for i in range(n_images):
        w, h = int(g.integers(200, 500)), int(g.integers(150, 400))
        n_gt = int(g.integers(0, 4)) if edge_cases else int(g.integers(1, 4))
        x1 = g.uniform(0, w * 0.6, n_gt)
        y1 = g.uniform(0, h * 0.6, n_gt)
        gt = np.stack([x1, y1, x1 + g.uniform(10, w * 0.4, n_gt), y1 + g.uniform(10, h * 0.4, n_gt)], 1).round()
        gl = g.integers(1, n_classes, n_gt)
        if edge_cases and i % 17 == 5:
            gl[:] = n_classes                    # a class no detection carries
        n_det = int(g.integers(0, 25)) if edge_cases and i % 11 else (1 if edge_cases else int(g.integers(5, 25)))
        src = g.integers(0, max(n_gt, 1), n_det)
        base = gt[src] if n_gt else np.tile([[10., 10., 60., 60.]], (n_det, 1))
        boxes = base + g.normal(0, 6, (n_det, 4))
        boxes[:, 2:] = np.maximum(boxes[:, 2:], boxes[:, :2] + 1)
        labels = np.where(g.random(n_det) < 0.7, gl[src] if n_gt else 1, g.integers(1, n_classes, n_det))
        scores = g.uniform(0.001, 1.0, n_det)
        scores = scores.round(decimals) if decimals is not None else scores
        motion = g.choice([0.3, 0.65, 0.7, 0.8, 0.9, 0.95, 1.0], n_gt).tolist()
        if edge_cases and i % 13 == 3:
            motion = motion[:max(n_gt - 1, 0)]
        images.append({"size": (w, h), "gt": torch.tensor(gt, dtype=torch.float32).reshape(-1, 4),
                       "gt_labels": torch.tensor(gl, dtype=torch.int64), "motion": motion,
                       "boxes": torch.tensor(boxes, dtype=torch.float32).reshape(-1, 4),
                       "labels": torch.tensor(labels, dtype=torch.int64),
                       "scores": torch.tensor(scores, dtype=torch.float32)})
    return images


def assert_same(dev, host):
    """bit-for-bit equality of two eval_detection_vid results with return_curves"""
    assert dev.keys() == host.keys()
    for r in host:
        a, b = dev[r], host[r]
        assert a["n_pos"] == {k: int(v) for k, v in b["n_pos"].items()}
        assert len(a["prec"]) == len(b["prec"]) and len(a["rec"]) == len(b["rec"])
        for x, y in zip(a["prec"] + a["rec"], b["prec"] + b["rec"]):
            assert (x is None) == (y is None)
            if x is not None:
                assert x.dtype == y.dtype == np.float64 and np.array_equal(x, y)
        assert np.array_equal(a["ap"], b["ap"], equal_nan=True)
        assert a["map"] == b["map"] or (np.isnan(a["map"]) and np.isnan(b["map"]))


def host_eval(preds, gts, motion, ranges, stable_ties=True, use_07_metric=False):
    from mega_core.data.datasets.evaluation.vid import eval_detection_vid
    return eval_detection_vid(preds, gts, 0.5, ranges, motion is not None, use_07_metric, motion_ious=motion,
                              stable_ties=stable_ties, return_curves=True)


@pytest.mark.parametrize("case", [0, 1])
def test_golden_cases_plain_and_four_ranges(case):
    images = torch.load(os.path.join(ROOT, "tests", "golden", "vid_eval.pt"), weights_only=False)[case]["images"]
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    assert_same(host_device_eval(preds, gts, None, [[0.0, 1.0]]), host_eval(preds, gts, None, [[0.0, 1.0]]))
    assert_same(host_device_eval(preds, gts, motion, RANGES4), host_eval(preds, gts, motion, RANGES4))


def test_tie_heavy_synthetic_with_edge_cases():
    images = synthetic(1)
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    ps = torch.cat([p.get_field("scores") for p in preds])
    assert ps.unique().numel() < ps.numel() // 10              # ties everywhere
    assert_same(host_device_eval(preds, gts, motion, RANGES4), host_eval(preds, gts, motion, RANGES4))
    assert_same(host_device_eval(preds, gts, None, RANGES4[:2]), host_eval(preds, gts, None, RANGES4[:2]))


def test_all_gt_ignored_and_empty_weight_one():
    """a range that ignores every GT (n_pos = 0: AP NaN) and one that keeps every motion value (the reference's
    empty_weight 1 becomes 0)"""
    images = synthetic(2, n_images=40, edge_cases=False)       # every GT has a motion value
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    ranges = [[2.0, 3.0], [0.0, 1.0]]
    dev = host_device_eval(preds, gts, motion, ranges)
    assert np.isnan(dev[0]["ap"]).all()
    assert_same(dev, host_eval(preds, gts, motion, ranges))


def test_voc07_metric_from_compacted_curve():
    images = synthetic(3, n_images=60)
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    dev = host_device_eval(preds, gts, motion, RANGES4, use_07_metric=True)
    host = host_eval(preds, gts, motion, RANGES4, use_07_metric=True)
    for r in host:
        assert np.array_equal(dev[r]["ap"], host[r]["ap"], equal_nan=True)


def test_resize_from_ratios_equals_boxlist_resize():
    """predictions in the network's input size, resized to the image's size by the evaluator: equal to evaluating
    prediction.resize(...) (do_vid_evaluation's host path), for boxes and hence every curve"""
    images = synthetic(4, n_images=80)
    g = np.random.default_rng(4)
    for im in images:
        w, h = im["size"]
        pw, ph = int(round(w * g.uniform(0.6, 2.5))), int(round(h * g.uniform(0.6, 2.5)))
        im["pred_size"] = (pw, ph)
        im["boxes"] = im["boxes"] * torch.tensor([pw / w, ph / h, pw / w, ph / h], dtype=torch.float32)
    gts, preds = _boxlists(images)
    sizes = [im["size"] for im in images]
    motion = [im["motion"] for im in images]
    resized = [p.resize(s) for p, s in zip(preds, sizes)]
    assert_same(host_device_eval(preds, gts, motion, RANGES4, image_sizes=sizes),
                host_eval(resized, gts, motion, RANGES4))
    # and the scaled boxes themselves: x * (float)(w / w_pred), as BoxList.resize computes them
    from mega_core.data.datasets.evaluation.vid.vid_eval import _VidEvalInputs
    x = _VidEvalInputs(preds, gts, motion, RANGES4, sizes, pin=False)
    sc = x.view(x.host, 4)
    off = x.view(x.host, 3)
    boxes = x.view(x.host, 0)
    for i in range(0, len(preds), 7):
        b = boxes[off[i]:off[i + 1]] * torch.cat([sc[i], sc[i]])
        assert torch.equal(b, resized[i].bbox)


def test_stable_ties_changes_nothing_without_ties():
    images = synthetic(5, n_images=60, decimals=None, edge_cases=False)
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    ps = torch.cat([p.get_field("scores") for p in preds])
    assert ps.unique().numel() == ps.numel()
    assert_same(host_eval(preds, gts, motion, RANGES4, stable_ties=True),
                host_eval(preds, gts, motion, RANGES4, stable_ties=False))


def test_vid_eval_default_is_host():
    from mega_core.config import cfg
    assert cfg.MODEL.B200.VID_EVAL == "host"
    import inspect
    from mega_core.engine.inference import inference_no_model
    from mega_core.data.datasets.evaluation.vid import do_vid_evaluation, eval_detection_vid
    assert inspect.signature(inference_no_model).parameters["vid_eval"].default == "host"
    assert inspect.signature(do_vid_evaluation).parameters["vid_eval"].default == "host"
    assert inspect.signature(eval_detection_vid).parameters["device"].default is False


def test_unknown_switch_value_is_refused():
    import logging
    from mega_core.data.datasets.evaluation.vid import do_vid_evaluation
    with pytest.raises(ValueError):
        do_vid_evaluation(None, [], None, False, False, logging.getLogger("t"), vid_eval="gpu")


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a CUDA device")
def test_device_without_gpu_raises():
    from mega_core import _lib
    from mega_core.data.datasets.evaluation.vid import eval_detection_vid
    images = synthetic(6, n_images=4)
    gts, preds = _boxlists(images)
    with pytest.raises(_lib.MegaError):
        eval_detection_vid(preds, gts, 0.5, [[0.0, 1.0]], device=True)


def test_workspace_query_bounds():
    from mega_core import _lib
    from mega_core.b200 import ops
    assert _lib.lib.mega_vid_eval_workspace_bytes(10, 5, 3, 31, 9) == -1      # at most 8 ranges
    assert _lib.lib.mega_vid_eval_workspace_bytes(10, 5, 1 << 20, 1 << 13, 4) == -1
    with pytest.raises(_lib.MegaError):
        ops.vid_eval_workspace_bytes(10, 5, 3, 31, 0)
