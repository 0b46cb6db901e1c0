"""The device VID evaluator (csrc/vid_eval.cu, MODEL.B200.VID_EVAL = "device") on the GPU: bit for bit equal to the host
evaluator with stable_ties=True -- n_pos, prec, rec and AP of every class and motion range -- on the golden cases, on a
seeded VID-shaped set of 20 k frames with the four ranges, and on the edge cases (images without detections or GT,
classes only in GT, all GT ignored, empty_weight 1 -> 0, single-detection classes, predictions resized in the kernel);
do_vid_evaluation / inference_no_model with vid_eval="device" write the host path's result.txt."""
import logging
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_vid_eval_device_cpu import RANGES4, _boxlists, assert_same, host_eval, synthetic  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def device_eval(preds, gts, motion, ranges, image_sizes=None, use_07_metric=False):
    from mega_core.data.datasets.evaluation.vid import eval_detection_vid
    return eval_detection_vid(preds, gts, 0.5, ranges, motion is not None, use_07_metric, motion_ious=motion,
                              device=True, return_curves=True, image_sizes=image_sizes)


@pytest.mark.parametrize("case", [0, 1])
def test_golden_cases(case):
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "vid_eval.pt"), weights_only=False)[case]
    gts, preds = _boxlists(gold["images"])
    motion = [im["motion"] for im in gold["images"]]
    assert_same(device_eval(preds, gts, None, [[0.0, 1.0]]), host_eval(preds, gts, None, [[0.0, 1.0]]))
    dev = device_eval(preds, gts, motion, RANGES4)
    assert_same(dev, host_eval(preds, gts, motion, RANGES4))
    # against the unmodified reference (numpy's default sort on its host): the difference tie order alone makes
    ref = gold["reference"]
    worst = 0.0
    for r, name in enumerate(("all", "fast", "medium", "slow")):
        a, b = dev[r]["ap"], ref[name]["ap"]
        assert np.array_equal(np.isnan(a), np.isnan(b))
        worst = max(worst, float(np.nanmax(np.abs(a - b))))
    print("vid_eval golden case %d: max |dAP| vs the reference from tie order = %.3g" % (case, worst))
    assert worst < 0.05


def test_vid_shaped_20k_frames_four_ranges():
    """555-video-like structure at 20 k frames, 60 detections per frame, 30 classes, 1-3 GT with motion IoUs"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_vid_eval
    preds, gt_src, sizes, motion = bench_vid_eval.workload(20000, 64, 60, seed=3)
    gts = [bench_vid_eval.make_gt(e) for e in gt_src]
    # ties: scores on a 1e-3 grid
    for p in preds:
        p.add_field("scores", (p.get_field("scores") * 1000).round() / 1000)
    resized = [p.resize(s) for p, s in zip(preds, sizes)]
    dev = device_eval(preds, gts, motion, RANGES4, image_sizes=sizes)
    assert_same(dev, host_eval(resized, gts, motion, RANGES4))


def test_edge_cases():
    images = synthetic(11, n_images=300)
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    assert_same(device_eval(preds, gts, motion, RANGES4), host_eval(preds, gts, motion, RANGES4))
    assert_same(device_eval(preds, gts, None, [[0.0, 1.0]]), host_eval(preds, gts, None, [[0.0, 1.0]]))
    images = synthetic(12, n_images=50, edge_cases=False)
    gts, preds = _boxlists(images)
    motion = [im["motion"] for im in images]
    ranges = [[2.0, 3.0], [0.0, 1.0]]                   # all GT ignored; empty_weight 1 -> 0
    dev = device_eval(preds, gts, motion, ranges)
    assert np.isnan(dev[0]["ap"]).all()
    assert_same(dev, host_eval(preds, gts, motion, ranges))
    dev07 = device_eval(preds, gts, motion, RANGES4, use_07_metric=True)
    host07 = host_eval(preds, gts, motion, RANGES4, use_07_metric=True)
    for r in host07:
        assert np.array_equal(dev07[r]["ap"], host07[r]["ap"], equal_nan=True)


def test_resize_in_kernel():
    images = synthetic(13, n_images=120)
    g = np.random.default_rng(13)
    for im in images:
        w, h = im["size"]
        pw, ph = int(round(w * g.uniform(0.6, 2.5))), int(round(h * g.uniform(0.6, 2.5)))
        im["pred_size"] = (pw, ph)
        im["boxes"] = im["boxes"] * torch.tensor([pw / w, ph / h, pw / w, ph / h], dtype=torch.float32)
    gts, preds = _boxlists(images)
    sizes = [im["size"] for im in images]
    motion = [im["motion"] for im in images]
    assert_same(device_eval(preds, gts, motion, RANGES4, image_sizes=sizes),
                host_eval([p.resize(s) for p, s in zip(preds, sizes)], gts, motion, RANGES4))


class _Dataset(object):
    def __init__(self, images):
        self.images = images
        self.gts, _ = _boxlists(images)

    def __len__(self):
        return len(self.images)

    def get_img_info(self, i):
        w, h = self.images[i]["size"]
        return {"width": w, "height": h}

    def get_groundtruth(self, i):
        return self.gts[i]

    def map_class_id_to_class_name(self, i):
        return "class_%d" % i


def _tie_free_run(seed):
    images = synthetic(seed, n_images=150, decimals=None)
    for im in images:                                   # network-size predictions: resized by the evaluator
        w, h = im["size"]
        im["pred_size"] = (2 * w, 2 * h)
        im["boxes"] = im["boxes"] * 2
    _, preds = _boxlists(images)
    return _Dataset(images), preds


def test_do_vid_evaluation_device_writes_host_result(tmp_path):
    from mega_core.data.datasets.evaluation.vid import do_vid_evaluation
    ds, preds = _tie_free_run(21)
    log = logging.getLogger("test_vid_eval_gpu")
    texts = {}
    for mode in ("host", "device"):
        out = tmp_path / mode
        out.mkdir()
        do_vid_evaluation(ds, preds, str(out), False, False, log, vid_eval=mode)
        texts[mode] = (out / "result.txt").read_text()
    assert texts["host"] == texts["device"]


def test_inference_no_model_device(tmp_path):
    from mega_core.engine.inference import inference_no_model
    ds, preds = _tie_free_run(22)
    torch.save(preds, str(tmp_path / "predictions.pth"))

    class _Loader(object):
        dataset = ds

    res_dev = inference_no_model(_Loader(), output_folder=str(tmp_path), vid_eval="device")
    text_dev = (tmp_path / "result.txt").read_text()
    res_host = inference_no_model(_Loader(), output_folder=str(tmp_path))
    assert (tmp_path / "result.txt").read_text() == text_dev
    assert np.array_equal(res_dev[0]["ap"], res_host[0]["ap"], equal_nan=True)
