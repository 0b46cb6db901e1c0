"""The evaluation loop around the hot path, with the reference's names and call contract (engine/inference.py:18-160):
`inference(cfg, model, data_loader, dataset_name, ...)` as tools/test_net.py:116-128 calls it.

Per batch the images go to the device and `model(images)` runs (the B200 engines behind the reference-named modules); the
per-rank `{image_id: BoxList}` results reach rank 0 through `utils.comm.gather_predictions` (typed tensor gathers instead
of the reference's pickled byte all-gather, :50-69) and are scored by the VID evaluator of this package. Timing is
reported the way the reference reports it (total and model-only seconds per image per device)."""
import logging
import os
import time

import torch

from ..data.datasets.evaluation.vid import vid_evaluation
from ..utils.comm import gather_predictions, get_world_size, is_main_process, synchronize
from .bbox_aug import im_detect_bbox_aug
from .seq_nms import seq_nms_predictions


class Timer(object):
    """utils/timer.py:9-46: accumulating tic / toc"""

    def __init__(self):
        self.total_time, self.calls, self._t0 = 0.0, 0, None

    def tic(self):
        self._t0 = time.time()

    def toc(self):
        dt = time.time() - self._t0
        self.total_time += dt
        self.calls += 1
        return dt


def _to_device(images, device, method):
    if method == "base":
        return images.to(device)
    if method not in ("rdn", "mega", "fgfa", "dff"):
        raise ValueError("method {} not supported yet.".format(method))
    move = lambda t: t.to(device) if hasattr(t, "to") else t                # noqa: E731
    images["cur"] = move(images["cur"])
    for key in ("ref", "ref_l", "ref_m", "ref_g"):
        if key in images:
            images[key] = [move(img) for img in images[key]]
    return images


def compute_on_dataset(model, data_loader, device, bbox_aug, method, timer=None):
    """engine/inference.py:18-47 -> {image_id: BoxList on the CPU}. bbox_aug: TEST.BBOX_AUG.ENABLED, the batches are
    BBoxAugCollator's (untransformed images) and im_detect_bbox_aug runs them; single-frame method only"""
    if bbox_aug and method != "base":
        raise NotImplementedError("TEST.BBOX_AUG.ENABLED: test-time box augmentation is defined for MODEL.VID.METHOD "
                                  "'base' only, not for '%s'" % method)
    model.eval()
    results = {}
    cpu = torch.device("cpu")
    for images, targets, image_ids in data_loader:
        with torch.no_grad():
            if timer:
                timer.tic()
            if bbox_aug:
                output = im_detect_bbox_aug(model, images, device)
            else:
                output = model(_to_device(images, device, method))
            if timer:
                if device.type != "cpu":
                    torch.cuda.synchronize()
                timer.toc()
            output = [o.to(cpu) for o in output]
        results.update({i: r for i, r in zip(image_ids, output)})
    return results


def _seconds(t):
    return time.strftime("%H:%M:%S", time.gmtime(t))


def _seq_nms_kwargs(settings):
    """MODEL.B200.SEQ_NMS (a CfgNode, or a dict with its keys ENABLED / LINK_IOU / NMS_IOU / RESCORE) -> keyword
    arguments of seq_nms_predictions, or None when absent or not enabled"""
    if settings is None:
        return None
    get = settings.get if isinstance(settings, dict) else lambda k, d=None: getattr(settings, k, d)
    if not get("ENABLED", False):
        return None
    return {"link_iou": float(get("LINK_IOU", 0.5)), "nms_iou": float(get("NMS_IOU", 0.3)),
            "rescore": str(get("RESCORE", "avg"))}


def _apply_seq_nms(predictions, dataset, kwargs, world, logger):
    """Seq-NMS over the videos of `predictions` ({image_id: BoxList}); logged like the other timings"""
    t0 = time.time()
    predictions = seq_nms_predictions(predictions, dataset, **kwargs)
    t = time.time() - t0
    logger.info("Seq-NMS time: {} ({} s / img per device, on {} devices)".format(
        _seconds(t), t * world / max(len(dataset), 1), world))
    return predictions


def inference(cfg, model, data_loader, dataset_name, iou_types=("bbox",), motion_specific=False, box_only=False,
              bbox_aug=False, device="cuda", expected_results=(), expected_results_sigma_tol=4, output_folder=None):
    """engine/inference.py:72-134; VID datasets only (`dataset` needs get_img_info / get_groundtruth /
    map_class_id_to_class_name, as data/datasets/vid.py provides)"""
    device = torch.device(device)
    world = get_world_size()
    logger = logging.getLogger("mega_core.inference")
    dataset = data_loader.dataset
    logger.info("Start evaluation on {} dataset({} images).".format(dataset_name, len(dataset)))
    total, model_only = Timer(), Timer()
    total.tic()
    predictions = compute_on_dataset(model, data_loader, device, bbox_aug, cfg.MODEL.VID.METHOD, model_only)
    synchronize()
    t = total.toc()
    logger.info("Total run time: {} ({} s / img per device, on {} devices)".format(_seconds(t), t * world / len(dataset), world))
    logger.info("Model inference time: {} ({} s / img per device, on {} devices)".format(
        _seconds(model_only.total_time), model_only.total_time * world / len(dataset), world))
    # per rank, before the gather: VIDTestDistributedSampler gives every rank whole videos
    seq = _seq_nms_kwargs(getattr(getattr(cfg.MODEL, "B200", None), "SEQ_NMS", None))
    if seq is not None:
        predictions = _apply_seq_nms(predictions, dataset, seq, world, logger)
    predictions = gather_predictions(predictions)
    if not is_main_process():
        return None
    if output_folder:
        torch.save(predictions, os.path.join(output_folder, "predictions.pth"))
    return vid_evaluation(dataset=dataset, predictions=predictions, output_folder=output_folder, box_only=box_only,
                          motion_specific=motion_specific, iou_types=iou_types, expected_results=expected_results,
                          expected_results_sigma_tol=expected_results_sigma_tol)


def inference_no_model(data_loader, iou_types=("bbox",), motion_specific=False, box_only=False, expected_results=(),
                       expected_results_sigma_tol=4, output_folder=None, seq_nms=None):
    """engine/inference.py:137-160: score the predictions.pth of an earlier run. `seq_nms`: a dict with the keys of
    MODEL.B200.SEQ_NMS (ENABLED, LINK_IOU, NMS_IOU, RESCORE), e.g. dict(cfg.MODEL.B200.SEQ_NMS), to rescore the saved
    predictions with Seq-NMS first (the file is not changed)"""
    predictions = torch.load(os.path.join(output_folder, "predictions.pth"), weights_only=False)
    seq = _seq_nms_kwargs(seq_nms)
    if seq is not None:
        by_id = _apply_seq_nms(dict(enumerate(predictions)), data_loader.dataset, seq, 1,
                               logging.getLogger("mega_core.inference"))
        predictions = [by_id[i] for i in range(len(predictions))]
    return vid_evaluation(dataset=data_loader.dataset, predictions=predictions, output_folder=output_folder,
                          box_only=box_only, motion_specific=motion_specific)
