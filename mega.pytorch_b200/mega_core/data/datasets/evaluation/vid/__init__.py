from .vid_eval import (calc_detection_vid_ap, calc_detection_vid_prec_rec, do_vid_evaluation,  # noqa: F401
                       eval_detection_vid, eval_proposals_vid)


def vid_evaluation(dataset, predictions, output_folder, box_only, motion_specific, **_):
    """data/datasets/evaluation/vid/__init__.py:6-16"""
    import logging
    logger = logging.getLogger("mega_core.inference")
    logger.info("performing vid evaluation, ignored iou_types.")
    return do_vid_evaluation(dataset=dataset, predictions=predictions, output_folder=output_folder, box_only=box_only,
                             motion_specific=motion_specific, logger=logger)
