"""Test-time box augmentation (TEST.BBOX_AUG) with the reference's name and call contract (engine/bbox_aug.py:11-68):
`im_detect_bbox_aug(model, images, device)` -> list[BoxList] (fields `scores`, `labels`) in the identity pass's size.

Passes, in the reference's order: identity at (INPUT.MIN_SIZE_TEST, INPUT.MAX_SIZE_TEST); its horizontal flip if H_FLIP;
for each of SCALES, (scale, BBOX_AUG.MAX_SIZE), then its flip if SCALE_H_FLIP. Each pass runs the device transform
(Resize -> optional flip -> ToTensor -> Normalize, bit-identical to the PIL pipeline) and the whole single-frame
detector; its raw post-processor output is mapped back to the identity frame on the device, and one merge applies the
post-processor's filter_results to all passes (BaseEngine.forward_bbox_aug, csrc/bbox_aug.cu). Single-frame method
("base") only: the reference's video datasets yield dicts its transforms cannot take, so it defines TTA for "base" only.
"""
import torch

from ..data.transforms.transforms import DeviceTestTransform, get_size


class AugPass(object):
    """one pass of the plan: the Resize arguments, the flip, the resized (w, h) and the ratios identity size / pass size
    (Python floats, as BoxList.resize computes them; `same_ratio` is its single-ratio branch)"""

    def __init__(self, min_size, max_size, hflip, size, identity_size):
        self.min_size, self.max_size, self.hflip, self.size = min_size, max_size, bool(hflip), size
        self.ratio_w = float(identity_size[0]) / float(size[0])
        self.ratio_h = float(identity_size[1]) / float(size[1])
        self.same_ratio = self.ratio_w == self.ratio_h

    def __repr__(self):
        return "AugPass(min_size=%d, max_size=%s, hflip=%s, size=%s)" % (self.min_size, self.max_size, self.hflip,
                                                                          self.size)


def aug_plan(image_size, min_size_test, max_size_test, h_flip, scales, max_size, scale_h_flip):
    """image_size (w, h) of the source image -> list[AugPass] in the reference's order"""
    settings = [(min_size_test, max_size_test, False)]
    if h_flip:
        settings.append((min_size_test, max_size_test, True))
    for s in scales:
        settings.append((s, max_size, False))
        if scale_h_flip:
            settings.append((s, max_size, True))
    sizes = [get_size(image_size, int(mn), mx)[::-1] for mn, mx, _ in settings]     # (w, h)
    return [AugPass(int(mn), mx, f, sz, sizes[0]) for (mn, mx, f), sz in zip(settings, sizes)]


def plan_from_cfg(cfg, image_size):
    aug = cfg.TEST.BBOX_AUG
    min_size = cfg.INPUT.MIN_SIZE_TEST
    if isinstance(min_size, (list, tuple)):
        assert len(min_size) == 1, "test-time augmentation: a single INPUT.MIN_SIZE_TEST"
        min_size = min_size[0]
    return aug_plan(image_size, min_size, cfg.INPUT.MAX_SIZE_TEST, aug.H_FLIP, tuple(aug.SCALES), aug.MAX_SIZE,
                    aug.SCALE_H_FLIP)


def _image_size(image):
    """(w, h) of a PIL image, a uint8 [H, W, 3] array / tensor or a planar uint8 [3, H, W] tensor"""
    if not torch.is_tensor(image) and hasattr(image, "convert"):          # PIL.Image
        return tuple(image.size)
    shape = tuple(image.shape)
    if len(shape) == 3 and shape[2] == 3:
        return shape[1], shape[0]
    return shape[2], shape[1]


_TRANSFORMS = {}


def _transform(cfg, p, device):
    key = (p.min_size, p.max_size, p.hflip, tuple(cfg.INPUT.PIXEL_MEAN), tuple(cfg.INPUT.PIXEL_STD),
           bool(cfg.INPUT.TO_BGR255), str(device))
    t = _TRANSFORMS.get(key)
    if t is None:
        t = _TRANSFORMS[key] = DeviceTestTransform(p.min_size, p.max_size, cfg.INPUT.PIXEL_MEAN, cfg.INPUT.PIXEL_STD,
                                                   cfg.INPUT.TO_BGR255, device=device, hflip=p.hflip)
    return t


def im_detect_bbox_aug(model, images, device, trace=None):
    """engine/bbox_aug.py:11-68. model: the single-frame detector (MODEL.VID.METHOD "base"); images: PIL images or
    uint8 RGB arrays / tensors (what DeviceTestTransform accepts). Settings are read from mega_core.config.cfg, as the
    reference reads them. trace: optional list, gets per image the engine's per-pass (proposals, count, predictor rows)"""
    from ..config import cfg
    from ..modeling.detector.generalized_rcnn import GeneralizedRCNN
    if not isinstance(model, GeneralizedRCNN):
        raise NotImplementedError("TEST.BBOX_AUG.ENABLED: test-time augmentation is defined for the single-frame method "
                                  "(MODEL.VID.METHOD 'base') only, not for %s" % type(model).__name__)
    device = torch.device(device)
    eng = model.engine
    results = []
    with torch.no_grad():
        for image in images:
            plan = plan_from_cfg(cfg, _image_size(image))
            passes = ((_transform(cfg, p, device)(image)[0][None], p.size[0], p.size[1], p.hflip) for p in plan)
            im_w, im_h = plan[0].size
            t = [] if trace is not None else None
            det = eng.forward_bbox_aug(passes, len(plan), im_w, im_h, trace=t)
            if trace is not None:
                trace.append(t)
            results.append(model._to_boxlist(det, im_w, im_h))
    return results
