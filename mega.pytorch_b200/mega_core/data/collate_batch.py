"""BatchCollator (data/collate_batch.py:5-38): dataset items -> (images, targets, image ids). Video methods carry one
image per GPU; every frame becomes an ImageList, the scalar fields pass through."""
from ..structures.image_list import to_image_list

_FRAME_LISTS = ("ref", "ref_l", "ref_m", "ref_g")


class BatchCollator(object):
    def __init__(self, size_divisible=0, method="base", is_train=True):
        self.size_divisible, self.method, self.is_train = size_divisible, method, is_train

    def __call__(self, batch):
        items, targets, ids = zip(*batch)
        if self.method == "base":
            return to_image_list(items, self.size_divisible), targets, ids
        if self.method not in ("rdn", "mega", "fgfa", "dff"):
            raise NotImplementedError("method {} not supported yet.".format(self.method))
        assert len(items) == 1, ("Currently 1 gpu could only hold 1 image. Please modify SOLVER.IMS_PER_BATCH and "
                                 "TEST.IMS_PER_BATCH to ensure this.")
        images = {}
        for key, value in items[0].items():
            if key == "cur":
                images[key] = to_image_list((value,), self.size_divisible)
            elif key in _FRAME_LISTS:
                images[key] = [to_image_list((img,), self.size_divisible) for img in value]
            else:
                images[key] = value
        return images, targets, ids


class BBoxAugCollator(object):
    """data/collate_batch.py:42-50: with TEST.BBOX_AUG.ENABLED the dataset yields untransformed images; the batch stays
    (images, targets, image ids) tuples and mega_core.engine.bbox_aug.im_detect_bbox_aug transforms every image itself"""

    def __call__(self, batch):
        return list(zip(*batch))
