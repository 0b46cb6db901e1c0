"""make_data_loader (data/build.py:18-192), test side: one DataLoader per dataset of cfg.DATASETS.TEST, one image per
GPU for the video methods, whole videos per rank when distributed."""
import torch.utils.data

from . import datasets as D
from .collate_batch import BatchCollator, BBoxAugCollator
from .samplers import VIDTestDistributedSampler
from .transforms import build_transforms
from ..utils.comm import get_world_size


def build_dataset(dataset_list, transforms, dataset_catalog, is_train=False, method="base"):
    if not isinstance(dataset_list, (list, tuple)):
        raise RuntimeError("dataset_list should be a list of strings, got {}".format(dataset_list))
    out = []
    for name in dataset_list:
        data = dataset_catalog.get(name, method)
        out.append(getattr(D, data["factory"])(transforms=transforms, is_train=is_train, **data["args"]))
    return out


def make_data_loader(cfg, is_train=False, is_distributed=False, start_iter=0, is_for_period=False, transforms=None,
                     dataset_catalog=None):
    """`transforms`: defaults to the device transform of this package (build_transforms(cfg, False): frames reach the
    model already on the GPU); pass the reference's CPU transform object to keep decoding + resizing on the workers.
    `dataset_catalog`: defaults to mega_core.config.paths_catalog.DatasetCatalog (cfg.PATHS_CATALOG in the reference)."""
    if is_train or is_for_period:
        raise NotImplementedError("mega_core.data (B200 build): test-time loaders only")
    world = get_world_size()
    per_batch = cfg.TEST.IMS_PER_BATCH
    assert per_batch % world == 0, \
        "TEST.IMS_PER_BATCH ({}) must be divisible by the number of GPUs ({}) used.".format(per_batch, world)
    if dataset_catalog is None:
        from ..config.paths_catalog import DatasetCatalog as dataset_catalog
    method = cfg.MODEL.VID.METHOD
    # TEST.BBOX_AUG.ENABLED (data/build.py:165, :175-176): no dataset transform, im_detect_bbox_aug transforms each pass
    bbox_aug = cfg.TEST.BBOX_AUG.ENABLED
    device_side = transforms is None and not bbox_aug
    if bbox_aug:
        transforms = None
    elif device_side:
        transforms = build_transforms(cfg, is_train=False)
    loaders = []
    for dataset in build_dataset(cfg.DATASETS.TEST, transforms, dataset_catalog, False, method):
        if is_distributed and method == "base":
            # make_data_sampler (data/build.py:62-77): the single-frame baseline shards IMAGES (the base VIDDataset has no
            # video index; samplers.DistributedSampler there == torch's, padding the tail so every rank gets equally many)
            from torch.utils.data.distributed import DistributedSampler
            from ..utils.comm import get_rank
            sampler = DistributedSampler(dataset, num_replicas=world, rank=get_rank(), shuffle=False)
        elif is_distributed:
            if method not in ("rdn", "mega", "fgfa", "dff"):
                raise NotImplementedError("Method {} is not implemented.".format(method))
            sampler = VIDTestDistributedSampler(dataset, shuffle=False)
        else:
            sampler = torch.utils.data.sampler.SequentialSampler(dataset)
        batches = torch.utils.data.sampler.BatchSampler(sampler, per_batch // world, drop_last=False)
        loaders.append(torch.utils.data.DataLoader(
            dataset, batch_sampler=batches,
            collate_fn=BBoxAugCollator() if bbox_aug else BatchCollator(cfg.DATALOADER.SIZE_DIVISIBILITY, method, False),
            num_workers=0 if device_side else cfg.DATALOADER.NUM_WORKERS))   # CUDA tensors cannot cross worker processes
    return loaders
