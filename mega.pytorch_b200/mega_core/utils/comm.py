"""Multi-process helpers with the reference's names (utils/comm.py:13-117) plus the packed prediction hand-off of
SURVEY.md section 8f row 2.

The reference moves the per-rank `{image_id: BoxList}` dicts to rank 0 by pickling them into byte tensors
(`all_gather`, comm.py:47-87; `_accumulate_predictions_from_multiple_gpus`, engine/inference.py:50-69): every box goes
through the pickler twice and through a padded byte all-gather. `gather_predictions` sends the same information as five
flat tensors (ids, sizes, counts, boxes | scores, labels) with two size exchanges and padded `all_gather`s of typed
tensors -- no pickling, works with NCCL (device tensors) and gloo (CPU tensors) alike -- and returns the reference's
result: on rank 0 the list of BoxLists ordered by image id, None elsewhere. The proposals of an MODEL.RPN_ONLY run
(BoxLists whose only field is `objectness`) travel the same way as four flat tensors (ids, sizes, counts, boxes |
objectness)."""
import logging
import pickle

import torch
import torch.distributed as dist

from ..structures.bounding_box import BoxList


def get_world_size():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def get_rank():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def is_main_process():
    return get_rank() == 0


def synchronize():
    if get_world_size() > 1:
        dist.barrier()


def _comm_device():
    return torch.device("cuda") if dist.get_backend() == "nccl" else torch.device("cpu")


def _gather_var(t, dev):
    """all-gather of 1-D / 2-D tensors whose first dimension differs per rank -> list of per-rank tensors"""
    world = get_world_size()
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=dev)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n)
    sizes = [int(s.item()) for s in sizes]
    pad = torch.zeros((max(sizes),) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
    pad[:t.shape[0]] = t.to(dev)
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return [p[:s].cpu() for p, s in zip(parts, sizes)]


def all_gather(data):
    """arbitrary picklable data from every rank (comm.py:47-87); kept for callers that gather small objects"""
    if get_world_size() == 1:
        return [data]
    dev = _comm_device()
    buf = torch.frombuffer(bytearray(pickle.dumps(data)), dtype=torch.uint8)
    return [pickle.loads(p.numpy().tobytes()) for p in _gather_var(buf, dev)]


def _objectness_only(predictions):
    """True when the predictions are proposals (field `objectness`, no `scores`) on any rank"""
    b = next(iter(predictions.values()), None)
    flag = int(b is not None and b.has_field("objectness") and not b.has_field("scores"))
    if get_world_size() > 1:
        t = torch.tensor([flag], dtype=torch.int64, device=_comm_device())
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        flag = int(t.item())
    return bool(flag)


def _gather_proposals(predictions):
    ids = sorted(predictions.keys())
    boxlists = [predictions[i].convert("xyxy") for i in ids]
    meta = torch.tensor([[i, b.size[0], b.size[1], len(b)] for i, b in zip(ids, boxlists)], dtype=torch.int64).reshape(-1, 4)
    floats = torch.cat([torch.cat([b.bbox.float().cpu().reshape(-1, 4),
                                   b.get_field("objectness").float().cpu().reshape(-1, 1)], 1)
                        for b in boxlists]) if boxlists else torch.zeros(0, 5)
    if get_world_size() > 1:
        dev = _comm_device()
        metas, floatss = _gather_var(meta, dev), _gather_var(floats, dev)
    else:
        metas, floatss = [meta], [floats]
    if not is_main_process():
        return None
    merged = {}
    for m, f in zip(metas, floatss):
        off = 0
        for image_id, w, h, n in m.tolist():
            b = BoxList(f[off:off + n, :4].clone(), (w, h), mode="xyxy")
            b.add_field("objectness", f[off:off + n, 4].clone())
            merged[image_id] = b
            off += n
    return [merged[i] for i in sorted(merged.keys())]


def gather_predictions(predictions):
    """{image_id: BoxList with `scores`, `labels`} per rank -> on rank 0 the list of BoxLists ordered by image id (what
    engine/inference.py:50-69 returns), None on the other ranks. BoxLists with the single field `objectness` (the
    proposals of an RPN-only model) are gathered as such."""
    if _objectness_only(predictions):
        return _gather_proposals(predictions)
    ids = sorted(predictions.keys())
    boxlists = [predictions[i].convert("xyxy") for i in ids]
    meta = torch.tensor([[i, b.size[0], b.size[1], len(b)] for i, b in zip(ids, boxlists)], dtype=torch.int64).reshape(-1, 4)
    floats = torch.cat([torch.cat([b.bbox.float().cpu().reshape(-1, 4), b.get_field("scores").float().cpu().reshape(-1, 1)], 1)
                        for b in boxlists]) if boxlists else torch.zeros(0, 5)
    labels = torch.cat([b.get_field("labels").long().cpu().reshape(-1) for b in boxlists]) if boxlists else \
        torch.zeros(0, dtype=torch.int64)
    if get_world_size() > 1:
        dev = _comm_device()
        metas, floatss, labelss = _gather_var(meta, dev), _gather_var(floats, dev), _gather_var(labels, dev)
    else:
        metas, floatss, labelss = [meta], [floats], [labels]
    if not is_main_process():
        return None
    merged = {}
    for m, f, l in zip(metas, floatss, labelss):
        off = 0
        for image_id, w, h, n in m.tolist():
            b = BoxList(f[off:off + n, :4].clone(), (w, h), mode="xyxy")
            b.add_field("scores", f[off:off + n, 4].clone())
            b.add_field("labels", l[off:off + n].clone())
            merged[image_id] = b                      # later ranks overwrite duplicates, like dict.update in the reference
            off += n
    image_ids = sorted(merged.keys())
    if image_ids and len(image_ids) != image_ids[-1] + 1:
        logging.getLogger("mega_core.inference").warning(
            "Number of images that were gathered from multiple processes is not a contiguous set. "
            "Some images might be missing from the evaluation")
    return [merged[i] for i in image_ids]
