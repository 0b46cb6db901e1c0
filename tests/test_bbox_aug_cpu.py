"""CPU checks of test-time box augmentation (TEST.BBOX_AUG; mega_core.engine.bbox_aug, csrc/bbox_aug.cuh):
  1. the pass plan equals the passes the reference's im_detect_bbox_aug makes (recorded in the fixture from its own
     control flow) over several source sizes, including MAX_SIZE hits and unequal x / y ratios;
  2. the kernels' mapping and merge bodies, built by g++ (tests/native/bbox_aug_host.cpp) and fed the reference's raw
     per-pass BoxLists, reproduce the reference's merged detections bit for bit (which also shows that BoxList.resize
     computes x * fl32(ratio));
  3. an 18 x 300 x 31 case with a class that keeps more than DETECTIONS_PER_IMG boxes and ties at the cap equals a
     PyTorch restatement of filter_results without any early stop;
  4. the data path: make_data_loader with BBOX_AUG.ENABLED, compute_on_dataset's dispatch;
  5. the C ABI: symbols, and capacity checks that need no device."""
import ctypes
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden", "bbox_aug_r50_240x400.pt")
_host = None


def host_lib():
    """g++ build of csrc/bbox_aug.cuh, cached in the temp directory under the digest of its sources"""
    global _host
    if _host is None:
        src = os.path.join(ROOT, "tests", "native", "bbox_aug_host.cpp")
        deps = [src] + [os.path.join(ROOT, "mega.pytorch_b200", "csrc", n) for n in
                        ("bbox_aug.cuh", "box_head.cuh", "iou.cuh")] + [os.path.join(ROOT, "include", "mega_b200.h")]
        digest = hashlib.sha256(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
        so_path = os.path.join(tempfile.gettempdir(), "mega_bbox_aug_host_%s_%d.so" % (digest, os.getuid()))
        if not os.path.exists(so_path):
            tmp = so_path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-I",
                                   os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                                   "-o", tmp, src])
            os.replace(tmp, so_path)
        _host = ctypes.CDLL(so_path)
        from mega_core import _lib
        for name in ("mega_bbox_aug_workspace_bytes", "mega_bbox_aug_collect", "mega_bbox_aug_merge"):
            fn, real = getattr(_host, name), getattr(_lib.lib, name)
            fn.argtypes, fn.restype = real.argtypes, real.restype
        _vp, _i, _d, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_float
        _host.bbox_aug_stage_raw_host.argtypes = [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _d, _d, _f, _vp]
        _host.bbox_aug_stage_raw_host.restype = _i
    return _host


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def host_merge(num_passes, r_max, ncls, nms, max_det, ws):
    lib = host_lib()
    cap = (ncls - 1) * num_passes * r_max
    ob, os_, ol, oc = torch.zeros(cap, 4), torch.zeros(cap), torch.zeros(cap, dtype=torch.int64), torch.zeros(1, dtype=torch.int32)
    assert lib.mega_bbox_aug_merge(num_passes, r_max, ncls, nms, max_det, _p(ws), ws.numel(), _p(ob), _p(os_), _p(ol),
                                   cap, _p(oc), None) == 0
    n = int(oc.item())
    return ob[:n], os_[:n], ol[:n]


def _gold():
    return torch.load(GOLD, weights_only=False)


def test_fixture_image_regenerates_from_its_seed():
    from mega_core.b200 import synth
    g = _gold()
    image = synth.synthetic_image_u8(*g["image_hw"], g["image_seed"])
    assert image.dtype == torch.uint8 and tuple(image.shape) == tuple(g["image_hw"]) + (3,)
    assert hashlib.sha256(image.numpy().tobytes()).hexdigest() == g["image_sha256"]


# ---------------------------------------------------------------- 1. plan
@pytest.mark.parametrize("case", range(6))
def test_plan_equals_the_reference_passes(case):
    from mega_core.engine.bbox_aug import aug_plan
    ref = _gold()["plans"][case]
    plan = aug_plan(ref["image_size"], ref["min_size_test"], ref["max_size_test"], ref["h_flip"], ref["scales"],
                    ref["max_size"], ref["scale_h_flip"])
    got = [{"min_size": p.min_size, "max_size": p.max_size, "hflip": p.hflip, "size": tuple(p.size)} for p in plan]
    assert got == [dict(r, size=tuple(r["size"])) for r in ref["passes"]]
    w0, h0 = ref["passes"][0]["size"]
    for p in plan:                                 # BoxList.resize: float(s) / float(s_orig), Python doubles
        assert p.ratio_w == float(w0) / float(p.size[0]) and p.ratio_h == float(h0) / float(p.size[1])
        assert p.same_ratio == (p.ratio_w == p.ratio_h)


def test_plan_cases_cover_both_ratio_branches_and_max_size():
    from mega_core.engine.bbox_aug import aug_plan
    same, differ, capped = 0, 0, 0
    for ref in _gold()["plans"]:
        plan = aug_plan(ref["image_size"], ref["min_size_test"], ref["max_size_test"], ref["h_flip"], ref["scales"],
                        ref["max_size"], ref["scale_h_flip"])
        for p in plan[1:]:
            same += p.same_ratio
            differ += not p.same_ratio
            capped += min(p.size) < p.min_size
    assert same and differ and capped


# ---------------------------------------------------------------- 2. mapping + merge vs the reference, bit for bit
def test_host_mapping_and_merge_reproduce_the_reference_detections():
    g = _gold()
    lib = host_lib()
    ncls, passes = g["num_classes"], g["passes"]
    A, R = len(passes), max(p["proposals"].shape[0] for p in passes)
    ws = torch.zeros(lib.mega_bbox_aug_workspace_bytes(A, R, ncls), dtype=torch.uint8)
    w0, h0 = g["size"]
    assert tuple(passes[0]["size"]) == (w0, h0)
    for a, p in enumerate(passes):
        w, h = p["size"]
        k = p["proposals"].shape[0]
        boxes, scores = p["raw_boxes"].contiguous(), p["raw_scores"].contiguous()
        assert lib.bbox_aug_stage_raw_host(_p(boxes), _p(scores), k, R, ncls, a, A, w, int(p["hflip"]),
                                           float(w0) / float(w), float(h0) / float(h), g["score_thresh"], _p(ws)) == 0
    b, s, l = host_merge(A, R, ncls, g["nms"], g["detections_per_img"], ws)
    rb, rs, rl = g["boxes"], g["scores"], g["labels"]
    assert b.shape[0] == rb.shape[0] > 0
    assert torch.equal(l, torch.sort(l).values)                     # class-major
    assert torch.equal(torch.sort(l).values, torch.sort(rl).values)

    def rows(bb, ss, ll):
        return sorted(zip(ll.tolist(), bb.view(torch.int32).tolist(), ss.view(torch.int32).tolist()))
    assert rows(b, s, l) == rows(rb, rs, rl)                        # the same (label, box, score) multiset, bitwise


def test_host_collect_follows_the_reference_post_processor():
    """collect on the reference's logits / deltas / proposals vs its raw BoxList (mapped): expf of libm vs torch's may
    differ in the last bit, so boxes to 1e-4 px and scores to 2 ulp-ish"""
    g = _gold()
    lib = host_lib()
    ncls, passes = g["num_classes"], g["passes"]
    A, R = len(passes), g["post_nms_top_n"]
    ws_c = torch.zeros(lib.mega_bbox_aug_workspace_bytes(A, R, ncls), dtype=torch.uint8)
    ws_r = torch.zeros_like(ws_c)
    w0, h0 = g["size"]
    for a, p in enumerate(passes):
        w, h = p["size"]
        k = p["proposals"].shape[0]
        lg, dl, pr = (p[n].contiguous().float() for n in ("class_logits", "box_regression", "proposals"))
        cnt = torch.tensor([k], dtype=torch.int32)
        wx, wy, ww, wh = g["bbox_reg_weights"]
        assert lib.mega_bbox_aug_collect(_p(lg), lg.shape[1], _p(dl), dl.shape[1], _p(pr), _p(cnt), R, ncls, a, A, w, h,
                                         int(p["hflip"]), float(w0) / w, float(h0) / h, g["score_thresh"], wx, wy, ww,
                                         wh, _p(ws_c), ws_c.numel(), None) == 0
        boxes, scores = p["raw_boxes"].contiguous(), p["raw_scores"].contiguous()
        lib.bbox_aug_stage_raw_host(_p(boxes), _p(scores), k, R, ncls, a, A, w, int(p["hflip"]), float(w0) / w,
                                    float(h0) / h, g["score_thresh"], _p(ws_r))
    slots = A * R * ncls
    nb = (16 * slots + 255) // 256 * 256
    bc, br = ws_c[:16 * slots].view(torch.float32), ws_r[:16 * slots].view(torch.float32)
    sc, sr = ws_c[nb:nb + 4 * slots].view(torch.float32), ws_r[nb:nb + 4 * slots].view(torch.float32)
    assert (bc - br).abs().max().item() < 1e-3
    assert (sc - sr).abs().max().item() < 1e-6


# ---------------------------------------------------------------- 3. capacity: 18 x 300 x 31, exact stop, ties at the cap
def _synthetic_staging(seed, A=18, R=300, ncls=31, thresh=0.05):
    g = torch.Generator().manual_seed(seed)
    rows = A * R
    boxes = torch.zeros(ncls, rows, 4)
    scores = torch.zeros(ncls, rows)
    xy = torch.rand(ncls, rows, 2, generator=g) * 600
    wh = torch.rand(ncls, rows, 2, generator=g) * 120 + 2
    boxes[..., :2], boxes[..., 2:] = xy, xy + wh
    scores[:] = torch.rand(ncls, rows, generator=g) * 0.12           # most rows below the threshold
    # class 1: 2000 disjoint small boxes on a grid with scores quantised to a few levels -> keeps > DETECTIONS_PER_IMG,
    # with many ties at the cap
    i = torch.arange(2000)
    gx, gy = (i % 50).float() * 12, (i // 50).float() * 12
    boxes[1, :2000] = torch.stack([gx, gy, gx + 8, gy + 8], 1)
    scores[1, :2000] = 0.5 + torch.randint(0, 4, (2000,), generator=g).float() / 8
    # class 2: a dense pile (heavy suppression) with a few ties
    boxes[2, :3000] = torch.tensor([100., 100., 200., 200.]) + torch.rand(3000, 4, generator=g) * 20
    scores[2, :3000] = 0.3 + torch.randint(0, 50, (3000,), generator=g).float() / 100
    cand = (scores > thresh).to(torch.uint8)
    cand[0] = 0
    return boxes, scores, cand


def _stage(boxes, scores, cand):
    ncls, rows = scores.shape
    slots = ncls * rows
    nb, ns = (16 * slots + 255) // 256 * 256, (4 * slots + 255) // 256 * 256
    ws = torch.zeros(nb + ns + (slots + 255) // 256 * 256, dtype=torch.uint8)
    ws[:16 * slots].view(torch.float32).copy_(boxes.reshape(-1))
    ws[nb:nb + 4 * slots].view(torch.float32).copy_(scores.reshape(-1))
    ws[nb + ns:nb + ns + slots].copy_(cand.reshape(-1))
    return ws


def _iou_gt(b, others, thresh):
    """IoU(b, others) > thresh, "+1" convention, fp32 ops in the reference's order (nms.cu:16-19)"""
    left, right = torch.maximum(b[0], others[:, 0]), torch.minimum(b[2], others[:, 2])
    top, bottom = torch.maximum(b[1], others[:, 1]), torch.minimum(b[3], others[:, 3])
    w = (right - left + 1).clamp(min=0)
    h = (bottom - top + 1).clamp(min=0)
    inter = w * h
    sa = (b[2] - b[0] + 1) * (b[3] - b[1] + 1)
    sb = (others[:, 2] - others[:, 0] + 1) * (others[:, 3] - others[:, 1] + 1)
    return inter / (sa + sb - inter) > thresh


def filter_results_restated(boxes, scores, cand, nms, max_det):
    """box_head/inference.py:108-149 over staged rows: per class NMS in (score desc, row asc) order, concatenation
    class-major in row order, kthvalue cap with ties kept. No early stop."""
    ncls, rows = scores.shape
    out_l, out_b, out_s = [], [], []
    for j in range(1, ncls):
        idx = torch.nonzero(cand[j]).squeeze(1)
        order = sorted(idx.tolist(), key=lambda r: (-scores[j, r].item(), r))
        keep = []
        kb = boxes[j, order]
        removed = torch.zeros(len(order), dtype=torch.bool)
        for q in range(len(order)):
            if removed[q]:
                continue
            keep.append(order[q])
            removed[q + 1:] |= _iou_gt(kb[q], kb[q + 1:], nms)
        keep.sort()
        out_l += [j] * len(keep)
        out_b.append(boxes[j, keep])
        out_s.append(scores[j, keep])
    b, s, l = torch.cat(out_b), torch.cat(out_s), torch.tensor(out_l, dtype=torch.int64)
    if b.shape[0] > max_det > 0:
        thr, _ = torch.kthvalue(s, b.shape[0] - max_det + 1)
        k = s >= thr.item()
        b, s, l = b[k], s[k], l[k]
    return b, s, l


@pytest.mark.parametrize("max_det", [300, 0])
def test_host_merge_at_capacity_with_exact_stop_and_ties(max_det):
    boxes, scores, cand = _synthetic_staging(7)
    A, R, ncls = 18, 300, 31
    ws = _stage(boxes, scores, cand)
    b, s, l = host_merge(A, R, ncls, 0.5, max_det, ws)
    rb, rs, rl = filter_results_restated(boxes, scores, cand, 0.5, max_det)
    assert torch.equal(l, rl) and torch.equal(b, rb) and torch.equal(s, rs)
    if max_det:
        kept1 = int((l == 1).sum())
        assert kept1 > max_det                       # class 1 alone passes the cap: the sweep stops early there
        thr = s.min().item()
        assert int((s == thr).sum()) > 1             # ties at the cap are kept


# ---------------------------------------------------------------- 4. data path
def test_make_data_loader_with_bbox_aug_yields_untransformed_batches(tmp_path):
    from PIL import Image
    from test_datasets_cpu import make_tree
    from mega_core.config import cfg
    from mega_core.config.paths_catalog import DatasetCatalog
    from mega_core.data import make_data_loader
    from mega_core.data.collate_batch import BBoxAugCollator
    n = make_tree(str(tmp_path))

    class Catalog(DatasetCatalog):
        DATA_DIR = str(tmp_path)

    c = cfg.clone()
    c.merge_from_dict({"DATASETS": {"TEST": ("VID_val_videos",)}, "TEST": {"IMS_PER_BATCH": 2, "BBOX_AUG": {"ENABLED": True}},
                       "MODEL": {"VID": {"METHOD": "base"}}, "DATALOADER": {"NUM_WORKERS": 0}})
    (loader,) = make_data_loader(c, is_train=False, dataset_catalog=Catalog)
    assert isinstance(loader.collate_fn, BBoxAugCollator) and loader.dataset.transforms is None
    images, targets, ids = next(iter(loader))
    assert all(isinstance(im, Image.Image) for im in images) and len(images) == 2 and tuple(ids) == (0, 1)
    assert images[0].size == (160, 96) and len(loader) == (n + 1) // 2
    assert BBoxAugCollator()([("a", "t", 3), ("b", "u", 4)]) == [("a", "b"), ("t", "u"), (3, 4)]


def test_compute_on_dataset_dispatches_base_and_refuses_video_methods(monkeypatch):
    from mega_core.engine import inference

    class Model(object):
        def eval(self):
            return self

        def __call__(self, images):
            raise AssertionError("model(images) must not run with bbox_aug")

    class Det(str):
        def to(self, device):
            return self

    monkeypatch.setattr(inference, "im_detect_bbox_aug", lambda m, ims, d: [Det("det-%s" % im) for im in ims])
    loader = [(("x", "y"), (None, None), (4, 5))]
    res = inference.compute_on_dataset(Model(), loader, torch.device("cpu"), True, "base")
    assert res == {4: "det-x", 5: "det-y"}
    with pytest.raises(NotImplementedError, match="TEST.BBOX_AUG.ENABLED.*mega"):
        inference.compute_on_dataset(Model(), loader, torch.device("cpu"), True, "mega")


def test_im_detect_bbox_aug_refuses_video_detectors():
    from mega_core.engine.bbox_aug import im_detect_bbox_aug
    with pytest.raises(NotImplementedError, match="TEST.BBOX_AUG.ENABLED"):
        im_detect_bbox_aug(object(), [], "cpu")


def test_config_defaults_match_the_reference():
    from mega_core.config import cfg
    a = cfg.TEST.BBOX_AUG
    assert (a.ENABLED, a.H_FLIP, tuple(a.SCALES), a.MAX_SIZE, a.SCALE_H_FLIP) == (False, False, (), 4000, False)


# ---------------------------------------------------------------- 5. ABI
def test_abi_symbols_and_capacity_without_device():
    from mega_core import _lib
    header = open(os.path.join(ROOT, "include", "mega_b200.h")).read()
    for name in ("mega_image_transform_u8_ex", "mega_bbox_aug_workspace_bytes", "mega_bbox_aug_collect",
                 "mega_bbox_aug_merge"):
        assert name + "(" in header and name in _lib.EXPORTS and hasattr(_lib.lib, name)
    assert _lib.lib.mega_abi_version() == 7
    L = _lib.lib
    assert L.mega_bbox_aug_workspace_bytes(18, 300, 31) > 0
    assert L.mega_bbox_aug_workspace_bytes(1, 8192, 31) > 0
    assert L.mega_bbox_aug_workspace_bytes(28, 300, 31) == -1         # 8400 merged rows > 8192
    assert L.mega_bbox_aug_workspace_bytes(18, 300, 1) == -1
    assert L.mega_bbox_aug_workspace_bytes(0, 300, 31) == -1
    st = L.mega_bbox_aug_merge(28, 300, 31, 0.5, 300, None, 0, None, None, None, 0, None, None)
    assert st != 0 and b"8192" in L.mega_last_error()
    st = L.mega_bbox_aug_collect(None, 31, None, 124, None, None, 300, 31, 0, 28, 100, 100, 0, 1.0, 1.0, 0.05, 10., 10.,
                                 5., 5., None, 0, None)
    assert st != 0 and b"8192" in L.mega_last_error()
    from mega_core.b200 import ops
    with pytest.raises(_lib.MegaError, match="8192"):
        ops.bbox_aug_workspace_bytes(28, 300, 31)
