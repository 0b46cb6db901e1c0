"""Seq-NMS without a GPU:
  1. the NumPy oracle (tests/seq_nms_oracle.py) on hand-built videos whose answers are derived by hand in the comments;
  2. the kernels' own bodies (csrc/seq_nms.cuh, built by g++ through tests/native/seq_nms_host.cpp with the C ABI's
     names) equal the oracle bit for bit on seeded random videos -- kept set and fp32 scores;
  3. the Python layer (mega_core.engine.seq_nms, inference(), inference_no_model()) driven end to end on the CPU with the
     host build patched over the library's entry points -- the patching exists in this test only, the product has no
     CPU path: without a GPU its calls raise."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import seq_nms_oracle as so  # noqa: E402

f32 = np.float32
_host = None


def host_lib():
    """g++ build of csrc/seq_nms.cuh, cached in the temp directory under the digest of its sources"""
    global _host
    if _host is None:
        src = os.path.join(ROOT, "tests", "native", "seq_nms_host.cpp")
        deps = [src] + [os.path.join(ROOT, "mega.pytorch_b200", "csrc", n) for n in ("seq_nms.cuh", "iou.cuh")] + [
            os.path.join(ROOT, "include", "mega_b200.h")]
        digest = hashlib.sha256(b"".join(open(p, "rb").read() for p in deps)).hexdigest()[:16]
        so_path = os.path.join(tempfile.gettempdir(), "mega_seq_nms_host_%s_%d.so" % (digest, os.getuid()))
        if not os.path.exists(so_path):
            tmp = so_path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-I",
                                   os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                                   "-o", tmp, src])
            os.replace(tmp, so_path)
        _host = ctypes.CDLL(so_path)
        from mega_core import _lib
        for name in ("mega_seq_nms", "mega_seq_nms_workspace_bytes"):
            fn, real = getattr(_host, name), getattr(_lib.lib, name)
            fn.argtypes, fn.restype = real.argtypes, real.restype
    return _host


def host_run(videos, link_iou=0.5, nms_iou=0.3, rescore="avg"):
    """the C ABI call on the host build, all videos in one call -> per video, per frame (keep, new_scores)"""
    lib = host_lib()
    boxes, scores, labels, counts, offsets, num_classes = so.pack(videos)
    F, D = scores.shape
    nbytes = lib.mega_seq_nms_workspace_bytes(F, D, num_classes)
    assert nbytes > 0
    ws = np.zeros(nbytes // 8 + 1, np.float64)
    out_scores = np.full((F, D), np.nan, f32)
    keep = np.full((F, D), 7, np.uint8)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)          # noqa: E731
    st = lib.mega_seq_nms(p(boxes), p(scores), p(labels), p(counts), F, D, p(offsets), len(videos), num_classes,
                          link_iou, nms_iou, {"avg": 0, "max": 1}[rescore], p(ws), nbytes, p(out_scores), p(keep), None)
    assert st == 0
    assert set(np.unique(keep)) <= {0, 1} and np.all(out_scores[keep == 0] == 0)
    return so.unpack(videos, keep, out_scores)


def box(x, w=10, y=0, h=10):
    """a box of w x h pixels ("+1" convention) at (x, y)"""
    return [x, y, x + w - 1, y + h - 1]


def frame(*dets):
    """dets: (box, score, label), given in class-major order"""
    if not dets:
        return (np.zeros((0, 4), f32), np.zeros(0, f32), np.zeros(0, np.int64))
    b, s, l = zip(*dets)
    return (np.array(b, f32), np.array(s, f32), np.array(l, np.int64))


def avg(*scores):
    """the avg rescore of a chain: fp64 sum from the last frame backward, divided, rounded to fp32"""
    acc = 0.0
    for s in reversed(scores):
        acc = float(np.float64(f32(s))) + acc
    return f32(acc / len(scores))


def check(result, want):
    """want: per frame, list of new scores with None for removed boxes"""
    assert len(result) == len(want)
    for (k, s), w in zip(result, want):
        assert list(k) == [x is not None for x in w], (k, w)
        assert np.array_equal(s[k], np.array([x for x in w if x is not None], f32)), (s, w)


# Width-10 boxes shifted by d pixels along x: IoU = (10 - d) / (10 + d): d=2 -> 0.667, d=3 -> 0.538 (links at 0.5),
# d=5 -> 0.333 (suppresses at 0.3, does not link), d=6 -> 0.25 (neither).
def test_oracle_two_crossing_tubes():
    # tube A moves right (x 0, 3, 6), tube B left (x 6, 3, 0); they coincide in frame 1, every box links to every box of
    # the next frame. Pass 1: best(A2) 0.8, best(B2) 0.4; best(A1) = 0.6 + 0.8, best(B1) = 0.7 + 0.8 (both -> A2);
    # best(A0) = 0.9 + 1.5 (-> B1), best(B0) = 0.5 + 1.5. Root A0: chain A0 -> B1 -> A2 switches tubes at the crossing;
    # A1 (IoU 1 with B1) is suppressed, B0 / B2 (IoU 0.25) are not. Frame 1 is then empty, so B0 and B2 are lone boxes.
    video = [frame((box(0), 0.9, 1), (box(6), 0.5, 1)),
             frame((box(3), 0.6, 1), (box(3), 0.7, 1)),
             frame((box(6), 0.8, 1), (box(0), 0.4, 1))]
    a = avg(0.9, 0.7, 0.8)
    check(so.seq_nms_video(video), [[a, f32(0.5)], [None, a], [a, f32(0.4)]])
    check(so.seq_nms_video(video, rescore="max"), [[f32(0.9), f32(0.5)], [None, f32(0.9)], [f32(0.9), f32(0.4)]])
    assert a != f32(0.9)


def test_oracle_gap_frame_and_empty_frames_break_chains():
    # class 1 at the same place in frames 0, 2 and 4; frame 1 holds only a class-2 box, frame 3 nothing: every class-1
    # box is a chain of length 1 and keeps its score (avg of one value = the value)
    video = [frame((box(0), 0.5, 1)), frame((box(0), 0.9, 2)), frame((box(0), 0.7, 1)), frame(), frame((box(0), 0.3, 1))]
    check(so.seq_nms_video(video), [[f32(0.5)], [f32(0.9)], [f32(0.7)], [], [f32(0.3)]])
    # without the gap the three frames form one chain
    joined = [frame((box(0), 0.5, 1)), frame((box(0), 0.9, 1)), frame((box(0), 0.7, 1))]
    a = avg(0.5, 0.9, 0.7)
    check(so.seq_nms_video(joined), [[a], [a], [a]])
    check(so.seq_nms_video([frame(), frame()]), [[], []])


def test_oracle_iou_exactly_at_the_thresholds_does_not_count():
    # [0,9]x[0,9] inside [0,19]x[0,9]: IoU = 100 / 200 = 0.5 exactly -> no link at LINK_IOU 0.5, a link just below
    video = [frame((box(0), 0.6, 1)), frame((box(0, w=20), 0.2, 1))]
    check(so.seq_nms_video(video), [[f32(0.6)], [f32(0.2)]])
    a = avg(0.6, 0.2)
    check(so.seq_nms_video(video, link_iou=0.4999), [[a], [a]])
    # [0,9] vs [4,19] (x), same rows: inter 60, union 100 + 160 - 60 = 200, IoU = 0.3 exactly -> no suppression at 0.3
    one = [frame((box(0), 0.9, 1), (box(4, w=16), 0.5, 1))]
    check(so.seq_nms_video(one), [[f32(0.9), f32(0.5)]])
    check(so.seq_nms_video(one, nms_iou=0.2999), [[f32(0.9), None]])


def test_oracle_dp_ties_go_to_the_smallest_index():
    # P (x 3) links to both boxes of frame 1 (x 6 and x 0, equal scores 0.5, IoU 0.25 between them): the successor is
    # the one listed first
    video = [frame((box(3), 0.7, 1)), frame((box(6), 0.5, 1), (box(0), 0.5, 1))]
    a = avg(0.7, 0.5)
    check(so.seq_nms_video(video), [[a], [a, f32(0.5)]])
    video = [frame((box(3), 0.7, 1)), frame((box(0), 0.5, 1), (box(6), 0.5, 1))]
    check(so.seq_nms_video(video), [[a], [a, f32(0.5)]])


def test_oracle_root_ties_go_to_the_smallest_frame_then_index():
    # one frame, two equal scores with IoU 0.667: the first listed is the root and suppresses the other
    check(so.seq_nms_video([frame((box(2), 0.5, 1), (box(0), 0.5, 1))]), [[f32(0.5), None]])
    # X (frame 0, 0.25) -> X1 (frame 1, x 3, 0.25): best 0.5 = best of Y (frame 1, x 5, 0.5; no link to X, IoU 0.667
    # with X1). The frame-0 root wins: chain X -> X1 (avg 0.25) suppresses Y.
    video = [frame((box(0), 0.25, 1)), frame((box(3), 0.25, 1), (box(5), 0.5, 1))]
    check(so.seq_nms_video(video), [[f32(0.25)], [f32(0.25), None]])


def test_oracle_one_frame_video_is_per_class_nms():
    # classes are independent: the class-2 box overlapping the class-1 box survives
    video = [frame((box(0), 0.9, 1), (box(1), 0.8, 1), (box(40), 0.3, 1), (box(0), 0.2, 2))]
    check(so.seq_nms_video(video), [[f32(0.9), None, f32(0.3), f32(0.2)]])


def test_oracle_avg_and_max_rescoring():
    video = [frame((box(0), 0.3, 1)), frame((box(2), 0.9, 1)), frame((box(4), 0.6, 1))]
    a = avg(0.3, 0.9, 0.6)
    check(so.seq_nms_video(video), [[a], [a], [a]])
    check(so.seq_nms_video(video, rescore="max"), [[f32(0.9)], [f32(0.9)], [f32(0.9)]])


HAND_BUILT = [
    [frame((box(0), 0.9, 1), (box(6), 0.5, 1)), frame((box(3), 0.6, 1), (box(3), 0.7, 1)),
     frame((box(6), 0.8, 1), (box(0), 0.4, 1))],
    [frame((box(0), 0.5, 1)), frame((box(0), 0.9, 2)), frame((box(0), 0.7, 1)), frame(), frame((box(0), 0.3, 1))],
    [frame((box(0), 0.6, 1)), frame((box(0, w=20), 0.2, 1))],
    [frame((box(0), 0.9, 1), (box(4, w=16), 0.5, 1))],
    [frame((box(0), 0.25, 1)), frame((box(3), 0.25, 1), (box(5), 0.5, 1))],
    [frame((box(2), 0.5, 1), (box(0), 0.5, 1))],
]


def _same(a, b):
    for (ka, sa), (kb, sb) in zip(a, b):
        assert np.array_equal(ka, kb) and np.array_equal(sa.view(np.uint32), sb.view(np.uint32))


@pytest.mark.parametrize("rescore", ["avg", "max"])
def test_host_build_equals_the_oracle_on_hand_built_videos(rescore):
    for thresholds in ((0.5, 0.3), (0.4999, 0.2999)):
        got = host_run(HAND_BUILT, *thresholds, rescore=rescore)
        for v, g in zip(HAND_BUILT, got):
            _same(g, so.seq_nms_video(v, *thresholds, rescore=rescore))


@pytest.mark.parametrize("seed", range(4))
def test_host_build_equals_the_oracle_bit_for_bit(seed):
    """seeded random videos of 1..40 frames, several per call; one with a dense class; thresholds and rescore vary"""
    rng = np.random.default_rng(seed)
    videos = [so.make_video(rng, int(n), int(rng.integers(5, 40)), 6, dense_class=2 if i == 0 else None)
              for i, n in enumerate([1, 2, 40, int(rng.integers(3, 30))])]
    link, nms = [(0.5, 0.3), (0.3, 0.5), (0.7, 0.1), (0.5, 0.3)][seed]
    rescore = ["avg", "max"][seed % 2]
    got = host_run(videos, link, nms, rescore)
    kept = 0
    for v, g in zip(videos, got):
        want = so.seq_nms_video(v, link, nms, rescore)
        _same(g, want)
        kept += sum(int(k.sum()) for k, _ in want)
    assert kept > 0
    # one video per call gives the same bits
    for v, g in zip(videos, got):
        _same(host_run([v], link, nms, rescore)[0], g)


def test_workspace_and_argument_checks_of_the_library():
    from mega_core import _lib
    lib = _lib.lib
    assert lib.mega_seq_nms_workspace_bytes(10, 300, 31) > 10 * 300 * (5 * 8 + 8 + 4)
    assert lib.mega_seq_nms_workspace_bytes(10, 513, 31) == -1
    assert lib.mega_seq_nms_workspace_bytes(0, 300, 31) == -1
    assert lib.mega_seq_nms(None, None, None, None, 4, 300, None, 1, 31, 0.5, 0.3, 2, None, 0, None, None, None) != 0
    assert b"rescore" in lib.mega_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without a GPU")
def test_no_cpu_fallback():
    from mega_core import _lib
    from mega_core.engine.seq_nms import seq_nms
    from mega_core.structures.bounding_box import BoxList
    b = BoxList(torch.tensor([[0.0, 0, 9, 9]]), (100, 100))
    b.add_field("scores", torch.tensor([0.5]))
    b.add_field("labels", torch.tensor([1]))
    with pytest.raises(_lib.MegaError):
        seq_nms([b, b])


@pytest.fixture
def host_seq_nms(monkeypatch):
    """mega_seq_nms served by the host build, the module's device set to the CPU"""
    from mega_core import _lib
    from mega_core.b200 import ops
    from mega_core.engine import seq_nms as sn
    host = host_lib()
    for name in ("mega_seq_nms", "mega_seq_nms_workspace_bytes"):
        monkeypatch.setattr(_lib.lib, name, getattr(host, name))
    monkeypatch.setattr(ops, "require_cuda", lambda *t: None)
    monkeypatch.setattr(ops, "stream_ptr", lambda: None)
    monkeypatch.setattr(sn, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(sn, "FRAMES_PER_LAUNCH", 7)     # several launches, each of whole videos
    return sn


def _boxlist(f, size=(1000, 600)):
    from mega_core.structures.bounding_box import BoxList
    b = BoxList(torch.from_numpy(f[0].copy()), size, mode="xyxy")
    b.add_field("scores", torch.from_numpy(f[1].copy()))
    b.add_field("labels", torch.from_numpy(f[2].copy()))
    return b


def test_seq_nms_api_keeps_input_order_and_fields(host_seq_nms):
    rng = np.random.default_rng(11)
    video = so.make_video(rng, 12, 30, 5)
    # shuffle the detections of each frame: the API takes any order and returns the input order
    shuffled = []
    for b, s, l in video:
        p = rng.permutation(len(s))
        shuffled.append((b[p], s[p], l[p]))
    want = so.seq_nms_video(shuffled, 0.5, 0.3, "avg")
    lists = [_boxlist(f) for f in shuffled]
    for bl in lists:
        bl.add_field("tag", torch.arange(len(bl)))
    out = host_seq_nms.seq_nms(lists)
    for bl, o, (k, s) in zip(lists, out, want):
        idx = torch.from_numpy(np.nonzero(k)[0])
        assert torch.equal(o.bbox, bl.bbox[idx]) and torch.equal(o.get_field("labels"), bl.get_field("labels")[idx])
        assert torch.equal(o.get_field("tag"), idx) and o.size == bl.size and o.mode == bl.mode
        assert np.array_equal(o.get_field("scores").numpy().view(np.uint32), s[k].view(np.uint32))


class _Dataset(object):
    """two videos of a VID-style list (pattern / frame_seg_id), frames interleaved in the index like no real list is"""

    def __init__(self, videos):
        self.pattern, self.frame_seg_id, self.frames = [], [], []
        for v, frames in enumerate(videos):
            for t, f in enumerate(frames):
                self.pattern.append("val/video_%d/%%06d" % v)
                self.frame_seg_id.append(t)
                self.frames.append(f)

    def __len__(self):
        return len(self.frames)

    def get_img_info(self, i):
        return {"width": 1000, "height": 600}

    def get_groundtruth(self, i):
        from mega_core.structures.bounding_box import BoxList
        b, _, l = self.frames[i]
        gt = BoxList(torch.from_numpy(b[:2].copy()).reshape(-1, 4), (1000, 600), mode="xyxy")
        gt.add_field("labels", torch.from_numpy(l[:2].copy()))
        return gt

    def map_class_id_to_class_name(self, i):
        return "class%d" % i


def _run_inference(tmp_path, cfg, videos):
    from mega_core.engine.inference import inference
    ds = _Dataset(videos)

    class Loader(object):
        dataset = ds

        def __iter__(self):
            for i in range(len(ds)):
                yield {"cur": torch.zeros(3, 4, 4), "frame_category": int(ds.frame_seg_id[i] > 0), "id": i}, None, [i]

    class Model(torch.nn.Module):
        def forward(self, batch):
            return [_boxlist(ds.frames[batch["id"]])]

    logging.getLogger("mega_core.inference").setLevel(logging.ERROR)
    inference(cfg, Model(), Loader(), "VID_val_synthetic", device="cpu", output_folder=str(tmp_path))
    return ds, torch.load(os.path.join(tmp_path, "predictions.pth"), weights_only=False)


def _cfg(**seq):
    from mega_core.config import cfg
    c = cfg.clone()
    c.MODEL.VID.METHOD = "mega"
    for k, v in seq.items():
        c.MODEL.B200.SEQ_NMS[k] = v
    return c


def _videos():
    rng = np.random.default_rng(5)
    return [so.make_video(rng, 9, 25, 4), so.make_video(rng, 6, 25, 4)]


def test_inference_applies_seq_nms_when_the_key_is_on(tmp_path, host_seq_nms):
    from mega_core.engine.inference import inference_no_model
    videos = _videos()
    ds, preds = _run_inference(tmp_path, _cfg(ENABLED=True, RESCORE="max", NMS_IOU=0.4), videos)
    want = [r for v in videos for r in so.seq_nms_video(v, 0.5, 0.4, "max")]
    assert len(preds) == len(want)
    changed = 0
    for p, f, (k, s) in zip(preds, ds.frames, want):
        assert torch.equal(p.bbox, torch.from_numpy(f[0][k])) and torch.equal(p.get_field("labels"), torch.from_numpy(f[2][k]))
        assert np.array_equal(p.get_field("scores").numpy().view(np.uint32), s[k].view(np.uint32))
        changed += int(len(p) != len(f[1]))
    assert changed > 0
    # rescoring the saved predictions of a run WITHOUT Seq-NMS gives the same detections
    plain = tmp_path / "plain"
    plain.mkdir()
    _run_inference(plain, _cfg(), videos)

    class Loader(object):
        dataset = ds

    import mega_core.engine.inference as inf
    captured = {}
    real = inf.vid_evaluation

    def capture(dataset, predictions, **kw):
        captured["p"] = predictions
        return real(dataset=dataset, predictions=predictions, **kw)

    inf.vid_evaluation = capture
    try:
        inference_no_model(Loader(), output_folder=str(plain),
                           seq_nms={"ENABLED": True, "LINK_IOU": 0.5, "NMS_IOU": 0.4, "RESCORE": "max"})
    finally:
        inf.vid_evaluation = real
    for a, b in zip(captured["p"], preds):
        assert torch.equal(a.bbox, b.bbox) and torch.equal(a.get_field("scores"), b.get_field("scores"))


@pytest.mark.parametrize("cfg_kind", ["absent", "off"])
def test_inference_without_the_key_returns_the_detections_unchanged(tmp_path, cfg_kind):
    class Bare:
        class MODEL:
            class VID:
                METHOD = "mega"

    videos = _videos()
    ds, preds = _run_inference(tmp_path, Bare if cfg_kind == "absent" else _cfg(), videos)
    for p, f in zip(preds, ds.frames):
        assert torch.equal(p.bbox, torch.from_numpy(f[0])) and torch.equal(p.get_field("scores"), torch.from_numpy(f[1]))
        assert torch.equal(p.get_field("labels"), torch.from_numpy(f[2]))
