"""Seq-NMS on the H100 (csrc/seq_nms.cu): the kernels equal the NumPy oracle (tests/seq_nms_oracle.py) bit for bit --
kept set and fp32 scores -- on seeded videos of 1, 2, 37 and 500 frames, at up to 300 detections per frame with a dense
class and junk-heavy scores; many videos per launch equal one video per launch; a side stream equals the default
stream; and Seq-NMS of the engine's own output (model(images) over a synthetic MEGA R-101 video) equals the oracle on the
same detections."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import seq_nms_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu


def _device_run(videos, link_iou=0.5, nms_iou=0.3, rescore="avg", stream=None):
    from mega_core.b200 import ops
    boxes, scores, labels, counts, offsets, num_classes = so.pack(videos)
    dev = torch.device("cuda")
    args = [torch.from_numpy(a).to(dev) for a in (boxes, scores, labels, counts, offsets)]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
        ns, keep = ops.seq_nms(*args, num_classes, link_iou=link_iou, nms_iou=nms_iou, rescore=rescore)
        ns, keep = ns.cpu(), keep.cpu()
    torch.cuda.synchronize()
    k = keep.numpy()
    assert set(np.unique(k)) <= {0, 1}
    return so.unpack(videos, k, ns.numpy())


def _same(got, want):
    for (kg, sg), (kw, sw) in zip(got, want):
        assert np.array_equal(kg, kw), (np.nonzero(kg != kw)[0][:10], len(kg))
        assert np.array_equal(sg.view(np.uint32), sw.view(np.uint32)), np.abs(sg - sw).max()


@pytest.mark.parametrize("n_frames,n_det,num_classes,rescore", [(1, 300, 31, "avg"), (2, 300, 31, "max"),
                                                                (37, 300, 31, "avg"), (500, 8, 4, "avg")])
def test_kernels_equal_the_oracle_bit_for_bit(cuda_dev, n_frames, n_det, num_classes, rescore):
    rng = np.random.default_rng(n_frames)
    video = so.make_video(rng, n_frames, n_det, num_classes, dense_class=7 if n_det >= 300 else None)
    if n_det >= 300:
        assert all(len(s) == 300 and int((l == 7).sum()) >= 100 for _, s, l in video)
        assert np.mean(np.concatenate([s for _, s, _ in video]) < 0.02) > 0.5      # junk-heavy
    got = _device_run([video], rescore=rescore)[0]
    want = so.seq_nms_video(video, rescore=rescore)
    _same(got, want)
    assert sum(int(k.sum()) for k, _ in want) > 0


def test_many_videos_per_launch_equal_one_per_launch_and_the_oracle(cuda_dev):
    rng = np.random.default_rng(3)
    videos = [so.make_video(rng, int(n), 60, 8, dense_class=3 if i == 2 else None)
              for i, n in enumerate([5, 1, 40, 33, 2, 17, 64])]
    together = _device_run(videos, 0.4, 0.35, "max")
    for v, t in zip(videos, together):
        _same(_device_run([v], 0.4, 0.35, "max")[0], t)
        _same(t, so.seq_nms_video(v, 0.4, 0.35, "max"))


def test_side_stream_equals_default_stream(cuda_dev):
    rng = np.random.default_rng(4)
    videos = [so.make_video(rng, 24, 120, 12, dense_class=5), so.make_video(rng, 9, 120, 12)]
    base = _device_run(videos)
    side = _device_run(videos, stream=torch.cuda.Stream())
    for a, b in zip(base, side):
        _same(a, b)


def test_public_api_on_the_device(cuda_dev):
    from mega_core.engine.seq_nms import seq_nms
    from mega_core.structures.bounding_box import BoxList
    rng = np.random.default_rng(8)
    video = so.make_video(rng, 12, 80, 6)
    lists = []
    for b, s, l in video:
        bl = BoxList(torch.from_numpy(b), (1000, 600), mode="xyxy")
        bl.add_field("scores", torch.from_numpy(s))
        bl.add_field("labels", torch.from_numpy(l))
        lists.append(bl)
    out = seq_nms(lists, link_iou=0.5, nms_iou=0.3, rescore="avg")
    for bl, o, (k, s) in zip(lists, out, so.seq_nms_video(video)):
        idx = torch.from_numpy(np.nonzero(k)[0])
        assert torch.equal(o.bbox, bl.bbox[idx]) and torch.equal(o.get_field("labels"), bl.get_field("labels")[idx])
        assert np.array_equal(o.get_field("scores").numpy().view(np.uint32), s[k].view(np.uint32))


def test_seq_nms_of_the_engines_own_output_equals_the_oracle(cuda_dev):
    """model(images) over a synthetic MEGA R-101 video (tiny body, 96x160), then Seq-NMS on the device, against the
    oracle applied to the very detections the engine returned"""
    from mega_core.b200 import synth
    from mega_core.engine.seq_nms import seq_nms
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    sd = synth.make_state_dict("mega_r101_tiny", seed=3)
    model = build_detection_model_from_state_dict(sd, method="mega", device=cuda_dev, precision="f16")
    h, w, total = 96, 160, 30
    frames = [synth.synthetic_frame(i, h, w)[0] for i in range(total)]
    common = {"seg_len": total, "pattern": "%06d", "img_dir": "/nonexistent/%s.JPEG"}
    dets = []
    with torch.no_grad():
        for t in range(16):
            if t == 0:
                images = {"cur": frames[0], "ref_l": [], "ref_g": [frames[j] for j in range(15, 25)], "frame_category": 0,
                          "lookahead": frames[1:13], **common}
            else:
                images = {"cur": frames[t], "ref_l": [frames[min(t + 12, total - 1)]],
                          "ref_g": [frames[(7 * t) % total]], "frame_category": 1, **common}
            dets.append(model({k: ([x.to(cuda_dev) for x in v] if isinstance(v, list) else
                                   v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in images.items()})[0].to("cpu"))
    assert sum(len(d) for d in dets) > 0
    video = [(d.bbox.numpy(), d.get_field("scores").numpy(), d.get_field("labels").numpy()) for d in dets]
    out = seq_nms(dets)
    want = so.seq_nms_video(video)
    for d, o, (k, s) in zip(dets, out, want):
        assert torch.equal(o.bbox, d.bbox[torch.from_numpy(np.nonzero(k)[0])])
        assert np.array_equal(o.get_field("scores").numpy().view(np.uint32), s[k].view(np.uint32))
