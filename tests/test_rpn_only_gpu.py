"""MODEL.RPN_ONLY and proposal recall on the H100:
  * the RPN-only engines (single-frame R-50, DFF R-101, FGFA R-101; fixtures of tests/golden) return, in both arithmetic
    modes, exactly the proposals the full engine's RPN stage produces on the same frames (last_props / last_cnt of
    _mlp_features), in descending objectness order, and they match the reference's proposals under the criterion of
    tests/test_engine_gpu.py;
  * the RPN-only engines hold none of the box head's buffers or weights;
  * the model returns objectness-only BoxLists;
  * mega_proposal_recall equals its g++ host build bit for bit on a VID-val-sized synthetic dataset (with a tail of
    images whose IoU matrices take the global-workspace path) and on the golden cases of tests/golden/rpn_only.pt."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu

BOX_HEAD_BUFFERS = ("pooled", "fc6", "fc7", "pred", "res5_out", "reduce", "det_boxes", "det_scores", "det_labels",
                    "det_count")


def _match_rows(a, b, tol=0.75):
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _snap(r):
    """a copy of a frame's result: the engine reuses its output buffers on the next frame"""
    from mega_core.b200 import engine
    return engine.Proposals(r.boxes.clone(), r.objectness.clone(), r.count.clone()) if isinstance(r, engine.Proposals) else None


def _runs(name, cuda_dev, precision, rpn_only):
    """the engine; per frame of the fixture: its result (copied), the reference's proposals, and (last_props, last_cnt)"""
    from mega_core.b200 import engine, synth
    gold = torch.load(os.path.join(ROOT, "tests", "golden", name + "_192x320.pt"))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    if rpn_only:
        sd = {k: v for k, v in sd.items() if not k.startswith("roi_heads.")}
    h, w = gold["h"], gold["w"]
    if name == "base_r50":
        eng = engine.BaseEngine(sd, engine.EngineConfig(precision=precision, rpn_only=rpn_only), device=cuda_dev)
        res = [_snap(eng.forward(synth.synthetic_frame(gold["frame_index"], h, w).to(cuda_dev), w, h))]
        refs = [gold["proposals"]]
        states = [(eng.last_props.clone(), eng.last_cnt.clone())]
    elif name == "dff_r101":
        eng = engine.DffEngine(sd, engine.EngineConfig(precision=precision, rpn_only=rpn_only), device=cuda_dev)
        res, refs, states = [], [], []
        for t, (key, ref) in enumerate(zip(gold["key_flags"], gold["frames"])):
            res.append(_snap(eng.forward(synth.synthetic_frame(gold["frame_stride"] * t, h, w).to(cuda_dev), key, w, h)))
            refs.append(ref["proposals"])
            states.append((eng.last_props.clone(), eng.last_cnt.clone()))
    else:
        total = gold["total"]
        frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(total)]
        eng = engine.FgfaEngine(sd, engine.EngineConfig(all_frame_interval=19, key_frame_location=9, precision=precision,
                                                        rpn_only=rpn_only), device=cuda_dev)
        res, refs, states = [], [], []
        for t, ref in enumerate(gold["frames"]):
            res.append(_snap(eng.start_video(frames[0], frames[1:10], w, h) if t == 0 else
                             eng.step(frames[min(t + 9, total - 1)], w, h)))
            refs.append(ref["proposals"])
            states.append((eng.last_props.clone(), eng.last_cnt.clone()))
    torch.cuda.synchronize()
    return eng, res, refs, states


@pytest.mark.parametrize("precision", ["fp32x3", "f16"])
@pytest.mark.parametrize("name", ["base_r50", "dff_r101", "fgfa_r101"])
def test_rpn_only_proposals_equal_the_full_engines_rpn_stage(cuda_dev, name, precision):
    from mega_core.b200 import engine
    full, _, _, full_states = _runs(name, cuda_dev, precision, rpn_only=False)
    eng, res, refs, states = _runs(name, cuda_dev, precision, rpn_only=True)
    bar = 0.95 if name == "fgfa_r101" else 0.9
    for t, (r, ref, (fp, fc), (op, oc)) in enumerate(zip(res, refs, full_states, states)):
        assert isinstance(r, engine.Proposals)
        k = int(r.count.item())
        assert k == int(fc[0].item()) == int(oc[0].item()) and k > 0
        assert torch.equal(r.boxes[:k], fp[:k]) and torch.equal(op[:k], fp[:k]), "frame %d: proposals differ" % t
        s = r.objectness[:k]
        assert bool((s[:-1] >= s[1:]).all()), "frame %d: not in descending objectness order" % t
        idx = _match_rows(r.boxes[:k].cpu(), ref)
        assert (idx >= 0).float().mean().item() >= bar, (t, (idx >= 0).float().mean().item())
    assert not [key for key in eng._bufs if key[0] in BOX_HEAD_BUFFERS], sorted(eng._bufs)
    for attr in ("res5", "pred_w", "fc6_w", "fc7_w", "red_w"):
        assert not hasattr(eng, attr), attr
    del full


def test_the_rpn_only_model_returns_objectness_boxlists(cuda_dev):
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model
    from mega_core.modeling.detector.detectors import vid_config
    cfg = vid_config("base", "R-50-C4", device=str(cuda_dev))
    cfg.MODEL.RPN_ONLY = True
    cfg.MODEL.B200.PRECISION = "f16"
    model = build_detection_model(cfg).eval()
    sd = synth.make_state_dict("base_r50", seed=1)
    missing = model.load_state_dict({k: v for k, v in sd.items() if not k.startswith("roi_heads.")}, strict=False)
    assert not [k for k in missing.missing_keys if "cell_anchors" not in k]
    img = synth.synthetic_frame(3, 192, 320)[0].to(cuda_dev)
    out = model([img])
    assert len(out) == 1 and out[0].fields() == ["objectness"] and out[0].size == (320, 192) and len(out[0]) > 0
    s = out[0].get_field("objectness")
    assert bool((s[:-1] >= s[1:]).all())


def _device_recall(pb, ps, gb, po, go, iou_thresh=0.5, limit=300):
    from mega_core.b200 import ops
    dev = torch.device("cuda")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)        # noqa: E731
    ov = torch.full((len(gb),), float("nan"), device=dev)
    stats = torch.zeros(3, dtype=torch.int64, device=dev)
    cnt_p, cnt_g = np.diff(po), np.diff(go)
    ops.proposal_recall(t(pb), t(ps), t(po), t(gb), t(go), int(cnt_p.max(initial=0)), int(cnt_g.max(initial=0)), limit,
                        iou_thresh, ov, stats)
    hits, num_pos, rejected = stats.cpu().tolist()
    return hits, num_pos, rejected, ov.cpu().numpy()


def _host_recall(pb, ps, gb, po, go, iou_thresh=0.5, limit=300):
    import ctypes
    import test_rpn_only_cpu as cpu
    lib = cpu.host_lib()
    mp, mg = int(np.diff(po).max(initial=0)), int(np.diff(go).max(initial=0))
    nbytes = lib.mega_proposal_recall_workspace_bytes(len(po) - 1, mp, mg, limit)
    ws = np.zeros(nbytes // 4 + 1, np.float32)
    ov = np.full(len(gb), np.nan, np.float32)
    stats = np.zeros(3, np.uint64)
    p = lambda a: np.ascontiguousarray(a).ctypes.data_as(ctypes.c_void_p)     # noqa: E731
    arrs = [np.ascontiguousarray(a) for a in (pb, ps, po, gb, go)]
    assert lib.mega_proposal_recall(*[p(a) for a in arrs[:5]], len(po) - 1, mp, mg, limit, iou_thresh, p(ws), nbytes,
                                    p(ov), p(stats), None) == 0
    return int(stats[0]), int(stats[1]), int(stats[2]), ov


def test_kernel_equals_the_host_build_on_a_vid_val_sized_dataset(cuda_dev):
    from mega_core.b200 import ops, synth
    data = synth.synthetic_proposal_dataset(seed=5)
    pb, ps, gb, po, go = data
    assert len(po) - 1 > 176000 and np.diff(po).max() > 300 and np.diff(go).max() > 100
    assert ops.proposal_recall_workspace_bytes(len(po) - 1, int(np.diff(po).max()), int(np.diff(go).max()), 300) > 0
    dev = _device_recall(pb, ps, gb, po, go)
    host = _host_recall(pb, ps, gb, po, go)
    assert dev[:3] == host[:3] and dev[2] == 0
    assert np.array_equal(dev[3].view(np.uint32), host[3].view(np.uint32))
    assert 0 < dev[0] < dev[1]


def test_kernel_equals_the_golden_cases_and_the_public_api(cuda_dev):
    from mega_core.data.datasets.evaluation.vid import eval_proposals_vid
    from mega_core.structures.bounding_box import BoxList
    import test_rpn_only_cpu as cpu
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "rpn_only.pt"), weights_only=False)
    size = gold["image_size"]
    for case in gold["recall_cases"]:
        ims = case["images"]
        images = [(im["boxes"].numpy(), im["objectness"].numpy(), im["gt"].numpy()) for im in ims]
        pb = np.concatenate([i[0].reshape(-1, 4) for i in images]).astype(np.float32)
        ps = np.concatenate([i[1] for i in images]).astype(np.float32)
        gb = np.concatenate([i[2].reshape(-1, 4) for i in images]).astype(np.float32)
        po = np.concatenate([[0], np.cumsum([len(i[1]) for i in images])]).astype(np.int64)
        go = np.concatenate([[0], np.cumsum([len(i[2]) for i in images])]).astype(np.int64)
        hits, num_pos, rejected, ov = _device_recall(pb, ps, gb, po, go, case["iou_thresh"], case["limit"])
        got = cpu.contributing(images, case["limit"], ov)
        for g, w in zip(got, case["gt_overlaps"]):
            assert np.array_equal(g.view(np.uint32), w.numpy().astype(np.float32).view(np.uint32))
        preds, gts = [], []
        for im in ims:
            b = BoxList(im["boxes"], size)
            b.add_field("objectness", im["objectness"])
            preds.append(b)
            gts.append(BoxList(im["gt"].reshape(-1, 4), size))
        recall = eval_proposals_vid(preds, gts, case["iou_thresh"], case["limit"])["recall"]
        assert torch.equal(recall, case["recall"]), (case["name"], recall, case["recall"])
