"""CPU tests of the shipped VID configs that use MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL, MEGA.GLOBAL.RES_STAGE = 0 or
ATTENTION.ADVANCED_STAGE = 0 (configs/MEGA/vid_R_50_C4_MEGA_1x.yaml, configs/RDN/vid_R_{101,50}_C4_RDN_base_1x.yaml):
the module tree of all 11 VID configs against the reference's parameter lists, the config checks, the engines' host logic
on the CPU stand-ins (tests/cpu_ops.py) against the fixtures tools/make_golden_configs.py wrote from the unmodified
reference, and the multi-GPU schedules of MEGA without the second global stage."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden")

from cpu_ops import cpu_ops  # noqa: E402

FIXTURES = ("mega_r50_192x320.pt", "rdnbase_r101_192x320.pt", "rdnbase_r50_192x320.pt")


def _vid_configs():
    with open(os.path.join(GOLD, "reference_configs.json")) as fh:
        yamls = json.load(fh)
    with open(os.path.join(GOLD, "vid_configs.json")) as fh:
        extra = json.load(fh)
    yamls.update(extra["yaml"])
    return yamls, extra["state_dict_shapes"]


def _cfg(tmp_path, yamls, name):
    """defaults <- BASE_RCNN_1gpu.yaml <- the method YAML, as tools/test_net.py merges them"""
    import yaml
    from mega_core.config import cfg as base
    c = base.clone()
    for tag, data in (("base", yamls["configs/BASE_RCNN_1gpu.yaml"]), ("method", yamls[name])):
        p = os.path.join(str(tmp_path), tag + ".yaml")
        with open(p, "w") as fh:
            yaml.safe_dump(data, fh)
        c.merge_from_file(p)
    c.MODEL.DEVICE = "cpu"
    return c


def test_every_vid_config_builds_the_reference_module_tree(tmp_path):
    """all 11 VID YAMLs: build_detection_model gives every key and shape of the reference's model, and the engines
    serve the config"""
    from mega_core.modeling.detector import build_detection_model
    from mega_core.modeling.nets import engine_config_from
    yamls, shapes = _vid_configs()
    assert len(shapes) == 11
    for name, want in shapes.items():
        cfg = _cfg(tmp_path, yamls, name)
        got = {k: list(v.shape) for k, v in build_detection_model(cfg).state_dict().items()}
        assert got == dict(want), name
        engine_config_from(cfg)


def test_fixture_configs_give_their_engine_layout(tmp_path):
    from mega_core.modeling.nets import engine_config_from
    yamls, _ = _vid_configs()
    mega = engine_config_from(_cfg(tmp_path, yamls, "configs/MEGA/vid_R_50_C4_MEGA_1x.yaml"))
    assert (mega.stage, mega.global_res_stage) == (3, 0)
    for name in ("configs/RDN/vid_R_101_C4_RDN_base_1x.yaml", "configs/RDN/vid_R_50_C4_RDN_base_1x.yaml"):
        rdn = engine_config_from(_cfg(tmp_path, yamls, name))
        assert (rdn.stage, rdn.advanced_stage, rdn.all_frame_interval, rdn.key_frame_location) == (2, 0, 37, 18)


@pytest.mark.parametrize("method,key,value", [
    ("mega", "MODEL.VID.ROI_BOX_HEAD.ATTENTION.STAGE", 2),
    ("mega", "MODEL.VID.ROI_BOX_HEAD.ATTENTION.STAGE", 4),
    ("mega", "MODEL.VID.MEGA.GLOBAL.RES_STAGE", 2),
    ("rdn", "MODEL.VID.ROI_BOX_HEAD.ATTENTION.STAGE", 3),
    ("rdn", "MODEL.VID.ROI_BOX_HEAD.ATTENTION.ADVANCED_STAGE", 2),
])
def test_unserved_layouts_are_rejected_naming_the_key(method, key, value):
    from mega_core.modeling.detector.detectors import vid_config
    from mega_core.modeling.nets import engine_config_from
    cfg = vid_config(method, "R-101-C4", "cpu")
    cfg.merge_from_list([key, value])
    with pytest.raises(NotImplementedError, match=key.split("MODEL.")[1].replace(".", r"\.")):
        engine_config_from(cfg)


@pytest.mark.parametrize("fixture", FIXTURES)
def test_state_dict_gives_the_config(fixture):
    """build_detection_model_from_state_dict infers REDUCE_CHANNEL, GLOBAL.RES_STAGE and ADVANCED_STAGE, loads the
    synthetic weights (which have the reference's keys and shapes) and its engine config is the YAML's"""
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = torch.load(os.path.join(GOLD, fixture))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    want = dict(gold["state_dict_shapes"])
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: v for k, v in want.items() if "cell_anchors" not in k}
    method = gold["arch"].split("_")[0]
    model = build_detection_model_from_state_dict(sd, method=method, device="cpu", precision="tf32")
    v = model.cfg.MODEL.VID
    assert v.ROI_BOX_HEAD.REDUCE_CHANNEL == gold["options"].get("reduce_channel", False)
    ec = engine_config_from(model.cfg)
    if method == "mega":
        assert v.MEGA.GLOBAL.RES_STAGE == ec.global_res_stage == gold["options"]["global_res_stage"]
    else:
        assert v.ROI_BOX_HEAD.ATTENTION.ADVANCED_STAGE == ec.advanced_stage == gold["options"]["advanced_stage"]


def test_served_r101_state_dicts_still_infer_their_layout():
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    for arch, method in (("mega_r101_tiny", "mega"), ("rdn_r101_tiny", "rdn")):
        model = build_detection_model_from_state_dict(synth.make_state_dict(arch, seed=0), method=method, device="cpu")
        v = model.cfg.MODEL.VID
        assert not v.ROI_BOX_HEAD.REDUCE_CHANNEL
        assert v.MEGA.GLOBAL.RES_STAGE == 1 and v.ROI_BOX_HEAD.ATTENTION.ADVANCED_STAGE == (1 if method == "rdn" else 0)


@pytest.mark.parametrize("fixture", FIXTURES)
def test_oracle_matches_the_reference_fixture(fixture):
    """the oracle (+ the reduction conv after res5) against the unmodified reference, first 2 frames"""
    from configs_oracle import oracle_for, reduced_res5
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(GOLD, fixture))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    orc = oracle_for(gold, sd)
    for t, ref in enumerate(gold["frames"][:2]):
        if "globals_per_frame" in gold:
            infos = {"frame_category": 0 if t == 0 else 1,
                     "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                     "ref_g": [frames[j] for j in gold["globals_per_frame"][t]]}
        else:
            infos = {"frame_category": 0 if t == 0 else 1, "ref": frames[1:19] if t == 0 else [frames[min(t + 18, total - 1)]]}
        with reduced_res5():
            b, s, l = orc.forward(frames[t], infos)
        assert torch.allclose(orc.trace["class_logits"], ref["class_logits"], atol=1e-5)
        assert torch.equal(l, ref["labels"]) and b.shape == ref["boxes"].shape
        assert torch.allclose(b, ref["boxes"], atol=2e-3)


def _match_rows(a, b, tol=0.75):
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _check_frame(eng, det, ref, t, logit_tol=1e-3):
    k = int(eng.cur_cnt.view(-1)[0])
    props = eng.Bq0[:k] if hasattr(eng, "Bq0") else eng.last_props[:k]
    idx = _match_rows(props, ref["proposals"])
    assert (idx >= 0).all() and k == ref["proposals"].shape[0], "frame %d: proposals differ" % t
    assert (eng.last_pred[:k][idx, :31] - ref["class_logits"]).abs().max() < logit_tol, "frame %d: class logits" % t
    n = int(det.count.reshape(-1)[0])
    assert n == ref["boxes"].shape[0] and torch.equal(det.labels[:n], ref["labels"]), "frame %d: detections" % t
    assert torch.allclose(det.boxes[:n], ref["boxes"], atol=2e-2)


def _engine_det(eng):
    from mega_core.b200.engine import Detections
    get = lambda tag: [v for (t, _, _), v in eng._bufs.items() if t == tag][0]        # noqa: E731
    return Detections(get("det_boxes"), get("det_scores"), get("det_labels"), get("det_count"))


def test_mega_r50_module_api_matches_reference_fixture():
    """configs/MEGA/vid_R_50_C4_MEGA_1x.yaml through build_detection_model / load_state_dict / model(images) with the
    dict VIDMEGADataset builds: frame 0 with look-ahead and global frames, then two steady frames (the reduction conv in
    the per-frame branch, no G1, the predictor behind stage 2)"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = torch.load(os.path.join(GOLD, "mega_r50_192x320.pt"))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    gpf = gold["globals_per_frame"]
    with cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="mega", device="cpu", precision="tf32")
        assert model.roi_heads.box.feature_extractor.conv is not None
        model._engine = eng = engine.MegaEngine(model.state_dict(), engine_config_from(model.cfg), "cpu")
        assert eng.reduce and len(eng.att_g) == 1 and eng.X4 is None and eng.pooled.shape[1] == 256 * 49
        eng.use_graph = False
        common = {"seg_len": total, "pattern": "%06d", "img_dir": "/nonexistent/%s.JPEG"}
        for t in range(3):
            if t == 0:
                images = {"cur": frames[0][0], "ref_l": [], "ref_g": [frames[j][0] for j in gpf[0]], "frame_category": 0,
                          "lookahead": [f[0] for f in frames[1:13]], **common}
            else:
                images = {"cur": frames[t][0], "ref_l": [frames[min(t + 12, total - 1)][0]],
                          "ref_g": [frames[gpf[t][0]][0]], "frame_category": 1, **common}
            out = model(images)
            ref = gold["frames"][t]
            assert len(out) == 1 and torch.equal(out[0].get_field("labels"), ref["labels"])
            assert torch.allclose(out[0].bbox, ref["boxes"], atol=2e-2)
            _check_frame(eng, _engine_det(eng), ref, t)


@pytest.mark.parametrize("fixture", ["rdnbase_r101_192x320.pt", "rdnbase_r50_192x320.pt"])
def test_rdn_base_engine_matches_reference_fixture(fixture):
    """RdnEngine without the advanced stage (+ the reduction conv for R-50): start_video, then a steady frame"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = torch.load(os.path.join(GOLD, fixture))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    with cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="rdn", device="cpu", precision="tf32")
        eng = engine.RdnEngine(model.state_dict(), engine_config_from(model.cfg), device="cpu")
        assert len(eng.att) == 2 and len(eng.fc_w) == 2 and not hasattr(eng, "Xadv")
        assert eng.reduce == gold["options"].get("reduce_channel", False)
        eng.use_graph = False
        det = eng.start_video(frames[0], frames[1:19], w, h)
        _check_frame(eng, det, gold["frames"][0], 0)
        det = eng.step(frames[19], w, h)
        _check_frame(eng, det, gold["frames"][1], 1)


def test_roi_features_apply_the_reduction():
    """feature_extractor(x, proposals, pre_calculate=True) on an engine with REDUCE_CHANNEL: res5 -> conv + ReLU ->
    ROIAlign -> l_fcs[0] + ReLU, as the oracle computes it"""
    import mega_oracle as mo
    from configs_oracle import reduced_res5
    from mega_core.b200 import engine, synth
    sd = synth.make_state_dict("mega_r50_tiny", seed=2, reduce_channel=True, global_res_stage=0)
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(1, 1024, 12, 20, generator=g).relu()
    boxes = torch.tensor([[10.0, 12.0, 90.0, 140.0], [100.0, 40.0, 300.0, 180.0], [0.0, 0.0, 60.0, 60.0]])
    with cpu_ops():
        eng = engine.MegaEngine(sd, engine.EngineConfig(precision="tf32", global_res_stage=0), device="cpu")
        got = eng.roi_features(feats, boxes, torch.zeros(3, dtype=torch.int32))
    orc = mo.MegaOracle(sd, mo.Cfg(global_res_stage=0))
    with reduced_res5():
        ref = orc._roi_fc(feats, boxes)
    assert (got - ref).abs().max().item() < 1e-4 * max(ref.abs().max().item(), 1.0)


# ------------------------------------------------------------- multi-GPU schedules with GLOBAL.RES_STAGE = 0
W_IMG, H_IMG = 320, 192


def _make(sd, precision="tf32"):
    from mega_core.b200 import engine
    cfg = engine.EngineConfig(precision=precision, all_frame_interval=5, key_frame_location=2, memory_size=4, global_size=2,
                              post_nms_top_n=24, ref_post_nms_top_n=10, global_res_stage=0)
    eng = engine.MegaEngine(sd, cfg, device="cpu")
    eng.use_graph = False
    return eng


def _snap(eng, det, k=None):
    k = int(eng.cur_cnt.view(-1)[0]) if k is None else k
    n = int(det.count.reshape(-1)[0])
    return eng.last_pred[:k].clone(), det.boxes[:n].clone(), det.scores[:n].clone(), det.labels[:n].clone()


RINGS = ("E0", "B0", "Y1E", "Y2M", "B1", "B2", "win_x", "win_boxes", "win_cnt", "glob_x")


@pytest.mark.parametrize("world,precision", [(2, "tf32"), (3, "tf32"), (2, "f16")])
def test_no_g1_schedules_equal_the_sequential_step(world, precision):
    """GLOBAL.RES_STAGE = 0 on the stand-ins: the replicated-state step (owner / state split) and the wavefront step
    (parallel.play) over `world` ranks reproduce the 1-rank step bit for bit -- detections, predictor rows, rings"""
    from mega_core.b200 import parallel, synth
    sd = synth.make_state_dict("mega_r50_tiny", seed=3, reduce_channel=True, global_res_stage=0)
    frames = 2 * world if world == 3 else 3 * world          # > memory_size = 4: the memory ring wraps
    with cpu_ops():
        solo = _make(sd, precision)
        parallel.random_state(solo, 1, W_IMG, H_IMG)
        payloads = [parallel.random_payload(solo, 100 + t, W_IMG, H_IMG) for t in range(frames)]
        seq, seq_k = [], []
        for t in range(frames):
            seq.append(_snap(solo, solo.dist_step(None, W_IMG, H_IMG, rank=0, world=1, payloads=payloads[t][None])[0]))
            seq_k.append(int(solo.cur_cnt.view(-1)[0]))
        assert seq[-1][1].shape[0] > 0, "degenerate test: no detections"
        # replicated state: every rank runs the state rows of every frame, the key rows of its own
        for rank in range(world):
            e = _make(sd, precision)
            parallel.random_state(e, 1, W_IMG, H_IMG)
            for t0 in range(0, frames - world + 1, world):
                dets = e.dist_step(None, W_IMG, H_IMG, rank=rank, world=world, payloads=torch.stack(payloads[t0:t0 + world]))
                assert all(d is None for g, d in enumerate(dets) if g != rank)
                for a, b in zip(seq[t0 + rank], _snap(e, dets[rank], seq_k[t0 + rank])):
                    assert torch.equal(a, b), (rank, t0)
        # wavefront
        ranks = [_make(sd, precision) for _ in range(world)]
        for e in ranks:
            parallel.random_state(e, 1, W_IMG, H_IMG)
        for t0 in range(0, frames, world):
            dets = parallel.play([ranks[r]._wave(None, W_IMG, H_IMG, r, world, payload=payloads[t0 + r])
                                  for r in range(world)])
            for r in range(world):
                for a, b in zip(seq[t0 + r], _snap(ranks[r], dets[r])):
                    assert torch.equal(a, b), "key frame %d: wavefront differs from the sequential step" % (t0 + r)
        offs = {"E0": solo.KP + solo.nl0, "B0": solo.KP + solo.nl0, "Y1E": solo.nq, "Y2M": solo.nq, "B1": solo.nl12,
                "B2": solo.nl12}
        for name in RINGS:
            o = offs.get(name, 0)
            assert torch.equal(getattr(ranks[0], name)[o:], getattr(solo, name)[o:]), name
