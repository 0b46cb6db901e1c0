"""CPU tests of MEGA without long-range memory (MODEL.VID.MEGA.MEMORY.ENABLE False): the config is served and passed to
the engine, GLOBAL.ENABLE False stays refused, the memory-on config is unchanged; the oracle without memory
(tests/mega_nomem_oracle.py) and MegaEngine's host logic on the CPU stand-ins (tests/cpu_ops.py) against the fixtures
tools/make_golden_mega_nomem.py wrote from the unmodified reference; the wavefront schedule without increment stages,
symbolically and as the engine's real code, against the sequential step; the dataset's test items with the key off."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLD = os.path.join(ROOT, "tests", "golden")

from configs_oracle import reduced_res5  # noqa: E402
from cpu_ops import cpu_ops  # noqa: E402
from mega_nomem_oracle import MegaNoMemOracle  # noqa: E402
import mega_oracle as mo  # noqa: E402

FIXTURES = ("mega_r101_nomem_192x320.pt", "mega_r50_nomem_192x320.pt")
W_IMG, H_IMG = 320, 192


def _config(method="mega", body="R-101-C4", memory=False, **kw):
    from mega_core.modeling.detector.detectors import vid_config
    cfg = vid_config(method, body, "cpu", **kw)
    cfg.MODEL.VID.MEGA.MEMORY.ENABLE = memory
    return cfg


@pytest.mark.parametrize("res_stage", [0, 1])
def test_config_is_served_and_passed_to_the_engine(res_stage):
    from mega_core.modeling.nets import engine_config_from
    cfg = _config()
    cfg.MODEL.VID.MEGA.GLOBAL.RES_STAGE = res_stage
    ec = engine_config_from(cfg)
    assert ec.memory is False and ec.global_res_stage == res_stage


@pytest.mark.parametrize("body", ["deformable", "x101", "x101_s3x3"])
def test_config_is_served_on_other_bodies(body):
    from mega_core.modeling.nets import engine_config_from
    if body == "deformable":
        cfg = _config()
        cfg.MODEL.RESNETS.STAGE_WITH_DCN = (False, True, True, False)
        cfg.MODEL.RESNETS.WITH_MODULATED_DCN = True
    else:
        cfg = _config(num_groups=32, width_per_group=8, stride_in_1x1=body != "x101_s3x3")
    for precision in ("f16", "fp32x3"):
        cfg.MODEL.B200.PRECISION = precision
        ec = engine_config_from(cfg)
        assert ec.memory is False and ec.precision == precision


def test_global_disabled_is_still_refused_naming_it():
    from mega_core.modeling.nets import engine_config_from
    for memory in (True, False):
        cfg = _config(memory=memory)
        cfg.MODEL.VID.MEGA.GLOBAL.ENABLE = False
        with pytest.raises(NotImplementedError, match="GLOBAL.ENABLE") as e:
            engine_config_from(cfg)
        assert "MEMORY" not in str(e.value)


def test_memory_on_config_builds_the_same_engine_config():
    """the default (MEMORY.ENABLE True) passes no `memory` option: the EngineConfig is the one it always was"""
    from mega_core.b200 import engine
    from mega_core.modeling.nets import engine_config_from
    on = engine_config_from(_config(memory=True))
    assert "memory" not in vars(on) and on.memory is True and engine.EngineConfig.memory is True
    off = engine_config_from(_config(memory=False))
    assert {k: v for k, v in vars(off).items() if k != "memory"} == vars(on)


def test_other_methods_ignore_the_key():
    from mega_core.modeling.nets import engine_config_from
    for method in ("base", "dff", "fgfa", "rdn"):
        assert "memory" not in vars(engine_config_from(_config(method)))


def test_engine_without_memory_allocates_no_rings():
    from mega_core.b200 import engine, synth
    sd = synth.make_state_dict("mega_r101_tiny", seed=3)
    with cpu_ops():
        on = engine.MegaEngine(sd, engine.EngineConfig(precision="tf32"), device="cpu")
        off = engine.MegaEngine(sd, engine.EngineConfig(precision="tf32", memory=False), device="cpu")
    assert off.MEMF == off.mem_cap0 == off.mem_cap12 == 0 and on.MEMF == 25
    assert off.E0.shape[0] == 300 + 1875 and off.Y1E.shape[0] == off.nq == 675 and off.B1.shape[0] == 375
    assert (off.ld_0, off.ld_12) == (1888, 384) and (on.ld_0, on.ld_12) == (3776, 768)


# ------------------------------------------------------------------------------------------------- fixtures
def _gold(fixture):
    """the fixture, with its stored frames by frame index (the first three are always stored)"""
    gold = torch.load(os.path.join(GOLD, fixture))
    assert gold["memory"] is False
    gold["by_t"] = {f["t"]: f for f in gold["frames"]}
    assert all(t in gold["by_t"] for t in range(3))
    return gold


def _infos(gold, frames, t):
    total, gpf = gold["total"], gold["globals_per_frame"]
    return {"frame_category": 0 if t == 0 else 1,
            "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
            "ref_g": [frames[j] for j in gpf[t]]}


def _res5(gold):
    import contextlib
    return reduced_res5() if gold["options"].get("reduce_channel") else contextlib.nullcontext()


@pytest.mark.parametrize("fixture", FIXTURES)
def test_oracle_matches_the_reference_fixture(fixture):
    """the oracle without memory against the unmodified reference (first three frames: memory would be non-empty from
    frame 1 on)"""
    from mega_core.b200 import synth
    gold = _gold(fixture)
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, gold["h"], gold["w"]) for i in range(gold["total"])]
    orc = MegaNoMemOracle(sd, mo.Cfg(global_res_stage=gold["options"].get("global_res_stage", 1)), record=True)
    for t in range(3):
        ref = gold["by_t"][t]
        with _res5(gold):
            b, s, l = orc.forward(frames[t], _infos(gold, frames, t))
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
    idx = _match_rows(eng.Bq0[:k], ref["proposals"])
    assert (idx >= 0).all() and k == ref["proposals"].shape[0], "frame %d: proposals differ" % t
    assert (eng.last_pred[:k][idx, :31] - ref["class_logits"]).abs().max() < logit_tol, "frame %d: class logits" % t
    n = int(det.count.reshape(-1)[0])
    assert n == ref["boxes"].shape[0] and torch.equal(det.labels[:n], ref["labels"]), "frame %d: detections" % t
    assert torch.allclose(det.boxes[:n], ref["boxes"], atol=2e-2)


@pytest.mark.parametrize("fixture", FIXTURES)
def test_engine_matches_the_reference_fixture(fixture):
    """a reference-format checkpoint loaded into the model with MEMORY.ENABLE False, its engine (from
    engine_config_from) on the stand-ins: frame 0 with look-ahead and global frames, then steady frames"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model
    from mega_core.modeling.nets import engine_config_from
    gold = _gold(fixture)
    h, w, total, gpf = gold["h"], gold["w"], gold["total"], gold["globals_per_frame"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    cfg = _config(body="R-50-C4" if "r50" in gold["arch"] else "R-101-C4")
    cfg.MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL = gold["options"].get("reduce_channel", False)
    cfg.MODEL.VID.MEGA.GLOBAL.RES_STAGE = gold["options"].get("global_res_stage", 1)
    cfg.MODEL.B200.PRECISION = "tf32"
    model = build_detection_model(cfg)
    full = dict(sd)
    full["rpn.anchor_generator.cell_anchors.0"] = model.state_dict()["rpn.anchor_generator.cell_anchors.0"]
    model.load_state_dict(full, strict=True)
    with cpu_ops():
        eng = engine.MegaEngine(model.state_dict(), engine_config_from(model.cfg), device="cpu")
        assert eng.MEMF == 0
        eng.use_graph = False
        for t in range(3):
            det = (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
                   eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))
            _check_frame(eng, det, gold["by_t"][t], t)


# -------------------------------------------------------------------- wavefront schedule without increments
def test_wave_tables_of_a_schedule_without_memory_are_empty():
    from mega_core.b200 import parallel
    for world in (1, 2, 3, 8, 30):           # no ring: a group of any size fits
        for rank in range(world):
            tabs = parallel.wave_tables(17, rank, world, 75, 15, 0, 2175, 675, 375)
            assert set(tabs) == {"valid"} and tabs["valid"].tolist() == [0] * world


def _symbolic_sequential(payloads, L):
    """frame t's result is a function of the window (the last L payloads) alone"""
    win, out = [], []
    for p in payloads:
        win = (win + [p])[-L:]
        out.append(hash(tuple(win)))
    return out


def _symbolic_wave(window, rank, world, own):
    """one rank of the no-increment schedule: one gather of the payloads, ingest up to the own frame, aggregate, ingest
    the rest; `window` is the rank's replica (a list, updated in place)"""
    L = len(window)
    got = yield torch.tensor([own]), torch.zeros(world, 1, dtype=torch.long)
    pays = got.reshape(-1).tolist()
    for p in pays[:rank + 1]:
        window[:] = (window + [p])[-L:]
    res = hash(tuple(window))
    for p in pays[rank + 1:]:
        window[:] = (window + [p])[-L:]
    return res


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_symbolic_schedule_without_increments_equals_sequential(world):
    from mega_core.b200 import parallel
    L, groups = 5, 4                         # groups * world > L: the window wraps
    start = list(range(-L, 0))
    payloads = [1000 + t for t in range(groups * world)]
    seq = _symbolic_sequential(start + payloads, L)[L:]
    ranks = [list(start) for _ in range(world)]
    for g in range(groups):
        outs = parallel.play([_symbolic_wave(ranks[r], r, world, payloads[g * world + r]) for r in range(world)])
        assert outs == seq[g * world:(g + 1) * world]
        assert all(w == ranks[0] for w in ranks)


def _make(sd, precision="tf32", memory=False):
    from mega_core.b200 import engine
    cfg = engine.EngineConfig(precision=precision, all_frame_interval=5, key_frame_location=2, memory_size=4, global_size=2,
                              post_nms_top_n=24, ref_post_nms_top_n=10, memory=memory)          # R = 10, A = 2, KP = 24
    eng = engine.MegaEngine(sd, cfg, device="cpu")
    eng.use_graph = False
    return eng


def _snap(eng, det, k=None):
    k = int(eng.cur_cnt.view(-1)[0]) if k is None else k
    n = int(det.count.reshape(-1)[0])
    return eng.last_pred[:k].clone(), det.boxes[:n].clone(), det.scores[:n].clone(), det.labels[:n].clone()


@pytest.mark.parametrize("world,precision", [(2, "tf32"), (3, "tf32"), (2, "f16")])
def test_engine_schedules_without_memory_equal_the_sequential_step(world, precision):
    """the engine's real host code on the stand-ins, memory off: the replicated-state step and the wavefront step (one
    gather per group, no increments) over `world` ranks give the 1-rank results bit for bit, across window wrap-around;
    and the results are not those of the engine with memory"""
    from mega_core.b200 import parallel, synth
    sd = synth.make_state_dict("mega_r101_tiny", seed=3)
    frames = 2 * world if world == 3 else 3 * world      # > all_frame_interval = 5: the window ring wraps
    with cpu_ops():
        solo = _make(sd, precision)
        parallel.random_state(solo, 1, W_IMG, H_IMG)
        payloads = [parallel.random_payload(solo, 100 + t, W_IMG, H_IMG) for t in range(frames)]
        seq, seq_k = [], []
        for t in range(frames):
            seq.append(_snap(solo, solo.dist_step(None, W_IMG, H_IMG, rank=0, world=1, payloads=payloads[t][None])[0]))
            seq_k.append(int(solo.cur_cnt.view(-1)[0]))
        assert seq[-1][1].shape[0] > 0, "degenerate test: no detections"
        with_mem = _make(sd, precision, memory=True)
        parallel.random_state(with_mem, 1, W_IMG, H_IMG)
        mem = [_snap(with_mem, with_mem.dist_step(None, W_IMG, H_IMG, rank=0, world=1, payloads=payloads[t][None])[0])
               for t in range(3)]
        # frame 0 reads an empty memory either way; later frames relate their rows to it
        assert torch.allclose(mem[0][0], seq[0][0], atol=1e-5) and (mem[2][0] - seq[2][0]).abs().max() > 1e-4
        for rank in range(world):
            e = _make(sd, precision)
            parallel.random_state(e, 1, W_IMG, H_IMG)
            for t0 in range(0, frames, world):
                dets = e.dist_step(None, W_IMG, H_IMG, rank=rank, world=world, payloads=torch.stack(payloads[t0:t0 + world]))
                assert all(d is None for g, d in enumerate(dets) if g != rank)
                for a, b in zip(seq[t0 + rank], _snap(e, dets[rank], seq_k[t0 + rank])):
                    assert torch.equal(a, b), (rank, t0)
        ranks = [_make(sd, precision) for _ in range(world)]
        for e in ranks:
            parallel.random_state(e, 1, W_IMG, H_IMG)
        collectives = []

        def counted(gen):
            msg = next(gen)
            try:
                while True:
                    collectives.append(msg[0].numel())
                    msg = gen.send((yield msg))
            except StopIteration as stop:
                return stop.value
        for t0 in range(0, frames, world):
            dets = parallel.play([counted(ranks[r]._wave(None, W_IMG, H_IMG, r, world, payload=payloads[t0 + r]))
                                  for r in range(world)])
            for r in range(world):
                for a, b in zip(seq[t0 + r], _snap(ranks[r], dets[r])):
                    assert torch.equal(a, b), "key frame %d: wavefront differs from the sequential step" % (t0 + r)
        # one all-gather per group, of the frame payloads: no increment stages
        assert collectives == [solo.payload_in.numel()] * (frames // world * world)
        for r in range(world):
            for name in ("win_x", "win_boxes", "win_cnt", "glob_x"):
                assert torch.equal(getattr(ranks[r], name), getattr(solo, name)), (name, r)
            assert list(ranks[r].win_slots) == list(solo.win_slots)


def test_wave_selfcheck_without_memory():
    """parallel.wave_selfcheck on engines without memory: passes on the real schedule, and reports a broken one in
    which every rank ingests the whole group before it aggregates its key frame"""
    from mega_core.b200 import engine, parallel, synth
    sd = synth.make_state_dict("mega_r101_tiny", seed=3)
    with cpu_ops():
        for world in (2, 3):
            ok, msg = parallel.wave_selfcheck(lambda: _make(sd), W_IMG, H_IMG, world=world, groups=3, use_graph=False)
            assert ok, msg
        orig = engine.MegaEngine._wave

        def broken(self, imgs, im_w, im_h, rank, world, payload=None):
            return orig(self, imgs, im_w, im_h, world - 1, world, payload)
        engine.MegaEngine._wave = broken
        try:
            ok, msg = parallel.wave_selfcheck(lambda: _make(sd), W_IMG, H_IMG, world=2, groups=3, use_graph=False)
        finally:
            engine.MegaEngine._wave = orig
        assert not ok and "differs" in msg


# ------------------------------------------------------------------------------------------------- data
def test_dataset_test_items_do_not_depend_on_the_key(tmp_path):
    """the reference's VIDMEGADataset reads MEMORY.ENABLE only for training-time memory frames (vid_mega.py:47-76):
    the package's test items are the same with the key off"""
    from test_datasets_cpu import _datasets, make_tree
    from mega_core.config import cfg
    make_tree(str(tmp_path))
    items = {}
    saved = cfg.MODEL.VID.MEGA.MEMORY.ENABLE
    try:
        for memory in (True, False):
            cfg.MODEL.VID.MEGA.MEMORY.ENABLE = memory
            ds = _datasets(str(tmp_path))["mega"]
            np.random.seed(1)
            items[memory] = [ds[i] for i in range(len(ds))]
    finally:
        cfg.MODEL.VID.MEGA.MEMORY.ENABLE = saved
    assert len(items[True]) == len(items[False]) > 0
    for (a, ta, ia), (b, tb, ib) in zip(items[True], items[False]):
        assert ia == ib and sorted(a) == sorted(b) and torch.equal(a["cur"], b["cur"])
        assert a["frame_category"] == b["frame_category"]
        for key in ("ref_l", "ref_g"):
            assert len(a[key]) == len(b[key]) and all(torch.equal(x, y) for x, y in zip(a[key], b[key]))
        assert torch.equal(ta.bbox, tb.bbox)
