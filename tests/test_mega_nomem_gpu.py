"""GPU tests of MEGA without long-range memory (MODEL.VID.MEGA.MEMORY.ENABLE False): both fixtures written from the
unmodified reference (tools/make_golden_mega_nomem.py) in the strict and the throughput arithmetic, under the bars of
the memory-on fixture tests; the difference from the memory-on engine; CUDA-graph replay, stepn_batched, and the
replicated-state and wavefront multi-GPU steps (ranks played on one device) against the single-frame step."""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FIXTURES = ("mega_r101_nomem_192x320.pt", "mega_r50_nomem_192x320.pt")


def _match_rows(a, b, tol=0.75):
    """for each row of b (reference boxes) the index of an identical-within-tol row of a, or -1"""
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _load(fixture, cuda_dev):
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(GOLD, fixture))
    assert gold["memory"] is False
    gold["by_t"] = {f["t"]: f for f in gold["frames"]}
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, gold["h"], gold["w"]).to(cuda_dev) for i in range(gold["total"])]
    return gold, sd, frames


def _cfg(sd, precision, memory=False):
    """the EngineConfig model(images) builds for the fixture's checkpoint with MEMORY.ENABLE set to `memory`"""
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    cfg = build_detection_model_from_state_dict(sd, method="mega", device="cpu", precision=precision).cfg.clone()
    cfg.defrost()
    cfg.MODEL.VID.MEGA.MEMORY.ENABLE = memory
    return engine_config_from(cfg)


def _steps(gold, eng, frames, n=None):
    h, w, total, gpf = gold["h"], gold["w"], gold["total"], gold["globals_per_frame"]
    for t in range(n or gold["n_frames"]):
        yield t, (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
                  eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))


def _snap(eng, det):
    torch.cuda.synchronize()
    k = int(eng.cur_cnt.view(-1)[0].item())
    return (eng.last_pred[:k].clone().cpu(),) + det.to_host()


@pytest.mark.parametrize("fixture", FIXTURES)
@pytest.mark.parametrize("precision", ["fp32x3", "f16"])
def test_matches_reference_fixture(cuda_dev, fixture, precision):
    """all frames of the fixture's stream, checked at the frames it stores: strict mode: every proposal and every
    detection, logits within 1e-2 (the bar of the memory-on fixtures); f16: the statistical bars of the memory-on f16
    tests"""
    from mega_core.b200 import engine
    gold, sd, frames = _load(fixture, cuda_dev)
    cfg = _cfg(sd, precision)
    assert cfg.memory is False and cfg.global_res_stage == gold["options"].get("global_res_stage", 1)
    eng = engine.MegaEngine(sd, cfg, device=cuda_dev)
    assert eng.MEMF == 0
    checked = []
    for t, det in _steps(gold, eng, frames):
        ref = gold["by_t"].get(t)
        if ref is None:
            continue
        checked.append(t)
        torch.cuda.synchronize()
        k = int(eng.cur_cnt.view(-1)[0].item())
        idx = _match_rows(eng.Bq0[:k].cpu(), ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].float().cpu()
        assert torch.isfinite(pred).all()
        dabs = (pred[idx[m], :31] - ref["class_logits"][m]).abs()
        b, s, l = det.to_host()
        f = {"t": t, "proposals": k, "ref_proposals": int(ref["proposals"].shape[0]), "matched": m.float().mean().item(),
             "logits_maxabs": dabs.max().item(), "logits_p99": torch.quantile(dabs.flatten(), 0.99).item(),
             "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0])}
        print(fixture, precision, json.dumps(f))
        assert f["proposals"] == f["ref_proposals"], f
        if precision == "fp32x3":
            assert f["matched"] == 1.0 and f["dets"] == f["ref_dets"] and f["logits_maxabs"] < 1e-2, f
        else:
            assert f["matched"] >= 0.95 and f["logits_p99"] < 3e-2 and f["logits_maxabs"] < 0.5, f
    assert checked == sorted(gold["by_t"])


def test_detections_differ_from_the_memory_on_engine(cuda_dev):
    """same checkpoint, same stream: frame 0 reads an empty memory either way; with a memory of 8 and 9 frames the
    reference's logits differ by 4.2e-2 and 4.5e-2 between memory on and off (tools/make_golden_mega_nomem.py), four
    times the strict mode's bar against the reference, and so do the engines'"""
    from mega_core.b200 import engine
    gold, sd, frames = _load("mega_r101_nomem_192x320.pt", cuda_dev)
    outs = {}
    for memory in (False, True):
        eng = engine.MegaEngine(sd, _cfg(sd, "fp32x3", memory), device=cuda_dev)
        outs[memory] = [_snap(eng, det) for _, det in _steps(gold, eng, frames, 10)]
        del eng
    for t in (0, 8, 9):
        a, b = outs[False][t], outs[True][t]
        diff = (a[0] - b[0]).abs().max().item() if a[0].shape == b[0].shape else float("inf")
        if t == 0:
            assert diff < 1e-2 and torch.equal(a[3], b[3]), diff
        else:
            assert diff > 2e-2, (t, diff)
            assert a[1].shape != b[1].shape or not torch.equal(a[2], b[2]), t


@pytest.mark.parametrize("fixture", FIXTURES)
@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_graph_replay_equals_eager(cuda_dev, fixture, precision):
    """the steady frames as captured CUDA graphs (eager on first use, captured on the second, replayed on the third) and
    as eager launches: identical detections and predictor rows"""
    from mega_core.b200 import engine, ops
    gold, sd, frames = _load(fixture, cuda_dev)
    outs = []
    for use_graph in (False, True):
        eng = engine.MegaEngine(sd, _cfg(sd, precision), device=cuda_dev)
        ops.AUTOTUNE[0] = False
        eng.use_graph = use_graph
        outs.append([_snap(eng, det) for _, det in _steps(gold, eng, frames, 4)])
        if use_graph:
            assert eng._graphs, "no graph was captured"
        del eng
    for t, (a, b) in enumerate(zip(*outs)):
        for x, y in zip(a, b):
            assert torch.equal(x, y), "frame %d: graph replay differs from eager" % t


def _stream(gold, frames):
    total = gold["total"]
    glob0 = [frames[(3 * j + 1) % total] for j in range(10)]
    pair = lambda t: torch.cat([frames[(t + 12) % total], frames[(5 * t + 3) % total]], 0)      # noqa: E731
    return glob0, pair


@pytest.mark.parametrize("precision", ["fp32x3", "f16"])
def test_stepn_batched_equals_one_step_per_frame(cuda_dev, precision):
    """four key frames per call against four step_batched calls: a different batch moves the stream-K split points of
    the per-frame branch, so the comparison has the bounds of the memory-on pipelined-step test"""
    from mega_core.b200 import engine
    gold, sd, frames = _load("mega_r101_nomem_192x320.pt", cuda_dev)
    h, w = gold["h"], gold["w"]
    glob0, pair = _stream(gold, frames)
    cfg = _cfg(sd, precision)
    a, b = engine.MegaEngine(sd, cfg, device=cuda_dev), engine.MegaEngine(sd, cfg, device=cuda_dev)
    for e in (a, b):
        e.start_video(frames[0], frames[1:13], glob0, w, h)
    tol, cnt_tol = (2e-3, 0) if precision == "fp32x3" else (2e-2, 3)
    for s in range(2):
        ts = range(1 + 4 * s, 5 + 4 * s)
        want = []
        for t in ts:
            det = a.step_batched(pair(t), w, h)
            torch.cuda.synchronize()
            k = int(a.cur_cnt.view(-1)[0].item())
            want.append((int(det.count.item()), a.last_pred[:k].float().cpu(), a.Bq0[:k].cpu()))
        dets = b.stepn_batched(torch.cat([pair(t) for t in ts], 0), w, h)
        torch.cuda.synchronize()
        assert all(abs(int(d.count.item()) - x[0]) <= cnt_tol for d, x in zip(dets, want))
        k = int(b.cur_cnt.view(-1)[0].item())
        idx = _match_rows(b.Bq0[:k].cpu(), want[-1][2])
        m = idx >= 0
        assert m.float().mean().item() >= (1.0 if precision == "fp32x3" else 0.95)
        d = (b.last_pred[:k].float().cpu()[idx[m], :31] - want[-1][1][m, :31]).abs()
        assert torch.quantile(d.flatten(), 0.99).item() < tol


@pytest.mark.parametrize("fixture", FIXTURES)
@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_multi_gpu_steps_equal_one_rank(cuda_dev, fixture, precision):
    """two ranks played on one device: the replicated-state step (dist_step) gives the 1-rank results bit for bit; the
    wavefront step (what dist_step_wave / dist_stepn_wave drive, one all-gather of the payloads per group) gives the
    sequential step's results bit for bit; parallel.wave_selfcheck passes for two and three ranks"""
    from mega_core.b200 import engine, parallel
    gold, sd, frames = _load(fixture, cuda_dev)
    h, w = gold["h"], gold["w"]
    glob0, pair = _stream(gold, frames)
    cfg = _cfg(sd, precision)
    steps = 6

    def make():
        e = engine.MegaEngine(sd, cfg, device=cuda_dev)
        e.start_video(frames[0], frames[1:13], glob0, w, h)
        return e

    ranker = make()
    payloads = [ranker.ref_payload(pair(t), w, h) for t in range(1, steps + 1)]
    solo = make()
    out_solo = [_snap(solo, solo.dist_step(None, w, h, rank=0, world=1, payloads=payloads[t][None])[0])
                for t in range(steps)]
    assert out_solo[-1][1].shape[0] > 0
    for rank in (0, 1):
        e = make()
        for t in range(0, steps, 2):
            dets = e.dist_step(None, w, h, rank=rank, world=2, payloads=torch.stack(payloads[t:t + 2]))
            assert dets[1 - rank] is None
            k = out_solo[t + rank][0].shape[0]
            got = (e.last_pred[:k].clone().cpu(),) + dets[rank].to_host()
            for a, b in zip(out_solo[t + rank], got):
                assert torch.equal(a, b), "frame %d differs between 1 and 2 ranks" % (t + rank)
    ranks = [make(), make()]
    for t in range(0, steps, 2):
        dets = parallel.play([ranks[r]._wave(None, w, h, r, 2, payload=payloads[t + r]) for r in range(2)])
        for r in range(2):
            for a, b in zip(out_solo[t + r], _snap(ranks[r], dets[r])):
                assert torch.equal(a, b), "frame %d differs between the sequential and the wavefront schedule" % (t + r)
    for name in ("win_x", "win_boxes", "win_cnt", "glob_x"):
        for r in range(2):
            assert torch.equal(getattr(ranks[r], name), getattr(solo, name)), (name, r)
    for world in (2, 3):
        ok, msg = parallel.wave_selfcheck(lambda: engine.MegaEngine(sd, cfg, device=cuda_dev), w, h, world=world,
                                          groups=2)
        assert ok, msg
