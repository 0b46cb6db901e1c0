"""GPU tests of the shipped VID configs with REDUCE_CHANNEL, MEGA.GLOBAL.RES_STAGE = 0 or ATTENTION.ADVANCED_STAGE = 0
(configs/MEGA/vid_R_50_C4_MEGA_1x.yaml, configs/RDN/vid_R_{101,50}_C4_RDN_base_1x.yaml) against the fixtures written from
the unmodified reference (tools/make_golden_configs.py), in every arithmetic; the f16 res5 + reduction layer chain
against per-layer launches; CUDA-graph replay against eager runs; MEGA R-50's multi-GPU schedules played on one GPU."""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FIXTURES = ("mega_r50_192x320.pt", "rdnbase_r101_192x320.pt", "rdnbase_r50_192x320.pt")


def _match_rows(a, b, tol=0.75):
    """for each row of b (reference boxes) the index of an identical-within-tol row of a, or -1"""
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _load(fixture, cuda_dev):
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(GOLD, fixture))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], **gold["options"])
    frames = [synth.synthetic_frame(i, gold["h"], gold["w"]).to(cuda_dev) for i in range(gold["total"])]
    return gold, sd, frames


def _engine(gold, sd, precision, cuda_dev):
    """the engine model(images) builds for the fixture's config (layout inferred from the state dict)"""
    from mega_core.b200 import engine
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    method = gold["arch"].split("_")[0]
    cfg = engine_config_from(build_detection_model_from_state_dict(sd, method=method, device="cpu",
                                                                   precision=precision).cfg)
    cls = engine.MegaEngine if method == "mega" else engine.RdnEngine
    return cls(sd, cfg, device=cuda_dev)


def _steps(gold, eng, frames):
    """the fixture's frame sequence through the engine: yields (t, Detections)"""
    h, w, total = gold["h"], gold["w"], gold["total"]
    for t in range(len(gold["frames"])):
        if "globals_per_frame" in gold:
            gpf = gold["globals_per_frame"]
            det = (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
                   eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))
        else:
            det = eng.start_video(frames[0], frames[1:19], w, h) if t == 0 else eng.step(frames[min(t + 18, total - 1)], w, h)
        yield t, det


def _run(cuda_dev, fixture, precision):
    if precision == "shadow":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from fp32_shadow import fp32_shadow
        with fp32_shadow():
            return _run(cuda_dev, fixture, "tf32")
    gold, sd, frames = _load(fixture, cuda_dev)
    eng = _engine(gold, sd, precision, cuda_dev)
    per_frame = []
    for t, det in _steps(gold, eng, frames):
        ref = gold["frames"][t]
        torch.cuda.synchronize()
        k = int(eng.cur_cnt.view(-1)[0].item())
        props = (eng.Bq0 if hasattr(eng, "Bq0") else eng.last_props)[:k].cpu()
        idx = _match_rows(props, ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].float().cpu()
        assert torch.isfinite(pred).all()
        dabs = (pred[idx[m], :31] - ref["class_logits"][m]).abs()
        b, s, l = det.to_host()
        per_frame.append({"proposals": k, "ref_proposals": int(ref["proposals"].shape[0]),
                          "matched_frac": m.float().mean().item(), "logits_maxabs": dabs.max().item(),
                          "logits_p99": torch.quantile(dabs.flatten(), 0.99).item(),
                          "deltas_maxabs": (pred[idx[m], 31:155] - ref["box_regression"][m]).abs().max().item(),
                          "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0]),
                          "logit_rms": ref["class_logits"].pow(2).mean().sqrt().item()})
        print(fixture, precision, json.dumps(per_frame[-1]))
    return per_frame


@pytest.mark.parametrize("fixture", FIXTURES)
def test_exact_fp32_contractions_match_reference(cuda_dev, fixture):
    """the engine's orchestration (reduction conv, ROIAlign at 256 channels, l_fcs[0] at 196 k-blocks, no G1 / no
    advanced stage) with exact-fp32 contractions: every proposal, logits and deltas within 1e-3, same detection count"""
    for f in _run(cuda_dev, fixture, "shadow"):
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["logits_maxabs"] < 1e-3, f
        assert f["deltas_maxabs"] < 1e-3, f
        assert f["dets"] == f["ref_dets"], f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_fp32x3_matches_reference(cuda_dev, fixture):
    """strict mode (split-fp16 res5 + reduction, split-fp16 ROIAlign at 256 channels): every proposal and detection,
    logits within 1e-2, deltas within 5e-3"""
    for f in _run(cuda_dev, fixture, "fp32x3"):
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["dets"] == f["ref_dets"], f
        assert f["logits_maxabs"] < 1e-2, f
        assert f["deltas_maxabs"] < 5e-3, f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_tf32_matches_reference(cuda_dev, fixture):
    """the R-101 statistical bars of tests/test_engine_gpu.py"""
    for f in _run(cuda_dev, fixture, "tf32"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_maxabs"] < 0.15, f
        assert f["proposals"] == f["ref_proposals"], f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_f16_matches_reference(cuda_dev, fixture):
    """the R-101 statistical bars of tests/test_engine_gpu.py (MEGA's, RDN's for the RDN configs)"""
    p99, mx = (3e-2, 0.5) if fixture.startswith("mega") else (5e-2, 1.0)
    for f in _run(cuda_dev, fixture, "f16"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_p99"] < p99, f
        assert f["logits_maxabs"] < mx, f
        assert f["proposals"] == f["ref_proposals"], f


@pytest.mark.parametrize("n", [2, 4])
def test_f16_res5_reduction_chain_equals_per_layer_launches(cuda_dev, n):
    """res5 + the 2048 -> 256 reduction conv as one persistent chain kernel (n = 4: two interleaved lanes, each lane's
    reduction after its own res5 layers) and as per-layer launches over the same images: bit-identical"""
    from mega_core.b200 import ops
    gold, sd, _ = _load("mega_r50_192x320.pt", cuda_dev)
    g = torch.Generator().manual_seed(n)
    feats = (torch.randn(n, 12, 20, 1024, generator=g).relu()).half().to(cuda_dev)
    saved = ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0], ops.DUAL_CHAIN[0]
    try:
        eng = _engine(gold, sd, "f16", cuda_dev)
        ops.AUTOTUNE[0], ops.DUAL_CHAIN[0] = False, True
        dual = n >= ops.DUAL_MIN_IMAGES

        def run(x):
            with ops.chain(eng._chains, ("test_res5", tuple(x.shape), dual), eng.dev, enabled=True, interleave=dual) as ch:
                y = eng.res5_reduced(x, ch if dual else None)
            return y.clone()            # (the recorded chain runs when the block exits)
        y_chain, y_chain2 = run(feats), run(feats)
        ops.CHAINS_ENABLED[0] = False
        ops.MAX_BN[0] = 128                             # the widest tile a chain layer may pick
        ref = eng.__class__(sd, eng.cfg, device=cuda_dev)
        ops.AUTOTUNE[0] = False
        halves = (feats[:n // 2], feats[n // 2:]) if dual else (feats,)     # a lane's launches see its half of the batch
        y_layers = torch.cat([ref.res5_reduced(x.contiguous()).clone() for x in halves])
    finally:
        ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0], ops.DUAL_CHAIN[0] = saved
    torch.cuda.synchronize()
    assert y_chain.shape == (n, 12, 20, 256) and len(eng._chains) == 1
    assert torch.isfinite(y_chain.float()).all() and (y_chain > 0).any()
    assert torch.equal(y_chain, y_chain2)
    assert torch.equal(y_chain, y_layers), (y_chain.float() - y_layers.float()).abs().max().item()


@pytest.mark.parametrize("fixture", FIXTURES)
@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_graph_replay_equals_eager(cuda_dev, fixture, precision):
    """the steady frames as captured CUDA graphs and as eager launches: identical detections and predictor rows"""
    from mega_core.b200 import ops
    gold, sd, frames = _load(fixture, cuda_dev)
    outs = []
    for use_graph in (False, True):
        eng = _engine(gold, sd, precision, cuda_dev)
        ops.AUTOTUNE[0] = False
        eng.use_graph = use_graph
        snaps = []
        for t, det in _steps(gold, eng, frames):
            torch.cuda.synchronize()
            k = int(eng.cur_cnt.view(-1)[0].item())
            snaps.append((eng.last_pred[:k].clone().cpu(),) + det.to_host())
        outs.append(snaps)
        if use_graph:
            assert eng._graphs, "no graph was captured"
        del eng
    for t, (a, b) in enumerate(zip(*outs)):
        for x, y in zip(a, b):
            assert torch.equal(x, y), "frame %d: graph replay differs from eager" % t


def test_mega_r50_frame_parallel_and_wavefront_equal_one_rank(cuda_dev):
    """MEGA R-50 (no G1: the predictor behind stage 2) across world sizes, two and three ranks played on one GPU: the
    replicated-state step gives the 1-rank results bit for bit on real frames; the wavefront step passes the self-check
    that bench.py runs before it uses it (parallel.wave_selfcheck: bit-identical to the sequential step)"""
    from mega_core.b200 import engine, parallel
    gold, sd, frames = _load("mega_r50_192x320.pt", cuda_dev)
    h, w = gold["h"], gold["w"]
    cfg = _engine(gold, sd, "f16", cuda_dev).cfg
    assert cfg.global_res_stage == 0
    glob0 = [frames[(3 * j + 1) % 24] for j in range(10)]
    pair = lambda t: torch.cat([frames[(t + 12) % 24], frames[(5 * t + 3) % 24]], 0)      # noqa: E731
    steps = 4

    def make():
        e = engine.MegaEngine(sd, cfg, device=cuda_dev)
        e.start_video(frames[0], frames[1:13], glob0, w, h)
        return e

    def snap(e, det):
        torch.cuda.synchronize()
        k = int(e.cur_cnt.view(-1)[0].item())
        return (e.last_pred[:k].clone().cpu(),) + det.to_host()

    ranker = make()
    payloads = [ranker.ref_payload(pair(t), w, h) for t in range(1, steps + 1)]
    solo = make()
    out_solo = [snap(solo, solo.dist_step(None, w, h, rank=0, world=1, payloads=payloads[t][None])[0])
                for t in range(steps)]
    for rank in (0, 1):
        e = make()
        for t in range(0, steps, 2):
            dets = e.dist_step(None, w, h, rank=rank, world=2, payloads=torch.stack(payloads[t:t + 2]))
            assert dets[1 - rank] is None
            for a, b in zip(out_solo[t + rank], snap(e, dets[rank])):
                assert torch.equal(a, b), "frame %d differs between 1 and 2 ranks" % (t + rank)
    assert out_solo[-1][1].shape[0] > 0
    for world in (2, 3):
        ok, msg = parallel.wave_selfcheck(lambda: engine.MegaEngine(sd, cfg, device=cuda_dev), w, h, world=world,
                                          groups=2)
        assert ok, msg
