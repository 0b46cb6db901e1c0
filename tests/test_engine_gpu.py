"""End-to-end GPU parity of the B200 engine against the REFERENCE's outputs (fixtures produced by
oracle/make_golden.py from the unmodified reference) and against the oracle run live.

Dense contractions run in TF32 (10-bit mantissa operands, fp32 accumulate), so upstream scores
differ from fp32 at the 1e-3 relative level and a few near-tied proposals may be selected
differently; the comparison therefore (a) matches proposals geometrically, (b) compares class
logits / box deltas on matched rows with the tolerance from BASELINE.json's north_star (1e-3 abs
is the target; the measured value is written to gpurun_out/engine_parity.json and asserted
against the bound stated in each test).
"""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
_METRICS = {}


def _dump():
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "engine_parity.json"), "w") as fh:
        json.dump(_METRICS, fh, indent=1)


def _match_rows(a, b, tol=0.75):
    """for each row of b (reference boxes) the index of an identical-within-tol row of a, or -1"""
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)       # [na, nb]
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def test_backbone_matches_oracle(cuda_dev):
    import mega_oracle as mo
    from mega_core.b200 import engine, synth
    sd = synth.make_state_dict("mega_r101_tiny", seed=2)
    img = synth.synthetic_frame(1, 96, 160)
    ref = mo.resnet_c4_body(img, sd)                                       # [1,1024,6,10]
    bb = engine.Backbone({k: v for k, v in sd.items()}, cuda_dev)
    got = bb.forward(img.to(cuda_dev)).permute(0, 3, 1, 2).cpu()
    rel = ((got - ref).abs().max() / ref.pow(2).mean().sqrt()).item()
    _METRICS["backbone_tiny_relerr"] = rel
    _dump()
    assert rel < 2e-2, rel


def test_base_r50_matches_reference_fixture(cuda_dev):
    from mega_core.b200 import engine, synth
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "base_r50_192x320.pt"))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    img = synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"]).to(cuda_dev)
    eng = engine.BaseEngine(sd, device=cuda_dev)
    det = eng.forward(img, gold["w"], gold["h"])
    torch.cuda.synchronize()
    k = int(eng.last_cnt[0].item())
    props = eng.last_props[:k].cpu()
    idx = _match_rows(props, gold["proposals"])
    frac = (idx >= 0).float().mean().item()
    pred = eng.last_pred[:k].cpu()
    m = idx >= 0
    dl = (pred[idx[m], :31] - gold["class_logits"][m]).abs().max().item()
    db = (pred[idx[m], 31:155] - gold["box_regression"][m]).abs().max().item()
    b, s, l = det.to_host()
    _METRICS["base_r50"] = {"proposals": k, "ref_proposals": int(gold["proposals"].shape[0]), "matched_frac": frac,
                            "logits_maxabs": dl, "deltas_maxabs": db, "dets": int(b.shape[0]),
                            "ref_dets": int(gold["boxes"].shape[0]),
                            "logit_rms": gold["class_logits"].pow(2).mean().sqrt().item()}
    _dump()
    assert frac > 0.9, frac
    assert dl < 5e-3, dl


def _run_mega_against_fixture(cuda_dev, label, precision="tf32"):
    from mega_core.b200 import engine, synth
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "mega_r101_192x320.pt"))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(total)]
    eng = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev)
    gpf = gold["globals_per_frame"]
    per_frame = []
    for t, ref in enumerate(gold["frames"]):
        if t == 0:
            det = eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h)
        else:
            det = eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h)
        torch.cuda.synchronize()
        k = int(eng.cur_cnt.view(-1)[0].item())
        props = eng.Bq0[:k].cpu()
        idx = _match_rows(props, ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].cpu()
        assert torch.isfinite(pred).all()
        dabs = (pred[idx[m], :31] - ref["class_logits"][m]).abs()
        dl = dabs.max().item()
        db = (pred[idx[m], 31:155] - ref["box_regression"][m]).abs().max().item()
        b, s, l = det.to_host()
        per_frame.append({"proposals": k, "ref_proposals": int(ref["proposals"].shape[0]),
                          "matched_frac": m.float().mean().item(), "logits_maxabs": dl, "deltas_maxabs": db,
                          "logits_p99": torch.quantile(dabs.flatten(), 0.99).item(),
                          "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0]),
                          "labels_equal": bool(b.shape[0] == ref["boxes"].shape[0] and torch.equal(l, ref["labels"])),
                          "logit_rms": ref["class_logits"].pow(2).mean().sqrt().item()})
        _METRICS[label] = per_frame
        _dump()
    return per_frame


def test_mega_r101_logic_matches_reference_with_exact_fp32_contractions(cuda_dev):
    """The whole MEGA engine (window / global pool / long-range memory state machine, RPN selection, ROIAlign,
    relation soft-max with on-the-fly position bias, post-processing -- all our kernels) against the
    REFERENCE's outputs over 4 frames, with only the dense contractions swapped for exact-fp32 torch ops
    (tests/fp32_shadow.py). This is the north-star parity bar: every proposal identical, class logits
    within 1e-3 (measured ~2e-4)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from fp32_shadow import fp32_shadow
    with fp32_shadow():
        frames = _run_mega_against_fixture(cuda_dev, "mega_r101_fp32_shadow")
    for f in frames:
        assert f["matched_frac"] == 1.0, f
        assert f["logits_maxabs"] < 1e-3, f
        assert f["deltas_maxabs"] < 1e-3, f
        assert f["dets"] == f["ref_dets"], f


def test_mega_r101_tf32_matches_reference_fixture(cuda_dev):
    """Same run on the product path (TF32 tensor-core contractions, fp32 accumulate).
    TF32 rounding moves RPN box coordinates by ~0.1 px; the reference's own position embedding
    (sin/cos of 100 * log-ratios of box geometry, roi_box_feature_extractors.py:125-176) is chaotic
    under such shifts for near-coincident boxes, so end-to-end logits are only reproducible to a few
    percent of their RMS (0.76 here) for ANY arithmetic that is not bit-identical upstream -- the
    previous test shows the pipeline itself is exact. The summation order of a TF32 contraction also depends on the
    tile configuration the on-device autotuner picks for these small shapes, so the figures move a little from run to
    run (matched 0.96 .. 1.0, max logit difference 3e-2 .. 5e-2). Bounds asserted: >= 95 % of the reference's
    proposals reproduced within 0.75 px, matched class logits within 0.15, finite everywhere."""
    frames = _run_mega_against_fixture(cuda_dev, "mega_r101_tf32")
    for f in frames:
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_maxabs"] < 0.15, f
        assert f["proposals"] == f["ref_proposals"], f


def test_mega_r101_fp32x3_product_path_matches_reference_fixture(cuda_dev):
    """The PRODUCT path in its strict-parity arithmetic (EngineConfig(precision="fp32x3"): every dense contraction on
    the wgmma tensor cores as a 3xTF32 split with the accumulator re-started every 4 k-blocks, ~2e-6 relative error)
    against the reference's outputs: every proposal and every detection reproduced; class logits within 1e-2
    (measured 1.2e-3 .. 5.9e-3, logit RMS 0.76). The 1e-3 bar of the north star is met by the exact-fp32 shadow test
    above (<= 7e-4, i.e. two fp32 evaluations that merely SUM in a different order already differ by ~1e-3 on this
    randomly initialised model: the relu/log gate and the 100x sin/cos position features of the relation module,
    roi_box_feature_extractors.py:125-176, :593-633, amplify 1e-6 relative perturbations by ~1e3)."""
    frames = _run_mega_against_fixture(cuda_dev, "mega_r101_fp32x3", precision="fp32x3")
    for f in frames:
        assert f["matched_frac"] == 1.0, f
        assert f["logits_maxabs"] < 1e-2, f
        assert f["deltas_maxabs"] < 5e-3, f
        assert f["dets"] == f["ref_dets"], f


def test_mega_r101_f16_matches_reference_fixture(cuda_dev):
    """The throughput mode (EngineConfig(precision="f16"): activations / weights of the GEMM chain stored in fp16,
    kind::f16 tensor-core MMAs with fp32 accumulation). fp16 has the same 10-bit mantissa as TF32, so the same
    statistical bounds as the TF32 test are asserted; the measured numbers land in gpurun_out/engine_parity.json."""
    frames = _run_mega_against_fixture(cuda_dev, "mega_r101_f16", precision="f16")
    for f in frames:
        # fp16 STORAGE also rounds the residual chain of the 33 bottleneck blocks (TF32 rounds conv operands only),
        # so a few more near-tied RPN proposals swap than under TF32 (measured 0.967..1.0 vs 0.987..0.997)
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_p99"] < 3e-2, f
        assert f["logits_maxabs"] < 0.5, f
        assert f["proposals"] == f["ref_proposals"], f


def test_backbone_f16_matches_oracle(cuda_dev):
    import mega_oracle as mo
    from mega_core.b200 import engine, synth
    sd = synth.make_state_dict("mega_r101_tiny", seed=2)
    img = synth.synthetic_frame(1, 96, 160)
    ref = mo.resnet_c4_body(img, sd)
    bb = engine.Backbone({k: v for k, v in sd.items()}, cuda_dev, dtype=torch.float16)
    got = bb.forward(img.to(cuda_dev)).float().permute(0, 3, 1, 2).cpu()
    rel = ((got - ref).abs().max() / ref.pow(2).mean().sqrt()).item()
    _METRICS["backbone_tiny_relerr_f16"] = rel
    _dump()
    assert rel < 2e-2, rel


def _run_rdn_against_fixture(cuda_dev, label, precision):
    from mega_core.b200 import engine, synth
    if precision == "shadow":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from fp32_shadow import fp32_shadow
        with fp32_shadow():
            return _run_rdn_against_fixture(cuda_dev, label, "tf32")
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "rdn_r101_192x320.pt"))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(total)]
    eng = engine.RdnEngine(sd, engine.EngineConfig(all_frame_interval=37, key_frame_location=18, stage=2,
                                                   advanced_stage=1, precision=precision), device=cuda_dev)
    per_frame = []
    for t, ref in enumerate(gold["frames"]):
        if t == 0:
            det = eng.start_video(frames[0], frames[1:19], w, h)
        else:
            det = eng.step(frames[min(t + 18, total - 1)], w, h)
        torch.cuda.synchronize()
        k = int(eng.cur_cnt.view(-1)[0].item())
        props = eng.last_props[:k].cpu()
        idx = _match_rows(props, ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].cpu()
        assert torch.isfinite(pred).all()
        b, s, l = det.to_host()
        per_frame.append({"proposals": k, "ref_proposals": int(ref["proposals"].shape[0]),
                          "matched_frac": m.float().mean().item(),
                          "logits_maxabs": (pred[idx[m], :31] - ref["class_logits"][m]).abs().max().item(),
                          "logits_p99": torch.quantile((pred[idx[m], :31] - ref["class_logits"][m]).abs().flatten(), 0.99).item(),
                          "deltas_maxabs": (pred[idx[m], 31:155] - ref["box_regression"][m]).abs().max().item(),
                          "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0]),
                          "logit_rms": ref["class_logits"].pow(2).mean().sqrt().item()})
        _METRICS[label] = per_frame
        _dump()
    return per_frame


def test_rdn_r101_logic_matches_reference_with_exact_fp32_contractions(cuda_dev):
    """RDN R-101 (BASELINE configs[3]): the whole engine (37-frame ring, RPN selection, ROIAlign, relation soft-max,
    advanced stage, post-processing -- all our kernels) against the REFERENCE's outputs with only the dense
    contractions swapped for exact-fp32 torch ops: every proposal identical, class logits within the north star's
    1e-3."""
    for f in _run_rdn_against_fixture(cuda_dev, "rdn_r101_fp32_shadow", "shadow"):
        assert f["matched_frac"] == 1.0, f
        assert f["logits_maxabs"] < 1e-3, f
        assert f["deltas_maxabs"] < 1e-3, f
        assert f["dets"] == f["ref_dets"], f


def test_rdn_r101_strict_matches_reference_fixture(cuda_dev):
    """same on the product path in the strict arithmetic (3xTF32): all proposals / detections reproduced, class
    logits within 3e-2 (measured 5e-3 .. 1.6e-2 at logit RMS 1.07; see the MEGA strict test for why not 1e-3)"""
    for f in _run_rdn_against_fixture(cuda_dev, "rdn_r101_fp32x3", "fp32x3"):
        assert f["matched_frac"] == 1.0, f
        assert f["logits_maxabs"] < 3e-2, f
        assert f["deltas_maxabs"] < 2e-2, f
        assert f["dets"] == f["ref_dets"], f


def test_rdn_r101_f16_matches_reference_fixture(cuda_dev):
    """same in the throughput mode (fp16 operands): statistical bounds as for MEGA"""
    for f in _run_rdn_against_fixture(cuda_dev, "rdn_r101_f16", "f16"):
        assert f["matched_frac"] >= 0.95, f
        # the relu/log gate of the position bias makes single logits chaotic under 2^-11 operand rounding (max over
        # 9300 logits measured 0.05 .. 0.39 at RMS 1.07); the bulk is tight: 99th percentile of |diff| asserted
        assert f["logits_p99"] < 5e-2, f
        assert f["logits_maxabs"] < 1.0, f
        assert f["proposals"] == f["ref_proposals"], f


def _run_fgfa_against_fixture(cuda_dev, label, precision):
    from mega_core.b200 import engine, synth
    if precision == "shadow":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from fp32_shadow import fp32_shadow
        with fp32_shadow():
            return _run_fgfa_against_fixture(cuda_dev, label, "tf32")
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "fgfa_r101_192x320.pt"))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(total)]
    eng = engine.FgfaEngine(sd, engine.EngineConfig(all_frame_interval=19, key_frame_location=9, precision=precision),
                            device=cuda_dev)
    per_frame = []
    for t, ref in enumerate(gold["frames"]):
        det = eng.start_video(frames[0], frames[1:10], w, h) if t == 0 else eng.step(frames[min(t + 9, total - 1)], w, h)
        torch.cuda.synchronize()
        k = int(eng.last_cnt[0].item())
        idx = _match_rows(eng.last_props[:k].cpu(), ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].cpu()
        assert torch.isfinite(pred).all()
        flow = eng.last_flow[..., :2].permute(0, 3, 1, 2).float().cpu()
        feats = eng.last_feats.float().permute(0, 3, 1, 2).cpu()[:, ::64]
        b, s, l = det.to_host()
        per_frame.append({"proposals": k, "ref_proposals": int(ref["proposals"].shape[0]), "matched_frac": m.float().mean().item(),
                          "logits_maxabs": (pred[idx[m], :31] - ref["class_logits"][m]).abs().max().item(),
                          "flow_maxabs": (flow - ref["flow"]).abs().max().item(),
                          "flow_rms": ref["flow"].pow(2).mean().sqrt().item(),
                          "feats_maxabs": (feats - ref["feats_sample"]).abs().max().item(), "feats_rms": ref["feats_rms"],
                          "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0]),
                          "logit_rms": ref["class_logits"].pow(2).mean().sqrt().item()})
        _METRICS[label] = per_frame
        _dump()
    return per_frame


def test_fgfa_r101_logic_matches_reference_with_exact_fp32_contractions(cuda_dev):
    """FGFA R-101 (BASELINE configs[4]): frame / image rings, pair building, FlowNetS wiring (strided convs, the four
    parity classes of every transposed convolution, crops, concats), warp + adaptive weights + aggregation, box head --
    against the REFERENCE's outputs with exact-fp32 contractions: flow within 1e-4 cells, every proposal reproduced,
    class logits within 1e-3"""
    for f in _run_fgfa_against_fixture(cuda_dev, "fgfa_r101_fp32_shadow", "shadow"):
        assert f["flow_maxabs"] < 1e-4, f
        assert f["feats_maxabs"] < 1e-3 * max(f["feats_rms"], 1.0), f
        assert f["matched_frac"] == 1.0, f
        assert f["logits_maxabs"] < 1e-3, f
        assert f["dets"] == f["ref_dets"], f


@pytest.mark.parametrize("precision", ["f16", "tf32", "fp32x3"])
def test_fgfa_r101_product_path_matches_reference_fixture(cuda_dev, precision):
    """same on the tensor-core arithmetic: flow within 2 % of its RMS-scaled range, >= 95 % of the proposals reproduced"""
    for f in _run_fgfa_against_fixture(cuda_dev, "fgfa_r101_" + precision, precision):
        assert f["flow_maxabs"] < 0.05, f
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_maxabs"] < 0.3, f


def test_mega_frame_parallel_results_do_not_depend_on_world_size(cuda_dev):
    """Frame-parallel mode (SURVEY.md section 8e): a rank runs only the memory-feeding rows of a foreign key frame
    (MegaEngine._aggregate_split, mode "state") and the full row set of its own ("owner"). One GPU plays, in turn, the
    single rank of a 1-GPU group and both ranks of a 2-GPU group (payloads handed over instead of all-gathered):
    every detection and predictor output must be BIT-identical between the two group sizes, and agree with the fused
    single-GPU launch sequence within the fp16 re-association noise."""
    from mega_core.b200 import engine, synth
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "mega_r101_192x320.pt"))
    h, w = gold["h"], gold["w"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(24)]
    glob0 = [frames[(3 * j + 1) % 24] for j in range(10)]
    pair = lambda t: torch.cat([frames[(t + 12) % 24], frames[(5 * t + 3) % 24]], 0)
    steps = 6

    def make():
        e = engine.MegaEngine(sd, engine.EngineConfig(precision="f16"), device=cuda_dev)
        e.start_video(frames[0], frames[1:13], glob0, w, h)
        return e

    def snap(e, det):
        torch.cuda.synchronize()
        b, s, l = det.to_host()
        k = int(e.cur_cnt.view(-1)[0].item())        # live key proposals; rows beyond are padding nobody reads
        return e.last_pred[:k].clone().cpu(), b, s, l

    fused = make()
    out_fused = [snap(fused, fused.step_batched(pair(t), w, h)) for t in range(1, steps + 1)]

    ranker = make()                                  # stateless use: the per-frame branch only
    payloads = [ranker.ref_payload(pair(t), w, h) for t in range(1, steps + 1)]

    solo = make()
    out_solo = []
    for t in range(steps):
        det = solo.dist_step(None, w, h, rank=0, world=1, payloads=payloads[t][None])[0]
        out_solo.append(snap(solo, det))

    out_duo = [None] * steps
    for rank in (0, 1):
        e = make()
        for t in range(0, steps, 2):
            dets = e.dist_step(None, w, h, rank=rank, world=2, payloads=torch.stack(payloads[t:t + 2]))
            assert dets[1 - rank] is None
            out_duo[t + rank] = snap(e, dets[rank])

    worst = 0.0
    for t in range(steps):
        for a, b in zip(out_solo[t], out_duo[t]):
            assert torch.equal(a, b), "frame %d differs between 1 and 2 ranks" % t
        assert out_fused[t][0].shape == out_solo[t][0].shape
        assert abs(out_fused[t][1].shape[0] - out_solo[t][1].shape[0]) <= 2
        d = (out_fused[t][0][:, :31] - out_solo[t][0][:, :31]).abs()
        worst = max(worst, torch.quantile(d.flatten(), 0.99).item())
    _METRICS["mega_frame_parallel_split_vs_fused_logits_p99"] = worst
    _dump()
    assert worst < 2e-2, worst
