"""End-to-end parity at the BASELINE configuration: MEGA R-101, 600x1000, 42 key frames (25-frame local window, 10-frame
global pool, long-range memory FULL from key frame 25 on), product path through the C-ABI kernels, against the outputs of
the UNMODIFIED reference on the same seeded video (tests/golden/mega_r101_600x1000.pt, oracle/make_golden_full.py).

The parity point is the north star's: class logits of `FPNPredictor.forward` (roi_box_predictors.py:50-57), compared on
proposals matched by box. The fixture also carries the same logits from the reference run in fp64, and
profiles/r02_parity_floor.json the distance between the reference's own fp32 / fp64 / other-thread-count evaluations:
the bars below are stated next to that floor. Measured values land in gpurun_out/parity_full.json.
"""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "mega_r101_600x1000.pt")
_OUT = {}

# Bars, stated next to the floor (profiles/r02_parity_floor.json = the UNMODIFIED reference against itself on the same 42
# key frames: fp32 vs fp64 -> all proposals and detections equal, logits p99 <= 7.7e-5, p99.9 <= 5.5e-3, max 1.05e-2 with 2
# frames holding a logit beyond 1e-3; 8 vs 4 threads -> max 2.3e-6). A single logit can move by 1e-2 between two exact-ish
# evaluations (a proposal pair crossing the relu gate of the position bias), so the north star's 1e-3 is asserted at the
# 99th percentile of every check frame, and the maximum against the floor's own maximum.
STRICT_LOGITS_P99 = 1e-3        # north star tolerance, strict tensor-core mode (fp32x3), 99th percentile per frame
STRICT_LOGITS_MAX = 2e-2        # ~2x the reference's own fp32-vs-fp64 maximum
FAST_LOGITS_P99 = 5e-2          # 10-bit-mantissa operand modes (f16 / tf32): statistical bound (measured <= 2.9e-2)
FAST_MATCHED = 0.90             # share of the reference's proposals reproduced within 0.75 px (measured >= 0.937)


def _dump():
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "parity_full.json"), "w") as fh:
        json.dump(_OUT, fh, indent=1)


@pytest.fixture(scope="module")
def gold_and_frames(cuda_dev):
    from mega_core.b200 import synth
    gold = torch.load(FIXTURE)
    frames = [synth.synthetic_frame(i, gold["h"], gold["w"]).to(cuda_dev) for i in range(gold["total"])]
    return gold, frames


def _run(cuda_dev, gold_and_frames, precision):
    from mega_core.b200 import engine, parity, synth
    gold, frames = gold_and_frames
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    eng = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev)
    rows = parity.replay(eng, gold, cuda_dev, frames=frames)
    _OUT[precision] = {"summary": parity.summarize(rows), "frames": rows}
    _dump()
    del eng
    torch.cuda.empty_cache()
    return rows


def test_fixture_covers_the_baseline_configuration():
    gold = torch.load(FIXTURE)
    assert (gold["h"], gold["w"]) == (600, 1000) and len(gold["frames"]) >= 40
    chk = [t for t, f in enumerate(gold["frames"]) if "class_logits" in f]
    assert max(chk) >= 38 and sum(t >= 26 for t in chk) >= 4, "check frames must include key frames with a FULL memory"


def test_mega_600x1000_strict_mode_meets_the_logit_bar(cuda_dev, gold_and_frames):
    """fp32x3 (every contraction on the wgmma tensor cores as a 3xTF32 split): every proposal and every detection of the
    reference reproduced on every check frame (memory empty, filling and full), class logits within the north star's 1e-3
    at the 99th percentile and within 2e-2 at the maximum (the reference's own fp32-vs-fp64 distances: 7.7e-5 / 1.05e-2)"""
    rows = _run(cuda_dev, gold_and_frames, "fp32x3")
    for r in rows:
        assert r["finite"] and r["matched_frac"] == 1.0, r
        assert r["dets"] == r["ref_dets"], r
        assert r["logits_p99"] < STRICT_LOGITS_P99, r
        assert r["logits_max"] < STRICT_LOGITS_MAX, r


@pytest.mark.parametrize("precision", ["f16", "tf32"])
def test_mega_600x1000_throughput_modes_stay_within_the_statistical_bound(cuda_dev, gold_and_frames, precision):
    """f16 / tf32 operands (10-bit mantissa): >= 90 % of the reference's proposals reproduced within 0.75 px on every
    check frame incl. the full-memory ones (measured 0.937 .. 0.99), the same number of proposals and detections, 99th
    percentile of |logit difference| within 5e-2 (measured <= 2.9e-2 at logit RMS ~0.8). These modes do NOT meet the
    north star's 1e-3; bench.py therefore never prints them as the headline while a stricter mode passes."""
    rows = _run(cuda_dev, gold_and_frames, precision)
    for r in rows:
        assert r["finite"], r
        assert r["matched_frac"] >= FAST_MATCHED, r
        assert r["logits_p99"] < FAST_LOGITS_P99, r
        assert r["proposals"] == r["ref_proposals"], r
