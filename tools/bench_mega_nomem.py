#!/usr/bin/env python
"""Key frames/s of MEGA R-101 with and without the long-range memory (MODEL.VID.MEGA.MEMORY.ENABLE), on bench.py's
600x1000 synthetic stream, in the strict (fp32x3) and the throughput (f16) mode.

    python tools/bench_mega_nomem.py [--precision fp32x3 f16] [--steps 20] [--reps 5] [--json FILE]

Per mode both engines are built from the same checkpoint and primed with the same frames (the first frame of the video,
then 27 key frames: the memory-on engine's memory is full). Then `--reps` rounds alternate memory on / off, each a
device-timed window of `--steps` stepn_batched calls (4 key frames per call, CUDA graphs and tiles picked by the
autotuner, as bench.py's headline step);
every round is reported, then the median and the spread (min / max). Last, one eager step of each engine with a CUDA
event pair around every relation call (MegaEngine._attention: G0, the local stages L0-L2, G1) gives the per-stage
relation times; eager launches include the host gaps between them, so these rows are for comparison between the two
engines, not absolute kernel times. The card's name, power limit and max SM clock are printed with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402
from mega_core.modeling.detector import build_detection_model_from_state_dict  # noqa: E402


def card():
    """name, power limit and max SM clock of the current GPU"""
    import subprocess
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    out = subprocess.run(q, capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    return out[torch.cuda.current_device()].strip()


def build(mb, precision, memory):
    model = build_detection_model_from_state_dict(mb.sd, method="mega", device=mb.dev, precision=precision)
    model.cfg.defrost()
    model.cfg.MODEL.VID.MEGA.MEMORY.ENABLE = memory
    eng = model.engine
    assert eng.cfg.memory is memory
    eng.use_graph = True
    with torch.no_grad():
        model(mb.infos_first())
        for t in range(1, 28):
            model(mb.infos_next(t))
    return model, eng


def stage_times(eng, step, fps):
    """one eager step of `fps` key frames with an event pair around each relation call -> {stage: ms per key frame}"""
    names = {id(a): "G%d" % i for i, a in enumerate(eng.att_g)}
    names.update({id(a): "L%d" % i for i, a in enumerate(eng.att_l)})
    rec = []
    inner = eng._attention

    def timed(att, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = inner(att, *a, **k)
        e1.record()
        rec.append((names[id(att)], e0, e1))
        return out
    graphs, eng._graphs, eng.use_graph = eng._graphs, {}, False
    eng._attention = timed
    try:
        step()
        torch.cuda.synchronize()
    finally:
        del eng._attention
        eng._graphs, eng.use_graph = graphs, True
    out = {}
    for name, e0, e1 in rec:
        out[name] = out.get(name, 0.0) + e0.elapsed_time(e1) / fps
    return out


def run_mode(mb, precision, args):
    fps = mb.fps
    nb = 16 // fps
    batches = [torch.cat([mb.pairs_dev[(fps * i + j) % 16] for j in range(fps)], 0) for i in range(nb)]
    engines = {m: build(mb, precision, m) for m in (True, False)}
    rates = {True: [], False: []}
    with torch.no_grad():
        for m, (_, eng) in engines.items():
            for i in range(4 + args.warmup):
                eng.stepn_batched(batches[i % nb], mb.w, mb.h)
        torch.cuda.synchronize()
        for rep in range(args.reps):
            for m in (True, False):
                eng = engines[m][1]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.steps):
                    eng.stepn_batched(batches[i % nb], mb.w, mb.h)
                e1.record()
                torch.cuda.synchronize()
                rates[m].append(1000.0 * fps * args.steps / e0.elapsed_time(e1))
        stages = {m: stage_times(eng, lambda: eng.stepn_batched(batches[0], mb.w, mb.h), fps)
                  for m, (_, eng) in engines.items()}
    del engines
    torch.cuda.empty_cache()
    res = {"precision": precision, "key_frames_per_step": fps}
    for m in (True, False):
        r = rates[m]
        key = "memory_on" if m else "memory_off"
        res[key] = {"key_frames_per_s": r, "median": statistics.median(r), "min": min(r), "max": max(r),
                    "relation_ms_per_key_frame": stages[m]}
        print("%s %-10s key frames/s: median %.1f (min %.1f, max %.1f) over %d rounds: %s" % (
            precision, key, statistics.median(r), min(r), max(r), len(r), " ".join("%.1f" % v for v in r)))
        print("    relation ms per key frame (eager): " + ", ".join("%s %.3f" % kv for kv in sorted(stages[m].items())))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["fp32x3", "f16"], choices=["fp32x3", "f16"])
    ap.add_argument("--steps", type=int, default=20, help="stepn_batched calls per timed round")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="timed rounds per engine, memory on and off alternating")
    ap.add_argument("--json", default=None, metavar="FILE")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    ba = argparse.Namespace(arch="mega_r101", height=bench.H, width=bench.W, frames_per_step=bench.DEFAULT_FPS,
                            no_parity=True)
    mb = bench.MegaBench(ba, 0, 1)
    result = {"card": card(), "modes": [run_mode(mb, p, args) for p in args.precision]}
    print("card (name, power limit, max SM clock): %s" % result["card"])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
