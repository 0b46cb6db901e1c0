"""What the 3x3-strided bottleneck layout (MODEL.RESNETS.STRIDE_IN_1X1 False) costs against the MSRA layout at 600x1000:
steady-state key frames/s of MEGA R-101 and MEGA X-101 32x8d in f16 and fp32x3, the two layouts alternated in one
process, and the time of each launch of the two blocks that differ (the first bottleneck of res3 and of res4: conv1,
conv2, downsample, conv3), launched one by one.

    python tools/bench_stride3x3.py [--steps 20] [--warmup 5] [--rounds 3] [--out results.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "mega.pytorch_b200"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

from bench_resnext import H, W, card, per_layer, time_steps  # noqa: E402

LAYOUTS = {"msra": True, "s3x3": False}       # name -> stride_in_1x1
NAMES = ("conv1", "conv2", "downsample", "conv3")


def make_engine(sd, precision, stride_in_1x1, dev):
    from mega_core.b200 import engine, synth
    total = 40
    frames = [synth.synthetic_frame(i, H, W).to(dev) for i in range(total)]
    eng = engine.MegaEngine(sd, engine.EngineConfig(precision=precision, stride_in_1x1=stride_in_1x1), device=dev)
    gidx = synth.global_frame_indices(total, seed=0)
    eng.start_video(frames[0], frames[1:13], [frames[j] for j in gidx[:10]], W, H)
    step = [0]

    def run():
        t = step[0] = step[0] + 1
        return eng.step(frames[(t + 12) % total], frames[gidx[t % total]], W, H)
    return eng, run


def first_block_launches(eng):
    """indices, in the launch order of one key frame, of the launches of res3's and res4's first blocks (the stem is
    launch 0, the body follows block by block: conv1, conv2, downsample if any, conv3)"""
    out, i = {}, 1
    for si, blocks in enumerate(eng.backbone.stages.stages):
        for bi, blk in enumerate(blocks):
            names = NAMES if blk.wd is not None else ("conv1", "conv2", "conv3")
            if bi == 0 and si > 0:
                out["res%d" % (si + 2)] = dict(zip(names, range(i, i + len(names))))
            i += len(names)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for the full results (default: none)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    from mega_core.b200 import synth
    dev = torch.device("cuda:0")
    res = {"card": card(), "input": [H, W], "steps": args.steps, "rounds": args.rounds, "bodies": {}}
    print("card:", res["card"])
    for arch, body in (("mega_r101", "R-101"), ("mega_x101", "X-101 32x8d")):
        sd = synth.make_state_dict(arch, seed=0)
        res["bodies"][body] = {}
        for precision in ("f16", "fp32x3"):
            engines = {name: make_engine(sd, precision, s, dev) for name, s in LAYOUTS.items()}
            ms = {name: [] for name in LAYOUTS}
            for _ in range(args.rounds):                     # the two layouts alternated
                for name, (eng, run) in engines.items():
                    ms[name].append(time_steps(run, args.steps, args.warmup))
            row = {}
            for name, (eng, run) in engines.items():
                rows = per_layer(eng, run)
                blocks = {}
                for stage, idx in first_block_launches(eng).items():
                    assert rows[idx["conv2"]]["taps"] == 9, "launch order of the body changed"
                    blocks[stage] = {conv: rows[i] for conv, i in idx.items()}
                best = min(ms[name])
                row[name] = {"key_frame_ms": ms[name], "key_frames_per_s": 1000.0 / best, "first_blocks": blocks,
                             "first_blocks_ms": sum(r["ms"] for b in blocks.values() for r in b.values())}
            res["bodies"][body][precision] = row
            a, b = row["msra"], row["s3x3"]
            print("%-11s %-7s key frames/s MSRA %.1f / 3x3-strided %.1f (%+.1f %%; best of %d x %d steps, alternated); "
                  "first blocks of res3 + res4, launched one by one: %.3f / %.3f ms"
                  % (body, precision, a["key_frames_per_s"], b["key_frames_per_s"],
                     100.0 * (b["key_frames_per_s"] / a["key_frames_per_s"] - 1), args.rounds, args.steps,
                     a["first_blocks_ms"], b["first_blocks_ms"]))
            for stage in ("res3", "res4"):
                for conv in NAMES:
                    ra, rb = a["first_blocks"][stage][conv], b["first_blocks"][stage][conv]
                    print("    %s %-10s MSRA %.4f ms (%5.2f GFLOP)   3x3-strided %.4f ms (%5.2f GFLOP)"
                          % (stage, conv, ra["ms"], ra["gflop"], rb["ms"], rb["gflop"]))
            del engines
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
