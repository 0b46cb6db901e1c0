"""What deformable backbone stages (MODEL.RESNETS.STAGE_WITH_DCN) cost at 600x1000:
  * whole model: steady-state key frames/s of MEGA R-101 through MegaEngine.step() in f16 and fp32x3, the bodies
    alternated round by round (device time: CUDA events around `steps` steps). --set dcn: plain, DCN v1 on res3 + res4
    and modulated DCN v2 on res3 + res4; --set groups: DCN v1 on res3 + res4 with 1, 2 and 4 deformable groups
    (MODEL.RESNETS.DEFORMABLE_GROUPS);
  * per launch: the three launches of a deformable conv2 (offset conv, sampling, contraction) of one res3 and one res4
    block of every deformable body, each launched alone and timed with CUDA events. The offset conv and the sampling
    against their HBM byte floors at 3.35 TB/s -- offset conv: its input map read once and the fp32 offset rows written;
    sampling: the columns written, the input map and the offset rows read once -- and the sampling against its gather
    traffic (four corner vectors per sample read, the columns written).
The card line (name, power limit, max SM clock) is read by the same run.

    python tools/bench_dcn.py [--set dcn|groups] [--steps 20] [--warmup 5] [--rounds 3] [--out results.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "mega.pytorch_b200"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

from bench_resnext import H, W, card, time_steps  # noqa: E402

RES34 = (False, True, True, False)
SETS = {"dcn": {"plain": ((False,) * 4, False, 1), "v1 res3+res4": (RES34, False, 1), "v2 res3+res4": (RES34, True, 1)},
        "groups": {"v1 res3+res4 dg1": (RES34, False, 1), "v1 res3+res4 dg2": (RES34, False, 2),
                   "v1 res3+res4 dg4": (RES34, False, 4)}}
HBM = 3.35e12


def make_engine(sd, precision, dev):
    from mega_core.b200 import engine, synth
    total = 40
    frames = [synth.synthetic_frame(i, H, W).to(dev) for i in range(total)]
    eng = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=dev)
    gidx = synth.global_frame_indices(total, seed=0)
    eng.start_video(frames[0], frames[1:13], [frames[j] for j in gidx[:10]], W, H)
    step = [0]

    def run():
        t = step[0] = step[0] + 1
        return eng.step(frames[(t + 12) % total], frames[gidx[t % total]], W, H)
    return eng, run


def event_ms(fn, reps=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def block_launches(stages, blk, n, h, w, stride):
    """the three launches of blk's deformable conv2 on an n-image map of h x w (conv2's input), each timed alone"""
    from mega_core.b200 import ops
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    t1 = stages._buf("bench_t1", (n, h, w, blk.mid))
    t1.copy_(torch.rand(t1.shape, device=t1.device).to(t1.dtype) if not ops.is_split16(t1) else
             ops.split16_encode(torch.rand(t1.shape, device=t1.device)))
    t2 = stages._buf("t2", (n, ho, wo, blk.mid))
    off = stages._buf("dcn_off", (n, ho, wo, blk.off_rows), fp32=True)
    cols = stages._buf("dcn_cols", (n, ho, wo, 9 * blk.mid))
    kw = {"deformable_groups": blk.dg} if blk.dg > 1 else {}
    ms = {"offset conv": event_ms(lambda: ops.conv_gemm(t1, blk.wo, off, taps=(3, 3), pad=1, stride=(stride, stride),
                                                        bias=blk.bo)),
          "sampling": event_ms(lambda: ops.dcn_sample(t1, off, cols, blk.modulated, stride, **kw)),
          "contraction": event_ms(lambda: ops.conv_gemm(cols, blk.w2, t2, scale=blk.s2, bias=blk.b2, relu=True))}
    el = 4 if t1.dtype == torch.float32 else 2          # split-fp16 keeps 4 bytes per value
    col_bytes = cols.numel() * el
    off_bytes = off.numel() * 4
    floor = col_bytes + t1.numel() * el + off_bytes
    off_floor = t1.numel() * el + off_bytes
    gather = col_bytes + 4 * cols.numel() * el
    return {"ms": ms, "col_bytes": col_bytes, "offset_bytes": off_bytes, "floor_bytes": floor,
            "offset_conv_floor_bytes": off_floor, "deformable_groups": blk.dg,
            "sampling_floor_share": floor / HBM / (ms["sampling"] * 1e-3),
            "offset_conv_floor_share": off_floor / HBM / (ms["offset conv"] * 1e-3),
            "sampling_gather_TBps": gather / (ms["sampling"] * 1e-3) / 1e12}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--set", choices=sorted(SETS), default="dcn")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for the full results (default: none)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    from mega_core.b200 import ops, synth
    dev = torch.device("cuda:0")
    bodies = SETS[args.set]
    res = {"card": card(), "set": args.set, "input": [H, W], "steps": args.steps, "rounds": args.rounds, "model": {},
           "launches": {}}
    print("card:", res["card"])
    for precision in ("f16", "fp32x3"):
        engines = {}
        for name, (stages, modulated, dg) in bodies.items():
            sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=stages, modulated_dcn=modulated,
                                       deformable_groups=dg)
            engines[name] = make_engine(sd, precision, dev)
        ms = {name: [] for name in engines}
        for _ in range(args.rounds):
            for name, (eng, run) in engines.items():
                ms[name].append(time_steps(run, args.steps, args.warmup))
        res["model"][precision] = {name: {"key_frame_ms": v, "key_frames_per_s": 1000.0 / min(v)} for name, v in ms.items()}
        print("%-7s key frames/s (best of %d x %d steps, alternated): %s" % (
            precision, args.rounds, args.steps, ", ".join("%s %.1f" % (k, r["key_frames_per_s"])
                                                          for k, r in res["model"][precision].items())))
        hp, wp = (H - 1) // 4 + 1, (W - 1) // 4 + 1           # res2's map (after the stem and the max pool)
        res["launches"][precision] = {}
        for name, (eng, _) in engines.items():
            st = eng.backbone.stages
            if not st.has_dcn:
                continue
            rows = {}
            with ops.precision(precision):
                for si, stride, (h, w) in ((1, 1, ((hp - 1) // 2 + 1, (wp - 1) // 2 + 1)),
                                           (2, 1, ((hp - 1) // 4 + 1, (wp - 1) // 4 + 1))):
                    blk = st.stages[si][1]                          # a non-first block: conv2 at the stage's resolution
                    r = block_launches(st, blk, 1, h, w, stride)
                    rows["res%d" % (si + 2)] = r
                    print("    %s res%d block, 1 image %dx%d, C %d: offset conv %.4f ms (%.0f %% of its floor), sampling "
                          "%.4f ms (%.1f MB of columns; %.0f %% of the HBM floor at 3.35 TB/s, gather traffic %.2f "
                          "TB/s), contraction %.4f ms"
                          % (name, si + 2, h, w, blk.mid, r["ms"]["offset conv"], 100 * r["offset_conv_floor_share"],
                             r["ms"]["sampling"], r["col_bytes"] / 1e6, 100 * r["sampling_floor_share"],
                             r["sampling_gather_TBps"], r["ms"]["contraction"]))
            res["launches"][precision][name] = rows
        del engines
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
