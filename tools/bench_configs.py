"""Steady-state key frames/s of the shipped VID configs served since REDUCE_CHANNEL, MEGA.GLOBAL.RES_STAGE = 0 and
ATTENTION.ADVANCED_STAGE = 0 run (configs/MEGA/vid_R_50_C4_MEGA_1x.yaml, configs/RDN/vid_R_{101,50}_C4_RDN_base_1x.yaml),
with MEGA R-101 (configs/MEGA/vid_R_101_C4_MEGA_1x.yaml) as the control in the same process; 600x1000 synthetic frames,
seeded synthetic weights, f16 and fp32x3, every steady frame a captured CUDA graph. Device time with CUDA events over
--steps key frames after --warmup; the configs of one arithmetic are measured in turn, --rounds times, and the best
round is reported.

    python tools/bench_configs.py [--steps 30] [--warmup 5] [--rounds 3] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mega.pytorch_b200"))

import torch  # noqa: E402

H, W = 600, 1000
# name -> (synth arch, seed, make_state_dict options)
CONFIGS = {
    "MEGA R-101 (control)": ("mega_r101", 0, {}),
    "MEGA R-50": ("mega_r50", 5, {"reduce_channel": True, "global_res_stage": 0}),
    "RDN-base R-101": ("rdn_r101", 6, {"advanced_stage": 0}),
    "RDN-base R-50": ("rdn_r50", 7, {"reduce_channel": True, "advanced_stage": 0}),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def make_runner(name, precision, frames, dev):
    """the engine model(images) runs for the config, its video started; returns (engine, one-key-frame step)"""
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    arch, seed, opts = CONFIGS[name]
    method = arch.split("_")[0]
    sd = synth.make_state_dict(arch, seed=seed, **opts)
    eng = build_detection_model_from_state_dict(sd, method=method, device=dev, precision=precision).engine
    eng.use_graph = True
    total = len(frames)
    step = [0]
    if method == "mega":
        gidx = synth.global_frame_indices(total, seed=0)
        eng.start_video(frames[0], frames[1:13], [frames[j] for j in gidx[:10]], W, H)

        def run():
            t = step[0] = step[0] + 1
            return eng.step(frames[(t + 12) % total], frames[gidx[t % total]], W, H)
    else:
        eng.start_video(frames[0], frames[1:19], W, H)

        def run():
            t = step[0] = step[0] + 1
            return eng.step(frames[(t + 18) % total], W, H)
    return eng, run


def time_steps(run, steps, warmup):
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        run()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="JSON file for the results (default: none)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    from mega_core.b200 import synth
    dev = torch.device("cuda:0")
    frames = [synth.synthetic_frame(i, H, W).to(dev) for i in range(40)]
    res = {"card": card(), "input": [H, W], "steps": args.steps, "rounds": args.rounds, "modes": {}}
    print("card (name, power limit, max SM clock):", res["card"])
    for precision in ("f16", "fp32x3"):
        runners = {name: make_runner(name, precision, frames, dev) for name in CONFIGS}
        ms = {name: [] for name in CONFIGS}
        for _ in range(args.rounds):
            for name, (_, run) in runners.items():
                ms[name].append(time_steps(run, args.steps, args.warmup))
        res["modes"][precision] = {}
        for name in CONFIGS:
            best = min(ms[name])
            res["modes"][precision][name] = {"key_frame_ms": best, "key_frames_per_s": 1000.0 / best, "rounds_ms": ms[name]}
            print("%-7s %-21s %7.2f ms/key frame  %6.1f key frames/s   (rounds: %s)"
                  % (precision, name, best, 1000.0 / best, ", ".join("%.2f" % v for v in ms[name])))
        del runners
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
