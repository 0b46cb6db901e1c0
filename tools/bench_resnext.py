"""MEGA on a ResNeXt-101 32x8d body (MODEL.RESNETS.NUM_GROUPS 32, WIDTH_PER_GROUP 8) at 600x1000: steady-state key-frame
device time in f16 and fp32x3, the time of every grouped conv layer of one key frame (launched one by one) with the
diagonal-block MMA issue on and off (ops.GROUP_DIAG, alternated), and the GFLOP per frame computed from the shapes --
the useful ones and the ones the 64-channel chunked (block-diagonal) form of the grouped layers holds.

    python tools/bench_resnext.py [--steps 20] [--out results.json]

The summary goes to stdout; --out also writes every layer's row as JSON.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


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


def per_layer(eng, run, reps=5):
    """every tensor-core launch of one key frame, eager and unchained, each timed with CUDA events over `reps` repeats"""
    from mega_core.b200 import ops
    rows = []

    def hook(launch, flops, info):
        launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            launch()
        e1.record()
        e1.synchronize()
        rows.append(dict(info, ms=e0.elapsed_time(e1) / reps, gflop=flops / 1e9))
    saved = eng.use_graph, ops.CHAINS_ENABLED[0]
    eng.use_graph, ops.CHAINS_ENABLED[0] = False, False
    ops.TIMING_HOOK[0] = hook
    try:
        run()
        torch.cuda.synchronize()
    finally:
        ops.TIMING_HOOK[0] = None
        eng.use_graph, ops.CHAINS_ENABLED[0] = saved
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="JSON file for the full results (default: none)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    from mega_core.b200 import synth
    dev = torch.device("cuda:0")
    sd = synth.make_state_dict("mega_x101", seed=0)
    res = {"card": card(), "input": [H, W], "body": "X-101 32x8d", "modes": {}}
    print("card:", res["card"])
    from mega_core.b200 import ops
    for precision in ("f16", "fp32x3"):
        eng, run = make_engine(sd, precision, dev)
        key_ms = {True: [], False: []}
        grouped_ms = {True: [], False: []}
        for _ in range(3):                      # diagonal issue on / off, alternated
            for diag in (True, False):
                ops.GROUP_DIAG[0] = diag
                key_ms[diag].append(time_steps(run, args.steps, args.warmup))
                rows = per_layer(eng, run)
                grouped = [r for r in rows if r["taps"] == 9 and r["batch"] > 1 and r["cout"] == 64 and r["k"] == 64]
                grouped_ms[diag].append([r["ms"] for r in grouped])
        ops.GROUP_DIAG[0] = True
        ms = min(key_ms[True])
        for i, r in enumerate(grouped):
            r["ms_diag"] = min(g[i] for g in grouped_ms[True])
            r["ms_dense"] = min(g[i] for g in grouped_ms[False])
            r["group_width"] = r["batch"] * 64 // 32          # 32 groups: gw = C / 32
            r["useful_gflop"] = r["gflop"] * min(r["group_width"], 64) / 64
        m = {"key_frame_ms": ms, "key_frame_ms_diag_off": min(key_ms[False]),
             "conv_launches": len(rows), "conv_ms_sum": sum(r["ms"] for r in rows),
             "grouped_launches": len(grouped), "grouped_ms_sum": sum(r["ms_diag"] for r in grouped),
             "grouped_ms_sum_diag_off": sum(r["ms_dense"] for r in grouped),
             "gflop_executed": sum(r["gflop"] for r in rows),
             "gflop_useful": sum(r["gflop"] for r in rows) - sum(r["gflop"] - r["useful_gflop"] for r in grouped),
             "grouped_layers": grouped}
        res["modes"][precision] = m
        print("%-7s key frame %.2f ms (diagonal issue off: %.2f ms; device, steady state, best of 3 x %d steps); conv "
              "launches one by one: %.2f ms in %d, of which grouped 3x3: %.2f ms in %d; GFLOP/frame useful %.1f, chunked %.1f"
              % (precision, ms, m["key_frame_ms_diag_off"], args.steps, m["conv_ms_sum"], len(rows), m["grouped_ms_sum"],
                 len(grouped), m["gflop_useful"], m["gflop_executed"]))
        for gw in (8, 16, 32, 64):
            sel = [r for r in grouped if r["group_width"] == gw]
            if sel:
                print("    gw %2d: %3d launches, diagonal issue %.3f ms / whole chunks %.3f ms, %.2f GFLOP chunked / %.2f "
                      "useful" % (gw, len(sel), sum(r["ms_diag"] for r in sel), sum(r["ms_dense"] for r in sel),
                                  sum(r["gflop"] for r in sel), sum(r["useful_gflop"] for r in sel)))
        del eng
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
