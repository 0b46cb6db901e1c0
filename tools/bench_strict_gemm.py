#!/usr/bin/env python
"""Where the strict (fp32x3) step's time goes: every tensor-core launch of one 4-key-frame MEGA R-101 step at 600x1000
(MegaEngine.stepn_batched, as bench.py's roofline pass runs it), timed with a CUDA event pair per launch.

    python tools/bench_strict_gemm.py [--steps 20] [--warmup 5] [--reps 5] [--json FILE]

Prints one row per launch -- shape (m, cout, k, taps), block_n, stream-K, precision, ms and executed TFLOP/s (3 tensor-core
products per multiply-add in the strict modes) -- then the sum over the 3xFP16 launches (conv_gemm_kernel<.., kModeF16x3>)
and its share of the device-timed step (CUDA graphs, device-resident inputs: the step bench.py times), and the card's
name / power limit / max SM clock. The JSON written with --json also holds a SHA-256 digest of the output tensor of every
3xFP16 launch of one further step: two builds that compute the same bits give the same list.

Tiles come from the fixed heuristic (MEGA_B200_AUTOTUNE=0), so every run launches the same kernels on the same shapes.
The per-launch times come from eager launches (one event pair each, no overlap between kernels), the step time from graph
replays in which consecutive kernels overlap (programmatic dependent launch), so the share can exceed 1.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["MEGA_B200_AUTOTUNE"] = "0"

import torch  # noqa: E402

import bench  # noqa: E402
from mega_core.b200 import ops  # noqa: E402
from mega_core.modeling.detector import build_detection_model_from_state_dict  # noqa: E402

PRECISION_NAME = {0: "tf32", 1: "3xTF32", 2: "f16", 3: "3xFP16"}


def card():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    try:
        out = subprocess.run(q, capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired):
        return None
    idx = torch.cuda.current_device()
    return out[idx].strip() if idx < len(out) else None


def launch_times(step, reps):
    """[(info, flops, ms averaged over reps)] for every tensor-core launch of one eager step"""
    rec = []

    def hook(run, flops, info):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        rec.append((a, b, flops, info))

    ops.TIMING_HOOK[0] = hook
    try:
        step(0)
        rec.clear()
        for i in range(reps):
            torch.cuda._sleep(100_000_000)    # the whole step is queued before it runs: the events bracket kernels only
            step(i + 1)
            torch.cuda.synchronize()
    finally:
        ops.TIMING_HOOK[0] = None
    n = len(rec) // reps
    assert n * reps == len(rec), "launch sequence differs between steps"
    return [(rec[i][3], rec[i][2], sum(r[0].elapsed_time(r[1]) for r in rec[i::n]) / reps) for i in range(n)]


def output_digests(step):
    """SHA-256 of the output of every 3xFP16 conv_gemm call of one eager step, in launch order"""
    digests = []
    orig, depth = ops.conv_gemm, [0]

    def conv_gemm(a, w, out, **kw):
        depth[0] += 1          # grouped convolutions call conv_gemm again: digest the outermost call
        try:
            r = orig(a, w, out, **kw)
        finally:
            depth[0] -= 1
        if depth[0] == 0 and ops._split16_fmt(a) is not None:
            cout = kw.get("cout") or w.shape[1]
            cols = min(out.shape[-1], -(-cout // 32) * 32)
            digests.append(hashlib.sha256(out[..., :cols].contiguous().cpu().numpy().tobytes()).hexdigest())
        return r

    ops.conv_gemm = conv_gemm
    try:
        step(0)
        torch.cuda.synchronize()
    finally:
        ops.conv_gemm = orig
    return digests


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="device-timed steps")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="eager steps whose per-launch times are averaged")
    ap.add_argument("--json", default=None, metavar="FILE", help="write the result (with the output digests) to FILE")
    args = ap.parse_args()

    ba = argparse.Namespace(arch="mega_r101", height=bench.H, width=bench.W, frames_per_step=bench.DEFAULT_FPS,
                            no_parity=True)
    mb = bench.MegaBench(ba, 0, 1)
    model = build_detection_model_from_state_dict(mb.sd, method="mega", device=mb.dev, precision="fp32x3")
    eng, fps = model.engine, mb.fps
    eng.use_graph = True
    nb = 16 // fps
    batches = [torch.cat([mb.pairs_dev[(fps * i + j) % 16] for j in range(fps)], 0) for i in range(nb)]

    def step(i):
        return eng.stepn_batched(batches[i % nb], mb.w, mb.h)

    with torch.no_grad():
        model(mb.infos_first())                  # first frame, then fill the long-range memory as bench.py does
        for t in range(1, eng.MEMF + 3):
            model(mb.infos_next(t))
        for i in range(4 + args.warmup):         # every CUDA graph captured and replayed
            step(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            step(i)
        e1.record()
        torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1) / args.steps

        graphs, eng._graphs = eng._graphs, {}
        eng.use_graph = False
        try:
            launches = launch_times(step, args.reps)
            digests = output_digests(step)
        finally:
            eng._graphs, eng.use_graph = graphs, True

    rows = []
    print("%4s %7s %5s %5s %4s %4s %3s %7s %9s %9s" % ("#", "m", "cout", "k", "taps", "bn", "sk", "prec", "ms", "TFLOP/s"))
    for i, (info, flops, ms) in enumerate(launches):
        if "chain_layers" in info:
            row = {"kind": "conv_chain", "layers": info["chain_layers"], "ms": ms, "flops": flops, "executed_tflops": None}
            print("%4d conv_chain_kernel (%d layers) %34.4f" % (i, info["chain_layers"], ms))
        else:
            prec = PRECISION_NAME.get(info.get("precision"), "?")
            products = 3 if prec in ("3xFP16", "3xTF32") else 1
            row = {"kind": "conv_gemm", "m": info["m"] * info["batch"], "cout": info["cout"], "k": info["k"],
                   "taps": info["taps"], "block_n": info["bn"], "stream_k": info["sk"], "precision": prec, "ms": ms,
                   "flops": flops, "executed_tflops": products * flops / (ms * 1e-3) / 1e12}
            print("%4d %7d %5d %5d %4d %4d %3d %7s %9.4f %9.1f" % (i, row["m"], row["cout"], row["k"], row["taps"],
                                                                 row["block_n"], row["stream_k"], prec, ms,
                                                                 row["executed_tflops"]))
        rows.append(row)
    f16x3 = [r for r in rows if r.get("precision") == "3xFP16"]
    f16x3_ms = sum(r["ms"] for r in f16x3)
    kernel_ms = sum(r["ms"] for r in rows)
    exec_tflops = 3 * sum(r["flops"] for r in f16x3) / (f16x3_ms * 1e-3) / 1e12 if f16x3_ms else None
    result = {"card": card(), "key_frames_per_step": fps, "step_ms": step_ms, "tensor_core_launches": len(rows),
              "tensor_core_ms_per_step": kernel_ms, "f16x3_launches": len(f16x3), "f16x3_ms_per_step": f16x3_ms,
              "f16x3_share_of_step": f16x3_ms / step_ms, "f16x3_executed_tflops": exec_tflops,
              "launches": rows, "f16x3_output_sha256": digests}
    print("card (name, power limit, max SM clock): %s" % result["card"])
    print("device-timed step: %.3f ms (%d key frames)  tensor-core launches: %d, %.3f ms" % (step_ms, fps, len(rows), kernel_ms))
    print("3xFP16 launches: %d, %.3f ms per step = %.1f %% of the step, %.1f executed TFLOP/s" % (
        len(f16x3), f16x3_ms, 100.0 * f16x3_ms / step_ms, exec_tflops or 0.0))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps({k: v for k, v in result.items() if k not in ("launches", "f16x3_output_sha256")}))


if __name__ == "__main__":
    main()
