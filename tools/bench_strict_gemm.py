#!/usr/bin/env python
"""Where the strict (fp32x3) step's time goes: every tensor-core launch of one 4-key-frame MEGA R-101 step at 600x1000
(MegaEngine.stepn_batched, as bench.py's roofline pass runs it), timed with a CUDA event pair per launch.

    python tools/bench_strict_gemm.py [--steps 20] [--warmup 5] [--reps 5] [--json FILE]

Prints one row per launch -- shape (m, cout, k, taps), block_n, stream-K, precision, ms and executed TFLOP/s (3 tensor-core
products per multiply-add in the strict modes) -- then the sum over the 3xFP16 launches (conv_gemm_kernel<.., kModeF16x3>)
and its share of the device-timed step (CUDA graphs, device-resident inputs: the step bench.py times), and the card's
name / power limit / max SM clock. The JSON written with --json also holds a SHA-256 digest of the output tensor of every
3xFP16 launch of one further step: two builds that compute the same bits give the same list.

Each launch also gets its floor: the compute floor (executed fp16 products over the dense fp16 peak) and the HBM floor
(bytes it must move over the HBM bandwidth; A once, B, the output and the residual, 4 bytes per value as in the
split-fp16 format), which of the two bounds it, and the measured time over that floor. The peaks are bench.py's:
MEASURED_PEAKS.json when present, else the H100 SXM data sheet. The 3xFP16 launches are then summed per layer family
(stem, res2-4 1x1 and 3x3, RPN, res5, l_fcs[0], relation, predictor), named from the engine functions that made them.

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


FAMILY_OF = {"res5_reduced": "res5", "_reduce": "res5", "rpn_head": "RPN", "_fc0": "l_fcs[0]", "predict_gemm": "predictor",
             "_attention": "relation", "aggregate": "relation", "_aggregate_split": "relation"}


def family(frame, taps):
    """layer family of a launch, from the engine functions on its call stack (innermost first); None if unknown"""
    body = None
    while frame is not None:
        name, loc = frame.f_code.co_name, frame.f_locals
        if name in FAMILY_OF:
            return FAMILY_OF[name]
        if name == "forward" and "si" in loc and "blk" in loc:     # ResNetStages.forward: res2-4, or res5 further out
            body = "res2-4 %s" % ("1x1" if taps == 1 else "3x3")
        elif name == "forward" and type(loc.get("self")).__name__ == "Backbone":
            return body or "stem"
        frame = frame.f_back
    return body


def launch_bytes(info):
    """bytes a conv_gemm launch must move through HBM: A once, B, the output and the residual, 4 bytes per value"""
    m = info["m"] * info["batch"]
    n = m * info["k"] + info["batch"] * info["cout"] * info["k"] * info["taps"] + m * info["cout"] * (2 if info["res"] else 1)
    return 4 * n


def launch_times(step, reps):
    """[(info, flops, ms averaged over reps, layer family)] for every tensor-core launch of one eager step"""
    rec = []

    def hook(run, flops, info):
        fam = family(sys._getframe(1), info.get("taps", 1))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        rec.append((a, b, flops, info, fam))

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
    return [(rec[i][3], rec[i][2], sum(r[0].elapsed_time(r[1]) for r in rec[i::n]) / reps, rec[i][4]) for i in range(n)]


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

    pk = bench.peaks()
    flop_rate, byte_rate = pk["tflops"] * 1e12, pk["hbm_gbs"] * 1e9
    rows = []
    print("%4s %7s %5s %5s %4s %4s %3s %7s %9s %9s %8s %9s %9s %5s %6s  %s" % (
        "#", "m", "cout", "k", "taps", "bn", "sk", "prec", "ms", "TFLOP/s", "MB", "tc_ms", "hbm_ms", "bound", "x", "family"))
    for i, (info, flops, ms, fam) in enumerate(launches):
        if "chain_layers" in info:
            row = {"kind": "conv_chain", "layers": info["chain_layers"], "ms": ms, "flops": flops, "executed_tflops": None}
            print("%4d conv_chain_kernel (%d layers) %34.4f" % (i, info["chain_layers"], ms))
        else:
            prec = PRECISION_NAME.get(info.get("precision"), "?")
            products = 3 if prec in ("3xFP16", "3xTF32") else 1
            nbytes = launch_bytes(info)
            tc_ms, hbm_ms = products * flops / flop_rate * 1e3, nbytes / byte_rate * 1e3
            row = {"kind": "conv_gemm", "m": info["m"] * info["batch"], "cout": info["cout"], "k": info["k"],
                   "taps": info["taps"], "block_n": info["bn"], "stream_k": info["sk"], "precision": prec, "ms": ms,
                   "flops": flops, "executed_tflops": products * flops / (ms * 1e-3) / 1e12, "family": fam,
                   "bytes": nbytes, "compute_floor_ms": tc_ms, "hbm_floor_ms": hbm_ms,
                   "bound": "tc" if tc_ms >= hbm_ms else "hbm", "over_floor": ms / max(tc_ms, hbm_ms)}
            print("%4d %7d %5d %5d %4d %4d %3d %7s %9.4f %9.1f %8.1f %9.4f %9.4f %5s %6.2f  %s" % (
                i, row["m"], row["cout"], row["k"], row["taps"], row["block_n"], row["stream_k"], prec, ms,
                row["executed_tflops"], nbytes / 1e6, tc_ms, hbm_ms, row["bound"], row["over_floor"], fam))
        rows.append(row)
    f16x3 = [r for r in rows if r.get("precision") == "3xFP16"]
    f16x3_ms = sum(r["ms"] for r in f16x3)
    kernel_ms = sum(r["ms"] for r in rows)
    exec_tflops = 3 * sum(r["flops"] for r in f16x3) / (f16x3_ms * 1e-3) / 1e12 if f16x3_ms else None
    result = {"card": card(), "key_frames_per_step": fps, "step_ms": step_ms, "tensor_core_launches": len(rows),
              "tensor_core_ms_per_step": kernel_ms, "f16x3_launches": len(f16x3), "f16x3_ms_per_step": f16x3_ms,
              "f16x3_share_of_step": f16x3_ms / step_ms, "f16x3_executed_tflops": exec_tflops,
              "launches": rows, "f16x3_output_sha256": digests}
    fams = {}
    for r in f16x3:
        f = fams.setdefault(r["family"] or "other", {"launches": 0, "ms": 0.0, "floor_ms": 0.0, "compute_floor_ms": 0.0,
                                                     "hbm_floor_ms": 0.0, "hbm_bound_launches": 0})
        f["launches"] += 1
        f["ms"] += r["ms"]
        f["floor_ms"] += max(r["compute_floor_ms"], r["hbm_floor_ms"])
        f["compute_floor_ms"] += r["compute_floor_ms"]
        f["hbm_floor_ms"] += r["hbm_floor_ms"]
        f["hbm_bound_launches"] += r["bound"] == "hbm"
    result["f16x3_families"] = fams
    result["peaks"] = pk
    print("3xFP16 launches per layer family (floors from %s: %.0f TFLOP/s, %.0f GB/s)" % (pk["src"], pk["tflops"],
                                                                                          pk["hbm_gbs"]))
    print("%-12s %4s %9s %9s %9s %9s %6s %4s" % ("family", "n", "ms", "floor_ms", "tc_ms", "hbm_ms", "x", "hbm"))
    for name, f in sorted(fams.items(), key=lambda kv: -kv[1]["ms"]):
        print("%-12s %4d %9.3f %9.3f %9.3f %9.3f %6.2f %4d" % (name, f["launches"], f["ms"], f["floor_ms"],
                                                              f["compute_floor_ms"], f["hbm_floor_ms"],
                                                              f["ms"] / f["floor_ms"], f["hbm_bound_launches"]))
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
