#!/usr/bin/env python
"""Where the relation module's time goes: every launch of MegaEngine._attention (Q / K / V' projections, Q.K^T, the
position-biased soft-max, P.V') of one 4-key-frame MEGA R-101 step at 600x1000, in the strict (fp32x3) and the throughput
(f16) mode, each timed with a CUDA event pair.

    python tools/bench_relation.py [--precision fp32x3 f16] [--reps 5] [--json FILE]

One row per launch: the attention it belongs to (G0, L0-L2, G1, named from the engine's att_g / att_l), the launch kind
(proj, qk, pv, or chain for the fp16 chain kernels; softmax), its shape, ms, and the bytes and FLOPs it must move /
compute from its shapes:
  - tensor-core launches: bytes as tools/bench_strict_gemm.py counts them (A once, B, output, residual; 4 B per value),
    FLOPs 2 * m * n * k (algorithmic, not the 3 executed products of the strict mode);
  - soft-max launches: the logits read once and the probabilities written once (fp32 or split-fp16: 4 B, fp16: 2 B), and
    2 * 64 * 16 FLOPs of the position-bias product per (query, key) pair. A kernel that keeps a row's logits in global
    memory between its passes moves three times the logits' bytes more than this.
Each launch's floor is the larger of FLOPs over the fp32 SIMT peak (soft-max) or the dense fp16 peak x 3 products
(strict tensor-core launches) and bytes over the HBM bandwidth; the peaks are bench.peaks().
Then the sums per kind, the device-timed step (CUDA graphs; as bench.py times it) and the card's name / power limit /
max SM clock. Per-launch times come from eager launches with the queue filled ahead (torch.cuda._sleep), so kernels do
not overlap and launch gaps are not counted.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_strict_gemm as bsg  # noqa: E402  (sets MEGA_B200_AUTOTUNE=0: fixed tile heuristic)
import torch  # noqa: E402

import bench  # noqa: E402
from mega_core.b200 import ops  # noqa: E402
from mega_core.modeling.detector import build_detection_model_from_state_dict  # noqa: E402

FP32_SIMT_TFLOPS = 67.0      # H100 SXM data sheet, fp32 (not a measured rate)


def attention_frame(frame):
    while frame is not None:
        if frame.f_code.co_name == "_attention":
            return frame
        frame = frame.f_back
    return None


def att_name(eng, att):
    for i, a in enumerate(eng.att_g):
        if a is att:
            return "G%d" % i
    for i, a in enumerate(eng.att_l):
        if a is att:
            return "L%d" % i
    return "?"


def gemm_kind(info):
    if "chain_layers" in info:
        return "chain-qk" if info["layers"][0]["batch"] == 1 else "chain-pv"
    if info["batch"] == 16:
        return "pv" if info["cout"] == 64 else "qk"
    return "proj"


def record_step(eng, step, reps):
    """[(row dict, ms averaged over reps)] for every launch inside MegaEngine._attention of one eager step"""
    rec = []

    def where():
        fr = attention_frame(sys._getframe(2))
        if fr is None:
            return None
        loc = fr.f_locals
        return "%s nq=%d nref=%d" % (att_name(eng, loc["att"]), loc["nq"], loc["nref"])

    def hook(run, flops, info):
        tag = where()
        if tag is None:
            run()
            return
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        if "chain_layers" in info:
            nbytes = sum(bsg.launch_bytes(li) for li in info["layers"])
            shape = "%d layers" % info["chain_layers"]
        else:
            nbytes = bsg.launch_bytes(info)
            shape = "m=%d n=%d k=%d b=%d sk=%d" % (info["m"], info["cout"], info["k"], info["batch"], info["sk"])
        prec = info.get("precision", info["layers"][0].get("precision") if "layers" in info else None)
        rec.append((a, b, {"att": tag, "kind": gemm_kind(info), "shape": shape, "bytes": nbytes, "flops": flops,
                           "products": 3 if prec == 3 else 1}))

    orig_sm = ops.relation_softmax

    def softmax(logits, n_rows, ldm, scale, **kw):
        tag = where()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = orig_sm(logits, n_rows, ldm, scale, **kw)
        b.record()
        pr = kw.get("probs_f16")
        out_b = 2 if (pr is not None and pr.dtype == torch.float16) else 4
        m = kw.get("m_host", ldm)
        pe = kw.get("boxes_q") is not None
        rec.append((a, b, {"att": tag, "kind": "softmax", "shape": "rows=%d ldm=%d pe=%d" % (n_rows, ldm, pe),
                           "bytes": 16 * n_rows * ldm * (4 + out_b), "flops": 2 * 64 * 16 * n_rows * m if pe else 0,
                           "products": 0}))
        return r

    ops.TIMING_HOOK[0] = hook
    ops.relation_softmax = softmax
    try:
        step(0)
        torch.cuda.synchronize()
        rec.clear()
        for i in range(reps):
            torch.cuda._sleep(100_000_000)
            step(i + 1)
            torch.cuda.synchronize()
    finally:
        ops.TIMING_HOOK[0] = None
        ops.relation_softmax = orig_sm
    n = len(rec) // reps
    assert n * reps == len(rec), "launch sequence differs between steps"
    return [(rec[i][2], sum(r[0].elapsed_time(r[1]) for r in rec[i::n]) / reps) for i in range(n)]


def run_mode(mb, precision, args, pk):
    model = build_detection_model_from_state_dict(mb.sd, method="mega", device=mb.dev, precision=precision)
    eng, fps = model.engine, mb.fps
    eng.use_graph = True
    nb = 16 // fps
    batches = [torch.cat([mb.pairs_dev[(fps * i + j) % 16] for j in range(fps)], 0) for i in range(nb)]

    def step(i):
        return eng.stepn_batched(batches[i % nb], mb.w, mb.h)

    with torch.no_grad():
        model(mb.infos_first())
        for t in range(1, eng.MEMF + 3):
            model(mb.infos_next(t))
        for i in range(4 + args.warmup):
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
            launches = record_step(eng, step, args.reps)
        finally:
            eng._graphs, eng.use_graph = graphs, True
    del model, eng
    torch.cuda.empty_cache()

    tc_rate, simt_rate, byte_rate = pk["tflops"] * 1e12, FP32_SIMT_TFLOPS * 1e12, pk["hbm_gbs"] * 1e9
    rows, kinds = [], {}
    print("== %s (%d key frames per step)" % (precision, fps))
    print("%-20s %-9s %-32s %9s %9s %9s %9s %6s" % ("attention", "kind", "shape", "ms", "MB", "GFLOP", "floor_ms", "x"))
    for r, ms in launches:
        comp_ms = (r["flops"] / simt_rate if r["kind"] == "softmax" else r["products"] * r["flops"] / tc_rate) * 1e3
        floor = max(comp_ms, r["bytes"] / byte_rate * 1e3)
        row = dict(r, ms=ms, floor_ms=floor, bound="compute" if comp_ms >= r["bytes"] / byte_rate * 1e3 else "hbm")
        rows.append(row)
        k = kinds.setdefault(r["kind"], {"launches": 0, "ms": 0.0, "floor_ms": 0.0})
        k["launches"] += 1
        k["ms"] += ms
        k["floor_ms"] += floor
        print("%-20s %-9s %-32s %9.4f %9.1f %9.2f %9.4f %6.2f" % (r["att"], r["kind"], r["shape"], ms, r["bytes"] / 1e6,
                                                                r["flops"] / 1e9, floor, ms / floor if floor else 0.0))
    total = sum(r["ms"] for r in rows)
    for name, k in sorted(kinds.items()):
        print("  %-9s %3d launches %9.3f ms (floor %.3f)" % (name, k["launches"], k["ms"], k["floor_ms"]))
    print("  relation launches %.3f ms of a %.3f ms device-timed step" % (total, step_ms))
    return {"precision": precision, "key_frames_per_step": fps, "step_ms": step_ms, "relation_ms": total,
            "kinds": kinds, "launches": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", nargs="+", default=["fp32x3", "f16"], choices=["fp32x3", "f16"])
    ap.add_argument("--steps", type=int, default=20, help="device-timed steps")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5, help="eager steps whose per-launch times are averaged")
    ap.add_argument("--json", default=None, metavar="FILE")
    args = ap.parse_args()
    ba = argparse.Namespace(arch="mega_r101", height=bench.H, width=bench.W, frames_per_step=bench.DEFAULT_FPS,
                            no_parity=True)
    mb = bench.MegaBench(ba, 0, 1)
    pk = bench.peaks()
    result = {"card": bsg.card(), "peaks": pk, "modes": [run_mode(mb, p, args, pk) for p in args.precision]}
    print("card (name, power limit, max SM clock): %s" % result["card"])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)
    print(json.dumps({"card": result["card"], "modes": {m["precision"]: {"step_ms": m["step_ms"],
                                                                        "relation_ms": m["relation_ms"],
                                                                        "kinds": m["kinds"]} for m in result["modes"]}}))


if __name__ == "__main__":
    main()
