"""Fill and save the autotuned (block_n, stream_k) table of every contraction shape the repo's GPU tests, smoke() and
bench.py launch, so that tile choices -- hence summation orders, hence parity numbers -- are pinned:
    python tools/tune_all.py            -> gpurun_out/tuned_b200.json  (copy to mega.pytorch_b200/mega_core/b200/)
Runs the GPU test-suite in-process (its engines autotune every new shape), then the benchmark configurations
(MEGA R-101 at 600x1000 in f16 and fp32x3 with 1 / 2 / 4 key frames per step, tf32; the frame-parallel row splits;
MEGA R-101 / X-101 with 3x3-strided bottlenecks;
RDN / FGFA), and dumps the union."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "mega.pytorch_b200")):
    sys.path.insert(0, p)
import pytest  # noqa: E402
import torch  # noqa: E402

from mega_core.b200 import engine, ops, synth  # noqa: E402

out = os.path.join(ROOT, "gpurun_out", "tuned_b200.json")
os.makedirs(os.path.dirname(out), exist_ok=True)
if "--no-tests" not in sys.argv:
    rc = pytest.main(["-q", "-m", "gpu", "-p", "no:cacheprovider", "--no-header", "-x", os.path.join(ROOT, "tests")])
    print("pytest rc", rc, "entries", len(ops.TUNED))
    ops.save_tuned(out)
dev = torch.device("cuda:0")
h, w = 600, 1000
frames = [synth.synthetic_frame(i, h, w).to(dev) for i in range(16)]
pairs = [torch.cat([frames[(i + 12) % 16], frames[(5 * i + 3) % 16]], 0) for i in range(16)]
sd = synth.make_state_dict("mega_r101", seed=0)
with torch.no_grad():
    for prec in ("f16", "fp32x3", "tf32"):
        eng = engine.MegaEngine(sd, engine.EngineConfig(precision=prec), device=dev)
        eng.start_video(frames[0], frames[1:13], [frames[(3 * j + 1) % 16] for j in range(10)], w, h)
        for i in range(2):
            eng.step_batched(pairs[i], w, h)
        if prec in ("f16", "fp32x3"):
            for n in (2, 4):
                eng.stepn_batched(torch.cat([pairs[j] for j in range(n)], 0), w, h)
            pl = torch.stack([eng.ref_payload(pairs[j], w, h) for j in range(2)])
            eng.dist_step(None, w, h, rank=0, world=2, payloads=pl)      # owner + state row splits of the multi-GPU paths
            eng.dist_step(None, w, h, rank=1, world=2, payloads=pl)
        torch.cuda.synchronize()
        print(prec, "entries", len(ops.TUNED), flush=True)
        del eng
        torch.cuda.empty_cache()
        ops.save_tuned(out)
    # MODEL.RESNETS.STRIDE_IN_1X1 False, dense and X-101 32x8d: the full-resolution conv1 and the 3x3 / stride-2 conv2 of
    # res3 / res4's first blocks (150x250 -> 75x125, 75x125 -> 38x63)
    for arch in ("mega_r101", "mega_x101"):
        sdx = synth.make_state_dict(arch, seed=0)
        for prec in ("f16", "fp32x3"):
            eng = engine.MegaEngine(sdx, engine.EngineConfig(precision=prec, stride_in_1x1=False), device=dev)
            eng.start_video(frames[0], frames[1:13], [frames[(3 * j + 1) % 16] for j in range(10)], w, h)
            eng.step_batched(pairs[0], w, h)
            eng.stepn_batched(torch.cat([pairs[j] for j in range(4)], 0), w, h)
            torch.cuda.synchronize()
            print(arch, prec, "stride_in_1x1 False: entries", len(ops.TUNED), flush=True)
            del eng
            torch.cuda.empty_cache()
            ops.save_tuned(out)
    for arch, cls, kw in (("rdn_r101", engine.RdnEngine, dict(all_frame_interval=37, key_frame_location=18, stage=2, advanced_stage=1)),
                          ("fgfa_r101", engine.FgfaEngine, dict(all_frame_interval=19, key_frame_location=9))):
        sdx = synth.make_state_dict(arch, seed=4)
        eng = cls(sdx, engine.EngineConfig(precision="f16", **kw), device=dev)
        look = eng.L - eng.cfg.key_frame_location - 1
        eng.start_video(frames[0], [frames[(j + 1) % 16] for j in range(look)], w, h)
        eng.step(frames[3], w, h)
        torch.cuda.synchronize()
        print(arch, "entries", len(ops.TUNED), flush=True)
        del eng
        torch.cuda.empty_cache()
        ops.save_tuned(out)
print("saved", out, len(ops.TUNED))
