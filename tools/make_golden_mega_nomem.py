"""Generate the fixtures of MEGA without long-range memory (MODEL.VID.MEGA.MEMORY.ENABLE False, the paper's ablation) by
running the UNMODIFIED reference with that key on seeded synthetic weights (mega_core.b200.synth), and check the oracle
without memory (tests/mega_nomem_oracle.py) against it on the way with the tolerances of oracle/make_golden.py:

  tests/golden/mega_r101_nomem_192x320.pt   configs/MEGA/vid_R_101_C4_MEGA_1x.yaml (GLOBAL.RES_STAGE 1), 26 frames: with
                                            memory, the last one would read a full memory of 25 frames; on the weights
                                            of tests/golden/mega_r101_192x320.pt. The outputs of 8 of them are stored
                                            (the first four, 12 / 13 around the window's turn-over, 24 / 25 with a
                                            full memory), which keeps the file small; a test runs all 26 and checks those
  tests/golden/mega_r50_nomem_192x320.pt    configs/MEGA/vid_R_50_C4_MEGA_1x.yaml (REDUCE_CHANNEL, GLOBAL.RES_STAGE 0),
                                            4 frames, on the weights of tests/golden/mega_r50_192x320.pt

Each fixture must exercise the key: the oracle WITH memory (checked against the reference by the fixtures above) on the
same weights and frames gives the same class logits at frame 0, whose memory is empty, and different ones at every later
frame (R-101: 3.1e-3 at frame 1, growing to 0.12 with a full memory; R-50: 9.2e-4 at frame 1); the generator asserts
both. Only outputs are stored.

Run where the reference checkout exists:   python tools/make_golden_mega_nomem.py [out_dir [fixture ...]]
"""
import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
GOLD = os.path.join(ROOT, "tests", "golden")

import make_golden as mg  # noqa: E402
import mega_oracle as mo  # noqa: E402
from configs_oracle import reduced_res5  # noqa: E402
from make_golden_configs import config_instead_of  # noqa: E402
from make_golden_stride3x3 import extra_opts  # noqa: E402
from mega_nomem_oracle import MegaNoMemOracle  # noqa: E402

NOMEM_OPTS = ("MODEL.VID.MEGA.MEMORY.ENABLE", False)
R101 = "configs/MEGA/vid_R_101_C4_MEGA_1x.yaml"

# fixture -> (config, synth arch, seed, make_state_dict options, frames, frames whose outputs are stored (None: all))
CASES = {
    "mega_r101_nomem_192x320.pt": (R101, "mega_r101", 0, {}, 26, (0, 1, 2, 3, 12, 13, 24, 25)),
    "mega_r50_nomem_192x320.pt": ("configs/MEGA/vid_R_50_C4_MEGA_1x.yaml", "mega_r50", 5,
                                  {"reduce_channel": True, "global_res_stage": 0}, 4, None),
}


def golden(config_file, arch, seed, options, n_frames, keep=None, h=192, w=320, total=40):
    print("  %s, MEMORY.ENABLE False @%dx%d: reference vs oracle, %d frames" % (config_file, h, w, n_frames))
    sd = mg.synth.make_state_dict(arch, seed=seed, **options)
    frames = [mg.synth.synthetic_frame(i, h, w) for i in range(total)]
    gidx = mg.synth.global_frame_indices(total, seed=seed)
    globals_per_frame = [gidx[:10]] + [[gidx[(10 + t - 1) % total]] for t in range(1, n_frames)]
    with config_instead_of(R101, config_file), extra_opts(NOMEM_OPTS):
        cfg = mg.ref_import.build_cfg(R101)
        assert not cfg.MODEL.VID.MEGA.MEMORY.ENABLE and cfg.MODEL.VID.MEGA.GLOBAL.ENABLE
        ref = mg.run_reference_mega(sd, frames, globals_per_frame, n_frames)
    ocfg = mo.Cfg(global_res_stage=options.get("global_res_stage", 1))
    orc, with_mem = MegaNoMemOracle(sd, ocfg, record=True), mo.MegaOracle(sd, ocfg, record=True)
    gold = []
    for t in range(n_frames):
        infos = {"frame_category": 0 if t == 0 else 1,
                 "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                 "ref_g": [frames[j] for j in globals_per_frame[t]]}
        with reduced_res5() if options.get("reduce_channel") else contextlib.nullcontext():
            b, s, l = orc.forward(frames[t], infos)
            with_mem.forward(frames[t], infos)
        r = ref[t]
        assert r["class_logits"].shape == orc.trace["class_logits"].shape, "proposal count differs"
        mg.close(orc.trace["class_logits"], r["class_logits"], 2e-5, "frame %d class_logits" % t)
        mg.close(orc.trace["box_regression"], r["box_regression"], 2e-5, "frame %d box_regression" % t)
        assert torch.equal(l, r["labels"]) and b.shape == r["boxes"].shape, "detections differ (frame %d)" % t
        mg.close(b, r["boxes"], 1e-4, "frame %d det boxes" % t)
        mg.close(s, r["scores"], 1e-5, "frame %d det scores" % t)
        diff = (with_mem.trace["class_logits"] - r["class_logits"]).abs().max().item()
        print("  frame %2d: memory-on class logits differ by %.3e" % (t, diff))
        # (2e-5: the oracle's tolerance against the reference; a real difference is more than 5 times that)
        assert (diff < 2e-5) if t == 0 else (diff > 1e-4), "frame %d: memory off and on give %s logits" % (
            t, "different" if t == 0 else "the same")
        if keep is None or t in keep:
            gold.append({"t": t, "class_logits": r["class_logits"], "proposals": orc.trace["proposals"],
                         "boxes": r["boxes"], "scores": r["scores"], "labels": r["labels"]})
    return {"arch": arch, "seed": seed, "options": options, "config": config_file, "memory": False, "h": h, "w": w,
            "total": total, "n_frames": n_frames, "globals_per_frame": globals_per_frame, "frames": gold}


def main():
    torch.set_num_threads(8)
    out = sys.argv[1] if len(sys.argv) > 1 else GOLD
    only = sys.argv[2:]
    for name, case in CASES.items():
        if not only or name in only:
            torch.save(golden(*case), os.path.join(out, name))


if __name__ == "__main__":
    main()
