"""Generate the fixtures of the shipped VID configs that need REDUCE_CHANNEL, MEGA.GLOBAL.RES_STAGE = 0 or
ATTENTION.ADVANCED_STAGE = 0, by running the UNMODIFIED reference with those YAMLs on seeded synthetic weights
(mega_core.b200.synth), and check the oracle (with the reduction conv after res5, tests/configs_oracle.py) against it on
the way with the tolerances of oracle/make_golden.py:

  tests/golden/mega_r50_192x320.pt        configs/MEGA/vid_R_50_C4_MEGA_1x.yaml, 4 frames (the memory fills)
  tests/golden/rdnbase_r101_192x320.pt    configs/RDN/vid_R_101_C4_RDN_base_1x.yaml, 3 frames
  tests/golden/rdnbase_r50_192x320.pt     configs/RDN/vid_R_50_C4_RDN_base_1x.yaml, 3 frames
  tests/golden/vid_configs.json           the YAML contents of the VID configs that reference_configs.json does not
                                          hold, and the reference model's parameter / buffer shapes for all 11

Only outputs are stored, plus the reference model's parameter / buffer list, which the package's module tree must equal.

Run where the reference checkout exists:   python tools/make_golden_configs.py
"""
import contextlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
GOLD = os.path.join(ROOT, "tests", "golden")

import make_golden as mg  # noqa: E402
import ref_import  # noqa: E402
from configs_oracle import oracle_for, reduced_res5  # noqa: E402

VID_CONFIGS = ("configs/vid_R_50_C4_1x.yaml", "configs/vid_R_101_C4_1x.yaml",
               "configs/DFF/vid_R_50_C4_DFF_1x.yaml", "configs/DFF/vid_R_101_C4_DFF_1x.yaml",
               "configs/FGFA/vid_R_50_C4_FGFA_1x.yaml", "configs/FGFA/vid_R_101_C4_FGFA_1x.yaml",
               "configs/MEGA/vid_R_50_C4_MEGA_1x.yaml", "configs/MEGA/vid_R_101_C4_MEGA_1x.yaml",
               "configs/RDN/vid_R_101_C4_RDN_1x.yaml", "configs/RDN/vid_R_101_C4_RDN_base_1x.yaml",
               "configs/RDN/vid_R_50_C4_RDN_base_1x.yaml")

# fixture -> (config, synth arch, seed, make_state_dict options, frames)
CASES = {
    "mega_r50_192x320.pt": ("configs/MEGA/vid_R_50_C4_MEGA_1x.yaml", "mega_r50", 5,
                            {"reduce_channel": True, "global_res_stage": 0}, 4),
    "rdnbase_r101_192x320.pt": ("configs/RDN/vid_R_101_C4_RDN_base_1x.yaml", "rdn_r101", 6, {"advanced_stage": 0}, 3),
    "rdnbase_r50_192x320.pt": ("configs/RDN/vid_R_50_C4_RDN_base_1x.yaml", "rdn_r50", 7,
                               {"reduce_channel": True, "advanced_stage": 0}, 3),
}


@contextlib.contextmanager
def config_instead_of(served, config_file):
    """oracle/make_golden.py's reference runners build `served`; inside, they build `config_file`"""
    saved = ref_import.build_cfg

    def build_cfg(name, opts=()):
        return saved(config_file if name == served else name, opts)
    ref_import.build_cfg = build_cfg
    try:
        yield
    finally:
        ref_import.build_cfg = saved


def ref_state_dict_shapes(config_file):
    cfg = ref_import.build_cfg(config_file)            # imports the reference's mega_core
    from mega_core.modeling.detector import build_detection_model
    model = build_detection_model(cfg)
    return [[k, list(v.shape)] for k, v in model.state_dict().items()]


def golden(config_file, arch, seed, options, n_frames, h=192, w=320):
    print("  %s @%dx%d: reference vs oracle, %d frames" % (config_file, h, w, n_frames))
    mega = arch.startswith("mega")
    total = 40
    sd = mg.synth.make_state_dict(arch, seed=seed, **options)
    frames = [mg.synth.synthetic_frame(i, h, w) for i in range(total)]
    if mega:
        gidx = mg.synth.global_frame_indices(total, seed=seed)
        globals_per_frame = [gidx[:10]] + [[gidx[(10 + t - 1) % total]] for t in range(1, n_frames)]
        with config_instead_of("configs/MEGA/vid_R_101_C4_MEGA_1x.yaml", config_file):
            ref = mg.run_reference_mega(sd, frames, globals_per_frame, n_frames)
    else:
        with config_instead_of("configs/RDN/vid_R_101_C4_RDN_1x.yaml", config_file):
            ref = mg.run_reference_rdn(sd, frames, n_frames)
    gold = {"arch": arch, "seed": seed, "options": options, "config": config_file, "h": h, "w": w, "total": total}
    if mega:
        gold["globals_per_frame"] = globals_per_frame
    orc = oracle_for(gold, sd)
    out = []
    for t in range(n_frames):
        if mega:
            infos = {"frame_category": 0 if t == 0 else 1,
                     "ref_l": frames[1:13] if t == 0 else [frames[min(t + 12, total - 1)]],
                     "ref_g": [frames[j] for j in globals_per_frame[t]]}
        else:
            infos = {"frame_category": 0 if t == 0 else 1,
                     "ref": frames[1:19] if t == 0 else [frames[min(t + 18, total - 1)]]}
        with reduced_res5():
            b, s, l = orc.forward(frames[t], infos)
        r = ref[t]
        assert r["class_logits"].shape == orc.trace["class_logits"].shape, "proposal count differs"
        mg.close(orc.trace["class_logits"], r["class_logits"], 2e-5, "frame %d class_logits" % t)
        mg.close(orc.trace["box_regression"], r["box_regression"], 2e-5, "frame %d box_regression" % t)
        assert torch.equal(l, r["labels"]) and b.shape == r["boxes"].shape, "detections differ (frame %d)" % t
        mg.close(b, r["boxes"], 1e-4, "frame %d det boxes" % t)
        mg.close(s, r["scores"], 1e-5, "frame %d det scores" % t)
        out.append({"class_logits": r["class_logits"], "box_regression": r["box_regression"],
                    "proposals": orc.trace["proposals"], "boxes": r["boxes"], "scores": r["scores"],
                    "labels": r["labels"]})
    gold["frames"] = out
    gold["state_dict_shapes"] = [(k, tuple(s)) for k, s in ref_state_dict_shapes(config_file)]
    return gold


def vid_configs_json():
    import yaml
    with open(os.path.join(GOLD, "reference_configs.json")) as fh:
        stored = json.load(fh)
    yamls = {}
    for name in VID_CONFIGS:
        if name not in stored:
            with open(os.path.join(ref_import.REFERENCE, name)) as fh:
                yamls[name] = yaml.safe_load(fh)
    return {"yaml": yamls, "state_dict_shapes": {name: ref_state_dict_shapes(name) for name in VID_CONFIGS}}


def main():
    torch.set_num_threads(8)
    out = sys.argv[1] if len(sys.argv) > 1 else GOLD
    only = sys.argv[2:]
    if not only or "json" in only:
        with open(os.path.join(out, "vid_configs.json"), "w") as fh:
            json.dump(vid_configs_json(), fh, separators=(",", ":"))
    for name, case in CASES.items():
        if not only or name in only:
            torch.save(golden(*case), os.path.join(out, name))


if __name__ == "__main__":
    main()
