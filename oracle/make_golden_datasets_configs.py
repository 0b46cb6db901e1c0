"""Regenerate tests/golden/reference_datasets.pt and tests/golden/reference_configs.json from the UNMODIFIED reference
(where it is importable, see ref_import.py).

    python oracle/make_golden_datasets_configs.py [scratch_dir]

reference_datasets.pt: what the reference's own dataset classes return over the synthetic ImageNet-VID tree of
tests/test_datasets_cpu.make_tree (oracle/run_ref_datasets.py), with image tensors reduced to (shape, dtype, SHA-256) and
paths made relative to the tree root ("<tree>"), which is what test_datasets_equal_the_reference_classes compares.
reference_configs.json: the key/value contents of the reference's configs/*.yaml that
test_reference_yaml_configs_merge_and_drive_the_loader merges."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.environ.get("MEGA_REFERENCE", "/root/reference")
GOLD = os.path.join(ROOT, "tests", "golden")
CONFIGS = ["configs/BASE_RCNN_1gpu.yaml", "configs/MEGA/vid_R_101_C4_MEGA_1x.yaml", "configs/RDN/vid_R_101_C4_RDN_1x.yaml",
           "configs/FGFA/vid_R_101_C4_FGFA_1x.yaml", "configs/DFF/vid_R_101_C4_DFF_1x.yaml", "configs/vid_R_50_C4_1x.yaml"]


def digest(a, tree):
    if hasattr(a, "tensors"):
        a = a.tensors
    if torch.is_tensor(a):
        t = a.contiguous()
        return ("tensor", tuple(t.shape), str(t.dtype), hashlib.sha256(t.numpy().tobytes()).hexdigest())
    if isinstance(a, (list, tuple)):
        return ("seq", [digest(x, tree) for x in a])
    if isinstance(a, str):
        a = a.replace(tree, "<tree>")
    return ("value", a)


def main():
    work = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "mega.pytorch_b200"))
    from test_datasets_cpu import make_tree
    tree = os.path.join(work, "ds")
    make_tree(tree)
    raw = os.path.join(work, "ref_items.pt")
    subprocess.run([sys.executable, os.path.join(ROOT, "oracle", "run_ref_datasets.py"), tree, raw], check=True)
    ref = torch.load(raw, weights_only=False)
    out = {}
    for key, d in ref.items():
        items = []
        for it in d["items"]:
            it = dict(it)
            imgs = it["images"]
            it["images"] = {k: digest(v, tree) for k, v in imgs.items()} if isinstance(imgs, dict) else digest(imgs, tree)
            items.append(it)
        out[key] = dict(d, items=items)
    torch.save(out, os.path.join(GOLD, "reference_datasets.pt"))
    configs = {n: yaml.safe_load(open(os.path.join(REFERENCE, n))) for n in CONFIGS}
    with open(os.path.join(GOLD, "reference_configs.json"), "w") as fh:
        json.dump(configs, fh, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
