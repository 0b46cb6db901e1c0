"""The oracle's res5 head (oracle/mega_oracle.py) with MODEL.VID.ROI_BOX_HEAD.REDUCE_CHANNEL for the windowed methods:
when the state dict holds roi_heads.box.feature_extractor.conv, its 1x1 conv + ReLU follows res5, before ROIAlign, in
both the per-frame (_forward_ref) and the key-frame (_forward_test) paths of MEGAFeatureExtractor / RDNFeatureExtractor
(roi_box_feature_extractors.py:274-283, :474-483). reduced_res5() makes MegaOracle and RdnOracle use it. BaseOracle
applies the conv itself and must not run inside it."""
import contextlib

import torch.nn.functional as F


@contextlib.contextmanager
def reduced_res5():
    import mega_oracle as mo
    saved = mo.res5_head

    def res5_head(x, sd, prefix, dilation=2):
        y = saved(x, sd, prefix, dilation)
        if prefix == mo.FE + "head." and (mo.FE + "conv.weight") in sd:
            y = F.relu(F.conv2d(y, sd[mo.FE + "conv.weight"], sd[mo.FE + "conv.bias"]))
        return y

    mo.res5_head = res5_head
    try:
        yield
    finally:
        mo.res5_head = saved


def oracle_for(gold, sd):
    """the oracle of a fixture written by tools/make_golden_configs.py (its "options" are make_state_dict's)"""
    import mega_oracle as mo
    opts = gold["options"]
    if gold["arch"].startswith("mega"):
        return mo.MegaOracle(sd, mo.Cfg(global_res_stage=opts.get("global_res_stage", 1)), record=True)
    return mo.RdnOracle(sd, record=True, advanced_stage=opts.get("advanced_stage", 1))
