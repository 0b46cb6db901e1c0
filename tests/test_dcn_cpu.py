"""CPU tests of deformable backbone stages (MODEL.RESNETS.STAGE_WITH_DCN, DCN v1 and modulated v2): which configs the
engines serve and which they refuse, the module tree against the reference's parameter lists, the Caffe2 loader's nested
names, the g++ build of the shared sampling header (csrc/dcn_sample.cuh) against the fp32 restatement of
oracle/train_ops_oracle.py, and the engines' DCN host logic on the CPU stand-ins (tests/cpu_ops.py, plus a stand-in for
ops.dcn_sample defined here) against the fixtures written from the unmodified reference (tools/make_golden_dcn.py)."""
import contextlib
import ctypes
import os
import subprocess
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]

import train_ops_oracle as to  # noqa: E402
from cpu_ops import cpu_ops  # noqa: E402

FIXTURES = ("base_r101_dcn_192x320.pt", "mega_r101_mdcn_192x320.pt", "base_r101_s3x3_mdcn_192x320.pt")


def _gold(fixture):
    return torch.load(os.path.join(GOLD, fixture))


def _sd(gold):
    from mega_core.b200 import synth
    return synth.make_state_dict(gold["arch"], seed=gold["seed"], stage_with_dcn=gold["stage_with_dcn"],
                                 modulated_dcn=gold["modulated"])


def _cfg(method="mega", stages=(False, True, True, False), modulated=False, stride_in_1x1=True, groups=1, wpg=64,
         deformable_groups=1):
    from mega_core.modeling.detector.detectors import vid_config
    cfg = vid_config(method, "R-101-C4", "cpu", num_groups=groups, width_per_group=wpg, stride_in_1x1=stride_in_1x1)
    cfg.MODEL.RESNETS.STAGE_WITH_DCN = tuple(stages)
    cfg.MODEL.RESNETS.WITH_MODULATED_DCN = modulated
    cfg.MODEL.RESNETS.DEFORMABLE_GROUPS = deformable_groups
    return cfg


# ----------------------------------------------------------------------------------------------------------- config
@pytest.mark.parametrize("stride_in_1x1", [True, False])
@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("stages", [(True, False, False, False), (False, True, False, False),
                                    (False, False, True, False), (False, True, True, False), (True, True, True, False)])
def test_served_stage_tuples_are_accepted(stages, modulated, stride_in_1x1):
    from mega_core.modeling.nets import engine_config_from
    for method in ("base", "mega", "rdn", "fgfa", "dff"):
        cfg = engine_config_from(_cfg(method, stages, modulated, stride_in_1x1))
        assert cfg.stride_in_1x1 is stride_in_1x1


def test_res5_entry_is_refused():
    from mega_core.modeling.nets import engine_config_from
    with pytest.raises(NotImplementedError, match="STAGE_WITH_DCN") as e:
        engine_config_from(_cfg(stages=(False, True, True, True)))
    assert "res5" in str(e.value) and "False" in str(e.value)


def test_grouped_deformable_body_is_refused():
    from mega_core.modeling.nets import engine_config_from
    with pytest.raises(NotImplementedError, match="STAGE_WITH_DCN") as e:
        engine_config_from(_cfg(stages=(False, True, True, False), groups=32, wpg=8, stride_in_1x1=False))
    assert "NUM_GROUPS" in str(e.value) and "STRIDE_IN_1X1" not in str(e.value)


def test_deformable_groups_are_refused():
    from mega_core.modeling.nets import engine_config_from
    with pytest.raises(NotImplementedError, match="MODEL.RESNETS.DEFORMABLE_GROUPS"):
        engine_config_from(_cfg(modulated=True, deformable_groups=2))
    engine_config_from(_cfg(stages=(False,) * 4, deformable_groups=2))         # read only with a deformable stage


# ------------------------------------------------------------------------------------------------------ module tree
@pytest.mark.parametrize("fixture", FIXTURES)
def test_module_tree_has_the_reference_parameters(fixture):
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    gold = _gold(fixture)
    model = build_detection_model_from_state_dict(_sd(gold), method=gold["arch"].split("_")[0], device="cpu",
                                                  precision="tf32", stride_in_1x1=gold["stride_in_1x1"])
    r = model.cfg.MODEL.RESNETS
    assert tuple(r.STAGE_WITH_DCN) == tuple(gold["stage_with_dcn"]) and bool(r.WITH_MODULATED_DCN) == gold["modulated"]
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == dict(gold["state_dict_shapes"])
    from mega_core.layers import DFConv2d
    conv2 = model.backbone.body.layer2[0].conv2
    assert isinstance(conv2, DFConv2d) and conv2.stride == (1 if gold["stride_in_1x1"] else 2)


def test_caffe2_nested_names_load_into_the_module_tree():
    """_nest_dcn_convs moves the 3x3 weights of deformable stages to conv2.conv.*; with the offset convs they load"""
    from mega_core.modeling.detector import build_detection_model
    from mega_core.b200 import synth
    from mega_core.utils.c2_model_loading import _nest_dcn_convs
    stages = (False, True, True, False)
    sd = synth.make_state_dict("base_r101", seed=1, stage_with_dcn=stages)
    flat = {k.replace("conv2.conv.weight", "conv2.weight"): v for k, v in sd.items()}
    nested = _nest_dcn_convs(dict(flat), stages + (False,))
    assert set(nested) == set(sd)
    model = build_detection_model(_cfg("base", stages))
    missing = model.load_state_dict(nested, strict=False)
    assert not missing.unexpected_keys and not [k for k in missing.missing_keys if "cell_anchors" not in k]


# --------------------------------------------------------------------------------------- sampling header, g++ build
_HOST = {}


def _host_lib():
    if "lib" not in _HOST:
        so = os.path.join(tempfile.mkdtemp(), "libdcn_sample_host.so")
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-I",
                               os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               "-o", so, os.path.join(ROOT, "tests", "native", "dcn_sample_host.cpp")])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def _identity_weight(c, dtype):
    w = torch.zeros(9 * c, c, 3, 3, dtype=dtype)
    idx = torch.arange(9 * c)
    w.view(9 * c, c, 9)[idx, idx // 9, idx % 9] = 1.0
    return w


def columns(x_nhwc, offset, modulated, stride, dil=1, dtype=torch.float32):
    """the tap-major columns of mega_dcn_sample_nhwc by the oracle's restatement: x [N,H,W,C], offset [N,Ho,Wo,>=18/27]"""
    x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    o = offset.permute(0, 3, 1, 2).to(dtype)
    if dtype == torch.float64:          # the positions as the kernel forms them: one fp32 rounding of base + offset
        n, _, ho, wo = o.shape
        tap = torch.arange(9)
        bh = (torch.arange(ho).view(1, 1, ho, 1) * stride - dil + (tap // 3 * dil).view(1, 9, 1, 1)).double()
        bw = (torch.arange(wo).view(1, 1, 1, wo) * stride - dil + (tap % 3 * dil).view(1, 9, 1, 1)).double()
        o = o.clone()
        o[:, 0:18:2] = (bh + o[:, 0:18:2]).float().double() - bh
        o[:, 1:18:2] = (bw + o[:, 1:18:2]).float().double() - bw
    mask = o[:, 18:27].sigmoid().contiguous() if modulated else None
    c = x.shape[1]
    out = to.deform_conv2d(x, o[:, :18].contiguous(), mask, _identity_weight(c, dtype), None, (stride, stride),
                           (dil, dil), (dil, dil), 1, 1)
    n, _, ho, wo = out.shape
    return out.view(n, c, 9, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, 9 * c)


@pytest.mark.parametrize("dil", [1, 2])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("modulated", [False, True])
def test_host_build_of_the_sampling_header_matches_the_oracle(modulated, stride, dil):
    """every column element within the fp32 rounding of the interpolation, 2^-21 sum |w v| (x mask), against the fp64
    restatement at the kernel's fp32 sample positions; the fp32 restatement sums the same products in another order"""
    g = torch.Generator().manual_seed(3 + stride + 2 * dil)
    n, h, w, c = 2, 23, 37, 32
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = torch.randn(n, h, w, c, generator=g)
    off = torch.randn(n, ho, wo, 32, generator=g) * 2.0
    off[..., :18] += torch.randint(-1, 2, (n, ho, wo, 18), generator=g).float()
    off[0, 0, 0, :18] = torch.tensor([-1.0, 0.0] * 9)                   # the gate's edge: h = -1 reads nothing
    got = torch.zeros(n, ho, wo, 9 * c)
    vp = ctypes.c_void_p
    assert _host_lib().mega_dcn_sample_nhwc(vp(x.data_ptr()), 0, n, h, w, c, vp(off.data_ptr()), 32, int(modulated),
                                            stride, dil, vp(got.data_ptr()), None) == 0
    ref = columns(x, off, modulated, stride, dil, torch.float64)
    S = columns(x.abs(), off, modulated, stride, dil, torch.float64)
    err = (got.double() - ref).abs()
    assert bool((err <= 2.0 ** -21 * S + 1e-30).all()), (err / S.clamp_min(1e-30)).max().item()
    ref32 = columns(x, off, modulated, stride, dil, torch.float32)
    assert bool(((got - ref32).abs().double() <= 2.0 ** -20 * S + 1e-30).all())
    outside = (ref == 0).float().mean().item()
    assert 0 < outside < 0.2, outside


# -------------------------------------------------------------------------------------- engines on the stand-ins
def dcn_sample_stand_in(x, offset, cols, modulated, stride=1, dil=1):
    """ops.dcn_sample on CPU tensors: the restatement's columns, rounded to the storage format of cols"""
    cols.copy_(columns(x.float(), offset, modulated, stride, dil).to(cols.dtype))
    return cols


@contextlib.contextmanager
def dcn_cpu_ops():
    from mega_core.b200 import ops
    saved = ops.dcn_sample
    with cpu_ops():
        ops.dcn_sample = dcn_sample_stand_in
        try:
            yield
        finally:
            ops.dcn_sample = saved


def _match_rows(a, b, tol=0.75):
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _check(eng, det, ref, k, props, logit_tol=1e-3):
    idx = _match_rows(props, ref["proposals"])
    assert (idx >= 0).all() and k == ref["proposals"].shape[0], "proposals differ"
    assert (eng.last_pred[:k][idx, :31] - ref["class_logits"]).abs().max() < logit_tol, "class logits"
    n = int(det.count.reshape(-1)[0])
    assert n == ref["boxes"].shape[0] and torch.equal(det.labels[:n], ref["labels"]), "detections"
    assert torch.allclose(det.boxes[:n], ref["boxes"], atol=2e-2)


@pytest.mark.parametrize("fixture", [FIXTURES[0], FIXTURES[2]])
def test_base_engine_matches_reference_fixture(fixture):
    """BaseEngine from the model's config: v1 on res3 + res4, and modulated with the 3x3-strided layout (stride-2
    sampling in the first res3 / res4 block)"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = _gold(fixture)
    sd = _sd(gold)
    img = synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"])
    with dcn_cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="base", device="cpu", precision="tf32",
                                                      stride_in_1x1=gold["stride_in_1x1"])
        eng = engine.BaseEngine(sd, engine_config_from(model.cfg), device="cpu")
        blocks = [blk for s in eng.backbone.stages.stages for blk in s]
        assert sum(blk.dcn for blk in blocks) == 4 + 23 and all(blk.modulated == gold["modulated"]
                                                                for blk in blocks if blk.dcn)
        det = eng.forward(img, gold["w"], gold["h"])
        k = int(eng.last_cnt[0])
        _check(eng, det, gold, k, eng.last_props[:k])


def test_mega_engine_matches_reference_fixture():
    """MegaEngine, modulated res3 + res4: start_video (look-ahead and global frames), then a steady frame"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = _gold(FIXTURES[1])
    h, w, total, gpf = gold["h"], gold["w"], gold["total"], gold["globals_per_frame"]
    sd = _sd(gold)
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    with dcn_cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="mega", device="cpu", precision="tf32")
        eng = engine.MegaEngine(sd, engine_config_from(model.cfg), device="cpu")
        eng.use_graph = False
        for t in range(2):
            det = (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
                   eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))
            k = int(eng.cur_cnt.view(-1)[0])
            _check(eng, det, gold["frames"][t], k, eng.Bq0[:k])


def test_deformable_block_launch_sequence():
    """a deformable conv2 is the offset conv (3x3, bias, no activation, DCN_OFFSET_ROWS fp32 rows, conv2's stride), the
    sampling at that stride, and a 1x1 contraction with K = 9 C carrying bn2 and the ReLU; plain blocks are unchanged"""
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict("mega_r50_tiny", seed=2, stage_with_dcn=(False, True, False, False), modulated_dcn=True)
    calls = []
    with dcn_cpu_ops():
        conv, samp = ops.conv_gemm, ops.dcn_sample

        def rec(a, wt, out, **kw):
            calls.append(("gemm", tuple(a.shape), tuple(wt.shape), out.dtype, kw.get("stride", (1, 1)),
                          kw.get("relu", False)))
            return conv(a, wt, out, **kw)

        def rec_s(x, off, cols, modulated, stride=1, dil=1):
            calls.append(("sample", tuple(x.shape), tuple(cols.shape), modulated, stride))
            return samp(x, off, cols, modulated, stride, dil)
        ops.conv_gemm, ops.dcn_sample = rec, rec_s
        bb = engine.Backbone(sd, "cpu", stride_in_1x1=False)
        bb.forward(torch.zeros(1, 3, 64, 96))
    i = next(j for j, c in enumerate(calls) if c[0] == "sample")
    off_call, sample, contraction = calls[i - 1], calls[i], calls[i + 1]
    assert off_call == ("gemm", (1, 16, 24, 128), (9, engine.DCN_OFFSET_ROWS, 128), torch.float32, (2, 2), False)
    assert sample == ("sample", (1, 16, 24, 128), (1, 8, 12, 9 * 128), True, 2)
    assert contraction[:3] == ("gemm", (1, 8, 12, 9 * 128), (1, 128, 9 * 128)) and contraction[5] is True
    assert sum(c[0] == "sample" for c in calls) == 1
