"""CPU tests of DCN v1 backbone stages with several deformable groups (MODEL.RESNETS.DEFORMABLE_GROUPS > 1): which
configs the engines serve and which they refuse, the module tree and the state-dict loader against the fixtures, the
g++ build of the grouped sampling (tests/native/dcn_sample_groups_host.cpp) against the restatement of
oracle/train_ops_oracle.py, and the engines' host logic on the CPU stand-ins against the fixtures written from the
unmodified reference (tools/make_golden_dcn.py)."""
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
from test_dcn_cpu import _check, _identity_weight, columns as columns_v2  # noqa: E402

FIXTURES = ("base_r101_dcn_g4_192x320.pt", "mega_r101_dcn_g2_192x320.pt", "base_r101_s3x3_dcn_g8_192x320.pt")
METHODS = ("base", "mega", "rdn", "fgfa", "dff")
RES234, RES34, RES4 = (True, True, True, False), (False, True, True, False), (False, False, True, False)


def gold_of(fixture):
    return torch.load(os.path.join(GOLD, fixture))


def state_dict_of(gold):
    from mega_core.b200 import synth
    return synth.make_state_dict(gold["arch"], seed=gold["seed"], stage_with_dcn=gold["stage_with_dcn"],
                                 modulated_dcn=gold["modulated"], deformable_groups=gold["deformable_groups"])


def _cfg(method, stages, dg, modulated=False):
    from mega_core.modeling.detector.detectors import vid_config
    cfg = vid_config(method, "R-101-C4", "cpu")
    cfg.MODEL.RESNETS.STAGE_WITH_DCN = tuple(stages)
    cfg.MODEL.RESNETS.WITH_MODULATED_DCN = modulated
    cfg.MODEL.RESNETS.DEFORMABLE_GROUPS = dg
    return cfg


# ----------------------------------------------------------------------------------------------------------- config
@pytest.mark.parametrize("stages, dg", [(RES234, 2), (RES234, 4), (RES234, 8), (RES34, 16), (RES4, 32),
                                        ((True, False, False, False), 8), (RES34, 4)])
def test_v1_deformable_groups_are_served(stages, dg):
    """any group count that cuts every deformable conv2 width (64 / 128 / 256 for res2 / res3 / res4) into multiples
    of 8 channels"""
    from mega_core.modeling.nets import engine_config_from
    for method in METHODS:
        engine_config_from(_cfg(method, stages, dg))


@pytest.mark.parametrize("stages, dg, width", [(RES234, 16, "64"), (RES34, 32, "128"), (RES4, 64, "256"),
                                               (RES34, 3, "128"), (RES234, 6, "64"), (RES34, 0, "128")])
def test_groups_that_do_not_divide_are_refused(stages, dg, width):
    from mega_core.modeling.nets import engine_config_from
    for method in METHODS:
        with pytest.raises(NotImplementedError, match="MODEL.RESNETS.DEFORMABLE_GROUPS = %d " % dg) as e:
            engine_config_from(_cfg(method, stages, dg))
        assert "multiple" in str(e.value) and width in str(e.value)


@pytest.mark.parametrize("dg", [2, 4])
def test_modulated_groups_stay_refused(dg):
    from mega_core.modeling.nets import engine_config_from
    for method in METHODS:
        with pytest.raises(NotImplementedError, match="MODEL.RESNETS.DEFORMABLE_GROUPS = %d with "
                                                      "MODEL.RESNETS.WITH_MODULATED_DCN" % dg) as e:
            engine_config_from(_cfg(method, RES34, dg, modulated=True))
        assert "one deformable group" in str(e.value)


def test_res5_and_grouped_refusals_keep_their_messages():
    """the res5 and NUM_GROUPS refusals read as before with several deformable groups; the group count adds nothing"""
    from mega_core.modeling.nets import engine_config_from
    with pytest.raises(NotImplementedError) as e:
        engine_config_from(_cfg("mega", (False, True, True, True), 2))
    assert "res5" in str(e.value) and "DEFORMABLE_GROUPS" not in str(e.value)
    cfg = _cfg("mega", RES34, 2)
    cfg.MODEL.RESNETS.NUM_GROUPS, cfg.MODEL.RESNETS.WIDTH_PER_GROUP = 32, 8
    with pytest.raises(NotImplementedError) as e:
        engine_config_from(cfg)
    assert "NUM_GROUPS = 32" in str(e.value) and "DEFORMABLE_GROUPS" not in str(e.value)


def test_synthetic_offsets_keep_group_0():
    """group 0 of a several-group state dict is the one-group offset conv; the other tensors are the same"""
    from mega_core.b200 import synth
    one = synth.make_state_dict("base_r50_tiny", seed=5, stage_with_dcn=RES234)
    four = synth.make_state_dict("base_r50_tiny", seed=5, stage_with_dcn=RES234, deformable_groups=4)
    assert set(one) == set(four)
    for k, v in one.items():
        if ".conv2.offset." in k:
            assert four[k].shape[0] == 72 and torch.equal(four[k][:18], v)
            assert not torch.equal(four[k][18:36], v)
        else:
            assert torch.equal(four[k], v), k


# ------------------------------------------------------------------------------------------------------ module tree
@pytest.mark.parametrize("fixture", FIXTURES)
def test_module_tree_and_loader_read_the_groups(fixture):
    from mega_core.layers import DFConv2d
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = gold_of(fixture)
    model = build_detection_model_from_state_dict(state_dict_of(gold), method=gold["arch"].split("_")[0],
                                                  device="cpu", precision="tf32", stride_in_1x1=gold["stride_in_1x1"])
    r = model.cfg.MODEL.RESNETS
    assert r.DEFORMABLE_GROUPS == gold["deformable_groups"] and not r.WITH_MODULATED_DCN
    assert tuple(r.STAGE_WITH_DCN) == tuple(gold["stage_with_dcn"])
    got = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert got == dict(gold["state_dict_shapes"])
    conv2 = model.backbone.body.layer3[0].conv2
    assert isinstance(conv2, DFConv2d) and conv2.offset.out_channels == 18 * gold["deformable_groups"]
    engine_config_from(model.cfg)


# ---------------------------------------------------------------------------------- grouped sampling, g++ build
_HOST = {}


def host_lib(name="dcn_sample_groups_host"):
    """the g++ build of tests/native/<name>.cpp"""
    if name not in _HOST:
        so = os.path.join(tempfile.mkdtemp(), "lib%s.so" % name)
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-I",
                               os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               "-o", so, os.path.join(ROOT, "tests", "native", name + ".cpp")])
        _HOST[name] = ctypes.CDLL(so)
    return _HOST[name]


def host_columns(x, off, dg, stride, dil=1, modulated=False):
    """columns of the g++ build: x [N,H,W,C] fp32, off [N,Ho,Wo,ld] fp32"""
    n, h, w, c = x.shape
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    out = torch.zeros(n, ho, wo, 9 * c)
    vp = ctypes.c_void_p
    assert host_lib().mega_dcn_sample_nhwc_groups(vp(x.data_ptr()), 0, n, h, w, c, dg, vp(off.data_ptr()),
                                                  off.shape[3], int(modulated), stride, dil, vp(out.data_ptr()),
                                                  None) == 0
    return out


def columns(x_nhwc, offset, dg, stride, dil=1, dtype=torch.float32):
    """the tap-major columns of mega_dcn_sample_nhwc_groups (DCN v1) by the oracle's restatement: x [N,H,W,C],
    offset [N,Ho,Wo,>=18 dg]; in fp64 the sample positions are the kernel's, one fp32 rounding of base + offset"""
    x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    o = offset.permute(0, 3, 1, 2)[:, :18 * dg].to(dtype).contiguous()
    if dtype == torch.float64:
        n, _, ho, wo = o.shape
        tap = torch.arange(9)
        bh = (torch.arange(ho).view(1, 1, ho, 1) * stride - dil + (tap // 3 * dil).view(1, 9, 1, 1)).double()
        bw = (torch.arange(wo).view(1, 1, 1, wo) * stride - dil + (tap % 3 * dil).view(1, 9, 1, 1)).double()
        g = o.view(n, dg, 18, ho, wo).clone()
        g[:, :, 0::2] = (bh.unsqueeze(1) + g[:, :, 0::2]).float().double() - bh.unsqueeze(1)
        g[:, :, 1::2] = (bw.unsqueeze(1) + g[:, :, 1::2]).float().double() - bw.unsqueeze(1)
        o = g.view(n, 18 * dg, ho, wo)
    c = x.shape[1]
    out = to.deform_conv2d(x, o, None, _identity_weight(c, dtype), None, (stride, stride), (dil, dil), (dil, dil), 1,
                           dg)
    n, _, ho, wo = out.shape
    return out.view(n, c, 9, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, 9 * c)


def _sampling_case(seed, n, h, w, c, dg, stride, ld=None):
    g = torch.Generator().manual_seed(seed)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = torch.randn(n, h, w, c, generator=g)
    off = torch.randn(n, ho, wo, ld or 18 * dg, generator=g) * 2.0
    off[..., :18 * dg] += torch.randint(-1, 2, (n, ho, wo, 18 * dg), generator=g).float()    # some integer positions
    return x, off


@pytest.mark.parametrize("dil", [1, 2])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("dg, c", [(2, 64), (4, 64), (8, 64), (4, 32)])
def test_host_build_of_grouped_sampling_matches_the_oracle(dg, c, stride, dil):
    """every column element within the fp32 rounding of the interpolation, 2^-21 sum |w v|, against the fp64
    restatement at the kernel's fp32 sample positions, and within 2^-20 sum |w v| of the fp32 restatement"""
    x, off = _sampling_case(17 + dg + stride + 2 * dil, 2, 21, 34, c, dg, stride, ld=-(-18 * dg // 32) * 32)
    off[1, 0, 0, :18 * dg] = torch.tensor([-1.0, 0.0] * 9 * dg)                   # the gate's edge: h = -1 reads nothing
    got = host_columns(x, off, dg, stride, dil)
    ref = columns(x, off, dg, stride, dil, torch.float64)
    S = columns(x.abs(), off, dg, stride, dil, torch.float64)
    err = (got.double() - ref).abs()
    assert bool((err <= 2.0 ** -21 * S + 1e-30).all()), (err / S.clamp_min(1e-30)).max().item()
    ref32 = columns(x, off, dg, stride, dil, torch.float32)
    assert bool(((got - ref32).abs().double() <= 2.0 ** -20 * S + 1e-30).all())
    # each group samples at its own positions: group 0's offsets everywhere give other columns
    same = off.clone()
    same[..., :18 * dg] = off[..., :18].repeat(1, 1, 1, dg)
    other = host_columns(x, same, dg, stride, dil).view(*got.shape[:3], 9, dg, c // dg)
    g = got.view(*got.shape[:3], 9, dg, c // dg)
    assert torch.equal(other[..., 0, :], g[..., 0, :])
    assert all(not torch.equal(other[..., k, :], g[..., k, :]) for k in range(1, dg))


@pytest.mark.parametrize("modulated", [False, True])
def test_one_group_host_build_equals_the_plain_entry(modulated):
    """deformable_groups = 1 is mega_dcn_sample_nhwc bit for bit (tests/native/dcn_sample_host.cpp)"""
    x, off = _sampling_case(23, 2, 19, 27, 64, 1, 2, ld=32)
    new = host_columns(x, off, 1, 2, 1, modulated)
    old = torch.zeros_like(new)
    vp = ctypes.c_void_p
    assert host_lib("dcn_sample_host").mega_dcn_sample_nhwc(vp(x.data_ptr()), 0, 2, 19, 27, 64, vp(off.data_ptr()), 32,
                                                            int(modulated), 2, 1, vp(old.data_ptr()), None) == 0
    assert torch.equal(new.view(torch.int32), old.view(torch.int32))


def test_host_build_refuses_what_the_entry_point_refuses():
    x = torch.zeros(1, 5, 5, 64)
    vp = ctypes.c_void_p
    for dg, ld, modulated in ((16, 288, 0), (3, 54, 0), (2, 35, 0), (2, 54, 1)):    # 4 channels, 64 % 3, ld, v2
        off = torch.zeros(1, 5, 5, ld)
        out = torch.zeros(1, 5, 5, 9 * 64)
        assert host_lib().mega_dcn_sample_nhwc_groups(vp(x.data_ptr()), 0, 1, 5, 5, 64, dg, vp(off.data_ptr()), ld,
                                                      modulated, 1, 1, vp(out.data_ptr()), None) == 1


# -------------------------------------------------------------------------------------- engines on the stand-ins
def dcn_sample_stand_in(x, offset, cols, modulated, stride=1, dil=1, deformable_groups=1):
    """ops.dcn_sample on CPU tensors: the restatement's columns, rounded to the storage format of cols (v1)"""
    assert not modulated or deformable_groups == 1
    if modulated:
        cols.copy_(columns_v2(x.float(), offset, True, stride, dil).to(cols.dtype))
    else:
        cols.copy_(columns(x.float(), offset, deformable_groups, stride, dil).to(cols.dtype))
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


def _dcn_blocks(eng):
    return [blk for s in eng.backbone.stages.stages for blk in s if blk.dcn]


@pytest.mark.parametrize("fixture", [FIXTURES[0], FIXTURES[2]])
def test_base_engine_matches_reference_fixture(fixture):
    """BaseEngine from the model's config: 4 groups on res3 + res4, and 8 groups on res2 - res4 with the 3x3-strided
    layout (8 channels per group in res2, stride-2 sampling in the first res3 / res4 block)"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = gold_of(fixture)
    sd = state_dict_of(gold)
    img = synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"])
    with dcn_cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="base", device="cpu", precision="tf32",
                                                      stride_in_1x1=gold["stride_in_1x1"])
        eng = engine.BaseEngine(sd, engine_config_from(model.cfg), device="cpu")
        blocks = _dcn_blocks(eng)
        assert len(blocks) == sum(n for n, on in zip((3, 4, 23), gold["stage_with_dcn"]) if on)
        assert all(blk.dg == gold["deformable_groups"] and not blk.modulated for blk in blocks)
        det = eng.forward(img, gold["w"], gold["h"])
        k = int(eng.last_cnt[0])
        _check(eng, det, gold, k, eng.last_props[:k])


def test_mega_engine_matches_reference_fixture():
    """MegaEngine, 2 groups on res2 - res4: start_video (look-ahead and global frames), then three steady frames"""
    from mega_core.b200 import engine, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    gold = gold_of(FIXTURES[1])
    h, w, total, gpf = gold["h"], gold["w"], gold["total"], gold["globals_per_frame"]
    sd = state_dict_of(gold)
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    with dcn_cpu_ops():
        model = build_detection_model_from_state_dict(sd, method="mega", device="cpu", precision="tf32")
        eng = engine.MegaEngine(sd, engine_config_from(model.cfg), device="cpu")
        eng.use_graph = False
        assert all(blk.dg == 2 for blk in _dcn_blocks(eng)) and len(_dcn_blocks(eng)) == 30
        for t in range(len(gold["frames"])):
            det = (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
                   eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))
            k = int(eng.cur_cnt.view(-1)[0])
            _check(eng, det, gold["frames"][t], k, eng.Bq0[:k])


@pytest.mark.parametrize("dg, rows", [(2, 64), (4, 96), (8, 160)])
def test_grouped_block_launch_sequence(dg, rows):
    """a grouped deformable conv2 is still three launches: the offset conv (3x3, bias, no activation, 18 dg rows padded
    to a multiple of 32, fp32, conv2's stride), the sampling with the group count, and the 1x1 contraction (K = 9 C)
    carrying bn2 and the ReLU"""
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict("mega_r50_tiny", seed=2, stage_with_dcn=(False, True, False, False),
                               deformable_groups=dg)
    calls = []
    with dcn_cpu_ops():
        conv, samp = ops.conv_gemm, ops.dcn_sample

        def rec(a, wt, out, **kw):
            calls.append(("gemm", tuple(a.shape), tuple(wt.shape), tuple(out.shape), out.dtype,
                          kw.get("stride", (1, 1)), kw.get("relu", False)))
            return conv(a, wt, out, **kw)

        def rec_s(x, off, cols, modulated, stride=1, dil=1, **kw):
            calls.append(("sample", tuple(x.shape), tuple(off.shape), tuple(cols.shape), modulated, stride, kw))
            return samp(x, off, cols, modulated, stride, dil, **kw)
        ops.conv_gemm, ops.dcn_sample = rec, rec_s
        bb = engine.Backbone(sd, "cpu", stride_in_1x1=False)
        bb.forward(torch.zeros(1, 3, 64, 96))
    i = next(j for j, c in enumerate(calls) if c[0] == "sample")
    off_call, sample, contraction = calls[i - 1], calls[i], calls[i + 1]
    assert off_call == ("gemm", (1, 16, 24, 128), (9, rows, 128), (1, 8, 12, rows), torch.float32, (2, 2), False)
    assert sample == ("sample", (1, 16, 24, 128), (1, 8, 12, rows), (1, 8, 12, 9 * 128), False, 2,
                      {"deformable_groups": dg})
    assert contraction[:3] == ("gemm", (1, 8, 12, 9 * 128), (1, 128, 9 * 128)) and contraction[6] is True
    assert sum(c[0] == "sample" for c in calls) == 1
    blk = bb.stages.stages[1][0]
    w = sd["backbone.body.layer2.0.conv2.offset.weight"]
    assert torch.equal(blk.wo[:, :18 * dg].cpu(), w.permute(2, 3, 0, 1).reshape(9, 18 * dg, 128))
    assert not blk.wo[:, 18 * dg:].any() and not blk.bo[18 * dg:].any()
