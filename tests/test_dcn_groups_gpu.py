"""GPU tests of DCN v1 backbone stages with several deformable groups (MODEL.RESNETS.DEFORMABLE_GROUPS > 1):
  * the deformable conv2 layer as the engines launch it (offset conv with 18 dg rows, grouped sampling, contraction with
    FrozenBN and ReLU) for dg 2 / 4 / 8 in tf32, split-fp16 (fp32x3) and f16, stride 1 / 2, on odd map sizes: each
    launch against float64 with the bounds of tests/test_dcn_gpu.py;
  * the grouped sampling kernel against the g++ build (tests/native/dcn_sample_groups_host.cpp), bit for bit in fp32,
    and its one-group form against mega_dcn_sample_nhwc, bit for bit in every storage format;
  * the base and MEGA engines against the fixtures of tools/make_golden_dcn.py in f16 and fp32x3;
  * the f16 body as chain segments against per-layer launches, CUDA-graph replay against eager runs,
    model.forward_frames against one model(images) call per frame;
  * the DFF / FGFA backbones against the base engine's, RDN's against MEGA's; parallel.wave_selfcheck with 2 groups."""
import ctypes
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]

import train_ops_oracle as to  # noqa: E402
from conv_gemm_ref import conv_gemm_ref  # noqa: E402
from test_conv_gemm_conformance_gpu import _bound_check  # noqa: E402
from test_dcn_gpu import _decode, _steps  # noqa: E402
from test_dcn_groups_cpu import FIXTURES, gold_of, host_columns, state_dict_of  # noqa: E402
from test_stride3x3_gpu import _match_rows  # noqa: E402

MODES = {"tf32": (0, 0), "split16": (1, 3), "f16": (0, 2)}     # -> (ops.precision, conformance mode of the bound)
RES34, RES234 = (False, True, True, False), (True, True, True, False)


def _block_sd(c, dg, seed):
    """one bottleneck, c channels throughout, whose conv2 is a DCN v1 DFConv2d with dg groups (offsets ~1.5 pixels)"""
    from mega_core.b200 import synth
    g = torch.Generator().manual_seed(seed)
    sd = {}
    p = "layer2.0."
    sd[p + "conv1.weight"] = synth._kaiming((c, c, 1, 1), g)
    sd[p + "conv2.conv.weight"] = synth._kaiming((c, c, 3, 3), g)
    sd[p + "conv2.offset.weight"] = synth._kaiming((18 * dg, c, 3, 3), g, gain=2.0)
    sd[p + "conv2.offset.bias"] = torch.randn(18 * dg, generator=g) * 0.5
    sd[p + "conv3.weight"] = synth._kaiming((c, c, 1, 1), g)
    for bn in ("bn1.", "bn2.", "bn3."):
        synth._bn(sd, p + bn, c, g)
    return sd


def _cols64(x64, offset, dg, stride):
    """[N,C,H,W] fp64 -> columns [N,Ho,Wo,9C] tap-major (fp64 restatement of the grouped sampling, on the host)"""
    c = x64.shape[1]
    cpu = torch.device("cpu")
    w = torch.zeros(9 * c, c, 3, 3, dtype=torch.float64)
    idx = torch.arange(9 * c)
    w.view(9 * c, c, 9)[idx, idx // 9, idx % 9] = 1.0
    out = to.deform_conv2d(x64.to(cpu), offset.to(cpu), None, w, None, (stride, stride), (1, 1), (1, 1), 1, dg)
    n, _, ho, wo = out.shape
    return out.view(n, c, 9, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, 9 * c).to(x64.device)


@pytest.mark.parametrize("hw", [(75, 125), (38, 63)])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("dg", [2, 4, 8])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_grouped_deformable_conv2_layer_matches_fp64(cuda_dev, mode, dg, stride, hw):
    from mega_core.b200 import engine, ops
    prec, cmode = MODES[mode]
    c, n = 64, 1
    sd = _block_sd(c, dg, seed=7 * stride + hw[0] + 100 * dg)
    dtype = torch.float16 if mode == "f16" else torch.float32
    st = engine.ResNetStages(sd, "", (2,), cuda_dev, first_stride_of=lambda li: stride, dtype=dtype,
                             stride_in_1x1=False)
    blk = st.stages[0][0]
    rows = -(-18 * dg // 32) * 32
    assert blk.dcn and blk.dg == dg and not blk.modulated and blk.off_rows == rows
    if mode == "split16":
        st.use_split16()
    h, w = hw
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    g = torch.Generator(device=cuda_dev).manual_seed(11)
    x = torch.randn(n, h, w, c, device=cuda_dev, generator=g).relu()
    t1 = x.half() if mode == "f16" else (ops.pack_split16(x.contiguous()) if mode == "split16" else x)
    t2 = st._buf("t2", (n, ho, wo, c))
    with ops.precision(prec):
        st._dcn_conv2(blk, t1, t2, stride, 0)
    torch.cuda.synchronize()
    fmt = "f16" if mode == "f16" else ("split" if mode == "split16" else "f32")
    a64 = _decode(t1, fmt)
    off = st._bufs[("dcn_off", (n, ho, wo, rows), 0)]
    cols = st._bufs[("dcn_cols", (n, ho, wo, 9 * c), 0)]
    what = "%s dg %d stride %d %s" % (mode, dg, stride, hw)
    # 1. offset conv: 3x3, bias, fp32 output, 18 dg rows and zero padding
    acc = ops._split16_weight(blk.wo) if mode == "split16" else 1.0
    _, ref, P, Q = conv_gemm_ref(a64, _decode(blk.wo, fmt), taps=(3, 3), pad=1, stride=(stride, stride), k=c, n_img=n,
                                 out_hw=(ho, wo), cout=rows, bias=blk.bo, acc_scale=acc)[0]
    _bound_check(cmode, off.double(), ref, P, Q, "f32", "offset conv " + what)
    assert not off[..., 18 * dg:].any()
    # 2. sampling of t1's stored values at the stored offsets, each group at its own
    offset = off.double().permute(0, 3, 1, 2)[:, :18 * dg].contiguous()
    xin = a64.permute(0, 3, 1, 2).contiguous()
    ref = _cols64(xin, offset, dg, stride)
    S = _cols64(xin.abs(), offset, dg, stride)          # sum of |w v| over the four corners
    got = _decode(cols, fmt)
    pos = 2.0 ** -23 * (h + w + 4) * xin.abs().amax().item()
    bound = 2.0 ** -20 * S + pos + {"f16": 2.0 ** -11 * ref.abs() + 2.0 ** -24,
                                    "split": 2.0 ** -22 * ref.abs() + 2.0 ** -25, "f32": 1e-30}[fmt]
    err = (got - ref).abs()
    assert bool((err <= bound).all()), "sampling %s: max err %.3e, worst err / bound %.3f" % (
        what, err.max().item(), (err / bound).max().item())
    assert (ref == 0).float().mean().item() < 0.2 and (ref != 0).any()
    one = _cols64(xin, offset[:, :18].repeat(1, dg, 1, 1), dg, stride)      # group 0's positions everywhere
    per_group = (one - ref).abs().view(n, ho, wo, 9, dg, c // dg).amax((0, 1, 2, 3, 5))
    assert per_group[0] == 0 and bool((per_group[1:] > 1e-3).all()), per_group
    # 3. contraction over the columns (K = 9 C) with FrozenBN and ReLU
    acc = ops._split16_weight(blk.w2) if mode == "split16" else 1.0
    scale = None if mode == "split16" else blk.s2
    _, ref, P, Q = conv_gemm_ref(got, _decode(blk.w2, fmt), k=9 * c, n_img=n, out_hw=(ho, wo), cout=c, bias=blk.b2,
                                 scale=scale, relu=1, acc_scale=acc)[0]
    _bound_check(cmode, _decode(t2, fmt), ref, P, Q, fmt, "contraction " + what)


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("dg, c", [(2, 64), (4, 64), (8, 64), (16, 256), (32, 256)])
def test_grouped_sampling_kernel_equals_host_build(cuda_dev, dg, c, stride):
    """fp32, bit for bit against the g++ build of dcn_sample.cuh; 16 and 32 groups run one pixel per CTA"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(5 + dg)
    n, h, w = 2, 37, 61
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    ld = -(-18 * dg // 32) * 32
    x = torch.randn(n, h, w, c, generator=g)
    off = torch.randn(n, ho, wo, ld, generator=g) * 2.0
    off[..., :18 * dg] += torch.randint(-1, 2, (n, ho, wo, 18 * dg), generator=g).float()    # some integer positions
    cols = ops.dcn_sample(x.to(cuda_dev), off.to(cuda_dev), torch.zeros(n, ho, wo, 9 * c, device=cuda_dev), False,
                          stride, deformable_groups=dg).cpu()
    host = host_columns(x, off, dg, stride)
    assert torch.equal(cols.view(torch.int32), host.view(torch.int32))


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("fmt", ["f32", "f16", "split"])
def test_one_group_entry_equals_the_plain_entry(cuda_dev, fmt, modulated):
    """mega_dcn_sample_nhwc_groups with one group writes mega_dcn_sample_nhwc's bits in all three storage formats"""
    from mega_core import _lib
    from mega_core.b200 import ops
    g = torch.Generator(device=cuda_dev).manual_seed(9)
    n, h, w, c, stride = 2, 29, 47, 128, 2
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = torch.randn(n, h, w, c, device=cuda_dev, generator=g)
    off = torch.randn(n, ho, wo, 32, device=cuda_dev, generator=g) * 2.0
    code = {"f32": 0, "f16": 1, "split": 2}[fmt]
    if fmt == "f16":
        x = x.half()
    elif fmt == "split":
        x = ops.pack_split16(x.contiguous())
    outs = []
    for entry in ("plain", "groups"):
        cols = torch.full((n, ho, wo, 9 * c), float("nan"), device=cuda_dev, dtype=x.dtype)
        args = (ops.ptr(x), code, n, h, w, c)
        tail = (ops.ptr(off), 32, int(modulated), stride, 1, ops.ptr(cols), ops.stream_ptr())
        if entry == "plain":
            ops.check(_lib.lib.mega_dcn_sample_nhwc(*(args + tail)), "mega_dcn_sample_nhwc")
        else:
            ops.check(_lib.lib.mega_dcn_sample_nhwc_groups(*(args + (1,) + tail)), "mega_dcn_sample_nhwc_groups")
        torch.cuda.synchronize()
        outs.append(cols.view(torch.int16 if fmt == "f16" else torch.int32).cpu())
    assert torch.equal(outs[0], outs[1])


def test_entry_point_refuses_bad_groups(cuda_dev):
    from mega_core import _lib
    from mega_core.b200 import ops
    x = torch.zeros(1, 5, 5, 64, device=cuda_dev)
    cols = torch.zeros(1, 5, 5, 9 * 64, device=cuda_dev)
    off = torch.zeros(1, 5, 5, 64, device=cuda_dev)
    for dg, ld, modulated in ((16, 64, 0), (3, 64, 0), (4, 64, 0), (2, 64, 1)):  # 4 channels, 64 % 3, ld < 72, v2
        with pytest.raises(_lib.MegaError):
            ops.check(_lib.lib.mega_dcn_sample_nhwc_groups(ops.ptr(x), 0, 1, 5, 5, 64, dg, ops.ptr(off), ld, modulated,
                                                           1, 1, ops.ptr(cols), ops.stream_ptr()), "groups")


# ------------------------------------------------------------------------------------------------ engines vs fixtures
def _load(fixture, cuda_dev):
    from mega_core.b200 import synth
    gold = gold_of(fixture)
    sd = state_dict_of(gold)
    n = gold.get("total", gold.get("frame_index", 0) + 1)
    frames = [synth.synthetic_frame(i, gold["h"], gold["w"]).to(cuda_dev) for i in range(n)]
    return gold, sd, frames


def _engine(gold, sd, precision, cuda_dev):
    from mega_core.b200 import engine
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    method = gold["arch"].split("_")[0]
    model = build_detection_model_from_state_dict(sd, method=method, device="cpu", precision=precision,
                                                  stride_in_1x1=gold["stride_in_1x1"])
    assert model.cfg.MODEL.RESNETS.DEFORMABLE_GROUPS == gold["deformable_groups"]
    cfg = engine_config_from(model.cfg)
    cls = engine.MegaEngine if method == "mega" else engine.BaseEngine
    eng = cls(sd, cfg, device=cuda_dev)
    assert {blk.dg for s in eng.backbone.stages.stages for blk in s if blk.dcn} == {gold["deformable_groups"]}
    return eng


def _run(cuda_dev, fixture, precision):
    gold, sd, frames = _load(fixture, cuda_dev)
    eng = _engine(gold, sd, precision, cuda_dev)
    per_frame = []
    for t, det, ref in _steps(gold, eng, frames):
        torch.cuda.synchronize()
        k = int(eng.cur_cnt.view(-1)[0].item()) if hasattr(eng, "Bq0") else int(eng.last_cnt[0].item())
        props = (eng.Bq0 if hasattr(eng, "Bq0") else eng.last_props)[:k].cpu()
        idx = _match_rows(props, ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].float().cpu()
        assert torch.isfinite(pred).all()
        dabs = (pred[idx[m], :31] - ref["class_logits"][m]).abs()
        b, s, l = det.to_host()
        per_frame.append({"proposals": k, "ref_proposals": int(ref["proposals"].shape[0]),
                          "matched_frac": m.float().mean().item(), "logits_maxabs": dabs.max().item(),
                          "logits_p99": torch.quantile(dabs.flatten(), 0.99).item(),
                          "deltas_maxabs": (pred[idx[m], 31:155] - ref["box_regression"][m]).abs().max().item(),
                          "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0])})
        print(fixture, precision, per_frame[-1])
    return per_frame


@pytest.mark.parametrize("fixture", FIXTURES)
def test_fp32x3_matches_reference(cuda_dev, fixture):
    """strict mode: every proposal and detection, the logit / delta bars of tests/test_dcn_gpu.py"""
    for f in _run(cuda_dev, fixture, "fp32x3"):
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["dets"] == f["ref_dets"], f
        assert f["logits_p99"] < 1e-3, f
        assert f["logits_maxabs"] < 1e-2, f
        assert f["deltas_maxabs"] < 5e-3, f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_f16_matches_reference(cuda_dev, fixture):
    """the statistical bars of tests/test_dcn_gpu.py"""
    for f in _run(cuda_dev, fixture, "f16"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_p99"] < 3e-2, f
        assert f["logits_maxabs"] < 0.5, f


def _body(cuda_dev, n, chained, dg, stride_in_1x1=True):
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=RES234, deformable_groups=dg)
    img = torch.cat([synth.synthetic_frame(i, 192, 320) for i in range(n)]).to(cuda_dev)
    saved = ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0]
    ops.AUTOTUNE[0] = False
    try:
        if not chained:
            ops.CHAINS_ENABLED[0] = False
            ops.MAX_BN[0] = 128
        bb = engine.Backbone(sd, cuda_dev, dtype=torch.float16, stride_in_1x1=stride_in_1x1)
        ys = [bb.forward(img).clone() for _ in range(2 if chained else 1)]
    finally:
        ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0] = saved
    torch.cuda.synchronize()
    blocks = sum(len(s) for s in bb.stages.stages)
    assert len(bb._chains) == (blocks + 1 if chained else 0)        # one chain segment per sampling launch, plus one
    return ys


@pytest.mark.parametrize("stride_in_1x1, dg", [(True, 2), (False, 8)])
@pytest.mark.parametrize("n", [1, 4])
def test_body_chain_segments_equal_per_layer_launches(cuda_dev, n, stride_in_1x1, dg):
    """the f16 body with every res2..res4 conv2 deformable in dg groups: chain segments (twice) and per-layer launches
    with the same tile choices give the same bits"""
    y_chain, y_chain2 = _body(cuda_dev, n, True, dg, stride_in_1x1)
    y_layers, = _body(cuda_dev, n, False, dg, stride_in_1x1)
    assert y_chain.shape == (n, 12, 20, 1024) and torch.isfinite(y_chain.float()).all()
    assert torch.equal(y_chain, y_chain2)
    assert torch.equal(y_chain, y_layers), (y_chain.float() - y_layers.float()).abs().max().item()


@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_graph_replay_equals_eager(cuda_dev, precision):
    from mega_core.b200 import ops
    gold, sd, frames = _load(FIXTURES[1], cuda_dev)
    outs = []
    for use_graph in (False, True):
        eng = _engine(gold, sd, precision, cuda_dev)
        ops.AUTOTUNE[0] = False
        eng.use_graph = use_graph
        snaps = []
        for t, det, _ in _steps(gold, eng, frames):
            torch.cuda.synchronize()
            k = int(eng.cur_cnt.view(-1)[0].item())
            snaps.append((eng.last_pred[:k].clone().cpu(),) + det.to_host())
        outs.append(snaps)
        if use_graph:
            assert eng._graphs, "no graph was captured"
        del eng
    for t, (a, b) in enumerate(zip(*outs)):
        for x, y in zip(a, b):
            assert torch.equal(x, y), "frame %d: graph replay differs from eager" % t


def test_forward_frames_equals_one_call_per_frame(cuda_dev):
    """strict mode, module API, MEGA with 4 groups on res3 + res4"""
    from mega_core.b200 import ops, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    h, w, total = 192, 320, 24
    sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=RES34, deformable_groups=4)
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    glob0 = [frames[(3 * j + 1) % total][0] for j in range(10)]
    first = {"cur": frames[0][0], "ref_l": [], "ref_g": glob0, "frame_category": 0,
             "lookahead": [f[0] for f in frames[1:13]], "seg_len": total, "pattern": "%06d", "img_dir": "/nonexistent/%s"}
    steady = [{"cur": frames[t][0], "ref_l": [frames[t + 12][0]], "ref_g": [frames[(5 * t + 3) % total][0]],
               "frame_category": 1} for t in range(1, 5)]
    results = []
    for batched in (False, True):
        model = build_detection_model_from_state_dict(sd, method="mega", device=cuda_dev, precision="fp32x3")
        r = model.cfg.MODEL.RESNETS
        assert tuple(r.STAGE_WITH_DCN) == RES34 and r.DEFORMABLE_GROUPS == 4 and not r.WITH_MODULATED_DCN
        model(first)
        ops.AUTOTUNE[0] = False
        outs = [o[0] for o in model.forward_frames(steady)] if batched else [model(im)[0] for im in steady]
        results.append([(o.bbox.cpu(), o.get_field("scores").cpu(), o.get_field("labels").cpu()) for o in outs])
        del model
    for t, ((b0, s0, l0), (b1, s1, l1)) in enumerate(zip(*results)):
        assert b0.shape[0] > 0 and b0.shape == b1.shape, (t, b0.shape, b1.shape)
        idx = _match_rows(b1, b0, tol=1e-2)
        assert (idx >= 0).all(), "frame %d: detections differ" % t
        assert torch.equal(l1[idx], l0), t
        assert (s1[idx] - s0).abs().max().item() < 2e-3, t


@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_video_engines_share_the_grouped_backbone(cuda_dev, precision):
    """DFF, FGFA and RDN engines built from 2-group DCN state dicts: the backbone output of an image equals, bit for bit,
    that of the engine with the same body arithmetic -- the base engine for DFF / FGFA, the MEGA engine for RDN"""
    from mega_core.b200 import engine, ops, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    img = synth.synthetic_frame(2, 192, 320).to(cuda_dev)
    ops.AUTOTUNE[0] = False
    feats = {}
    body = None
    for arch, cls in (("base_r101", engine.BaseEngine), ("dff_r101", engine.DffEngine),
                      ("fgfa_r101", engine.FgfaEngine), ("mega_r101", engine.MegaEngine),
                      ("rdn_r101", engine.RdnEngine)):
        sd = synth.make_state_dict(arch, seed=4, stage_with_dcn=RES234, deformable_groups=2)
        if body is None:         # the offset convs are drawn last, after tensors that differ by method: share one body
            body = {k: v for k, v in sd.items() if k.startswith("backbone.")}
        sd.update(body)
        model = build_detection_model_from_state_dict(sd, method=arch.split("_")[0], device="cpu", precision=precision)
        assert model.cfg.MODEL.RESNETS.DEFORMABLE_GROUPS == 2
        eng = cls(sd, engine_config_from(model.cfg), device=cuda_dev)
        assert {blk.dg for s in eng.backbone.stages.stages for blk in s if blk.dcn} == {2}
        with ops.precision(precision):
            y = eng.backbone.forward(img)
            feats[arch] = (ops.unpack_split16(y, torch.empty_like(y)) if ops.is_split16(y) else y).float().cpu()
        del eng
    for arch, ref in (("dff_r101", "base_r101"), ("fgfa_r101", "base_r101"), ("rdn_r101", "mega_r101")):
        assert torch.equal(feats[arch], feats[ref]), arch
    if precision == "f16":
        assert torch.equal(feats["mega_r101"], feats["base_r101"])


def test_wave_selfcheck_on_grouped_dcn_mega_engine(cuda_dev):
    from mega_core.b200 import engine, parallel, synth
    sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=RES34, deformable_groups=2)
    cfg = engine.EngineConfig(precision="f16")
    ok, msg = parallel.wave_selfcheck(lambda: engine.MegaEngine(sd, cfg, device=cuda_dev), 320, 192, world=2, groups=2)
    assert ok, msg
