"""GPU tests of deformable backbone stages (MODEL.RESNETS.STAGE_WITH_DCN, DCN v1 and modulated v2):
  * the deformable conv2 layer as the engines launch it (offset conv, sampling, contraction with FrozenBN and ReLU) in
    tf32, split-fp16 (fp32x3) and f16, v1 / v2, stride 1 / 2, on odd map sizes: each launch against float64 -- the two
    conv_gemm launches with the per-element bounds of the conformance suite (K = 9 C for the contraction, on the
    columns the sampling wrote), the sampling against the fp64 restatement of oracle/train_ops_oracle on the
    offsets the offset conv wrote, within the fp32 rounding of its arithmetic and the column's storage rounding;
  * the sampling kernel alone against the g++ build of the same header (tests/native/dcn_sample_host.cpp) in fp32;
  * the base and MEGA engines against the fixtures of tools/make_golden_dcn.py in f16 and fp32x3;
  * the f16 body as chain segments against per-layer launches, CUDA-graph replay against eager runs,
    model.forward_frames against one model(images) call per frame;
  * the DFF / FGFA backbones against the base engine's, RDN's against MEGA's; parallel.wave_selfcheck on a DCN MEGA engine."""
import ctypes
import os
import subprocess
import sys
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]

import train_ops_oracle as to  # noqa: E402
from conv_gemm_ref import conv_gemm_ref  # noqa: E402
from test_conv_gemm_conformance_gpu import _bound_check  # noqa: E402
from test_stride3x3_gpu import _match_rows  # noqa: E402

MODES = {"tf32": (0, 0), "split16": (1, 3), "f16": (0, 2)}     # -> (ops.precision, conformance mode of the bound)
RES34 = (False, True, True, False)


def _block_sd(c, modulated, seed):
    """one bottleneck, c channels throughout, whose conv2 is a DFConv2d with offsets of about 1.5 pixels"""
    from mega_core.b200 import synth
    g = torch.Generator().manual_seed(seed)
    sd = {}
    p = "layer2.0."
    sd[p + "conv1.weight"] = synth._kaiming((c, c, 1, 1), g)
    sd[p + "conv2.conv.weight"] = synth._kaiming((c, c, 3, 3), g)
    sd[p + "conv2.offset.weight"] = synth._kaiming((27 if modulated else 18, c, 3, 3), g, gain=2.0)
    sd[p + "conv2.offset.bias"] = torch.randn(27 if modulated else 18, generator=g) * 0.5
    sd[p + "conv3.weight"] = synth._kaiming((c, c, 1, 1), g)
    for bn in ("bn1.", "bn2.", "bn3."):
        synth._bn(sd, p + bn, c, g)
    return sd


def _identity_weight(c, dev):
    """deform_conv2d with this weight returns the sampled columns: output channel c * 9 + tap = tap of channel c"""
    w = torch.zeros(9 * c, c, 3, 3, dtype=torch.float64, device=dev)
    idx = torch.arange(9 * c, device=dev)
    w.view(9 * c, c, 9)[idx, idx // 9, idx % 9] = 1.0
    return w


def _cols64(x64, offset, mask, stride, dev):
    """[N,C,H,W] fp64 -> columns [N,Ho,Wo,9C] tap-major (fp64 restatement of the sampling, run on the host)"""
    c = x64.shape[1]
    cpu = torch.device("cpu")
    out = to.deform_conv2d(x64.to(cpu), offset.to(cpu), None if mask is None else mask.to(cpu),
                           _identity_weight(c, cpu), None, (stride, stride), (1, 1), (1, 1), 1, 1)
    n, _, ho, wo = out.shape
    return out.view(n, c, 9, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, 9 * c).to(dev)


def _decode(t, fmt):
    from mega_core.b200 import ops
    return (ops.split16_decode(t) if fmt == "split" else t).double()


@pytest.mark.parametrize("hw", [(75, 125), (38, 63)])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_deformable_conv2_layer_matches_fp64(cuda_dev, mode, modulated, stride, hw):
    from mega_core.b200 import engine, ops
    prec, cmode = MODES[mode]
    c, n = 64, 1
    sd = _block_sd(c, modulated, seed=7 * stride + hw[0])
    dtype = torch.float16 if mode == "f16" else torch.float32
    st = engine.ResNetStages(sd, "", (2,), cuda_dev, first_stride_of=lambda li: stride, dtype=dtype,
                             stride_in_1x1=False)
    blk = st.stages[0][0]
    assert blk.dcn and blk.modulated == modulated
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
    off = st._bufs[("dcn_off", (n, ho, wo, engine.DCN_OFFSET_ROWS), 0)]
    cols = st._bufs[("dcn_cols", (n, ho, wo, 9 * c), 0)]
    what = "%s %s stride %d %s" % (mode, "v2" if modulated else "v1", stride, hw)
    # 1. offset conv: 3x3, bias, fp32 output
    acc = ops._split16_weight(blk.wo) if mode == "split16" else 1.0
    _, ref, P, Q = conv_gemm_ref(a64, _decode(blk.wo, fmt), taps=(3, 3), pad=1, stride=(stride, stride), k=c, n_img=n,
                                 out_hw=(ho, wo), cout=engine.DCN_OFFSET_ROWS, bias=blk.bo, acc_scale=acc)[0]
    _bound_check(cmode, off.double(), ref, P, Q, "f32", "offset conv " + what)
    # 2. sampling of t1's stored values at the stored offsets
    o64 = off.double().permute(0, 3, 1, 2)
    offset, mask = o64[:, :18].contiguous(), (o64[:, 18:27].sigmoid().contiguous() if modulated else None)
    xin = a64.permute(0, 3, 1, 2).contiguous()
    ref = _cols64(xin, offset, mask, stride, cuda_dev)
    S = _cols64(xin.abs(), offset, mask, stride, cuda_dev)          # sum of |w v| over the four corners (x mask)
    got = _decode(cols, fmt)
    # fp32 geometry (position rounding moves a sample by up to 2^-24 (|h| + |w| + 2)), four rounded products / sums
    # and the sigmoid, then the column's storage rounding
    pos = 2.0 ** -23 * (h + w + 4) * xin.abs().amax().item()
    bound = 2.0 ** -20 * S + pos + {"f16": 2.0 ** -11 * ref.abs() + 2.0 ** -24,
                                    "split": 2.0 ** -22 * ref.abs() + 2.0 ** -25, "f32": 1e-30}[fmt]
    err = (got - ref).abs()
    assert bool((err <= bound).all()), "sampling %s: max err %.3e, worst err / bound %.3f" % (
        what, err.max().item(), (err / bound).max().item())
    assert (ref == 0).float().mean().item() < 0.2 and (ref != 0).any()
    # 3. contraction over the columns (K = 9 C) with FrozenBN and ReLU
    acc = ops._split16_weight(blk.w2) if mode == "split16" else 1.0
    scale = None if mode == "split16" else blk.s2
    _, ref, P, Q = conv_gemm_ref(got, _decode(blk.w2, fmt), k=9 * c, n_img=n, out_hw=(ho, wo), cout=c, bias=blk.b2,
                                 scale=scale, relu=1, acc_scale=acc)[0]
    _bound_check(cmode, _decode(t2, fmt), ref, P, Q, fmt, "contraction " + what)


_HOST = {}


def _host_lib():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp()
        so = os.path.join(d, "libdcn_sample_host.so")
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-I",
                               os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                               "-o", so, os.path.join(ROOT, "tests", "native", "dcn_sample_host.cpp")])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("modulated", [False, True])
def test_sampling_kernel_equals_host_build(cuda_dev, modulated, stride):
    """fp32: bit for bit against the g++ build of dcn_sample.cuh. v2: the device's expf is within 2 ulp and the host
    library's within 1, and the sigmoid's add, reciprocal and the product with the sample round once more each, so the
    masked values are held to 8 ulp"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(5)
    n, h, w, c = 2, 37, 61, 64
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = torch.randn(n, h, w, c, generator=g)
    off = torch.randn(n, ho, wo, 32, generator=g) * 2.0
    off[..., :18] += torch.randint(-1, 2, (n, ho, wo, 18), generator=g).float()       # some integer positions
    cols = ops.dcn_sample(x.to(cuda_dev), off.to(cuda_dev), torch.zeros(n, ho, wo, 9 * c, device=cuda_dev), modulated,
                          stride).cpu()
    host = torch.zeros_like(cols)
    vp = ctypes.c_void_p
    fn = _host_lib().mega_dcn_sample_nhwc
    assert fn(vp(x.data_ptr()), 0, n, h, w, c, vp(off.data_ptr()), 32, int(modulated), stride, 1,
              vp(host.data_ptr()), None) == 0
    if not modulated:
        assert torch.equal(cols.view(torch.int32), host.view(torch.int32))
    else:
        ulp = (cols.view(torch.int32).long() - host.view(torch.int32).long()).abs()
        assert ulp.max().item() <= 8, ulp.max().item()


# ------------------------------------------------------------------------------------------------ engines vs fixtures
FIXTURES = ("base_r101_dcn_192x320.pt", "mega_r101_mdcn_192x320.pt", "base_r101_s3x3_mdcn_192x320.pt")


def _load(fixture, cuda_dev):
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(ROOT, "tests", "golden", fixture))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"], stage_with_dcn=gold["stage_with_dcn"],
                               modulated_dcn=gold["modulated"])
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
    assert tuple(model.cfg.MODEL.RESNETS.STAGE_WITH_DCN) == tuple(gold["stage_with_dcn"])
    cfg = engine_config_from(model.cfg)
    cls = engine.MegaEngine if method == "mega" else engine.BaseEngine
    eng = cls(sd, cfg, device=cuda_dev)
    assert eng.backbone.stages.has_dcn
    return eng


def _steps(gold, eng, frames):
    h, w = gold["h"], gold["w"]
    if "frames" not in gold:
        yield 0, eng.forward(frames[gold["frame_index"]], w, h), gold
        return
    total, gpf = gold["total"], gold["globals_per_frame"]
    for t, ref in enumerate(gold["frames"]):
        det = (eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h) if t == 0 else
               eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h))
        yield t, det, ref


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
    """strict mode: every proposal and detection, the logit / delta bars of tests/test_stride3x3_gpu.py"""
    for f in _run(cuda_dev, fixture, "fp32x3"):
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["dets"] == f["ref_dets"], f
        assert f["logits_p99"] < 1e-3, f
        assert f["logits_maxabs"] < 1e-2, f
        assert f["deltas_maxabs"] < 5e-3, f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_f16_matches_reference(cuda_dev, fixture):
    """the MEGA R-101 statistical bars of tests/test_engine_gpu.py"""
    for f in _run(cuda_dev, fixture, "f16"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_p99"] < 3e-2, f
        assert f["logits_maxabs"] < 0.5, f


def _body(cuda_dev, n, chained, stride_in_1x1=True):
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=(True, True, True, False), modulated_dcn=True)
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


@pytest.mark.parametrize("stride_in_1x1", [True, False])
@pytest.mark.parametrize("n", [1, 4])
def test_body_chain_segments_equal_per_layer_launches(cuda_dev, n, stride_in_1x1):
    """the f16 body with every res2..res4 conv2 deformable: chain segments (twice) and per-layer launches with the same
    tile choices give the same bits"""
    y_chain, y_chain2 = _body(cuda_dev, n, True, stride_in_1x1)
    y_layers, = _body(cuda_dev, n, False, stride_in_1x1)
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
    """strict mode, module API, MEGA with modulated res3 + res4"""
    from mega_core.b200 import ops, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    h, w, total = 192, 320, 24
    sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=RES34, modulated_dcn=True)
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    glob0 = [frames[(3 * j + 1) % total][0] for j in range(10)]
    first = {"cur": frames[0][0], "ref_l": [], "ref_g": glob0, "frame_category": 0,
             "lookahead": [f[0] for f in frames[1:13]], "seg_len": total, "pattern": "%06d", "img_dir": "/nonexistent/%s"}
    steady = [{"cur": frames[t][0], "ref_l": [frames[t + 12][0]], "ref_g": [frames[(5 * t + 3) % total][0]],
               "frame_category": 1} for t in range(1, 5)]
    results = []
    for batched in (False, True):
        model = build_detection_model_from_state_dict(sd, method="mega", device=cuda_dev, precision="fp32x3")
        assert tuple(model.cfg.MODEL.RESNETS.STAGE_WITH_DCN) == RES34 and model.cfg.MODEL.RESNETS.WITH_MODULATED_DCN
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
def test_video_engines_share_the_dcn_backbone(cuda_dev, precision):
    """DFF, FGFA and RDN engines built from DCN state dicts: the backbone output of an image equals, bit for bit, that
    of the engine with the same body arithmetic -- the base engine for DFF / FGFA, the MEGA engine for RDN (in fp32x3 the
    windowed engines run their body on split-fp16, the single-frame ones on 3xTF32; in f16 all five agree)"""
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
        sd = synth.make_state_dict(arch, seed=4, stage_with_dcn=RES34, modulated_dcn=True)
        if body is None:         # the offset convs are drawn last, after tensors that differ by method: share one body
            body = {k: v for k, v in sd.items() if k.startswith("backbone.")}
        sd.update(body)
        cfg = engine_config_from(build_detection_model_from_state_dict(sd, method=arch.split("_")[0], device="cpu",
                                                                       precision=precision).cfg)
        eng = cls(sd, cfg, device=cuda_dev)
        assert eng.backbone.stages.has_dcn
        with ops.precision(precision):
            y = eng.backbone.forward(img)
            feats[arch] = (ops.unpack_split16(y, torch.empty_like(y)) if ops.is_split16(y) else y).float().cpu()
        del eng
    for arch, ref in (("dff_r101", "base_r101"), ("fgfa_r101", "base_r101"), ("rdn_r101", "mega_r101")):
        assert torch.equal(feats[arch], feats[ref]), arch
    if precision == "f16":
        assert torch.equal(feats["mega_r101"], feats["base_r101"])


def test_wave_selfcheck_on_dcn_mega_engine(cuda_dev):
    from mega_core.b200 import engine, parallel, synth
    sd = synth.make_state_dict("mega_r101", seed=0, stage_with_dcn=RES34, modulated_dcn=True)
    cfg = engine.EngineConfig(precision="f16")
    ok, msg = parallel.wave_selfcheck(lambda: engine.MegaEngine(sd, cfg, device=cuda_dev), 320, 192, world=2, groups=2)
    assert ok, msg
