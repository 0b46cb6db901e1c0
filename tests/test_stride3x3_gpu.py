"""GPU tests of 3x3-strided bottlenecks (MODEL.RESNETS.STRIDE_IN_1X1 False): the stride-2 3x3 conv_gemm, dense and grouped,
against the fp64 reference of tests/conv_gemm_ref.py with the per-element bounds of the conformance suite in every operand
arithmetic; the f16 body as one layer chain against per-layer launches; the single-frame and MEGA engines against the
fixtures written from the unmodified reference (tools/make_golden_stride3x3.py); CUDA-graph replay against eager runs;
model.forward_frames against one model(images) call per frame."""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests"))

from conv_gemm_ref import conv_gemm_ref  # noqa: E402
from test_conv_gemm_conformance_gpu import _bound_check  # noqa: E402

# operand arithmetic -> (ops.precision, conformance mode of the bound): plain TF32, the 3xTF32 split of fp32 tensors,
# fp16 operands with fp16 output (the f16 body), and 3xFP16 on split-fp16 operands and output (the strict body)
MODES = {"tf32": (0, 0), "fp32x3": (1, 1), "f16": (0, 2), "split16": (1, 3)}
GROUP_WIDTHS = (0, 8, 16, 32, 64)         # 0: dense


def _strided_conv(dev, mode, gw, n, stream_k, c=128, hw=(75, 125)):
    """3x3 / stride 2 / pad 1 conv with FrozenBN scale / bias and ReLU over an odd-sized map (75x125 -> 38x63), dense or
    grouped with group width gw, as the engines launch a 3x3-strided conv2 -> (result, fp64 reference, P, Q, format)"""
    from mega_core.b200 import ops
    prec, cmode = MODES[mode]
    g = torch.Generator(device=dev).manual_seed(1000 * gw + 10 * n + stream_k)
    h, w = hw
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    x = torch.randn(n, h, w, c, device=dev, generator=g).relu()
    wl = torch.randn(c, gw or c, 3, 3, device=dev, generator=g) / (9 * (gw or c)) ** 0.5
    scale = torch.rand(c, device=dev, generator=g) + 0.5
    bias = torch.randn(c, device=dev, generator=g) * 0.1
    wp = ops.pack_grouped_conv(wl, c // gw, dev) if gw else wl.permute(2, 3, 0, 1).reshape(9, c, c).contiguous()
    kw = dict(taps=(3, 3), pad=1, stride=(2, 2), bias=bias, relu=True, stream_k=stream_k)
    if gw:
        kw["groups"] = c // gw
    else:
        kw["block_n"] = 128 if mode in ("f16", "tf32") else 64
    acc_scale, fmt = 1.0, "f32"
    if mode == "f16":
        a, b = x.half(), wp.half()
        if gw:
            b = ops.pack_grouped_conv(wl, c // gw, dev, torch.float16)
        out = torch.full((n, oh, ow, c), float("nan"), device=dev, dtype=torch.float16)
        kw["scale"], fmt = scale, "f16"
        A64, B64, S = a.double(), b.double(), scale
    elif mode == "split16":
        a = ops.pack_split16(x.contiguous())
        b = ops.pack_weights_split16(wp, scale=scale)
        out = ops.mark_split16(torch.zeros(n, oh, ow, c, device=dev))
        acc_scale, fmt = ops._split16_weight(b), "split"
        A64, B64, S = ops.split16_decode(a).double(), ops.split16_decode(b).double(), None
    else:
        a, b = x, wp
        out = torch.full((n, oh, ow, c), float("nan"), device=dev)
        kw["scale"] = scale
        A64, B64, S = a.double(), b.double(), scale
    with ops.precision(prec):
        ops.conv_gemm(a, b, out, **kw)
    torch.cuda.synchronize()
    got = (ops.split16_decode(out) if mode == "split16" else out).double()
    geo = dict(taps=(3, 3), pad=1, stride=(2, 2), n_img=n, out_hw=(oh, ow), bias=bias, scale=S, relu=1,
               acc_scale=acc_scale)
    if gw:
        z = 64
        blocks = conv_gemm_ref(A64, B64, k=z, cout=z, batch=c // z, a_c_off=z, b_n_off=z, out_c_off=z, bias_z_off=z, **geo)
        ref, P, Q = (torch.cat([blk[i] for blk in blocks], 3) for i in (1, 2, 3))
    else:
        _, ref, P, Q = conv_gemm_ref(A64, B64, k=c, cout=c, **geo)[0]
    return got, ref, P, Q, fmt, cmode


@pytest.mark.parametrize("n", [1, 2, 4])
@pytest.mark.parametrize("gw", GROUP_WIDTHS)
@pytest.mark.parametrize("mode", sorted(MODES))
def test_strided_3x3_matches_fp64(cuda_dev, mode, gw, n):
    """every element within the conformance suite's bound, stream-K on and off"""
    for stream_k in (0, 1):
        got, ref, P, Q, fmt, cmode = _strided_conv(cuda_dev, mode, gw, n, stream_k)
        assert not bool(torch.isnan(got).any()), "unwritten outputs"
        _bound_check(cmode, got, ref, P, Q, fmt, "%s gw %d n %d stream_k %d" % (mode, gw, n, stream_k))


def _body_outputs(cuda_dev, arch, n, chained):
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict(arch, seed=0)
    img = torch.cat([synth.synthetic_frame(i, 192, 320) for i in range(n)]).to(cuda_dev)
    saved = ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0]
    ops.AUTOTUNE[0] = False
    try:
        if not chained:
            ops.CHAINS_ENABLED[0] = False
            ops.MAX_BN[0] = 128                             # the widest tile a chain layer may pick
        bb = engine.Backbone(sd, cuda_dev, dtype=torch.float16, stride_in_1x1=False)
        ys = [bb.forward(img).clone() for _ in range(2 if chained else 1)]
    finally:
        ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0] = saved
    torch.cuda.synchronize()
    assert len(bb._chains) == (1 if chained else 0)
    if chained:
        depths = {ch.depth for ch in bb._chains.values()}
        assert depths == {2 if n >= ops.DUAL_MIN_IMAGES else 1}, depths
    return ys


@pytest.mark.parametrize("n", [2, 4])
@pytest.mark.parametrize("arch", ["mega_r101", "mega_x101"])
def test_body_chain_equals_per_layer_launches(cuda_dev, arch, n):
    """the 3x3-strided f16 body (dense R-101 / grouped X-101) as one persistent chain (n = 2: depth 1; n = 4: two
    interleaved lanes, depth 2), twice, and as per-layer launches with the same tile choices: bit-identical"""
    y_chain, y_chain2 = _body_outputs(cuda_dev, arch, n, True)
    y_layers, = _body_outputs(cuda_dev, arch, n, False)
    assert y_chain.shape == (n, 12, 20, 1024)
    assert torch.isfinite(y_chain.float()).all()
    assert torch.equal(y_chain, y_chain2)
    assert torch.equal(y_chain, y_layers), (y_chain.float() - y_layers.float()).abs().max().item()


# ------------------------------------------------------------------------------------------------ engines vs fixtures
FIXTURES = ("base_r101_s3x3_192x320.pt", "mega_r101_s3x3_192x320.pt", "mega_x101_s3x3_192x320.pt")


def _match_rows(a, b, tol=0.75):
    """for each row of b (reference boxes) the index of an identical-within-tol row of a, or -1"""
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _load(fixture, cuda_dev):
    from mega_core.b200 import synth
    gold = torch.load(os.path.join(GOLD, fixture))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    n = gold.get("total", gold.get("frame_index", 0) + 1)
    frames = [synth.synthetic_frame(i, gold["h"], gold["w"]).to(cuda_dev) for i in range(n)]
    return gold, sd, frames


def _engine(gold, sd, precision, cuda_dev):
    """the engine of the model build_detection_model_from_state_dict(stride_in_1x1=False) makes"""
    from mega_core.b200 import engine
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    from mega_core.modeling.nets import engine_config_from
    method = gold["arch"].split("_")[0]
    cfg = engine_config_from(build_detection_model_from_state_dict(sd, method=method, device="cpu", precision=precision,
                                                                   stride_in_1x1=False).cfg)
    assert cfg.stride_in_1x1 is False
    cls = engine.MegaEngine if method == "mega" else engine.BaseEngine
    return cls(sd, cfg, device=cuda_dev)


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
        print(fixture, precision, json.dumps(per_frame[-1]))
    return per_frame


@pytest.mark.parametrize("fixture", FIXTURES)
def test_exact_fp32_contractions_match_reference(cuda_dev, fixture):
    """the engines' orchestration of the 3x3-strided layout with exact-fp32 contractions (tests/fp32_shadow.py): every
    proposal and detection, the bars of the X-101 fixture's exact-fp32 run"""
    from fp32_shadow import fp32_shadow
    with fp32_shadow():
        frames = _run(cuda_dev, fixture, "tf32")
    for f in frames:
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["dets"] == f["ref_dets"], f
        assert f["logits_p99"] < 1e-4, f
        assert f["logits_maxabs"] < 1e-2, f
        assert f["deltas_maxabs"] < 5e-3, f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_fp32x3_matches_reference(cuda_dev, fixture):
    """strict mode: every proposal and detection; the logit / delta bars of the MEGA R-101 and X-101 fixtures"""
    mx, dmx = (3e-2, 1e-2) if "x101" in fixture else (1e-2, 5e-3)
    for f in _run(cuda_dev, fixture, "fp32x3"):
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["dets"] == f["ref_dets"], f
        assert f["logits_p99"] < 1e-3, f
        assert f["logits_maxabs"] < mx, f
        assert f["deltas_maxabs"] < dmx, f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_tf32_matches_reference(cuda_dev, fixture):
    """the R-101 statistical bars of tests/test_engine_gpu.py"""
    for f in _run(cuda_dev, fixture, "tf32"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_maxabs"] < 0.15, f


@pytest.mark.parametrize("fixture", FIXTURES)
def test_f16_matches_reference(cuda_dev, fixture):
    """the MEGA R-101 statistical bars of tests/test_engine_gpu.py"""
    for f in _run(cuda_dev, fixture, "f16"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_p99"] < 3e-2, f
        assert f["logits_maxabs"] < 0.5, f


@pytest.mark.parametrize("fixture", FIXTURES[1:])
@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_graph_replay_equals_eager(cuda_dev, fixture, precision):
    """the steady frames as captured CUDA graphs and as eager launches: identical detections and predictor rows"""
    from mega_core.b200 import ops
    gold, sd, frames = _load(fixture, cuda_dev)
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


@pytest.mark.parametrize("arch", ["mega_r101", "mega_x101"])
def test_forward_frames_equals_one_call_per_frame(cuda_dev, arch):
    """strict mode, module API: model.forward_frames over 4 steady frames (one batch of 8 images through the per-frame
    branch) against model(images) per frame: the same detections, up to the stream-K split points of the larger launches
    (scores within 2e-3)"""
    from mega_core.b200 import ops, synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    h, w, total = 192, 320, 24
    sd = synth.make_state_dict(arch, seed=0)
    frames = [synth.synthetic_frame(i, h, w) for i in range(total)]
    glob0 = [frames[(3 * j + 1) % total][0] for j in range(10)]
    first = {"cur": frames[0][0], "ref_l": [], "ref_g": glob0, "frame_category": 0,
             "lookahead": [f[0] for f in frames[1:13]], "seg_len": total, "pattern": "%06d", "img_dir": "/nonexistent/%s"}
    steady = [{"cur": frames[t][0], "ref_l": [frames[t + 12][0]], "ref_g": [frames[(5 * t + 3) % total][0]],
               "frame_category": 1} for t in range(1, 5)]
    results = []
    for batched in (False, True):
        model = build_detection_model_from_state_dict(sd, method="mega", device=cuda_dev, precision="fp32x3",
                                                      stride_in_1x1=False)
        assert model.cfg.MODEL.RESNETS.STRIDE_IN_1X1 is False
        model(first)
        ops.AUTOTUNE[0] = False
        if batched:
            outs = [o[0] for o in model.forward_frames(steady)]
        else:
            outs = [model(im)[0] for im in steady]
        results.append([(o.bbox.cpu(), o.get_field("scores").cpu(), o.get_field("labels").cpu()) for o in outs])
        del model
    for t, ((b0, s0, l0), (b1, s1, l1)) in enumerate(zip(*results)):
        assert b0.shape[0] > 0 and b0.shape == b1.shape, (t, b0.shape, b1.shape)
        idx = _match_rows(b1, b0, tol=1e-2)
        assert (idx >= 0).all(), "frame %d: detections differ" % t
        assert torch.equal(l1[idx], l0), t
        assert (s1[idx] - s0).abs().max().item() < 2e-3, t
