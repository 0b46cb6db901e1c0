"""GPU parity of the training-side half of `mega_core._C` through the C ABI: roi_align_backward, roi_pool_forward /
backward, deform_conv_backward_input / _parameters, modulated_deform_conv_backward, deform_psroi_pooling_backward
(SURVEY.md section 8b; 8f row 3). Oracles: oracle/train_ops_oracle.py (autograd of forward restatements anchored in
tests/test_train_ops_cpu.py). Scatter kernels accumulate with red.global.add.f32 in an unspecified order, as the
reference's atomicAdd does, so float results are compared to 1e-5-level tolerances; arg-max indices are exact.
Order inside the file (the GPU tier runs with -x): most certain first -- integer-exact image transform, the simple
scatter kernels, the engine-level wavefront / DFF checks (all-existing kernels in a new order), then the ops that also
drive the wgmma GEMM with shapes it has not seen (deformable-conv backward, the layer wrappers).
(This file sorts last on purpose: these kernels were added after the last full GPU session of round 1 and verified on
the CPU first, through their host builds; a surprise here must not hide the hot-path tests. First B200 run: 20 of 21
passed unchanged, see profiles/r01_summary.md.)"""
import os
import sys

import pytest
import torch

# first GPU run of these kernels happens without supervision: a generous per-test timeout that ends the PROCESS (thread
# method: a signal cannot interrupt a blocked CUDA call) keeps a surprise from stalling the whole GPU tier
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def _rois(g, k, n_img, w_img, h_img):
    x1 = torch.rand(k, generator=g) * w_img * 0.7 - 10
    y1 = torch.rand(k, generator=g) * h_img * 0.7 - 10
    bw = torch.rand(k, generator=g) * w_img * 0.6 + 1
    bh = torch.rand(k, generator=g) * h_img * 0.6 + 1
    b = torch.randint(0, n_img, (k,), generator=g).float()
    return torch.stack([b, x1, y1, x1 + bw, y1 + bh], 1)


def _rel_err(a, b):
    return ((a - b).abs().max() / b.pow(2).mean().sqrt().clamp_min(1e-12)).item()


@pytest.mark.parametrize("h,w", [(720, 1280), (480, 640), (600, 1000), (375, 500)])
def test_device_image_transform_matches_reference_pipeline(cuda_dev, h, w):
    """mega_image_transform_u8 vs the reference's CPU pipeline (PIL resize -> to_tensor -> BGR255 -> normalize), bit for
    bit, at ImageNet-VID frame sizes and MIN_SIZE_TEST / MAX_SIZE_TEST = 600 / 1000 (SURVEY.md section 8f row 1)"""
    import numpy as np
    import image_oracle as io
    from mega_core.data.transforms import DeviceTestTransform
    mean, std = [102.9801, 115.9465, 122.7717], [1.0, 1.0, 1.0]
    g = np.random.default_rng(h + w)
    base = g.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3), dtype=np.uint8)
    img = np.kron(base, np.ones((16, 16, 1), dtype=np.uint8))[:h, :w]
    img = np.clip(img.astype(np.int16) + g.integers(-20, 20, (h, w, 3), dtype=np.int16), 0, 255).astype(np.uint8)
    ref = io.reference_pipeline(img, 600, 1000, mean, std, True)
    tr = DeviceTestTransform(600, 1000, mean, std, True, device=cuda_dev)
    out, _ = tr(img)
    assert out.is_cuda and out.shape == ref.shape
    assert torch.equal(out.cpu(), ref)
    out2, _ = tr(torch.from_numpy(img).pin_memory())              # pinned host frame, tables cached from the first call
    assert torch.equal(out2.cpu(), ref)
    out3, _ = tr(torch.from_numpy(img).permute(2, 0, 1).contiguous().to(cuda_dev))      # planar [3, H, W] (nvJPEG layout)
    assert torch.equal(out3.cpu(), ref)



@pytest.mark.parametrize("sr,c", [(0, 5), (2, 19), (0, 16)])
def test_roi_align_backward(cuda_dev, sr, c):
    import train_ops_oracle as to
    from mega_core import _C
    g = torch.Generator().manual_seed(31 + c)
    n, h, w, k = 2, 12, 17, 6
    rois = _rois(g, k, n, w * 16, h * 16)
    rois[5] = torch.tensor([1.0, 250.0, 170.0, 252.0, 500.0])
    grad = torch.randn(k, c, 7, 7, generator=g)
    ref = to.roi_align_backward(grad, rois, 1 / 16.0, 7, 7, n, c, h, w, sr)
    got = _C.roi_align_backward(grad.to(cuda_dev), rois.to(cuda_dev), 1 / 16.0, 7, 7, n, c, h, w, sr).cpu()
    assert got.shape == (n, c, h, w)
    assert torch.allclose(got, ref, atol=2e-5, rtol=1e-5)
    empty = _C.roi_align_backward(torch.zeros(0, c, 7, 7, device=cuda_dev), torch.zeros(0, 5, device=cuda_dev),
                                  1 / 16.0, 7, 7, n, c, h, w, sr)
    assert empty.shape == (n, c, h, w) and empty.abs().sum().item() == 0


def test_roi_pool_forward_backward(cuda_dev):
    import train_ops_oracle as to
    from mega_core import _C
    g = torch.Generator().manual_seed(41)
    n, c, h, w, k = 2, 6, 13, 19, 7
    feat = torch.randn(n, c, h, w, generator=g)
    rois = _rois(g, k, n, w * 16, h * 16)
    rois[6] = torch.tensor([0.0, 400.0, 300.0, 420.0, 310.0])
    ref, ref_arg = to.roi_pool(feat, rois, 1 / 16.0, 7, 7)
    out, arg = _C.roi_pool_forward(feat.to(cuda_dev), rois.to(cuda_dev), 1 / 16.0, 7, 7)
    assert arg.dtype == torch.int32
    assert torch.equal(out.cpu(), ref) and torch.equal(arg.cpu(), ref_arg)
    grad = torch.randn(k, c, 7, 7, generator=g)
    gin = _C.roi_pool_backward(grad.to(cuda_dev), feat.to(cuda_dev), rois.to(cuda_dev), arg, 1 / 16.0, 7, 7, n, c, h, w)
    assert torch.allclose(gin.cpu(), to.roi_pool_backward(grad, feat, rois, 1 / 16.0, 7, 7), atol=1e-6)


@pytest.mark.parametrize("no_trans", [True, False])
def test_deform_psroi_pooling_backward(cuda_dev, no_trans):
    import train_ops_oracle as to
    from mega_core import _C
    g = torch.Generator().manual_seed(3)
    gs, ps, od, ncls = 3, 3, 4, 2
    data = torch.randn(2, od * gs * gs, 11, 13, generator=g)
    rois = torch.tensor([[0, 8.0, 10.0, 120.0, 90.0], [1, 40.2, 33.7, 150.9, 160.1], [0, -10.0, -5.0, 30.0, 20.0],
                         [1, 300.0, 300.0, 320.0, 330.0]])
    k = rois.shape[0]
    trans = torch.randn(k, 2 * ncls, ps, ps, generator=g) * 0.5
    og = torch.randn(k, od, ps, ps, generator=g)
    ref_in, ref_tr = to.deform_psroi_pool_grads(data, rois, trans, og, no_trans, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
    d = cuda_dev
    out = torch.zeros(k, od, ps, ps, device=d)
    cnt = torch.zeros(k, od, ps, ps, device=d)
    _C.deform_psroi_pooling_forward(data.to(d), rois.to(d), trans.to(d), out, cnt, no_trans, 1 / 16.0, od, gs, ps, ps, 4,
                                    0.1)
    gin = torch.zeros(data.shape, device=d)
    gtr = torch.zeros(trans.shape, device=d)
    _C.deform_psroi_pooling_backward(og.to(d), data.to(d), rois.to(d), trans.to(d), cnt, gin, gtr, no_trans, 1 / 16.0, od,
                                     gs, ps, ps, 4, 0.1)
    assert torch.allclose(gin.cpu(), ref_in, atol=2e-5, rtol=1e-4)
    if no_trans:
        assert gtr.abs().sum().item() == 0
    else:
        assert torch.allclose(gtr.cpu(), ref_tr, atol=2e-4, rtol=1e-3)


@pytest.mark.parametrize("precision", ["f16", "fp32x3"])
def test_mega_wavefront_step_equals_replicated_state_step(cuda_dev, precision):
    """MegaEngine._wave (SURVEY.md section 8e option ii; schedule verified symbolically in
    tests/test_wave_schedule_cpu.py): both ranks of a 2-GPU group played on one device with parallel.play() must give
    the detections and predictor outputs of the sequential owner-mode step BIT for bit, and leave the same memory."""
    from mega_core.b200 import engine, parallel, synth
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "mega_r101_192x320.pt"))
    h, w = gold["h"], gold["w"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(24)]
    glob0 = [frames[(3 * j + 1) % 24] for j in range(10)]
    pair = lambda t: torch.cat([frames[(t + 12) % 24], frames[(5 * t + 3) % 24]], 0)
    steps = 6

    def make():
        e = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev)
        e.start_video(frames[0], frames[1:13], glob0, w, h)
        return e

    def snap(e, det):
        torch.cuda.synchronize()
        b, s, l = det.to_host()
        k = int(e.cur_cnt.view(-1)[0].item())
        return e.last_pred[:k].clone().cpu(), b, s, l

    # what bench.py runs on every rank before a multi-GPU run adopts the wavefront schedule (seeded rows in the engine's
    # own row format: split-fp16 in the strict mode)
    ok, msg = parallel.wave_selfcheck(lambda: engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev),
                                      w, h, world=2, groups=2, use_graph=False)
    assert ok, msg
    ranker = make()
    payloads = [ranker.ref_payload(pair(t), w, h) for t in range(1, steps + 1)]
    solo = make()
    out_solo = [snap(solo, solo.dist_step(None, w, h, rank=0, world=1, payloads=payloads[t][None])[0])
                for t in range(steps)]
    ranks = [make(), make()]
    out_wave = [None] * steps
    for t in range(0, steps, 2):
        gens = [ranks[r]._wave(None, w, h, r, 2, payload=payloads[t + r]) for r in range(2)]
        dets = parallel.play(gens)
        for r in range(2):
            out_wave[t + r] = snap(ranks[r], dets[r])
    for t in range(steps):
        for a, b in zip(out_solo[t], out_wave[t]):
            assert torch.equal(a, b), "frame %d differs between the sequential and the wavefront schedule" % t
    torch.cuda.synchronize()
    for name in ("E0", "B0", "Y1E", "Y2M", "B1", "B2", "win_x", "glob_x"):
        ring = {"E0": solo.KP + solo.nl0, "B0": solo.KP + solo.nl0, "Y1E": solo.nq, "Y2M": solo.nq, "B1": solo.nl12,
                "B2": solo.nl12}.get(name, 0)
        for r in range(2):
            assert torch.equal(getattr(ranks[r], name)[ring:], getattr(solo, name)[ring:]), (name, r)


@pytest.mark.parametrize("precision", ["shadow", "fp32x3", "f16"])
def test_dff_r101_matches_reference_fixture(cuda_dev, precision):
    """DFF R-101 (SURVEY.md section 8f row 4; configs/DFF): DffEngine against the outputs of the unmodified reference's
    GeneralizedRCNNDFF (tests/golden/dff_r101_192x320.pt: key, non-key, non-key, key, non-key frames). "shadow": all
    kernels ours, dense contractions in exact fp32 (logic check: flow within 1e-4 cells, every proposal reproduced, class
    logits within 1e-3); product arithmetics with the statistical bounds of the FGFA tests."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from mega_core.b200 import engine, synth
    from test_engine_gpu import _match_rows
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "dff_r101_192x320.pt"))
    h, w = gold["h"], gold["w"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])

    def run(prec):
        eng = engine.DffEngine(sd, engine.EngineConfig(precision=prec), device=cuda_dev)
        out = []
        for t, (key, ref) in enumerate(zip(gold["key_flags"], gold["frames"])):
            img = synth.synthetic_frame(gold["frame_stride"] * t, h, w).to(cuda_dev)
            det = eng.forward(img, key, w, h)
            torch.cuda.synchronize()
            k = int(eng.last_cnt[0].item())
            idx = _match_rows(eng.last_props[:k].cpu(), ref["proposals"])
            m = idx >= 0
            pred = eng.last_pred[:k].cpu()
            assert torch.isfinite(pred).all()
            flow = eng.last_flow[..., :2].permute(0, 3, 1, 2).float().cpu()
            scale = eng.last_scale.float().permute(0, 3, 1, 2).cpu()[:, ::64]
            feats = eng.last_feats.float().permute(0, 3, 1, 2).cpu()[:, ::64]
            b, s, l = det.to_host()
            out.append({"matched_frac": m.float().mean().item(),
                        "logits_maxabs": (pred[idx[m], :31] - ref["class_logits"][m]).abs().max().item(),
                        "flow_maxabs": (flow - ref["flow"]).abs().max().item(),
                        "scale_maxabs": (scale - ref["scale_sample"]).abs().max().item(),
                        "feats_maxabs": (feats - ref["feats_sample"]).abs().max().item(), "feats_rms": ref["feats_rms"],
                        "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0])})
        return out

    if precision == "shadow":
        from fp32_shadow import fp32_shadow
        with fp32_shadow():
            frames = run("tf32")
        for f in frames:
            assert f["flow_maxabs"] < 1e-4 and f["scale_maxabs"] < 1e-4, f
            assert f["feats_maxabs"] < 1e-3 * max(f["feats_rms"], 1.0), f
            assert f["matched_frac"] == 1.0 and f["logits_maxabs"] < 1e-3 and f["dets"] == f["ref_dets"], f
    else:
        for f in run(precision):
            assert f["flow_maxabs"] < 0.05 and f["scale_maxabs"] < 0.05, f
            assert f["matched_frac"] >= 0.95 and f["logits_maxabs"] < 0.3, f


def test_dff_module_api(cuda_dev):
    """build_detection_model(cfg) for META_ARCHITECTURE GeneralizedRCNNDFF: reference state_dict keys, dataset dict in,
    list[BoxList] out; a non-key first frame is rejected"""
    from mega_core.b200 import synth
    from mega_core.modeling.detector import build_detection_model_from_state_dict
    sd = synth.make_state_dict("dff_r101", seed=6)
    model = build_detection_model_from_state_dict(sd, method="dff", device=cuda_dev)
    h, w = 192, 320
    with pytest.raises(RuntimeError):
        model({"cur": synth.synthetic_frame(0, h, w)[0], "is_key_frame": False})
    for t, key in enumerate((True, False)):
        out = model({"cur": synth.synthetic_frame(3 * t, h, w)[0], "is_key_frame": key})
        assert len(out) == 1 and out[0].bbox.shape[1] == 4 and out[0].has_field("scores") and out[0].has_field("labels")



@pytest.mark.parametrize("modulated,groups,dg,stride,pad,dil", [(False, 1, 1, 1, 1, 1), (True, 1, 1, 1, 1, 1),
                                                                (True, 2, 2, 2, 1, 1), (False, 2, 4, 1, 2, 2)])
def test_deform_conv_backward(cuda_dev, modulated, groups, dg, stride, pad, dil):
    import train_ops_oracle as to
    from mega_core import _C
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(60 + groups + dg)
    b, c, h, w, cout, k = 2, 32, 19, 23, 64, 3
    x = torch.randn(b, c, h, w, generator=g)
    wt = torch.randn(cout, c // groups, k, k, generator=g) / (c * 9 / groups) ** 0.5
    bias = torch.randn(cout, generator=g) if modulated else None
    ho = (h + 2 * pad - (dil * (k - 1) + 1)) // stride + 1
    wo = (w + 2 * pad - (dil * (k - 1) + 1)) // stride + 1
    off = torch.randn(b, dg * 2 * k * k, ho, wo, generator=g) * 2.0
    mask = torch.rand(b, dg * k * k, ho, wo, generator=g) if modulated else None
    go = torch.randn(b, cout, ho, wo, generator=g)
    ref = to.deform_conv2d_grads(x, off, mask, wt, bias, go, (stride, stride), (pad, pad), (dil, dil), groups, dg)
    d = cuda_dev
    xd, offd, wtd, god = x.to(d), off.to(d), wt.to(d), go.to(d)
    gin, goff, gw = torch.zeros_like(xd), torch.zeros_like(offd), torch.zeros_like(wtd)
    with ops.precision("fp32x3"):
        if modulated:
            maskd, biasd = mask.to(d), bias.to(d)
            gmask, gb = torch.zeros_like(maskd), torch.zeros_like(biasd)
            _C.modulated_deform_conv_backward(xd, wtd, biasd, None, offd, maskd, None, gin, gw, gb, goff, gmask, god, k, k,
                                              stride, stride, pad, pad, dil, dil, groups, dg, True)
        else:
            assert _C.deform_conv_backward_input(xd, offd, god, gin, goff, wtd, None, k, k, stride, stride, pad, pad, dil,
                                                 dil, groups, dg, b) == 1
            assert _C.deform_conv_backward_parameters(xd, offd, god, gw, None, None, k, k, stride, stride, pad, pad, dil,
                                                      dil, groups, dg, 1.0, b) == 1
    torch.cuda.synchronize()
    assert _rel_err(gin.cpu(), ref["input"]) < 2e-4
    assert _rel_err(goff.cpu(), ref["offset"]) < 2e-4
    assert _rel_err(gw.cpu(), ref["weight"]) < 2e-4
    if modulated:
        assert _rel_err(gmask.cpu(), ref["mask"]) < 2e-4
        assert _rel_err(gb.cpu(), ref["bias"]) < 1e-5


def test_layers_autograd_on_device(cuda_dev):
    """mega_core.layers wrappers: forward and backward both on the sm_90a kernels"""
    import train_ops_oracle as to
    from mega_core import layers
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(71)
    feat = torch.randn(2, 6, 12, 17, generator=g)
    rois = _rois(g, 5, 2, 17 * 16, 12 * 16)
    wgt = torch.randn(5, 6, 7, 7, generator=g)
    x = feat.to(cuda_dev).requires_grad_(True)
    out = layers.ROIAlign((7, 7), 1 / 16.0, 2)(x, rois.to(cuda_dev))
    (out * wgt.to(cuda_dev)).sum().backward()
    assert torch.allclose(out.detach().cpu(), to.roi_align(feat, rois, 1 / 16.0, 7, 7, 2), atol=2e-6)
    assert torch.allclose(x.grad.cpu(), to.roi_align_backward(wgt, rois, 1 / 16.0, 7, 7, 2, 6, 12, 17, 2), atol=2e-5)
    # ModulatedDeformConvPack starts as 0.5 * conv(x, w) + b (zero offsets, masks sigmoid(0))
    torch.manual_seed(5)
    m = layers.ModulatedDeformConvPack(32, 64, 3, stride=1, padding=1, deformable_groups=2).to(cuda_dev)
    with torch.no_grad():
        m.bias.normal_()
    xx = torch.randn(2, 32, 9, 11, device=cuda_dev, requires_grad=True)
    with ops.precision("fp32x3"):
        y = m(xx)
        y.sum().backward()
    xr = xx.detach().cpu().double().requires_grad_(True)
    wr = m.weight.detach().cpu().double().requires_grad_(True)
    ref = 0.5 * torch.nn.functional.conv2d(xr, wr, None, 1, 1) + m.bias.detach().cpu().double().view(1, -1, 1, 1)
    ref.sum().backward()
    assert _rel_err(y.detach().cpu(), ref.detach().float()) < 1e-4
    assert _rel_err(m.weight.grad.cpu(), wr.grad.float()) < 2e-4
    assert _rel_err(xx.grad.cpu(), xr.grad.float()) < 2e-4


def test_nvjpeg_decode_feeds_the_transform(cuda_dev):
    """encoded JPEG -> nvJPEG (torchvision.io.decode_jpeg on the device, a library decoder) -> planar uint8 [3, H, W] ->
    the device transform, without a host round trip or re-layout. The transform must be bit-exact on the pixels nvJPEG
    produced (checked against the reference pipeline fed with those very pixels). The decoders themselves are NOT
    pixel-identical -- libjpeg-turbo (PIL) interpolates the subsampled chroma, nvJPEG replicates it, +-80 in a channel at a
    sharp colour edge (first B200 run: mean |diff| 2.9 after the transform) -- so against the PIL-decoded frame only a
    loose sanity bound is asserted."""
    import io
    import numpy as np
    import image_oracle as io_
    from PIL import Image
    from mega_core.data.transforms import DeviceTestTransform, decode_jpeg
    mean, std = [102.9801, 115.9465, 122.7717], [1.0, 1.0, 1.0]
    g = np.random.default_rng(3)
    base = g.integers(0, 256, (46, 81, 3), dtype=np.uint8)
    img = np.kron(base, np.ones((16, 16, 1), dtype=np.uint8))[:720, :1280]
    buf = io.BytesIO()
    Image.fromarray(img, "RGB").save(buf, format="JPEG", quality=92)
    try:
        dec = decode_jpeg(buf.getvalue(), device=cuda_dev)
    except RuntimeError as e:                       # a torchvision build without nvJPEG: the library is absent, not ours
        pytest.skip("torchvision.io.decode_jpeg on the device is unavailable: %s" % str(e)[:80])
    assert dec.is_cuda and dec.dtype == torch.uint8 and tuple(dec.shape) == (3, 720, 1280)
    out, _ = DeviceTestTransform(600, 1000, mean, std, True, device=cuda_dev)(dec)
    same_pixels = io_.reference_pipeline(dec.permute(1, 2, 0).contiguous().cpu().numpy(), 600, 1000, mean, std, True)
    assert torch.equal(out.cpu(), same_pixels)
    pil = io_.reference_pipeline(np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGB")), 600, 1000, mean, std, True)
    assert (out.cpu() - pil).abs().mean() < 10.0


def test_two_key_frames_per_call_on_device(cuda_dev):
    """MegaEngine.step2_batched (per-frame branch of two key frames as one batch of four images; bit-identical to two
    step_batched calls on the CPU stand-ins) on the device: a different batch size moves the stream-K split points of the
    wgmma GEMMs, so the comparison with two single-frame steps is statistical (the fp16 re-association noise bound of
    the frame-parallel test); the window / global rings, which are plain copies of identical payload rows up to that
    noise, must stay close as well."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from mega_core.b200 import engine, synth
    from test_engine_gpu import _match_rows
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "mega_r101_192x320.pt"))
    h, w = gold["h"], gold["w"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(24)]
    glob0 = [frames[(3 * j + 1) % 24] for j in range(10)]
    pair = lambda t: torch.cat([frames[(t + 12) % 24], frames[(5 * t + 3) % 24]], 0)
    a = engine.MegaEngine(sd, engine.EngineConfig(precision="f16"), device=cuda_dev)
    b = engine.MegaEngine(sd, engine.EngineConfig(precision="f16"), device=cuda_dev)
    for e in (a, b):
        e.start_video(frames[0], frames[1:13], glob0, w, h)
    worst = 0.0
    for t in range(1, 5, 2):
        outs = []
        for i in range(2):
            det = a.step_batched(pair(t + i), w, h)
            torch.cuda.synchronize()
            k = int(a.cur_cnt.view(-1)[0].item())
            outs.append((a.last_pred[:k].float().cpu(), int(det.count.item()), a.Bq0[:k].cpu()))
        d0, d1 = b.step2_batched(torch.cat([pair(t), pair(t + 1)], 0), w, h)
        torch.cuda.synchronize()
        k = int(b.cur_cnt.view(-1)[0].item())
        idx = _match_rows(b.Bq0[:k].cpu(), outs[1][2])                 # a flipped NMS decision shifts rows: match by box
        m = idx >= 0
        assert m.float().mean().item() >= 0.95
        diff = (b.last_pred[:k].float().cpu()[idx[m], :31] - outs[1][0][m, :31]).abs()
        worst = max(worst, torch.quantile(diff.flatten(), 0.99).item())
        assert abs(int(d0.count.item()) - outs[0][1]) <= 3 and abs(int(d1.count.item()) - outs[1][1]) <= 3
    assert worst < 2e-2, worst
    # the window rings hold the same frames in the same slots; inside a slot a flipped near-tie of the RPN's NMS shifts the
    # rows behind it, so rows are matched by box (like the logits above), not by position (first B200 run: one swapped
    # proposal put a different row at the same position and the positional comparison failed)
    KP = a.KP
    ring_worst, matched = 0.0, []
    for slot in range(a.L):
        ba, bb = a.win_boxes[slot * KP:(slot + 1) * KP].cpu(), b.win_boxes[slot * KP:(slot + 1) * KP].cpu()
        ka, kb = int(a.win_cnt[slot, 0].item()), int(b.win_cnt[slot, 0].item())
        assert abs(ka - kb) <= 3, (slot, ka, kb)
        idx = _match_rows(bb[:kb], ba[:ka])
        m = idx >= 0
        matched.append(m.float().mean().item())
        xa = a.win_x[slot * KP:slot * KP + ka].float().cpu()[m]
        xb = b.win_x[slot * KP:slot * KP + kb].float().cpu()[idx[m]]
        ring_worst = max(ring_worst, torch.quantile((xa - xb).abs().flatten()[:4_000_000], 0.999).item())
    assert min(matched) >= 0.95, matched
    assert ring_worst < 2e-2, ring_worst
    # global pool (75 rows per frame, no boxes kept): a swap inside the first 75 proposals shifts a few rows of one frame
    assert ((a.glob_x.float() - b.glob_x.float()).abs() > 0.05).float().mean().item() < 0.05


@pytest.mark.parametrize("precision", ["fp32x3", "f16"])
def test_pipelined_steps_match_batched_steps(cuda_dev, precision):
    """MegaEngine.stepn_pipelined: the aggregation of a batch of key frames runs concurrently with the per-frame branch of the
    next batch (two streams, persistent grids capped so that they share the GPU by SMs). The arithmetic is that of
    stepn_batched up to the stream-K split points of the capped grids: strict mode -> every detection count equal and the
    predictor outputs within 2e-3; fp16 mode -> the re-association bound of the tests above. Eager and CUDA-graph replays."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from mega_core.b200 import engine, synth
    from test_engine_gpu import _match_rows
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "mega_r101_192x320.pt"))
    h, w = gold["h"], gold["w"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(24)]
    glob0 = [frames[(3 * j + 1) % 24] for j in range(10)]
    pair = lambda t: torch.cat([frames[(t + 12) % 24], frames[(5 * t + 3) % 24]], 0)
    batch = lambda s: torch.cat([pair(1 + 2 * s), pair(2 + 2 * s)], 0)
    a = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev)
    b = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev)
    for e in (a, b):
        e.start_video(frames[0], frames[1:13], glob0, w, h)
        e.use_graph = True
    steps = 5                       # a graph key runs eagerly once, is captured on its second use, replays from the third

    def snap(e, dets):
        torch.cuda.synchronize()
        k = int(e.cur_cnt.view(-1)[0].item())
        return [int(d.count.item()) for d in dets], e.last_pred[:k].float().cpu(), e.Bq0[:k].cpu()

    want = [snap(a, a.stepn_batched(batch(s), w, h)) for s in range(steps)]
    assert b.stepn_pipelined(batch(0), w, h) is None
    got = [snap(b, b.stepn_pipelined(batch(s + 1) if s + 1 < steps else None, w, h)) for s in range(steps)]
    tol, cnt_tol = (2e-3, 0) if precision == "fp32x3" else (2e-2, 3)
    for (ca, pa, ba), (cb, pb, bb) in zip(want, got):
        assert all(abs(x - y) <= cnt_tol for x, y in zip(ca, cb)), (ca, cb)
        idx = _match_rows(bb, ba)
        m = idx >= 0
        assert m.float().mean().item() >= (1.0 if precision == "fp32x3" else 0.95)
        d = (pb[idx[m], :31] - pa[m, :31]).abs()
        assert torch.quantile(d.flatten(), 0.99).item() < tol, torch.quantile(d.flatten(), 0.99).item()
