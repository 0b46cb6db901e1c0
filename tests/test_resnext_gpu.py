"""GPU tests of the grouped (ResNeXt) convolutions: ops.conv_gemm(groups=...) against torch's grouped conv in fp64 in
every operand arithmetic, the X-101 body as one layer chain against per-layer launches, and the MEGA / single-frame
engines on a ResNeXt-101 32x8d body against the fixtures written from the unmodified reference
(tools/make_golden_resnext.py)."""
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _rel_err(got, ref):
    ref = ref.double()
    return ((got.double().cpu() - ref).abs().max() / ref.pow(2).mean().sqrt().clamp_min(1e-12)).item()


# arithmetic -> bound on max|err| / RMS(output), the bars of the dense cases (test_conv_gemm_gpu.py, test_split16_gpu.py);
# fp16 output: one rounding of the fp32 result, checked element by element as there
_BOUNDS = {"tf32": 4e-3, "fp32x3": 5e-5, "split16": 1e-5, "f16": 2e-5, "f16_out16": None}


def _grouped_conv(cuda_dev, mode, gw, stream_k=None):
    """3x3 grouped conv, stride 2, dilation 2, scale / bias, residual and ReLU, 256 channels in 256 / gw groups ->
    (result as fp32 NCHW on the host, fp64 reference)"""
    from mega_core.b200 import ops
    g = torch.Generator().manual_seed(gw)
    n, h, w, c = 2, 37, 61, 256
    groups = c // gw
    f16 = mode.startswith("f16")
    x = torch.randn(n, c, h, w, generator=g).relu() * 2.0
    wt = torch.randn(c, gw, 3, 3, generator=g) / (9 * gw) ** 0.5
    res = torch.randn(n, c, (h + 1) // 2, (w + 1) // 2, generator=g)
    if f16:     # operands rounded up front: the fp64 reference isolates the kernel's own error
        x, wt, res = x.half().float(), wt.half().float(), res.half().float()
    scale = torch.rand(c, generator=g) + 0.5
    bias = torch.randn(c, generator=g)
    ref = F.conv2d(x.double(), wt.double(), None, 2, 2, 2, groups) * scale.double().view(1, -1, 1, 1) \
        + bias.double().view(1, -1, 1, 1)
    ref = (ref + res.double()).relu()
    dt = torch.float16 if f16 else torch.float32
    a = x.permute(0, 2, 3, 1).contiguous().to(cuda_dev).to(dt)
    wp = ops.pack_grouped_conv(wt, groups, cuda_dev, dt)
    r = res.permute(0, 2, 3, 1).contiguous().to(cuda_dev)
    out = torch.full((n, ref.shape[2], ref.shape[3], c), float("nan"), device=cuda_dev,
                     dtype=torch.float16 if mode == "f16_out16" else torch.float32)
    r = r.to(out.dtype)
    sc = scale.to(cuda_dev)
    if mode == "split16":
        a = ops.pack_split16(a)
        wp = ops.pack_weights_split16(wp, scale=sc)
        sc = None
    with ops.precision("fp32x3" if mode in ("fp32x3", "split16") else "tf32"):
        ops.conv_gemm(a, wp, out, taps=(3, 3), dil=2, pad=2, stride=(2, 2), scale=sc, bias=bias.to(cuda_dev),
                      residual=r, relu=True, groups=groups, stream_k=stream_k)
    torch.cuda.synchronize()
    got = out.float().permute(0, 3, 1, 2).cpu()
    assert torch.isfinite(got).all(), "kernel left unwritten / non-finite outputs"
    return got, ref


@pytest.mark.parametrize("gw", [8, 16, 32, 64])
@pytest.mark.parametrize("mode", sorted(_BOUNDS))
def test_grouped_conv_matches_fp64(cuda_dev, mode, gw):
    got, ref = _grouped_conv(cuda_dev, mode, gw)
    err = _rel_err(got, ref)
    print("grouped conv %s gw %d: max|err| / RMS %.3e" % (mode, gw, err))
    if _BOUNDS[mode] is None:
        bound = ref.abs() * 2.0 ** -11 + 2e-5 * ref.pow(2).mean().sqrt()
        excess = (got.double().cpu() - ref).abs() / bound
        assert (excess <= 1.01).all(), excess.max().item()
    else:
        assert err < _BOUNDS[mode], err


@pytest.mark.parametrize("gw", [8, 16, 32])
@pytest.mark.parametrize("mode", ["tf32", "fp32x3", "split16", "f16", "f16_out16"])
@pytest.mark.parametrize("stream_k", [0, 1])
def test_diagonal_issue_is_bit_identical(cuda_dev, mode, gw, stream_k):
    """group_width set (MMAs of the diagonal blocks only) vs 0 (the whole 64-channel chunk): the skipped products are
    exact zeros, so the outputs are equal bit for bit -- also under stream-K, whose segments may start on either half of
    a tap's channels"""
    from mega_core.b200 import ops
    outs = []
    for diag in (True, False):
        saved, ops.GROUP_DIAG[0] = ops.GROUP_DIAG[0], diag
        try:
            outs.append(_grouped_conv(cuda_dev, mode, gw, stream_k=stream_k)[0])
        finally:
            ops.GROUP_DIAG[0] = saved
    assert torch.equal(outs[0], outs[1]), (outs[0] - outs[1]).abs().max().item()


def test_group_width_is_validated(cuda_dev):
    """a group_width outside {8, 16, 32, 64}, or on a launch without the 64-channel batched layout, is refused"""
    from mega_core import _lib
    from mega_core.b200 import ops
    a = torch.zeros(1, 8, 8, 128, device=cuda_dev)
    w = ops.pack_grouped_conv(torch.zeros(128, 8, 3, 3), 16, cuda_dev)
    out = torch.zeros(1, 8, 8, 128, device=cuda_dev)
    saved = ops._launch_conv_gemm
    for bad in ({"group_width": 12}, {"group_width": 8, "b_k_off": 64}, {"group_width": 8, "a_c_off": 0}):
        def launch(d, bad=bad):
            for k, v in bad.items():
                setattr(d, k, v)
            saved(d)
        ops._launch_conv_gemm = launch
        try:
            with pytest.raises(_lib.MegaError, match="group_width"):
                ops.conv_gemm(a, w, out, taps=(3, 3), pad=1, groups=16)
        finally:
            ops._launch_conv_gemm = saved


@pytest.mark.parametrize("n", [2, 4])
def test_x101_body_chain_equals_per_layer_launches(cuda_dev, n):
    """the f16 X-101 body (grouped conv2 included) as one persistent chain kernel (n = 4: two interleaved lanes) and as
    per-layer launches with the same tile choices: bit-identical"""
    from mega_core.b200 import engine, ops, synth
    sd = synth.make_state_dict("mega_x101", seed=0)
    img = torch.cat([synth.synthetic_frame(i, 192, 320) for i in range(n)]).to(cuda_dev)
    saved = ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0]
    ops.AUTOTUNE[0] = False
    try:
        bb = engine.Backbone(sd, cuda_dev, dtype=torch.float16)
        y_chain = bb.forward(img).clone()
        y_chain2 = bb.forward(img).clone()              # replayed
        ops.CHAINS_ENABLED[0] = False
        ops.MAX_BN[0] = 128                             # the widest tile a chain layer may pick
        bb2 = engine.Backbone(sd, cuda_dev, dtype=torch.float16)
        y_layers = bb2.forward(img).clone()
    finally:
        ops.AUTOTUNE[0], ops.MAX_BN[0], ops.CHAINS_ENABLED[0] = saved
    torch.cuda.synchronize()
    assert len(bb._chains) == 1 and not bb2._chains
    assert torch.isfinite(y_chain.float()).all()
    assert torch.equal(y_chain, y_chain2)
    assert torch.equal(y_chain, y_layers), (y_chain.float() - y_layers.float()).abs().max().item()


def _match_rows(a, b, tol=0.75):
    """for each row of b (reference boxes) the index of an identical-within-tol row of a, or -1"""
    d = (a[:, None, :] - b[None, :, :]).abs().amax(2)
    val, idx = d.min(0)
    idx[val > tol] = -1
    return idx


def _run_mega_x101(cuda_dev, label, precision):
    from mega_core.b200 import engine, synth
    gold = torch.load(os.path.join(GOLD, "mega_x101_192x320.pt"))
    h, w, total = gold["h"], gold["w"], gold["total"]
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    frames = [synth.synthetic_frame(i, h, w).to(cuda_dev) for i in range(total)]
    eng = engine.MegaEngine(sd, engine.EngineConfig(precision=precision), device=cuda_dev)
    gpf = gold["globals_per_frame"]
    per_frame = []
    for t, ref in enumerate(gold["frames"]):
        if t == 0:
            det = eng.start_video(frames[0], frames[1:13], [frames[j] for j in gpf[0]], w, h)
        else:
            det = eng.step(frames[min(t + 12, total - 1)], frames[gpf[t][0]], w, h)
        torch.cuda.synchronize()
        k = int(eng.cur_cnt.view(-1)[0].item())
        props = eng.Bq0[:k].cpu()
        idx = _match_rows(props, ref["proposals"])
        m = idx >= 0
        pred = eng.last_pred[:k].float().cpu()
        assert torch.isfinite(pred).all()
        dabs = (pred[idx[m], :31] - ref["class_logits"][m]).abs()
        b, s, l = det.to_host()
        per_frame.append({"proposals": k, "ref_proposals": int(ref["proposals"].shape[0]),
                          "matched_frac": m.float().mean().item(), "logits_maxabs": dabs.max().item(),
                          "deltas_maxabs": (pred[idx[m], 31:155] - ref["box_regression"][m]).abs().max().item(),
                          "logits_p99": torch.quantile(dabs.flatten(), 0.99).item(),
                          "dets": int(b.shape[0]), "ref_dets": int(ref["boxes"].shape[0]),
                          "logit_rms": ref["class_logits"].pow(2).mean().sqrt().item()})
        print(label, json.dumps(per_frame[-1]))
    return per_frame


# The X-101 fixture's 4th frame holds one proposal row whose logits the reference itself does not pin down to better than
# ~1e-2: the oracle in fp32 with its input frames multiplied by (1 + 1e-6 noise) moves that row by 8.5e-3 (every other row
# by < 1e-3, p99 6.5e-5; the R-101 fixture has no such row). The max bars below are set above that row; the p99 bars are
# the R-101 ones or tighter.
def test_mega_x101_fp32x3_matches_reference_fixture(cuda_dev):
    """strict mode: every proposal and every detection of the reference; logits p99 < 1e-3 (measured <= 5.0e-4), max
    < 3e-2 (measured 2.0e-2 on the row above, <= 5.6e-3 on the first three frames), deltas < 1e-2 (measured 6.9e-3)"""
    for f in _run_mega_x101(cuda_dev, "mega_x101_fp32x3", "fp32x3"):
        assert f["matched_frac"] == 1.0 and f["proposals"] == f["ref_proposals"], f
        assert f["dets"] == f["ref_dets"], f
        assert f["logits_p99"] < 1e-3, f
        assert f["logits_maxabs"] < 3e-2, f
        assert f["deltas_maxabs"] < 1e-2, f


def test_mega_x101_f16_matches_reference_fixture(cuda_dev):
    for f in _run_mega_x101(cuda_dev, "mega_x101_f16", "f16"):
        assert f["matched_frac"] >= 0.95, f
        assert f["logits_p99"] < 3e-2, f


def test_mega_x101_logic_matches_reference_with_exact_fp32_contractions(cuda_dev):
    """the engine's orchestration of the grouped layers with exact-fp32 contractions (tests/fp32_shadow.py)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from fp32_shadow import fp32_shadow
    with fp32_shadow():
        frames = _run_mega_x101(cuda_dev, "mega_x101_fp32_shadow", "tf32")
    for f in frames:      # measured: p99 <= 4.9e-5, max 2.6e-4 .. 8.4e-4 and 7.7e-3 on the row above
        assert f["matched_frac"] == 1.0, f
        assert f["logits_p99"] < 1e-4, f
        assert f["logits_maxabs"] < 1e-2, f
        assert f["deltas_maxabs"] < 5e-3, f
        assert f["dets"] == f["ref_dets"], f


def test_base_x101_matches_reference_fixture(cuda_dev):
    """single-frame detector, strict mode: every proposal and detection, logits < 1e-2 (measured 2.4e-5)"""
    from mega_core.b200 import engine, synth
    gold = torch.load(os.path.join(GOLD, "base_x101_192x320.pt"))
    sd = synth.make_state_dict(gold["arch"], seed=gold["seed"])
    img = synth.synthetic_frame(gold["frame_index"], gold["h"], gold["w"]).to(cuda_dev)
    eng = engine.BaseEngine(sd, engine.EngineConfig(precision="fp32x3"), device=cuda_dev)
    det = eng.forward(img, gold["w"], gold["h"])
    torch.cuda.synchronize()
    k = int(eng.last_cnt[0].item())
    idx = _match_rows(eng.last_props[:k].cpu(), gold["proposals"])
    m = idx >= 0
    pred = eng.last_pred[:k].float().cpu()
    dl = (pred[idx[m], :31] - gold["class_logits"][m]).abs().max().item()
    b, s, l = det.to_host()
    print("base_x101_fp32x3", json.dumps({"proposals": k, "ref_proposals": int(gold["proposals"].shape[0]),
                                          "matched_frac": m.float().mean().item(), "logits_maxabs": dl,
                                          "dets": int(b.shape[0]), "ref_dets": int(gold["boxes"].shape[0])}))
    assert m.float().mean().item() == 1.0 and b.shape[0] == gold["boxes"].shape[0]
    assert dl < 1e-2, dl
