"""Conformance of every wgmma conv_gemm instantiation and of the layer chain against an fp64 reference of the descriptor
contract (include/mega_b200.h), element by element:

    |got - ref| <= ALPHA[mode] * P + out_rounding + tiny,     P = |scale| * conv(|a|, |b|)

out_rounding is the epilogue's own rounding: 2^-22 (|scale * acc| + |bias| + |residual|) for its fp32 fused multiply-add /
residual add, plus 2^-11 |ref| for fp16 outputs or the split-fp16 format's 2^-23 |ref| + 2^-25 (mega_b200.h). f16 and 3xFP16
operands are rounded to their storage format first, so the reference isolates the kernel's own error.

ALPHA per operand mode: >= 2x headroom over the largest err / P measured over the whole file on an NVIDIA H100 80GB HBM3
(SXM, 700 W):
    tf32   (round-to-nearest on load)       measured 3.3e-4    ALPHA 7e-4
    3xtf32 (hi*hi + hi*lo + lo*hi)          measured 7.6e-7    ALPHA 1.6e-6
    f16    (fp16 operands, fp32 accumulate) measured 9.9e-7    ALPHA 2e-6
    3xfp16 (split-fp16 operands)            measured 3.3e-7    ALPHA 7e-7

Besides the values every case checks: a sentinel bit pattern around the output view (channels past cout, skipped rows,
an extra column and image) is unchanged, no NaN is left inside the view, the operands and the residual are unchanged
and the stream-K tile counters are back to zero. A final test asserts that every one of the 42 instantiations ran with
stream-K on and off in a case that passed.
"""
import ctypes
import json
import os
import re

import pytest
import torch

from conv_gemm_ref import (COUNTER_INTS, MODES, VARIANTS, case_fields, case_problem, chain_rotation, conv_gemm_ref,
                           encoder_grid, make_cases, make_sk_cases, operand_extents, sk_label_holds, variant_of)

pytestmark = pytest.mark.gpu

ALPHA = {0: 7e-4, 1: 1.6e-6, 2: 2e-6, 3: 7e-7}
SENT32 = 0x7FA5A5A5         # a NaN payload no kernel produces
SENT16 = 0x7D5A
CASES = make_cases()
SK_CASES = make_sk_cases()
PASSED = set()              # (precision, block_n, out16, group_width, stream_k) launched by a case that passed
MEASURED = {}               # mode -> largest (err - out_rounding) / P seen


@pytest.fixture
def launches(monkeypatch):
    """records the instantiation of every conv_gemm launch, then launches it"""
    from mega_core.b200 import ops
    log = []
    orig = ops._launch_conv_gemm

    def wrapped(d):
        log.append(variant_of(d.precision, d.block_n, d.out_f16, d.group_width) + (d.stream_k,))
        return orig(d)
    monkeypatch.setattr(ops, "_launch_conv_gemm", wrapped)
    return log


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _counters_zero(dev):
    from mega_core.b200 import ops
    torch.cuda.synchronize()
    ws = ops.gemm_workspace(dev)
    cnt = ws[:COUNTER_INTS * 4].view(torch.int32)
    assert int(cnt.count_nonzero()) == 0, "stream-K tile counters left non-zero: %s" % cnt.nonzero()[:8].flatten().tolist()


def _bound_check(mode, got, ref, P, Q, fmt, what):
    """element-wise bound; returns the measured (err - rounding) / P"""
    err = (got - ref).abs()
    rnd = 2.0 ** -22 * Q
    if fmt == "f16":
        rnd = rnd + 2.0 ** -11 * 1.001 * ref.abs() + 2.0 ** -24
    elif fmt == "split":
        rnd = rnd + 2.0 ** -23 * ref.abs() + 2.0 ** -25
    else:
        rnd = rnd + 1e-30
    bound = ALPHA[mode] * P + rnd
    bad = ~(err <= bound)
    ratio = ((err - rnd).clamp_min(0) / P.clamp_min(1e-300)).max().item()
    MEASURED[mode] = max(MEASURED.get(mode, 0.0), ratio)
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        i = tuple(idx)
        raise AssertionError("%s: %d elements out of bound, first at %s: got %r ref %r |err| %.3e bound %.3e (P %.3e); "
                             "max (err - rounding) / P = %.3e vs ALPHA %.1e" % (
                                 what, int(bad.sum()), idx, got[i].item(), ref[i].item(), err[i].item(), bound[i].item(),
                                 P[i].item(), ratio, ALPHA[mode]))
    return ratio


def _fill_sentinel(buf):
    _bits(buf).fill_(SENT16 if buf.element_size() == 2 else SENT32)


def run_case(c, dev, repeats=1):
    """builds the operands of case `c`, launches it through ops.conv_gemm `repeats` times and checks every element of
    the output buffer; returns the output bits after each launch"""
    from mega_core.b200 import ops
    mode, out16 = c["mode"], c["out16"]
    g = torch.Generator(device=dev).manual_seed(c["seed"])
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    f = case_fields(c)
    (a_n, a_h, a_w, a_c), (taps, b_n, b_k), (on, oh, ow, oc), (rn, rc) = operand_extents(c)
    gw = c.get("group_width", 0)
    # ---- operands (rounded to their storage format; the reference reads the stored values)
    a32 = rnd(a_n, a_h, a_w, a_c)
    if gw:
        wl = rnd(c["channels"], gw, taps // c["taps"][1], c["taps"][1]) / (gw * taps) ** 0.5
        b32 = ops.pack_grouped_conv(wl, c["channels"] // gw, dev, torch.float16 if mode == 2 else torch.float32)
    else:
        b32 = rnd(taps, b_n, b_k) / (c["k"] * taps) ** 0.5
    acc_scale = 1.0
    if mode == 2:
        a = a32.half()
        b = b32.half() if not gw else b32
        A64, B64 = a.double(), b.double()
    elif mode == 3:
        a = ops.pack_split16(a32.contiguous())
        b = ops.pack_weights_split16(b32)
        acc_scale = ops._split16_weight(b)
        A64 = ops.split16_decode(a).double()
        B64 = ops.split16_decode(b).double()           # the stored weights; the kernel applies acc_scale
    else:
        a, b = a32, b32
        A64, B64 = a.double(), b.double()
    nsb = c["cout"] + (f["batch"] - 1) * f["bias_z_off"]
    scale = ((torch.rand(nsb, device=dev, generator=g) * 1.5 + 0.25) *
             torch.where(torch.rand(nsb, device=dev, generator=g) < 0.25, -1.0, 1.0)) if c["scale"] else None
    bias = rnd(nsb) * 0.5 if c["bias"] else None
    # ---- output: a view inside a sentinel-filled buffer with an extra image, row, column and channels
    split_out = mode == 3 and out16
    odt = torch.float16 if (mode == 2 and out16) else torch.float32
    rs = c["row_skip"]
    cq = 32 if split_out else 8
    buf = torch.empty(on + 1, oh * rs + 1, ow + 1, -(-oc // cq) * cq + cq, device=dev, dtype=odt)
    _fill_sentinel(buf)
    view = buf[:on, 0:oh * rs:rs, :ow, :oc]
    written = torch.zeros(on, oh, ow, oc, dtype=torch.bool, device=dev)
    cw = -(-c["cout"] // 32) * 32 if split_out else c["cout"]
    for z in range(f["batch"]):
        written[z * f["out_n_off"]:z * f["out_n_off"] + c["n_img"], :, :, z * f["out_c_off"]:z * f["out_c_off"] + cw] = True
    view.masked_fill_(written, float("nan"))
    if split_out:
        ops.mark_split16(buf)
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:on, 0:oh * rs:rs, :ow, :oc] = ~written
    # ---- residual: a view of its own padded buffer
    res = R64 = rbuf = None
    if c["res"] != "none":
        rdt = odt if c["res"] == "same" else torch.float32
        rq = 32 if c["res"] == "split" else 8
        rbuf = rnd(rn + 1, oh + 1, ow + 1, -(-rc // rq) * rq + rq).to(rdt)
        if c["res"] == "split":
            ops.pack_split16(rbuf)
            R64 = ops.split16_decode(rbuf).double()[:rn, :oh, :ow, :rc]
        else:
            R64 = rbuf.double()[:rn, :oh, :ow, :rc]
        res = rbuf[:rn, :oh, :ow, :rc]
    keep = [t.clone() for t in (a, b, rbuf) if t is not None]
    # ---- launch
    kw = dict(taps=c["taps"], dil=c["dil"], pad=c["pad"], stride=c["stride"], tile=c["tile"], n_img=c["n_img"],
              out_hw=c["out_hw"], max_ctas=c["max_ctas"], stream_k=c["stream_k"], scale=scale, bias=bias, residual=res,
              relu={0: False, 1: True, 2: "leaky"}[c["relu"]])
    if c["pad_w"] is not None:
        kw["pad_w"] = c["pad_w"]
    if gw:
        kw["groups"] = c["channels"] // gw
    else:
        kw.update(block_n=c["block_n"], cout=c["cout"], k=c["k"], batch=f["batch"])
        kw.update({key: f[key] for key in ("a_c_off", "a_n_off", "b_k_off", "b_n_off", "out_c_off", "out_n_off",
                                           "res_c_off", "res_n_off", "bias_z_off")})
    snaps = []
    with ops.precision(1 if mode == 1 else 0):
        for _ in range(repeats):
            ops.conv_gemm(a, b, view, **kw)
            torch.cuda.synchronize()
            snaps.append(_bits(buf).clone())
    _counters_zero(dev)
    # ---- guard band, unchanged inputs, no NaN left
    sent = SENT16 if odt == torch.float16 else SENT32
    changed = outside & (_bits(buf) != sent)
    assert not bool(changed.any()), "%s: wrote outside its output view (%d elements, channels %s, values %s)" % (
        c["id"], int(changed.sum()), sorted(set(changed.nonzero()[:, 3].tolist()))[:16], buf[changed][:8].tolist())
    for before, now in zip(keep, [t for t in (a, b, rbuf) if t is not None]):
        assert torch.equal(_bits(before), _bits(now)), "%s: an input tensor changed" % c["id"]
    got = (ops.split16_decode(view) if split_out else view).double()
    assert not bool(torch.isnan(got[written]).any()), "%s: NaN left inside the output view (%d elements)" % (
        c["id"], int(torch.isnan(got[written]).sum()))
    # ---- values
    if gw and mode != 3:      # the packed block-diagonal weights against a grouped convolution of the logical ones
        import torch.nn.functional as F
        wq = (wl.half() if mode == 2 else wl).double()
        x = F.pad(A64.permute(0, 3, 1, 2), (c["pad"],) * 4)
        want = F.conv2d(x, wq, dilation=c["dil"], groups=c["channels"] // gw).permute(0, 2, 3, 1)
        got_acc = torch.cat([v for _, v, _, _ in conv_gemm_ref(A64, B64, taps=c["taps"], dil=c["dil"], pad=c["pad"],
                                                               k=c["k"], n_img=c["n_img"], out_hw=c["out_hw"],
                                                               cout=c["cout"], **f)], 3)
        assert torch.allclose(got_acc, want, rtol=1e-12, atol=1e-12), "%s: pack_grouped_conv" % c["id"]
    blocks = conv_gemm_ref(A64, B64, taps=c["taps"], dil=c["dil"], pad=c["pad"], pad_w=c["pad_w"], stride=c["stride"],
                           k=c["k"], n_img=c["n_img"], out_hw=c["out_hw"], cout=c["cout"], scale=scale, bias=bias,
                           residual=R64, relu=c["relu"], acc_scale=acc_scale, **f)
    fmt = "split" if split_out else ("f16" if odt == torch.float16 else "f32")
    for z, ref, P, Q in blocks:
        gz = got[z * f["out_n_off"]:z * f["out_n_off"] + c["n_img"], :, :, z * f["out_c_off"]:z * f["out_c_off"] + c["cout"]]
        _bound_check(mode, gz, ref, P, Q, fmt, "%s batch %d" % (c["id"], z))
    return snaps


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_variant_sweep_matches_fp64(cuda_dev, launches, case):
    run_case(case, cuda_dev)
    want = variant_of(case["mode"], case["block_n"], case["out16"], case.get("group_width", 0)) + (case["stream_k"],)
    assert launches == [want], (launches, want)
    PASSED.add(want)


@pytest.mark.parametrize("label,case", SK_CASES, ids=[c["id"] for _, c in SK_CASES])
def test_stream_k_geometry(cuda_dev, launches, label, case):
    """stream-K splits (a) over >= 3 CTAs per tile, (bd) with a CTA spanning partial / whole / partial tiles on a grid
    that does not divide the units, (c) on one CTA, (e, f) of a 256-k-block reduction with and without the aligned grid:
    fp64 bound, two launches with identical bits, counters back at zero"""
    assert sk_label_holds(label, case), "the case no longer produces stream-K geometry (%s)" % label
    if torch.cuda.get_device_properties(cuda_dev).multi_processor_count < 132:
        pytest.skip("the stream-K geometry is worked out for the 132-CTA grid of an H100 SXM")
    snaps = run_case(case, cuda_dev, repeats=2)
    assert torch.equal(snaps[0], snaps[1]), "%s: two launches differ" % case["id"]
    assert len(set(launches)) == 1 and launches[0][-1] == 1
    PASSED.add(launches[0])


# ------------------------------------------------------------------------------------------------ layer chains
def _call_ref(a, w, out, kw):
    """fp64 reference of one ops.conv_gemm call (dense or grouped, fp16 operands) and its P / Q"""
    taps = kw.get("taps", (1, 1))
    cout = kw.get("cout") or w.shape[1]
    oh, ow = out.shape[1], out.shape[2]
    kk = dict(taps=taps, dil=kw.get("dil", 1), pad=kw.get("pad", 0), stride=kw.get("stride", (1, 1)), n_img=a.shape[0],
              out_hw=(oh, ow), scale=kw.get("scale"), bias=kw.get("bias"), relu={False: 0, True: 1, "leaky": 2}[kw.get("relu", False)])
    res = kw.get("residual")
    if kw.get("groups", 1) > 1:
        z = 64
        blocks = conv_gemm_ref(a.double(), w.double(), k=z, cout=z, batch=w.shape[1] // z, a_c_off=z, b_n_off=z,
                               out_c_off=z, res_c_off=z, bias_z_off=z, residual=None if res is None else res.double(), **kk)
        ref = torch.cat([b[1] for b in blocks], 3)
        P = torch.cat([b[2] for b in blocks], 3)
        Q = torch.cat([b[3] for b in blocks], 3)
        return ref, P, Q
    _, ref, P, Q = conv_gemm_ref(a.double(), w.double(), k=w.shape[2], cout=cout,
                                 residual=None if res is None else res.double(), **kk)[0]
    return ref, P, Q


def _chain_layers(dev, g):
    """weights of a chain mixing the layer kinds the engines record: 1x1, 3x3, grouped 3x3 (dilated), 1x1 + residual,
    strided 1x1 (first block of res3 / res4), dilated 3x3 (res5), 1x1 to 512, the REDUCE_CHANNEL 1x1 + ReLU and a
    ragged-cout fp32 head"""
    from mega_core.b200 import ops
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    w = lambda t, ci, co: (rnd(t, co, ci) / (t * ci) ** 0.5).half()
    sb = lambda co: dict(scale=torch.rand(co, device=dev, generator=g) * 0.5 + 0.75, bias=rnd(co) * 0.1)
    grp = ops.pack_grouped_conv(rnd(128, 32, 3, 3) / (9 * 32) ** 0.5, 4, dev, torch.float16)
    return [
        ("t1", w(1, 256, 128), dict(block_n=128, stream_k=0, relu=True, **sb(128))),
        ("t2", w(9, 128, 128), dict(taps=(3, 3), pad=1, block_n=64, stream_k=1, relu=True, **sb(128))),
        ("t3", grp, dict(taps=(3, 3), dil=2, pad=2, groups=4, stream_k=0, relu=True, **sb(128))),
        ("y", w(1, 128, 256), dict(block_n=128, stream_k=1, relu=True, residual="x", **sb(256))),
        ("s", w(1, 256, 128), dict(stride=(2, 2), block_n=128, stream_k=0, relu=True, **sb(128))),
        ("u", w(9, 128, 128), dict(taps=(3, 3), dil=2, pad=2, block_n=64, stream_k=1, relu=True, **sb(128))),
        ("v", w(1, 128, 512), dict(block_n=128, stream_k=0, relu=True, **sb(512))),
        ("rdc", w(1, 512, 256), dict(block_n=128, stream_k=1, relu=True, **sb(256))),
        ("head", w(1, 256, 64)[:, :60].contiguous(), dict(block_n=64, stream_k=0, cout=60, bias=rnd(60))),
    ]


def _chain_bufs(dev, n, h, w):
    hs, ws = h // 2, w // 2
    shapes = dict(t1=(n, h, w, 128), t2=(n, h, w, 128), t3=(n, h, w, 128), y=(n, h, w, 256), s=(n, hs, ws, 128),
                  u=(n, hs, ws, 128), v=(n, hs, ws, 512), rdc=(n, hs, ws, 256))
    d = {k: torch.full(s, float("nan"), device=dev, dtype=torch.float16) for k, s in shapes.items()}
    d["head"] = torch.full((n, hs, ws, 64), float("nan"), device=dev)
    return d


def _run_chain_lane(ops, layers, bufs, x, log=None):
    cur = x
    for name, wt, kw in layers:
        kw = dict(kw)
        if kw.get("residual") == "x":
            kw["residual"] = x
        out = bufs[name][..., :60] if name == "head" else bufs[name]
        ops.conv_gemm(cur, wt, out, tile=(8, 16), max_ctas=40, **kw)
        if log is not None:
            log.append((cur, wt, out, kw))
        cur = out


@pytest.mark.parametrize("depth", [1, 2])
def test_layer_chain_conformance(cuda_dev, depth):
    """the chain kernel against per-layer launches (identical bits over several replays) and every layer against the
    fp64 reference applied to the fp16 input the chain stored for it; the barrier words and the tile counters are zero
    after every replay. Grid capped at 40 CTAs: the whole-tile layers of the strided half use fewer (active_ctas < grid)
    and, at depth 2, start on rotated CTAs."""
    from mega_core.b200 import ops
    dev = cuda_dev
    g = torch.Generator(device=dev).manual_seed(77 + depth)
    layers = _chain_layers(dev, g)
    n, h, w = 2, 18, 24
    lanes = 2 if depth == 2 else 1
    xs = [torch.randn(n, h, w, 256, device=dev, generator=g).half() for _ in range(lanes)]
    # per-layer launches; their descriptors give the grid facts
    descs = []
    orig = ops._launch_conv_gemm

    def rec(d):
        descs.append((d.n_img, d.out_h, d.out_w, d.tile_h, d.tile_w, d.cout, d.block_n, d.batch, d.taps_r * d.taps_s,
                      d.k_per_tap, d.stream_k))
        orig(d)
    ref_bufs = [_chain_bufs(dev, n, h, w) for _ in range(lanes)]
    ops._launch_conv_gemm = rec
    try:
        with ops.sm_limit(40):
            for lane in range(lanes):
                _run_chain_lane(ops, layers, ref_bufs[lane], xs[lane])
    finally:
        ops._launch_conv_gemm = orig
    torch.cuda.synchronize()
    facts = []
    for (ni, oh, ow, th, tw, cout, bn, bt, taps, k, sk) in descs:
        tiles = bt * ni * -(-oh // th) * -(-ow // tw) * -(-cout // bn)
        kb = taps * -(-k // 64)
        facts.append((tiles, encoder_grid(tiles, kb, sk, 40)[0], sk))
    if depth == 2:       # interleaved A0 B0 A1 B1 ...
        facts = [f for pair in zip(facts[:len(layers)], facts[len(layers):]) for f in pair]
    grid = max(f[1] for f in facts)
    assert any(f[1] < grid for f in facts), facts
    if depth == 2:
        assert any(r != 0 for r in chain_rotation(facts, grid))
    # the chain
    got_bufs = [_chain_bufs(dev, n, h, w) for _ in range(lanes)]
    cache, logs = {}, [[] for _ in range(lanes)]
    for rep in range(3):
        with ops.sm_limit(40):
            with ops.chain(cache, "conformance", dev, interleave=depth == 2) as ch:
                for lane in range(lanes):
                    if lane:
                        ch.next_lane()
                    _run_chain_lane(ops, layers, got_bufs[lane], xs[lane], logs[lane] if rep == 0 else None)
        torch.cuda.synchronize()
        (chain_obj,) = cache.values()
        assert chain_obj.n == len(layers) * lanes and chain_obj.depth == depth and chain_obj.grid == grid
        assert int(chain_obj.sync[:depth + 1].count_nonzero()) == 0, chain_obj.sync.tolist()
        _counters_zero(dev)
        for lane in range(lanes):
            for name in ref_bufs[lane]:
                # equal values and NaN positions (the chain's ReLU stores +0 where conv_gemm's stores -0)
                gb, rb = got_bufs[lane][name], ref_bufs[lane][name]
                assert torch.equal(gb.isnan(), rb.isnan()) and torch.equal(gb.nan_to_num(7.0), rb.nan_to_num(7.0)), (
                    rep, lane, name, (gb.float() - rb.float()).abs().nan_to_num(0).max().item())
    for lane in range(lanes):
        for (a, wt, out, kw), (name, _, _) in zip(logs[lane], layers):
            ref, P, Q = _call_ref(a, wt, out, kw)
            got = out.double()
            assert not bool(torch.isnan(got).any()), name
            _bound_check(2, got, ref, P, Q, "f32" if name == "head" else "f16", "chain depth %d lane %d %s" % (depth, lane, name))


# ------------------------------------------------------------------------------------------------ host-side rejections
def _recorded_desc(ops, call):
    """the descriptor ops.conv_gemm builds for `call` (recorded, not launched)"""
    saved = ops._CHAIN_MODE[0], ops._CHAIN_REC[0]
    ops._CHAIN_MODE[0], ops._CHAIN_REC[0] = "record", []
    try:
        call()
        (d,) = ops._CHAIN_REC[0]
    finally:
        ops._CHAIN_MODE[0], ops._CHAIN_REC[0] = saved
    return d


@pytest.mark.parametrize("what", ["split16_channels", "strict_block_n_96", "f16_out_block_n_32", "group_width_layout",
                                  "b_lo_tap_off_batched", "depth2_chain_tiles"])
def test_descriptor_rejections(cuda_dev, what):
    from mega_core import _lib
    from mega_core._lib import MegaError, check, lib, stream_ptr
    from mega_core.b200 import ops
    dev = cuda_dev
    z32 = lambda *s: torch.zeros(*s, device=dev)
    z16 = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float16)
    raw = lambda d: check(lib.mega_conv_gemm(ctypes.byref(d), stream_ptr()), "mega_conv_gemm")
    if what == "split16_channels":
        a, wt = ops.pack_split16(z32(1, 8, 16, 64)), ops.pack_weights_split16(z32(1, 64, 64))
        msg, fn = "split-fp16 operands need channel counts / offsets in multiples of 32", \
            lambda: ops.conv_gemm(a, wt, z32(1, 8, 16, 64), k=48, block_n=64, stream_k=0)
    elif what == "strict_block_n_96":
        a, wt, out = z32(1, 8, 16, 64), z32(1, 96, 64), z32(1, 8, 16, 96)
        with ops.precision("fp32x3"):
            d = _recorded_desc(ops, lambda: ops.conv_gemm(a, wt, out, block_n=128, stream_k=0))
        d.block_n = 96
        msg, fn = "3xtf32 / 3xfp16 support block_n 64 / 128", lambda: raw(d)
    elif what == "f16_out_block_n_32":
        a, wt, out = z16(1, 8, 16, 64), z16(1, 32, 64), z16(1, 8, 16, 32)
        msg, fn = "fp16 output needs fp16 operands and block_n % 64 == 0", \
            lambda: ops.conv_gemm(a, wt, out, block_n=32, stream_k=0)
    elif what == "group_width_layout":
        a, wt, out = z16(1, 8, 16, 64), z16(1, 64, 64), z16(1, 8, 16, 64)
        d = _recorded_desc(ops, lambda: ops.conv_gemm(a, wt, out, block_n=64, stream_k=0))
        d.group_width = 16
        msg, fn = "group_width needs the 64-channel batched layout", lambda: raw(d)
    elif what == "b_lo_tap_off_batched":
        a, wt, out = z32(1, 8, 16, 128), z32(1, 64, 128), z32(1, 8, 16, 128)
        with ops.precision("fp32x3"):
            d = _recorded_desc(ops, lambda: ops.conv_gemm(a, wt, out, block_n=64, cout=64, k=64, batch=2, a_c_off=64,
                                                          b_k_off=64, out_c_off=64, stream_k=0))
        d.b_lo_tap_off = 1
        msg, fn = "b_lo_tap_off (1) needs precision 1, batch 1", lambda: raw(d)
    else:
        a, wt, out = z16(1, 8, 16, 64), z16(1, 64, 64), z16(1, 8, 16, 64)
        d = _recorded_desc(ops, lambda: ops.conv_gemm(a, wt, out, block_n=64, stream_k=0, tile=(8, 16)))
        d.batch = 33000          # 33000 tiles: within the single-launch counters, over a depth-2 chain's half
        msg, fn = "tiles exceed the 32768 counters of a depth-2 chain", lambda: ops.ConvChain([d], dev, depth=2)
    with pytest.raises(MegaError, match=re.escape(msg)):
        fn()
    torch.cuda.synchronize()
    assert _lib.lib.mega_device_ok() == 1


# ------------------------------------------------------------------------------------------------ coverage gate
def test_zz_every_instantiation_ran_both_schedules(cuda_dev):
    """runs last in this file: the 42 instantiations x stream-K {0, 1}, each launched by a case that passed. It reads the
    session-wide record of the sweep, so it fails when the file runs only in part (-k, a single case)."""
    want = {v + (sk,) for v in VARIANTS for sk in (0, 1)}
    assert len(VARIANTS) == 42 and len(want) == 84
    missing = sorted(want - PASSED)
    report = {"measured_err_over_P": {MODES[m]: r for m, r in sorted(MEASURED.items())},
              "alpha": {MODES[m]: a for m, a in ALPHA.items()}, "launched": len(want & PASSED), "missing": missing}
    path = os.environ.get("CONV_GEMM_CONFORMANCE_REPORT")
    if path:
        with open(path, "w") as fh:
            json.dump(report, fh, indent=1)
    print("conv_gemm conformance:", json.dumps(report))
    assert not missing, "instantiations without a passing case: %s" % missing
