"""Conformance of every ROIAlign forward kernel (csrc/roi_align.cu) against the fp64 reference of roi_align_ref.py,
element by element: each output lies in the interval of roi_align_ref.half_width.

A (roi_align_ref.A) is >= 2x the largest value the whole file measures, where "measured" is the smallest A every output
of a kernel still passes with (0: the A-free part of the interval, (u S + u |ref| + output rounding), already holds it).
Measured per kernel on an NVIDIA H100 80GB HBM3 (SXM, 700 W power limit), with A = 1 chosen (>= 2 x 0.31):
    kernel                                  measured A   max |got - ref| / half-width
    roi_align_nchw_kernel                   0.31         0.42
    roi_align_nhwc_kernel<float>            0.15         0.34
    roi_align_nhwc_cached_kernel<float>     0.31         0.42
    roi_align_nhwc_kernel<__half>           0            1.00   (the fp16 output rounding: half an ulp)
    roi_align_nhwc_cached_kernel<__half>    0            1.00
    roi_align_nhwc_f16_fast_kernel          0.003        1.00
    roi_align_nhwc_sep_kernel<false>        0.012        1.00
    roi_align_nhwc_sep_kernel<true>         0.095        1.00   (the split-fp16 output rounding)
    ops split-fp16 fallback                 0.24         1.00

Besides the interval, every case checks: the exact-order fp32 kernels equal the C oracle bit for bit (on a subset of
channels) and each other (on all of them); the per-sample fp16 kernels equal fp16(oracle on the same fp16 map); the
profiler sees exactly the kernel the restated dispatch rule predicts; the output is written into a view of a larger
buffer filled with a NaN sentinel (guard rows before and after, padding past ph * pw * C in each row) and the sentinel
survives; the inputs are bit-unchanged. The profiler watches every call of the table in a child process of its own
(fixture `observed`); the cases MEGA_B200_ROI_SEPARABLE=0 changes (read once per process) run in another. The last test asserts that every (kernel, sub-path) pair ran in a case that passed.
"""
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

import roi_align_ref as R

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
SENT32 = 0x7FA5A5A5         # a NaN payload no kernel produces
SENT16 = 0x7D5A
GUARD = 64                  # guard elements before and after (keeps split-fp16 views 128-byte aligned)
PAD = 32                    # padding elements past ph * pw * C in each output row
ORACLE_CH = 12              # channels of each case the C oracle recomputes
CASES = R.make_cases()
# cases whose fp16 call MEGA_B200_ROI_SEPARABLE=0 moves from the separable kernel to the fast kernel
NOSEP = ["map_64x64", "map_11x13_sr1", "map_12x11_sr2", "sr9_40x50", "sr17_40x50", "huge_20x30", "bins3x5", "map_1x1",
         "k0"]
PASSED = set()              # (kernel, sub-path) of calls in cases that passed
MEASURED = {}               # kernel -> largest A a passing output needed
DEV = {}                    # kernel -> largest |got - ref| / half-width
NAMES = {}                  # "case/format" -> roi_align kernels the profiler saw the call launch


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _kernel_names(prof):
    names = set()
    for e in prof.events():
        m = re.search(r"mega::(roi_align_\w+kernel(?:<[\w ]+>)?)\(", e.name)
        if m:
            names.add(m.group(1))
    return names


def _profiled(fn, k):
    """runs fn under the profiler; the roi_align kernel names it launched. CPU and CUDA activities together (a
    CUDA-only session took ~7x longer to set up and lost kernel records more often on an H100 with torch 2.11). A
    session now and then delivers no kernel record, and such losses come in bursts: one that saw none is retried after a
    growing pause."""
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for attempt in range(8):
        if attempt:
            time.sleep(0.05 * 2 ** attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = _kernel_names(prof)
        if names or k == 0:
            break
    return names


def _out_buffer(k, row, dtype, dev, pad):
    """(buffer, [k, row] view with rows of row + pad elements, GUARD sentinel elements before and after)"""
    rs = row + pad
    buf = torch.empty(k * rs + 2 * GUARD, dtype=dtype, device=dev)
    _bits(buf).fill_(SENT16 if dtype == torch.float16 else SENT32)
    return buf, buf[GUARD:GUARD + k * rs].view(k, rs)[:, :row]


def _sentinel_ok(buf, k, row, pad):
    b = _bits(buf)
    sent = SENT16 if buf.dtype == torch.float16 else SENT32
    ok = bool((b[:GUARD] == sent).all()) and bool((b[-GUARD:] == sent).all())
    if pad and k:
        ok &= bool((b[GUARD:-GUARD].view(k, row + pad)[:, row:] == sent).all())
    return ok


def _oracle_rows(feat, boxes, batch, c, chans):
    """C oracle on channels `chans` of an fp32 map: [K, ph * pw, len(chans)]"""
    import mega_oracle as mo
    rois = torch.cat([batch.float().view(-1, 1), boxes], 1)
    x = mo.roi_align(feat[..., chans].permute(0, 3, 1, 2).contiguous().cpu(), rois, R.SCALE, c["ph"], c["pw"], c["sr"])
    return x.permute(0, 2, 3, 1).reshape(x.shape[0], c["ph"] * c["pw"], len(chans))


def _record(kernel, got, ref, s, m, fmt):
    MEASURED[kernel] = max(MEASURED.get(kernel, 0.0), R.needed_a(got, ref, s, m, fmt))
    if got.numel():
        d = ((got.double() - ref).abs() / R.half_width(ref, s, m, fmt).clamp_min(1e-300)).max().item()
        DEV[kernel] = max(DEV.get(kernel, 0.0), d)


def run_case(c, dev, separable=True, formats=None, seen=None):
    """every check of one case over the formats it admits; records the (kernel, sub-path) pairs that passed. The
    kernel each call launched is what the profiler saw here (seen=None), or seen["case/format"] from a child process."""
    from mega_core.b200 import ops
    k, ph, pw, ch = c["k"], c["ph"], c["pw"], c["c"]
    row = ph * pw * ch
    feat, boxes, batch = R.build_inputs(c)
    geo = R.case_geometry(c, boxes)
    ay, ax = R.weight_matrices(geo)
    fd, bd, btd = feat.to(dev), boxes.to(dev), batch.to(dev)
    formats = [f for f in c["formats"] if formats is None or f in formats]
    packed = None
    if "split" in formats:     # the fp32 formats read the values a split-fp16 map holds
        packed = ops.pack_split16(fd.clone())
        fd = ops.unpack_split16(packed, torch.empty_like(fd))
    f16 = fd.half() if "f16" in formats else None
    refs = {}
    chans = sorted(set(np.random.default_rng(c["seed"]).choice(ch, min(ch, ORACLE_CH), replace=False).tolist())
                   | {0, ch - 1})
    oracle32 = _oracle_rows(fd, boxes, batch, c, chans)
    paths, exact32 = set(), []
    for fmt in formats:
        kernel, fallback = R.dispatch(fmt, ch, ph, pw, c["h"], c["w"], separable=separable)
        src = f16 if fmt == "f16" else fd
        key = "f16" if fmt == "f16" else "f32"
        if key not in refs:
            refs[key] = R.reference(src, batch, geo, ay, ax)
        ref, s = refs[key]
        m = R.m_tensor(R.chain_length(geo, ay, ax, kernel), geo, dev)
        keep = [(t, t.clone()) for t in (fd, f16, packed, bd, btd) if t is not None]
        if fmt == "nchw":
            inp = fd.permute(0, 3, 1, 2).contiguous()
            rois = torch.cat([btd.float().view(-1, 1), bd], 1)
            buf, out = _out_buffer(1, k * row, torch.float32, dev, 0)
            out = out.view(k, ch, ph, pw)
            fn = lambda: ops.roi_align_nchw(inp, rois, R.SCALE, ph, pw, c["sr"], out=out)
            pad = 0
            keep.append((inp, inp.clone()))
        else:
            pad = 0 if fallback else PAD
            dtype = torch.float16 if fmt == "f16" else torch.float32
            buf, out = _out_buffer(k, row, dtype, dev, pad)
            x = packed if fmt == "split" else src
            fn = lambda: ops.roi_align_nhwc(x, bd, btd, R.SCALE, ph, pw, c["sr"], out)
        if seen is None:
            names = _profiled(fn, k)
            NAMES["%s/%s" % (c["id"], fmt)] = sorted(names)
        else:
            fn()
            names = set(seen.get("%s/%s" % (c["id"], fmt), ["<no record>"]))
        torch.cuda.synchronize()
        if fmt == "nchw":
            got = out.permute(0, 2, 3, 1).reshape(k, ph * pw, ch)
        elif fmt == "split":
            assert ops.is_split16(out), c["id"]
            got = ops.split16_decode(out).view(k, ph * pw, ch)
        else:
            got = out.view(k, ph * pw, ch)
        want = {kernel} if k else set()
        assert names == want, "%s %s: launched %s, the dispatch rule says %s" % (c["id"], fmt, names, want)
        assert _sentinel_ok(buf, 1 if fmt == "nchw" else k, k * row if fmt == "nchw" else row, pad), \
            "%s %s: wrote outside its rows" % (c["id"], fmt)
        for t, before in keep:
            assert torch.equal(_bits(t), _bits(before)), "%s %s: an input changed" % (c["id"], fmt)
        ok = R.inside(got, ref, s, m, fmt)
        if not bool(ok.all()):
            i = tuple((~ok).nonzero()[0].tolist())
            hw = R.half_width(ref, s, m, fmt)
            raise AssertionError("%s %s (%s): %d of %d elements outside the interval, first (roi, bin, channel) %s: got "
                                 "%r fp64 %r half-width %r S %r box %s" % (
                                     c["id"], fmt, kernel, int((~ok).sum()), ok.numel(), i, got[i].item(),
                                     ref[i].item(), hw[i].item(), s[i].item(), boxes[i[0]].tolist()))
        _record(kernel if not fallback else R.FALLBACK, got, ref, s, m, fmt)
        if fmt in ("nchw", "f32"):
            assert torch.equal(_bits(got[..., chans].cpu()), _bits(oracle32)), "%s %s: != C oracle" % (c["id"], fmt)
            exact32.append(got)
        if fmt == "f16" and kernel in R.EXACT_ORDER:
            want16 = _oracle_rows(f16.float(), boxes, batch, c, chans).half()
            assert torch.equal(_bits(got[..., chans].cpu()), _bits(want16)), "%s f16: != fp16(C oracle)" % c["id"]
        paths |= R.roi_paths(kernel, geo)
        if fallback and k:
            paths.add((R.FALLBACK, "-"))
    if len(exact32) == 2:
        assert torch.equal(_bits(exact32[0]), _bits(exact32[1])), "%s: nchw and nhwc fp32 differ" % c["id"]
    PASSED.update(paths)


def _run_child(func, out, **env):
    """runs test_roi_align_conformance_gpu.<func>(out) in a fresh Python process; returns its JSON report"""
    env = dict(os.environ, **env,
               PYTHONPATH=os.pathsep.join([TESTS, ROOT, os.path.join(ROOT, "mega.pytorch_b200"), os.path.join(ROOT, "oracle")]
                                          + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    code = "import sys, test_roi_align_conformance_gpu as t; t.%s(sys.argv[1])" % func
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, str(out)]
    res = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stderr[-4000:]
    return json.loads(out.read_text())


def observe_child(out_path):
    """runs every case under the profiler in this (child) process and writes the kernels each call launched"""
    assert os.environ.get("MEGA_B200_ROI_SEPARABLE", "1") != "0"
    dev = torch.device("cuda:0")
    failed = {}
    for c in CASES:
        try:
            run_case(c, dev)
        except AssertionError as e:
            failed[c["id"]] = str(e)[:2000]
    with open(out_path, "w") as fh:
        json.dump(dict(names=NAMES, failed=failed), fh)


@pytest.fixture(scope="module")
def observed(cuda_dev, tmp_path_factory):
    """the kernel each call of the table launches, as torch.profiler sees it in a process of its own: in a long pytest
    process (after other suites have profiled, captured CUDA graphs, ...) the profiler can stop delivering kernel
    records for seconds at a time, which says nothing about the dispatch"""
    return _run_child("observe_child", tmp_path_factory.mktemp("roi_observe") / "names.json",
                      MEGA_B200_ROI_SEPARABLE="1")


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_roi_align_matches_fp64(cuda_dev, observed, case):
    try:
        run_case(case, cuda_dev, seen=observed["names"])
    except AssertionError as e:
        raise AssertionError("%s (under the profiler: %s)" % (e, observed["failed"].get(case["id"], "passed"))) from None


def nosep_child(out_path):
    """runs the NOSEP cases' fp16 and split-fp16 calls in this (child) process and writes what passed as JSON"""
    from mega_core import _lib
    assert os.environ.get("MEGA_B200_ROI_SEPARABLE") == "0"
    dev = torch.device("cuda:0")
    assert _lib.lib.mega_device_ok() == 1
    failed = {}
    for c in CASES:
        if c["id"] in NOSEP:
            try:
                run_case(c, dev, separable=False, formats=("f16", "split"))
            except AssertionError as e:
                failed[c["id"]] = str(e)[:2000]
    with open(out_path, "w") as fh:
        json.dump(dict(passed=sorted(PASSED), failed=failed, measured=MEASURED, dev=DEV), fh)


def test_separable_switch_off_in_child_process(cuda_dev, tmp_path):
    rep = _run_child("nosep_child", tmp_path / "nosep.json", MEGA_B200_ROI_SEPARABLE="0")
    assert not rep["failed"], rep["failed"]
    got = {tuple(p) for p in rep["passed"]}
    assert {(R.FAST, s) for s in ("cached", "global", "tabled", "inline")} <= got, got
    assert (R.SEPSPLIT, "tabled") in got and not any(kn == R.SEP16 for kn, _ in got), got
    for kn, v in rep["measured"].items():
        MEASURED[kn] = max(MEASURED.get(kn, 0.0), v)
    for kn, v in rep["dev"].items():
        DEV[kn] = max(DEV.get(kn, 0.0), v)
    PASSED.update(got)


# ------------------------------------------------------------------------------------------------ host-side rejections
ERRORS = ["f32_c_not_4", "f16_c_not_8", "f32_map_misaligned", "f16_map_misaligned", "f32_out_misaligned",
          "f16_out_misaligned", "split_entry_c64", "split_entry_map65", "split_entry_bins8", "nchw_bins0", "f32_bins0",
          "f16_bins0", "split_bins0"]


@pytest.mark.parametrize("what", ERRORS)
def test_argument_errors_before_launch(cuda_dev, what):
    from mega_core import _lib
    from mega_core._lib import MegaError, check, lib, ptr, stream_ptr
    from mega_core.b200 import ops
    dev = cuda_dev
    fmt = what.split("_")[0]
    c = {"f32_c_not_4": 6, "f16_c_not_8": 12}.get(what, 64 if what == "split_entry_c64" else 128)
    h = 65 if what == "split_entry_map65" else 9
    ph = 0 if what.endswith("bins0") else (8 if what == "split_entry_bins8" else 7)
    k = 5
    dtype = torch.float16 if fmt == "f16" else torch.float32
    fbuf = torch.randn(2 * h * 9 * c + 8, device=dev).to(dtype)
    off = 1 if what.endswith("map_misaligned") else 0
    feat = fbuf[off:off + 2 * h * 9 * c].view(2, h, 9, c)
    boxes = torch.tensor([[0.0, 0.0, 64.0, 64.0]] * k, device=dev)
    batch = torch.zeros(k, dtype=torch.int32, device=dev)
    row = max(ph * 7 * c, 1)
    obuf = torch.empty(k * row + 16, dtype=dtype, device=dev)
    _bits(obuf).fill_(SENT16 if dtype == torch.float16 else SENT32)
    ooff = 1 if what.endswith("out_misaligned") else 0
    out = obuf[ooff:ooff + k * row].view(k, row)
    before = _bits(obuf).clone()
    if fmt == "nchw":
        call = lambda: ops.roi_align_nchw(feat.permute(0, 3, 1, 2).contiguous(), torch.cat([batch.float().view(-1, 1), boxes], 1),
                                          R.SCALE, ph, 7, 0, out=out.view(-1))
    elif fmt == "split" and what != "split_bins0":
        call = lambda: check(lib.mega_roi_align_forward_nhwc_split16(
            ptr(feat), c, h, 9, feat.stride(0), ptr(boxes), 4, 0, ptr(batch), k, R.SCALE, ph, 7, 0, ptr(out), row,
            stream_ptr()), "mega_roi_align_forward_nhwc_split16")
    else:
        x = ops.pack_split16(feat.clone()) if fmt == "split" else feat
        call = lambda: ops.roi_align_nhwc(x, boxes, batch, R.SCALE, ph, 7, 0, out)
    with pytest.raises(MegaError):
        call()
    torch.cuda.synchronize()
    assert torch.equal(_bits(obuf), before)
    assert _lib.lib.mega_device_ok() == 1


LAYOUTS = ["feat_channel_slice", "boxes_f16", "boxes_column_stride", "batch_int64", "batch_strided", "batch_short",
           "out_inner_stride", "out_rows_short", "out_row_short", "split_fallback_strided_out"]


@pytest.mark.parametrize("what", LAYOUTS)
def test_ops_rejects_layouts_the_kernels_cannot_read(cuda_dev, what):
    from mega_core._lib import MegaError
    from mega_core.b200 import ops
    dev = cuda_dev
    k, c, h, w = 6, 128, 9, 11
    feat = torch.randn(1, h, w, c, device=dev)
    boxes = torch.tensor([[0.0, 0.0, 64.0, 64.0]] * k, device=dev)
    batch = torch.zeros(k, dtype=torch.int32, device=dev)
    out = torch.zeros(k, 49 * c, device=dev)
    if what == "feat_channel_slice":
        feat = torch.randn(1, h, w, 2 * c, device=dev)[..., :c]
    elif what == "boxes_f16":
        boxes = boxes.half()
    elif what == "boxes_column_stride":
        boxes = boxes.t().contiguous().t()
    elif what == "batch_int64":
        batch = batch.long()
    elif what == "batch_strided":
        batch = torch.zeros(2 * k, dtype=torch.int32, device=dev)[::2]
    elif what == "batch_short":
        batch = batch[:k - 1]
    elif what == "out_inner_stride":
        out = torch.zeros(49 * c, k, device=dev).t()
    elif what == "out_rows_short":
        out = out[:k - 1]
    elif what == "out_row_short":
        out = out[:, :49 * c - 8]
    else:
        feat = ops.pack_split16(torch.randn(1, 65, w, c, device=dev))
        out = torch.zeros(k, 49 * c + 32, device=dev)[:, :49 * c]
    before = out.clone()
    with pytest.raises(MegaError):
        ops.roi_align_nhwc(feat, boxes, batch, R.SCALE, 7, 7, 0, out)
    torch.cuda.synchronize()
    assert torch.equal(out, before)


# ------------------------------------------------------------------------------------------------ coverage gate
def test_zz_every_path_ran(cuda_dev):
    """runs last in this file: every (kernel, sub-path) pair, each taken by a roi of a case that passed. It reads the
    session-wide record, so it fails when the file runs in part."""
    missing = sorted(R.ALL_PATHS - PASSED)
    report = {"A": R.A, "measured_A": MEASURED, "max_dev_over_halfwidth": DEV, "paths": len(R.ALL_PATHS & PASSED),
              "of": len(R.ALL_PATHS), "missing": missing}
    path = os.environ.get("ROI_ALIGN_CONFORMANCE_REPORT")
    if path:
        with open(path, "w") as fh:
            json.dump(report, fh, indent=1)
    print("roi_align conformance:", json.dumps(report))
    assert not missing, "paths without a passing case: %s" % missing
