"""CPU half of the ROIAlign forward conformance suite: the fp64 reference and interval of
test_roi_align_conformance_gpu.py against the C oracle (mega_oracle.roi_align) and the host entry behind
`_C.roi_align_forward`, an exact-order fp32 restatement of the forward that both must equal bit for bit, mutations of
that restatement the interval must reject, and the restated dispatch rule against csrc/roi_align.cu and ops.py."""
import os
import re

import numpy as np
import pytest
import torch

import roi_align_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c["id"]: c for c in R.make_cases()}
# CPU-sized cases of the table (first CH channels): samples on -1 / H / integer cells, one-row / one-column maps with
# footprints of 191-193 cells, several images in a shuffled order, adaptive grids of 8 / 9 / 16 / 17, odd bins
FIXTURES = ["map_11x13_sr1", "map_12x11_sr2", "map_1x200", "map_200x1", "ch4", "ch8", "bins3x5", "sr9_40x50", "k1",
            "map_1x1"]
CH = 4


def fp32_forward(feat, boxes, batch, scale, ph, pw, sr, mutate=None):
    """ROIAlign forward in fp32 with the kernels' association order, one rounding per operation, vectorised over bins
    and channels: [K, ph * pw, C] bin-major rows. feat: [N, H, W, C]. `mutate` names a deliberate bug."""
    f = feat.numpy().astype(np.float32)
    n, h, w, c = f.shape
    b = boxes.numpy().astype(np.float32)
    k = b.shape[0]
    s = np.float32(scale)
    one = np.float32(1)
    out = np.zeros((k, ph, pw, c), np.float32)
    for i in range(k):
        sw, sh, ew, eh = b[i, 0] * s, b[i, 1] * s, b[i, 2] * s, b[i, 3] * s
        if mutate == "no_max_1":
            rw, rh = ew - sw, eh - sh
        else:
            rw, rh = max(ew - sw, one), max(eh - sh, one)
        bh, bw = rh / np.float32(ph), rw / np.float32(pw)
        rnd = np.floor if mutate == "grid_floor" else np.ceil
        gh = sr if sr > 0 else int(rnd(rh / np.float32(ph)))
        gw = sr if sr > 0 else int(rnd(rw / np.float32(pw)))
        off = np.float32(0) if mutate == "sample_at_i" else np.float32(0.5)

        def axis(start, bn, g, bins, size, it):
            cc = (start + np.arange(bins, dtype=np.float32) * bn) + ((np.float32(it) + off) * bn) / np.float32(g)
            empty = ((cc <= -one) if mutate == "empty_le_minus_1" else (cc < -one)) | \
                    ((cc >= np.float32(size)) if mutate == "empty_ge_size" else (cc > np.float32(size)))
            lo, hi, wlo, whi = R.axis_sample(cc, size)
            return empty, lo, hi, wlo, whi

        img = f[0 if mutate == "batch_ignored" else int(batch[i])]
        acc = np.zeros((ph, pw, c), np.float32)
        for iy in range(gh):
            ey, ylo, yhi, hy, ly = axis(sh, bh, gh, ph, h, iy)
            for ix in range(gw):
                ex, xlo, xhi, hx, lx = axis(sw, bw, gw, pw, w, ix)
                w1, w2 = (hy[:, None] * hx[None, :])[..., None], (hy[:, None] * lx[None, :])[..., None]
                w3, w4 = (ly[:, None] * hx[None, :])[..., None], (ly[:, None] * lx[None, :])[..., None]
                v1, v2 = img[ylo][:, xlo], img[ylo][:, xhi]
                v3, v4 = img[yhi][:, xlo], img[yhi][:, xhi]
                val = ((w1 * v1 + w2 * v2) + w3 * v3) + w4 * v4
                val[ey[:, None] | ex[None, :]] = 0
                acc = acc + val
        count = np.float32(gh * gw + (1 if mutate == "count_off_by_one" else 0))
        with np.errstate(divide="ignore", invalid="ignore"):
            out[i] = acc / count
    if mutate == "channel_major":
        out = np.ascontiguousarray(out.transpose(0, 3, 1, 2))
    return torch.from_numpy(out.reshape(k, ph * pw, c))


def _nchw_rows(x):
    """[K, C, ph, pw] -> [K, ph * pw, C]"""
    return x.permute(0, 2, 3, 1).reshape(x.shape[0], -1, x.shape[1])


def _inputs(cid):
    c = CASES[cid]
    feat, boxes, batch = R.build_inputs(c)
    feat = feat[..., :CH].contiguous()
    geo = R.case_geometry(c, boxes)
    ay, ax = R.weight_matrices(geo)
    ref, s = R.reference(feat, batch, geo, ay, ax)
    m = R.m_tensor(R.chain_length(geo, ay, ax, R.NCHW), geo, "cpu")
    return c, feat, boxes, batch, ref, s, m


@pytest.fixture(scope="module")
def fixtures():
    return {cid: _inputs(cid) for cid in FIXTURES}


@pytest.mark.parametrize("cid", FIXTURES)
def test_oracle_host_entry_and_restatement_agree_and_lie_inside(fixtures, cid):
    import mega_oracle as mo
    from mega_core import _C
    c, feat, boxes, batch, ref, s, m = fixtures[cid]
    rois = torch.cat([batch.float().view(-1, 1), boxes], 1)
    nchw = feat.permute(0, 3, 1, 2).contiguous()
    oracle = _nchw_rows(mo.roi_align(nchw, rois, R.SCALE, c["ph"], c["pw"], c["sr"]))
    host = _nchw_rows(_C.roi_align_forward(nchw, rois, R.SCALE, c["ph"], c["pw"], c["sr"]))
    mine = fp32_forward(feat, boxes, batch, R.SCALE, c["ph"], c["pw"], c["sr"])
    assert torch.equal(host.view(torch.int32), oracle.view(torch.int32)), cid
    assert torch.equal(mine.view(torch.int32), oracle.view(torch.int32)), cid
    ok = R.inside(oracle, ref, s, m, "f32")
    assert bool(ok.all()), "%s: %d elements outside the interval" % (cid, int((~ok).sum()))
    for fmt in ("f16", "split"):     # the output roundings: the fp32 result rounded once lies inside the wider intervals
        if fmt == "f16":
            r = oracle.half().float()
        else:
            hi = oracle.half()
            r = hi.float() + (oracle - hi.float()).half().float()
        assert bool(R.inside(r, ref, s, m, fmt).all()), (cid, fmt)


def test_fixtures_reach_the_edges(fixtures):
    """the CPU fixtures hold samples exactly on -1, on H, on integer cells, zero rows (rois outside the map), several
    images, footprints of 191 / 192 / 193 cells and adaptive grids on both sides of 8 and 16"""
    seen = dict(minus1=False, at_h=False, zero_row=False, multi=False)
    foot, grids = set(), set()
    for c, feat, boxes, batch, ref, s, m in fixtures.values():
        geo = R.case_geometry(c, boxes)
        for i in range(geo.k):
            y = geo.coords(i, "h")
            seen["minus1"] |= bool((y == -1).any())
            seen["at_h"] |= bool((y == c["h"]).any())
        seen["zero_row"] |= bool((s.flatten(1).amax(1) == 0).any())
        seen["multi"] |= len(set(batch.tolist())) > 1
        foot |= set(geo.footprint().tolist())
        if c["sr"] == 0:
            grids |= set(geo.grid_h.tolist()) | set(geo.grid_w.tolist())
    assert all(seen.values()), seen
    assert {191, 192, 193} <= foot
    assert {8, 9, 16, 17} <= grids


def test_interval_is_not_vacuous(fixtures):
    """the half-width is a small fraction of S: median <= 2^-16 S over elements with S > 0"""
    for c, feat, boxes, batch, ref, s, m in fixtures.values():
        live = s > 0
        if bool(live.any()):
            rel = (R.half_width(ref, s, m, "f32") / s.clamp_min(1e-300))[live]
            assert rel.median().item() <= 2.0 ** -16, (c["id"], rel.median().item())


MUTATIONS = ["sample_at_i", "empty_le_minus_1", "empty_ge_size", "no_max_1", "grid_floor", "count_off_by_one",
             "batch_ignored", "channel_major"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_are_rejected(fixtures, mutation):
    rejected = []
    for c, feat, boxes, batch, ref, s, m in fixtures.values():
        if mutation == "grid_floor" and c["sr"] > 0:
            continue
        got = fp32_forward(feat, boxes, batch, R.SCALE, c["ph"], c["pw"], c["sr"], mutate=mutation)
        if not bool(R.inside(got, ref, s, m, "f32").all()):
            rejected.append(c["id"])
    assert rejected, "%s passes the bound on every fixture" % mutation


def test_reference_weights_are_the_per_sample_weights():
    """Ay / Ax summed over a bin-row / bin-column are the number of samples inside the map (every live sample puts a
    total weight of 1 on its axis)"""
    c = CASES["map_11x13_sr1"]
    feat, boxes, batch = R.build_inputs(c)
    geo = R.case_geometry(c, boxes)
    ay, ax = R.weight_matrices(geo)
    for i in range(geo.k):
        for mat, axis, size in ((ay, "h", geo.h), (ax, "w", geo.w)):
            cc = geo.coords(i, axis)
            live = ((cc >= -1) & (cc <= size)).sum(1)
            assert np.allclose(mat[i].sum(1), live, rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------------ dispatch vs source
def _src():
    return open(os.path.join(ROOT, "mega.pytorch_b200", "csrc", "roi_align.cu")).read()


def test_constants_match_the_source():
    src = _src()
    for name, want in (("kRoiSliceBytes", R.K_ROI_SLICE_BYTES), ("kRoiMaxCells", R.K_ROI_MAX_CELLS),
                       ("kRoiMaxGrid", R.K_ROI_MAX_GRID), ("kSepMaxDim", R.K_SEP_MAX_DIM),
                       ("kSepMaxGrid", R.K_SEP_MAX_GRID)):
        got = re.findall(r"constexpr int %s = (\d+);" % name, src)
        assert got == [str(want)], (name, got)


def test_dispatch_restatement_matches_the_source():
    """the kernels roi_align.cu launches are the eight of the table, behind the branch conditions dispatch() restates"""
    src = re.sub(r"\s+", " ", _src())
    launched = set(re.findall(r"(roi_align_\w+kernel(?:<\w+>)?)<<<", src))
    assert launched == {R.NCHW, "roi_align_nhwc_cached_kernel<T>", "roi_align_nhwc_kernel<T>", R.SEP16, R.FAST,
                        R.SEPSPLIT}, launched
    assert set(re.findall(r"roi_align_nhwc_launch<(\w+)>\(", src)) == {"float", "__half"}
    for cond in (
            # roi_align_nhwc_launch<T>: channel check, slice kernel when C is a multiple of the 256-byte slice
            "MEGA_ARG_CHECK((channels % V) == 0,",
            "constexpr int kSlice = kRoiSliceBytes / static_cast<int>(sizeof(T)); MEGA_ARG_CHECK(pooled_h > 0",
            "if ((channels % kSlice) == 0) {",
            # the fp16 entry
            "const bool fast = (channels % 128) == 0 && pooled_h <= 7 && pooled_w <= 7 && "
            "(reinterpret_cast<uintptr_t>(input) & 15) == 0 && (reinterpret_cast<uintptr_t>(output) & 15) == 0 && "
            "(out_roi_stride % 8) == 0 && (in_img_stride % 8) == 0;",
            "if (fast && height <= kSepMaxDim && width <= kSepMaxDim && g_roi_separable) {",
            "return e != nullptr ? e[0] != '0' : true;",
            # the split-fp16 entry
            "MEGA_ARG_CHECK((channels % 128) == 0 && pooled_h <= 7 && pooled_w <= 7 && pooled_h > 0 && pooled_w > 0 && "
            "height <= kSepMaxDim && width <= kSepMaxDim",
            # per-roi sub-paths
            "const bool tabled = g.grid_h <= kRoiMaxGrid && g.grid_w <= kRoiMaxGrid;",
            "const bool tabled = g.grid_h <= kSepMaxGrid && g.grid_w <= kSepMaxGrid;",
            "r0 = min(max(r0, 0), height - 1); r1 = min(max(r1, 0), height - 1);",
            "int r0 = static_cast<int>(floorf(fmaxf(g.start_h, 0.f))), r1 = static_cast<int>(floorf(fmaxf(end_h, 0.f))) + 1;",
            "const float end_h = __fadd_rn(g.start_h, __fmul_rn(g.bin_h, static_cast<float>(ph)));"):
        assert cond in src, cond
    assert src.count("const bool cached = (rh * rw <= kRoiMaxCells);") == 2        # the cached kernel and the fast kernel
    assert 'getenv("MEGA_B200_ROI_SEPARABLE")' in src


def test_ops_split16_rule_matches_the_source():
    src = open(os.path.join(ROOT, "mega.pytorch_b200", "mega_core", "b200", "ops.py")).read()
    body = src[src.index("def roi_align_nhwc("):src.index("def stem_im2col(")]
    assert "if h <= 64 and w <= 64 and c % 128 == 0 and ph <= 7 and pw <= 7:" in body
    assert "fn = lib.mega_roi_align_forward_nhwc_split16" in body
    assert "plain = unpack_split16(" in body and "return pack_split16(out)" in body


def test_case_table_covers_every_path():
    """the table's restated dispatch reaches every (kernel, sub-path) pair (with MEGA_B200_ROI_SEPARABLE=0 for the
    f16 fast kernel's tabled / inline rois of maps <= 64 x 64 as well)"""
    paths = set()
    for c in CASES.values():
        _, boxes, _ = R.build_inputs(c)
        geo = R.case_geometry(c, boxes)
        for fmt in c["formats"]:
            kern, fb = R.dispatch(fmt, c["c"], c["ph"], c["pw"], c["h"], c["w"])
            paths |= R.roi_paths(kern, geo)
            if fb:
                paths.add((R.FALLBACK, "-"))
    assert paths == set(R.ALL_PATHS), set(R.ALL_PATHS) - paths
    chans = {(f, c["c"]) for c in CASES.values() for f in c["formats"]}
    for want in [("f32", x) for x in (4, 60, 64, 1024)] + [("f16", x) for x in (8, 120, 128, 2048)]:
        assert want in chans, want
    assert {(1, 1), (7, 7), (14, 14), (3, 5), (8, 7)} <= {(c["ph"], c["pw"]) for c in CASES.values()}
    assert {0, 1, 2, 8, 9, 16, 17} <= {c["sr"] for c in CASES.values()}
    assert {0, 1} <= {c["k"] for c in CASES.values()} and max(c["k"] for c in CASES.values()) > 1000
    maps = {(c["h"], c["w"]) for c in CASES.values()}
    assert {(1, 1), (64, 64), (65, 64), (64, 65), (38, 63), (75, 125)} <= maps
    assert any(h == 1 for h, _ in maps) and any(w == 1 for _, w in maps)
    assert {"randn", "hdr", "cancel"} == {c["values"] for c in CASES.values()}
    assert {"spans", "perm"} <= {c["batch"] for c in CASES.values()}
