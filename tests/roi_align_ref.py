"""Shared pieces of the ROIAlign forward conformance suite (test_roi_align_conformance_cpu.py / _gpu.py).

- geometry / reference / interval: an fp64 restatement of ROIAlign forward (ROIAlign_cuda.cu:62-115, oracle_ops.c
  oracle_roi_align_fwd) and a per-element interval that bounds what each kernel of csrc/roi_align.cu may return;
- dispatch / roi_paths: which kernel a call reaches and which sub-path each roi takes inside it;
- the committed case table: the engines' pooling geometries, map and channel edges, bins, sampling ratios, and rois
  placed where the kernels can go wrong.

Geometry. Everything up to the bilinear weights is computed in fp32, one rounding per operation, in the kernels' order:
start = x1 * scale, roi = max(end - start, 1), bin = roi / bins, grid = sr > 0 ? sr : ceil(roi / bins), each sample
coordinate start + p * bin + ((i + .5) * bin) / grid, the empty rule c < -1 || c > size, the clamps to 0 and to
size - 1, l = c - lo and 1 - l. The floor inside the bilinear set-up is discontinuous: an fp64 sample position could pick
another cell than the kernel does, and no error bound would then hold. Only the blend, the sum and the division by
count run in fp64, in the separable form out = (1 / count) Ay F Ax^T with per-roi [ph, H] and [pw, W] weight matrices
(Ay[p, y] = the sum of the fp32 row weights that bin-row p's samples put on map row y; samples outside the map add 0).

Interval. With u = 2^-24 and S the same reference applied to |F| (all weights are >= 0, so S bounds every partial sum):
    |got - ref| <= (A m + 1) u S + u |ref| + output rounding
output rounding: 0 for fp32, 2^-11 |ref| + 2^-25 for fp16, 2^-23 |ref| + 2^-25 for split-fp16 (hi = fp16(v), lo =
fp16(v - hi); hi + lo decodes exactly). The extra u S covers the exact products wy * wx of the reference where the kernels
round them; u |ref| covers the final division. m is the longest chain of fp32 roundings feeding one output, n = gh * gw:
  * exact-order kernels (nchw, nhwc<T>, nhwc_cached<T>): the weight product, the product with the value, three blend
    additions, n accumulations: m = n + 6;
  * f16 fast kernel: the weight product, 4 n chained FMAs, fl(1 / count) and the multiply by it: m = 4 n + 3;
  * separable kernels: the per-cell weight sums (at most 2 gh resp. 2 gw terms), the row pass over the bin-row's
    footprint rows (ry FMAs), the column pass over its footprint columns (rx FMAs), fl(1 / count) and its multiply:
    m = 2 gh + 2 gw + ry + rx + 2.
A is calibrated in test_roi_align_conformance_gpu.py.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mega_oracle  # noqa: E402,F401

U = 2.0 ** -24
A = 1.0                                    # calibration: test_roi_align_conformance_gpu.py
SCALE = 1.0 / 16
F32 = np.float32
FORMATS = ("nchw", "f32", "f16", "split")

# constants of csrc/roi_align.cu (test_roi_align_conformance_cpu.py reads them back from the source)
K_ROI_SLICE_BYTES = 256
K_ROI_MAX_CELLS = 192
K_ROI_MAX_GRID = 8
K_SEP_MAX_DIM = 64
K_SEP_MAX_GRID = 16

# ------------------------------------------------------------------------------------------------ dispatch
NCHW = "roi_align_nchw_kernel"
NHWC32 = "roi_align_nhwc_kernel<float>"
CACHED32 = "roi_align_nhwc_cached_kernel<float>"
NHWC16 = "roi_align_nhwc_kernel<__half>"
CACHED16 = "roi_align_nhwc_cached_kernel<__half>"
FAST = "roi_align_nhwc_f16_fast_kernel"
SEP16 = "roi_align_nhwc_sep_kernel<false>"
SEPSPLIT = "roi_align_nhwc_sep_kernel<true>"
KERNELS = (NCHW, NHWC32, CACHED32, NHWC16, CACHED16, FAST, SEP16, SEPSPLIT)
FALLBACK = "ops split-fp16 fallback"
SUBPATHS = {NCHW: ("-",), NHWC32: ("-",), NHWC16: ("-",), CACHED32: ("cached", "global"),
            CACHED16: ("cached", "global"), FAST: ("cached", "global", "tabled", "inline"),
            SEP16: ("tabled", "inline"), SEPSPLIT: ("tabled", "inline"), FALLBACK: ("-",)}
ALL_PATHS = frozenset((k, s) for k, subs in SUBPATHS.items() for s in subs)
EXACT_ORDER = (NCHW, NHWC32, CACHED32, NHWC16, CACHED16)


def dispatch(fmt, c, ph, pw, h, w, aligned=True, separable=True):
    """(kernel, through the ops split-fp16 fallback) a call reaches, or (None, False) when the entry rejects it.
    nchw: mega_roi_align_forward_nchw. f32: mega_roi_align_forward_nhwc -> roi_align_nhwc_launch<float>: the 256-byte
    slice kernel when C % 64 == 0, else one CTA per (roi, bin). f16: mega_roi_align_forward_nhwc_f16: with C % 128 == 0,
    bins <= 7 x 7 and 16-byte aligned pointers and strides, the separable kernel for maps <= 64 x 64 (unless
    MEGA_B200_ROI_SEPARABLE=0), else the fast kernel; otherwise roi_align_nhwc_launch<__half> (slice kernel when
    C % 128 == 0). split: ops.roi_align_nhwc sends maps <= 64 x 64 with C % 128 == 0 and bins <= 7 x 7 to
    mega_roi_align_forward_nhwc_split16, anything else unpacks, runs the fp32 path and packs the result."""
    if ph <= 0 or pw <= 0 or c <= 0 or h <= 0 or w <= 0:
        return None, False
    if fmt == "nchw":
        return NCHW, False
    if fmt == "split":
        if h <= K_SEP_MAX_DIM and w <= K_SEP_MAX_DIM and c % 128 == 0 and ph <= 7 and pw <= 7:
            return (SEPSPLIT if aligned else None), False
        return dispatch("f32", c, ph, pw, h, w, aligned)[0], True
    if fmt == "f16":
        fast = c % 128 == 0 and ph <= 7 and pw <= 7 and aligned
        if fast and h <= K_SEP_MAX_DIM and w <= K_SEP_MAX_DIM and separable:
            return SEP16, False
        if fast:
            return FAST, False
    v = 4 if fmt == "f32" else 8
    if c % v or not aligned:
        return None, False
    slice_c = K_ROI_SLICE_BYTES // (4 if fmt == "f32" else 2)
    if fmt == "f32":
        return (CACHED32 if c % slice_c == 0 else NHWC32), False
    return (CACHED16 if c % slice_c == 0 else NHWC16), False


# ------------------------------------------------------------------------------------------------ fp32 geometry
class Geometry:
    """per-roi fp32 geometry of a call (numpy arrays over K): start_*, bin_*, grid_* and the footprint r0, r1, c0, c1"""

    def __init__(self, boxes, scale, ph, pw, sr, h, w):
        b = np.ascontiguousarray(np.asarray(boxes, dtype=F32).reshape(-1, 4))
        s = F32(scale)
        self.k, self.ph, self.pw, self.h, self.w = b.shape[0], ph, pw, h, w
        self.start_w, self.start_h = b[:, 0] * s, b[:, 1] * s
        end_w, end_h = b[:, 2] * s, b[:, 3] * s
        roi_w = np.maximum(end_w - self.start_w, F32(1))
        roi_h = np.maximum(end_h - self.start_h, F32(1))
        self.bin_h, self.bin_w = roi_h / F32(ph), roi_w / F32(pw)
        if sr > 0:
            self.grid_h = np.full(self.k, sr, dtype=np.int64)
            self.grid_w = np.full(self.k, sr, dtype=np.int64)
        else:
            self.grid_h = np.ceil(roi_h / F32(ph)).astype(np.int64)
            self.grid_w = np.ceil(roi_w / F32(pw)).astype(np.int64)
        # footprint of the cached kernels: rows r0..r1, columns c0..c1
        fend_h = self.start_h + self.bin_h * F32(ph)
        fend_w = self.start_w + self.bin_w * F32(pw)
        self.r0 = np.clip(np.floor(np.maximum(self.start_h, F32(0))).astype(np.int64), 0, h - 1)
        self.r1 = np.clip(np.floor(np.maximum(fend_h, F32(0))).astype(np.int64) + 1, 0, h - 1)
        self.c0 = np.clip(np.floor(np.maximum(self.start_w, F32(0))).astype(np.int64), 0, w - 1)
        self.c1 = np.clip(np.floor(np.maximum(fend_w, F32(0))).astype(np.int64) + 1, 0, w - 1)

    def footprint(self):
        return (self.r1 - self.r0 + 1) * (self.c1 - self.c0 + 1)

    def coords(self, i, axis):
        """fp32 sample coordinates of roi i along an axis ('h' or 'w'): [bins, grid]"""
        start, bn, g, bins = ((self.start_h[i], self.bin_h[i], self.grid_h[i], self.ph) if axis == "h" else
                              (self.start_w[i], self.bin_w[i], self.grid_w[i], self.pw))
        p = np.arange(bins, dtype=F32)[:, None]
        it = np.arange(g, dtype=F32)[None, :] + F32(0.5)
        return (start + p * bn) + (it * bn) / F32(g)


def axis_sample(c, size):
    """fp32 coordinates -> (lo, hi, wlo, whi) with the kernels' empty rule and clamps; empty samples get weight 0"""
    c = np.asarray(c, dtype=F32)
    empty = (c < F32(-1)) | (c > F32(size))
    c = np.where(c <= F32(0), F32(0), c)
    lo = c.astype(np.int64)
    clamp = lo >= size - 1
    lo = np.where(clamp, size - 1, lo)
    hi = np.where(clamp, lo, lo + 1)
    c = np.where(clamp, lo.astype(F32), c)
    l = (c - lo.astype(F32)).astype(F32)
    wlo, whi = (F32(1) - l).astype(F32), l
    wlo = np.where(empty, F32(0), wlo)
    whi = np.where(empty, F32(0), whi)
    return lo, hi, wlo, whi


def weight_matrices(geo):
    """fp64 [K, ph, H] and [K, pw, W]: the total weight each bin-row / bin-column puts on each map row / column"""
    ay = np.zeros((geo.k, geo.ph, geo.h))
    ax = np.zeros((geo.k, geo.pw, geo.w))
    for i in range(geo.k):
        for mat, axis, size, bins in ((ay, "h", geo.h, geo.ph), (ax, "w", geo.w, geo.pw)):
            lo, hi, wlo, whi = axis_sample(geo.coords(i, axis), size)
            p = np.broadcast_to(np.arange(bins)[:, None], lo.shape)
            np.add.at(mat[i], (p, lo), wlo.astype(np.float64))
            np.add.at(mat[i], (p, hi), whi.astype(np.float64))
    return ay, ax


def chain_length(geo, ay, ax, kernel):
    """m per output, broadcastable to [K, ph, pw]"""
    n = (geo.grid_h * geo.grid_w).astype(np.float64)[:, None, None]
    if kernel in EXACT_ORDER:
        return n + 6
    if kernel == FAST:
        return 4 * n + 3
    def span(mat):
        nz = mat != 0
        size = mat.shape[2]
        first = np.where(nz.any(2), nz.argmax(2), 0)
        last = np.where(nz.any(2), size - 1 - nz[:, :, ::-1].argmax(2), -1)
        return (last - first + 1).astype(np.float64)
    ry, rx = span(ay)[:, :, None], span(ax)[:, None, :]
    return 2 * geo.grid_h[:, None, None] + 2 * geo.grid_w[:, None, None] + ry + rx + 2


# ------------------------------------------------------------------------------------------------ fp64 reference
def reference(feat, batch, geo, ay=None, ax=None, chunk_bytes=1 << 29):
    """fp64 (ref, S) [K, ph * pw, C] on feat's device. feat: [N, H, W, C] (any float dtype; the values it holds are the
    input), batch: int [K] image index per roi."""
    if ay is None:
        ay, ax = weight_matrices(geo)
    dev = feat.device
    k, (n, h, w, c) = geo.k, feat.shape
    ref = torch.zeros(k, geo.ph, geo.pw, c, dtype=torch.float64, device=dev)
    s = torch.zeros_like(ref)
    if k == 0:
        return ref.view(k, geo.ph * geo.pw, c), s.view(k, geo.ph * geo.pw, c)
    Ay = torch.from_numpy(ay).to(dev)
    Ax = torch.from_numpy(ax).to(dev)
    inv = torch.from_numpy(1.0 / (geo.grid_h * geo.grid_w).astype(np.float64)).to(dev)
    bt = torch.as_tensor(np.asarray(batch, dtype=np.int64))
    step = max(1, chunk_bytes // (8 * geo.ph * w * c))
    for b in range(n):
        idx = (bt == b).nonzero().flatten()
        if idx.numel() == 0:
            continue
        f = feat[b].to(torch.float64)
        for src, dst in ((f, ref), (f.abs(), s)):
            for j in range(0, idx.numel(), step):
                sel = idx[j:j + step].to(dev)
                t = torch.einsum("kpy,ywc->kpwc", Ay[sel], src)
                dst[sel] = torch.einsum("kqx,kpxc->kpqc", Ax[sel], t) * inv[sel].view(-1, 1, 1, 1)
    return ref.view(k, geo.ph * geo.pw, c), s.view(k, geo.ph * geo.pw, c)


def m_tensor(m, geo, dev):
    """chain_length's m as a [K, ph * pw, 1] fp64 tensor on dev"""
    mm = np.broadcast_to(m, (geo.k, geo.ph, geo.pw)).reshape(geo.k, geo.ph * geo.pw, 1)
    return torch.from_numpy(np.array(mm, dtype=np.float64)).to(dev)


def half_width(ref, s, m, fmt, a=A):
    """per-element half-width of the interval (m: m_tensor)"""
    hw = (a * m + 1) * U * s + U * ref.abs()
    if fmt == "f16":
        hw = hw + 2.0 ** -11 * ref.abs() + 2.0 ** -25
    elif fmt == "split":
        hw = hw + 2.0 ** -23 * ref.abs() + 2.0 ** -25
    return hw


def inside(got, ref, s, m, fmt, a=A):
    """boolean: every element of got within its interval"""
    return (got.double() - ref).abs() <= half_width(ref, s, m, fmt, a)


def needed_a(got, ref, s, m, fmt):
    """the smallest A every element of got passes with (0 when the A-free part of the interval already holds it)"""
    if got.numel() == 0:
        return 0.0
    base = half_width(ref, s, m, fmt, a=0.0)
    per = (m * U * s).clamp_min(1e-300)
    over = ((got.double() - ref).abs() - base).clamp_min(0)
    return (over / per).max().item()


# ------------------------------------------------------------------------------------------------ sub-paths
def roi_paths(kernel, geo):
    """set of (kernel, sub-path) the rois of a call take inside `kernel`"""
    if kernel not in (CACHED32, CACHED16, FAST, SEP16, SEPSPLIT):
        return {(kernel, "-")} if geo.k else set()
    out = set()
    if kernel in (CACHED32, CACHED16, FAST):
        cached = geo.footprint() <= K_ROI_MAX_CELLS
        out |= {(kernel, "cached" if x else "global") for x in cached.tolist()}
    if kernel in (FAST, SEP16, SEPSPLIT):
        g = K_ROI_MAX_GRID if kernel == FAST else K_SEP_MAX_GRID
        tabled = (geo.grid_h <= g) & (geo.grid_w <= g)
        out |= {(kernel, "tabled" if x else "inline") for x in tabled.tolist()}
    return out


# ------------------------------------------------------------------------------------------------ case table
def _exact_rois(h, w, sr):
    """boxes (px, scale 1/16) whose samples land where the kernels' rules switch"""
    W, H = 16.0 * w, 16.0 * h
    b = [
        [-32, -32, 192, 192],              # sr 1 / 2: samples exactly on -1 and on integers up to 11 / 12 (= H on 11 / 12)
        [8, 8, 120, 120],                  # sr 1: every sample on an integer cell (weight 0 on the high cell)
        [40, 40, 45, 44],                  # smaller than one cell
        [100, 90, 60, 50],                 # inverted
        [W + 32, H + 32, W + 300, H + 300],  # wholly beyond the bottom-right edge: zeros
        [-400, -400, -40, -40],            # wholly before the top-left edge: zeros
        [-100, 20, 100, 60], [20, -100, 60, 100],           # straddle the left / top border
        [W - 100, 20, W + 100, 60], [20, H - 100, 60, H + 100],  # straddle the right / bottom border
        [-100, -100, W + 100, H + 100],    # all four
        [0, 0, W - 1, H - 1],              # the whole image
        [-16, -16, W, H],                  # ends exactly on the map's far edge
        [16 * (w - 1), 16 * (h - 1), W + 16, H + 16],  # one corner cell
        [0, 0, 16, 16],                    # one cell at the origin
    ]
    # footprints around the cached kernels' 192-cell budget: rows r0..r0+a-1 x columns c0..c0+b-1 (the box ends mid-cell)
    # (a map of one row / column clamps that axis of the footprint to one cell)
    for fa, fb in ((12, 16), (13, 15), (11, 17), (1, 191), (1, 192), (1, 193), (191, 1), (192, 1), (193, 1)):
        if (h == 1 if fa == 1 else fa + 1 <= h) and (w == 1 if fb == 1 else fb + 1 <= w):
            b.append([16.0, 16.0, 16.0 * (fb - 0.5), 16.0 * (fa - 0.5)])
    # adaptive grids just below / above 8 and 16 on each axis (sr = 0): roi = 7 g - 0.5 cells
    if sr == 0:
        for gh, gw in ((8, 9), (9, 8), (16, 17), (17, 16), (7, 8)):
            b.append([8.0, 8.0, 8.0 + 16.0 * (7 * gw - 0.5), 8.0 + 16.0 * (7 * gh - 0.5)])
    return np.asarray(b, dtype=F32)


def _random_rois(k, h, w, rng, max_frac=1.0):
    W, H = 16.0 * w, 16.0 * h
    xy = rng.uniform(-0.1, 0.95, size=(k, 2)) * np.array([W, H])
    wh = rng.uniform(0.5, 16.0 + max_frac * max(W, H), size=(k, 2))
    b = np.concatenate([xy, xy + wh], 1)
    return b.astype(F32)


def _huge_rois(k, h, w, rng):
    """boxes far larger than the map: adaptive grids of 20 - 60 samples per bin and axis"""
    W, H = 16.0 * w, 16.0 * h
    c = rng.uniform(0.2, 0.8, size=(k, 2)) * np.array([W, H])
    half = rng.uniform(16 * 7 * 10, 16 * 7 * 30, size=(k, 2))
    return np.concatenate([c - half, c + half], 1).astype(F32)


def build_inputs(c):
    """(feat fp32 [N, H, W, C], boxes fp32 [K, 4], batch int32 [K]) of case `c`, on the CPU"""
    rng = np.random.default_rng(c["seed"])
    g = torch.Generator().manual_seed(c["seed"])
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    if c["values"] == "randn":
        f = torch.randn(n, h, w, ch, generator=g)
    elif c["values"] == "hdr":          # relu'd, magnitudes from 1e-4 to ~3e4 (inside fp16's range)
        f = torch.randn(n, h, w, ch, generator=g).relu() * torch.exp(torch.rand(n, h, w, ch, generator=g) * 18 - 9)
    else:                               # "cancel": a +-512 checkerboard, so bilinear sums cancel to ~1e-2 of their terms
        sign = (torch.arange(h).view(h, 1, 1) + torch.arange(w).view(1, w, 1)) % 2 * 2 - 1
        f = (512.0 * sign + torch.randn(n, h, w, ch, generator=g) * 2.0).float()
    parts = []
    if c["rois"] in ("exact", "mixed"):
        parts.append(_exact_rois(h, w, c["sr"]))
    if c["rois"] in ("random", "mixed"):
        parts.append(_random_rois(max(c["k"] - sum(len(p) for p in parts), 0), h, w, rng))
    if c["rois"] == "huge":
        parts.append(_huge_rois(c["k"], h, w, rng))
    boxes = np.concatenate(parts, 0)[:c["k"]] if parts else np.zeros((0, 4), F32)
    if c["k"] > len(boxes):
        boxes = np.concatenate([boxes] * (c["k"] // max(len(boxes), 1) + 1), 0)[:c["k"]]
    if c["batch"] == "spans":            # engine._roi_table: consecutive spans of 300 / 75 rows per image
        spans = c["spans"]
        batch = np.concatenate([np.full(r, i) for i, r in enumerate(spans)])
    elif c["batch"] == "perm":           # every image repeated, in a shuffled order
        batch = rng.permutation(np.arange(c["k"]) % n)
    else:
        batch = np.zeros(c["k"], np.int64)
    return f.contiguous(), torch.from_numpy(boxes.astype(F32)).reshape(-1, 4), torch.from_numpy(batch.astype(np.int32))


def _case(cid, *, n=1, h, w, c, ph=7, pw=7, sr=0, k, rois="mixed", values="randn", batch="none", spans=None, seed,
          formats=FORMATS):
    # split-fp16 tensors hold groups of 32 values; the engines' split-fp16 maps have C % 128 == 0
    fm = tuple(f for f in formats if dispatch(f, c, ph, pw, h, w)[0] is not None and (f != "split" or c % 128 == 0))
    if spans:
        k = sum(spans)
    return dict(id=cid, n=n, h=h, w=w, c=c, ph=ph, pw=pw, sr=sr, k=k, rois=rois, values=values, batch=batch,
                spans=spans, seed=seed, formats=fm)


def make_cases():
    """the committed case table (fixed seeds: every case is reproducible)"""
    C = []
    add = lambda *a, **kw: C.append(_case(*a, **kw))
    # engine geometries: res5 map of a 600 x 1000 frame, C = 2048 (and the 256-channel REDUCE_CHANNEL map), 7 x 7, sr 0
    add("eng_38x63_c2048_k75", h=38, w=63, c=2048, k=75, seed=1)
    add("eng_38x63_c256_k300", h=38, w=63, c=256, k=300, rois="random", values="hdr", seed=2)
    add("eng_batch3_spans", n=3, h=38, w=63, c=256, k=0, spans=(300, 75, 300), rois="random", batch="spans", seed=3)
    add("eng_batch3_perm", n=3, h=38, w=63, c=128, k=240, batch="perm", values="cancel", seed=4)
    add("bbox_aug_75x125_c256", h=75, w=125, c=256, k=150, seed=5)      # a rescaled TEST.BBOX_AUG pass (fast kernel)
    # map edges
    add("map_1x1", h=1, w=1, c=128, k=20, rois="exact", seed=10)
    add("map_1x200", h=1, w=200, c=128, k=40, seed=11)
    add("map_200x1", h=200, w=1, c=128, k=40, sr=2, seed=12)
    add("map_64x64", h=64, w=64, c=128, k=60, seed=13)
    add("map_65x64", h=65, w=64, c=128, k=60, sr=2, seed=14)
    add("map_64x65", h=64, w=65, c=128, k=60, values="hdr", seed=15)
    add("map_11x13_sr1", h=11, w=13, c=128, sr=1, k=30, rois="exact", values="hdr", seed=16)
    add("map_12x11_sr2", n=2, h=12, w=11, c=128, sr=2, k=30, rois="exact", batch="perm", seed=17)
    # channels
    add("ch4", n=2, h=13, w=17, c=4, k=40, batch="perm", seed=20)
    add("ch8", h=13, w=17, c=8, k=40, sr=2, values="cancel", seed=21)
    add("ch60", h=20, w=30, c=60, k=40, seed=22)
    add("ch64", n=2, h=20, w=30, c=64, k=40, batch="perm", values="hdr", seed=23)
    add("ch120", h=20, w=30, c=120, k=40, seed=24)
    add("ch1024", h=30, w=40, c=1024, k=40, values="cancel", seed=25)
    # bins
    add("bins14", h=38, w=63, c=256, ph=14, pw=14, sr=2, k=60, seed=30)
    add("bins1x1", h=20, w=30, c=128, ph=1, pw=1, k=40, seed=31)
    add("bins3x5", h=20, w=30, c=128, ph=3, pw=5, k=40, values="hdr", seed=32)
    add("bins8x7", h=20, w=30, c=128, ph=8, pw=7, k=40, seed=33)
    add("bins8x7_75x90", h=75, w=90, c=128, ph=8, pw=7, k=40, sr=3, seed=34)
    # sampling ratios (maps <= 64: separable; above: fast)
    add("sr1_40x50", h=40, w=50, c=128, sr=1, k=40, seed=40)
    add("sr8_40x50", h=40, w=50, c=128, sr=8, k=40, values="cancel", seed=41)
    add("sr9_40x50", h=40, w=50, c=128, sr=9, k=40, seed=42)
    add("sr16_40x50", h=40, w=50, c=128, sr=16, k=30, seed=43)
    add("sr17_40x50", h=40, w=50, c=128, sr=17, k=30, values="hdr", seed=44)
    add("sr8_72x80", h=72, w=80, c=128, sr=8, k=40, seed=45)
    add("sr9_72x80", h=72, w=80, c=128, sr=9, k=40, values="cancel", seed=46)
    add("sr17_72x80", h=72, w=80, c=128, sr=17, k=20, seed=47)
    add("huge_20x30", h=20, w=30, c=128, k=16, rois="huge", seed=48)
    add("huge_70x90", h=70, w=90, c=128, k=16, rois="huge", values="hdr", seed=49)
    add("huge_ch8", h=20, w=30, c=8, k=12, rois="huge", seed=50)
    # sizes
    add("k0", h=20, w=30, c=128, k=0, seed=60)
    add("k1", h=20, w=30, c=128, k=1, rois="random", seed=61)
    add("k1200", n=2, h=24, w=40, c=128, k=1200, rois="random", batch="perm", seed=62)
    return C


def case_geometry(c, boxes):
    return Geometry(boxes.numpy(), SCALE, c["ph"], c["pw"], c["sr"], c["h"], c["w"])
