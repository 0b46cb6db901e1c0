"""Shared pieces of the FGFA / DFF conformance suite (test_fgfa_conformance_cpu.py / _gpu.py).

- geometry: the warp's sample positions and corner weights, restated from csrc/fgfa.cu flow_corners;
- reference / interval: fp64 results of the five kernels of csrc/fgfa.cu and a per-element half-width each output must
  lie within;
- the committed case table: the engines' shapes, the kernels' limits and edges, flows and values placed where the
  kernels can go wrong.

Geometry. Everything up to the corner weights is computed in fp32, one rounding per operation, in the kernel's order:
    gx = fl(fl(fx + x) / ((w - 1) * 0.5)) - 1,  px = fl(fma(fl(gx + 1), w, -1)) * 0.5,  px = min(max(px, 0), w - 1),
    x0 = floor(px), x1 = min(x0 + 1, w - 1), lx = px - x0,  weights fl(fl(1 - lx) fl(1 - ly)), fl(lx fl(1 - ly)), ...
F.grid_sample rounds (gx + 1) * w and the subtraction of 1 separately: about 2 % of the positions of a random flow then
sit one ulp apart, and the sampled value moves by up to ~30 ulps of max|feature|, more than the whole blend's error.
numpy has no fma: the fp32 product (gx + 1) * w is exact in fp64, the fp64 sum with -1 is rounded once to fp32. That sum
is exact unless |gx + 1| is tiny, where the result is ~ -1 and clamped to 0 anyway; `geometry` asserts exactly this.
The floor is discontinuous, so only the blend and the sums run in fp64.

Reference and interval (u = 2^-24; Se = the same sample of |values|, so |each partial sum| <= Se; A scales every bound):
  * sample (both warps): one FMUL (w00 * v00) and three FFMA: |d sample| <= 4 u Se.
  * dff_warp_scale: the sample times scale, one more rounding: m = 5, S = Se |scale|.
  * fgfa_aggregate, per pixel, per = ceil(ce / 256) channels per thread, R = per + 13 (per FMAs, 5 shuffle levels,
    8 warp partials summed in order):
      dot_f  = sum_c e_f e_k             |d| <= (R + 8) u sum_c Se_f Se_k   (8: the two samples' 4 u each)
      |e_f|^2                            |d| <= (R + 8) u sum_c Se_f^2 =: D
      n_f = sqrt(|e_f|^2) + 1e-10f       |d| <= min(sqrt(D), D / (2 |e_f|)) + 2 u n_f   (sqrtf, the add)
      l_f = (dot_f / n_f) / n_k          |d l_f| <= |d dot_f| / (n_f n_k) + |l_f| (|d n_f| / n_f + |d n_k| / n_k + 2 u)
    soft-max: expf is within 2 ulp (no --use_fast_math), so 4 u relative; the subtraction of the maximum adds
    u |l_f - l_max| (the maximum itself cancels); the L-term sum of the exponentials, 1 / den and the product add (L + 1) u:
      eps_f = |d l_f| + u |l_f - l_max| + 4 u,     |d w_f| <= w_f (eps_f + sum_g w_g eps_g + (L + 1) u)
    out = sum_f w_f s_f (the weight times the sample, accumulated by L FMAs):
      |d out| <= sum_f |d w_f| Ss_f + (L + 5) u sum_f w_f Ss_f          (Ss_f: the sample of |feats|)
  * avgpool2_nhwc: <= 3 additions and the division: m = 4, S = mean |v|.
  * fgfa_pool_image: each v / 255, <= 3 additions, fl(1 / count) and the product: m = 6, S = mean |v| / 255.
  * fgfa_build_pairs is a copy: bit for bit, zero borders and channels 3 and 7 included.
The half-width is A times the bound above plus, for fp16 outputs, half an fp16 ulp of |ref| + that bound.

Domain. fp32 embeddings whose sum of squares at a pixel lies below 2^-126 underflow in the kernel's fp32 sums and not in
the fp64 reference; the case table's embeddings have a sum of squares of 0 or >= 2^-126 at every pixel
(check_domain). Maps of height or width 1 are outside the warp's domain (get_grid divides by zero), and so are NaN flows
in channels 0 and 1. A is calibrated in test_fgfa_conformance_gpu.py.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

U = 2.0 ** -24
# A per output (calibration: test_fgfa_conformance_gpu.py)
A = {"agg": 1.0, "weights": 1.0, "dff": 2.0, "pool": 2.0, "pool_image": 1.0}
F32 = np.float32
EPS_NORM = float(np.float32(1e-10))        # the kernel's 1e-10f
DTYPES = ("f32", "f16")

# constants of csrc/fgfa.cu (test_fgfa_conformance_cpu.py reads them back from the source)
K_AGG_THREADS = 256
K_AGG_MAX_FRAMES = 32
K_AGG_MAX_EMBED = 16 * K_AGG_THREADS
GRID_CAP = 132 * 16                        # grid_for: at most this many blocks of BLOCK threads
BLOCK = 256
KERNELS = ("fgfa_pool_image_kernel", "fgfa_build_pairs_kernel", "avgpool2_nhwc_kernel", "fgfa_aggregate_kernel",
           "dff_warp_scale_kernel")
INSTANTIATIONS = tuple("%s<%s>" % (k, t) for k in KERNELS for t in ("float", "__half"))
GEOMETRY_MODES = ("kernel", "fp64", "align_corners", "zeros", "unclamped", "no_fma")


# ------------------------------------------------------------------------------------------------ geometry
def _two_sum_err(a, b):
    s = a + b
    bb = s - a
    return (a - (s - bb)) + (b - bb)


def _axis(f, pos, size, mode):
    """flow component f (fp32 [..., P]) at integer coordinates pos -> (lo, hi, l, valid_lo, valid_hi); l is fp32 (fp64
    in mode 'fp64'); lo / hi may be out of range in modes 'zeros' / 'unclamped'"""
    f = np.asarray(f, dtype=F32)
    if mode == "fp64":
        g = (f.astype(np.float64) + pos) / ((size - 1) / 2.0) - 1.0
        p = np.clip(((g + 1.0) * size - 1.0) / 2.0, 0.0, size - 1.0)
        lo = np.floor(p)
        return lo.astype(np.int64), np.minimum(lo + 1, size - 1).astype(np.int64), p - lo, None, None
    with np.errstate(over="ignore", invalid="ignore"):
        s = (f + F32(pos)).astype(F32)
        g = (s / (F32(size - 1) * F32(0.5))).astype(F32) - F32(1)
        t = (g + F32(1)).astype(F32)
        if mode == "align_corners":
            p = ((t * F32(0.5)).astype(F32) * F32(size - 1)).astype(F32)
        elif mode == "no_fma":
            p = ((t * F32(size)).astype(F32) - F32(1)).astype(F32) * F32(0.5)
        else:
            prod = t.astype(np.float64) * float(size)
            r = prod - 1.0
            exact = _two_sum_err(prod, -1.0) == 0
            p = r.astype(F32) * F32(0.5)
            # fma rounds once: the fp64 sum is exact, or the result lies below 0 and is clamped
            assert bool(np.all(exact | (p < 0) | np.isnan(p))), "fma restatement: inexact fp64 sum inside the map"
    if mode == "zeros":                    # padding_mode="zeros": no clamp, corners outside the map weigh 0
        lo = np.floor(p)
        l = (p - lo).astype(F32)
        lo = lo.astype(np.int64)
        hi = lo + 1
        return lo, hi, l, (lo >= 0) & (lo < size), (hi >= 0) & (hi < size)
    p = np.minimum(np.maximum(p, F32(0)), F32(size - 1)).astype(F32)
    lo_f = np.floor(p).astype(F32)
    lo = lo_f.astype(np.int64)
    hi = lo + 1 if mode == "unclamped" else np.minimum(lo + 1, size - 1)
    return lo, hi, (p - lo_f).astype(F32), None, None


class Geometry:
    """corners of a warp: idx [4, ..., P] int64 flat pixel indices y * w + x (order 00, 01, 10, 11), wts [4, ..., P]
    (fp32 values in fp64, or fp64 in mode 'fp64'). flow: fp32 [..., h, w, >= 2] (channel 0 = x, 1 = y)."""

    def __init__(self, flow, mode="kernel", swap_xy=False):
        flow = np.asarray(flow, dtype=F32)
        h, w = flow.shape[-3], flow.shape[-2]
        assert h >= 2 and w >= 2, "the warp needs maps of at least 2 x 2 cells"
        self.h, self.w = h, w
        fx, fy = flow[..., 0], flow[..., 1]
        if swap_xy:
            fx, fy = fy, fx
        ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        x0, x1, lx, vx0, vx1 = _axis(fx, xs, w, mode)
        y0, y1, ly, vy0, vy1 = _axis(fy, ys, h, mode)
        if mode == "fp64":
            hx, hy = 1.0 - lx, 1.0 - ly
            ws = [hx * hy, lx * hy, hx * ly, lx * ly]
        else:
            hx, hy = (F32(1) - lx).astype(F32), (F32(1) - ly).astype(F32)
            ws = [(hx * hy).astype(F32), (lx * hy).astype(F32), (hx * ly).astype(F32), (lx * ly).astype(F32)]
        corners = [(y0, x0), (y0, x1), (y1, x0), (y1, x1)]
        if mode == "zeros":
            valid = [vy0 & vx0, vy0 & vx1, vy1 & vx0, vy1 & vx1]
            ws = [np.where(v, wt, F32(0)) for v, wt in zip(valid, ws)]
            corners = [(np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)) for yy, xx in corners]
        lead = flow.shape[:-3]
        self.idx = np.stack([(yy * w + xx).reshape(lead + (h * w,)) for yy, xx in corners])
        self.wts = np.stack([np.asarray(wt, np.float64).reshape(lead + (h * w,)) for wt in ws])
        self.px = (xs, x0, lx)

    def torch(self, dev):
        return torch.from_numpy(self.idx).to(dev), torch.from_numpy(self.wts).to(dev)


def sample64(m, idx, wts):
    """fp64 bilinear samples of m [P', C] (any float dtype; P' >= max index + 1) at corners idx / wts [4, P] (torch)"""
    m = m.double()
    out = wts[0].unsqueeze(1) * m[idx[0]]
    for k in (1, 2, 3):
        out = out + wts[k].unsqueeze(1) * m[idx[k]]
    return out


# ------------------------------------------------------------------------------------------------ fp64 references
def half_ulp16(x):
    """half an fp16 ulp at |x| (fp64 tensor): 2^-25 below 2^-14, else 2^(floor(log2 |x|) - 11)"""
    m, e = torch.frexp(x.abs())
    return torch.where(x.abs() < 2.0 ** -14, torch.full_like(x, 2.0 ** -25), torch.ldexp(torch.ones_like(x), e - 12))


def half_width(bound, ref, dtype, a):
    hw = a * bound
    if dtype == "f16":
        hw = hw + half_ulp16(ref.abs() + hw)
    return hw


def inside(got, ref, bound, dtype, a):
    return (got.double() - ref).abs() <= half_width(bound, ref, dtype, a)


def needed_a(got, ref, bound, dtype):
    """the smallest A every element passes with (0 when the A-free part, the fp16 output rounding, holds it)"""
    if got.numel() == 0:
        return 0.0
    err = (got.double() - ref).abs()
    if dtype == "f16":
        err = (err - half_ulp16(ref.abs())).clamp_min(0)
    return (err / bound.clamp_min(1e-300)).max().item()


def aggregate_reference(ring, slots, key_pos, flow, cf, ce):
    """fp64 (out [P, cf], out_bound, weights [L, P], weights_bound) of fgfa_aggregate. ring: [S, h, w, >= cf + ce] (the
    values the kernel reads, any float dtype, on the device to compute on); slots: list of L ints; flow: fp32 numpy
    [>= L, h, w, >= 2] (position f warps window frame f)."""
    dev = ring.device
    s_, h, w, _ = ring.shape
    L, P = len(slots), h * w
    geo = Geometry(np.asarray(flow)[:L])
    idx, wts = geo.torch(dev)
    per = (ce + K_AGG_THREADS - 1) // K_AGG_THREADS
    red = per + 13 + 8
    flat = ring.reshape(s_, P, ring.shape[3])

    def emb(f):
        m = flat[slots[f], :, cf:cf + ce]
        return sample64(m, idx[:, f], wts[:, f]), sample64(m.abs(), idx[:, f], wts[:, f])

    def norm(e, se):
        d = red * U * (se * se).sum(1)
        n = (e * e).sum(1).sqrt()
        dn = torch.minimum(d.sqrt(), d / (2 * n).clamp_min(1e-300)) + 2 * U * (n + EPS_NORM)
        return n + EPS_NORM, dn

    ek, sk = emb(key_pos)
    nk, dnk = norm(ek, sk)
    logit = torch.empty(L, P, dtype=torch.float64, device=dev)
    dlogit = torch.empty_like(logit)
    feats = torch.empty(L, P, cf, dtype=torch.float64, device=dev)
    sfeats = torch.empty_like(feats)
    for f in range(L):
        e, se = emb(f)
        nf, dnf = norm(e, se)
        dot = (e * ek).sum(1)
        ddot = red * U * (se * sk).sum(1)
        l = dot / (nf * nk)
        logit[f], dlogit[f] = l, ddot / (nf * nk) + l.abs() * (dnf / nf + dnk / nk + 2 * U)
        m = flat[slots[f], :, :cf]
        feats[f] = sample64(m, idx[:, f], wts[:, f])
        sfeats[f] = sample64(m.abs(), idx[:, f], wts[:, f])
    wt = torch.softmax(logit, 0)
    eps = dlogit + U * (logit - logit.max(0).values).abs() + 4 * U
    dwt = wt * (eps + (wt * eps).sum(0) + (L + 1) * U)
    out = (wt.unsqueeze(2) * feats).sum(0)
    bound = (dwt.unsqueeze(2) * sfeats).sum(0) + (L + 5) * U * (wt.unsqueeze(2) * sfeats).sum(0)
    return out, bound, wt, dwt


def dff_reference(key, flow, scale):
    """fp64 (out [P, C], bound) of dff_warp_scale. key [h, w, C], scale [h, w, >= C] (values the kernel reads, on the
    device to compute on); flow fp32 numpy [h, w, >= 2]"""
    h, w, c = key.shape
    idx, wts = Geometry(np.asarray(flow)).torch(key.device)
    k = key.reshape(h * w, c)
    sc = scale[..., :c].reshape(h * w, c).double()
    return sample64(k, idx, wts) * sc, 5 * U * sample64(k.abs(), idx, wts) * sc.abs()


def _pool_windows(x):
    """x [N, H, W, C] fp64 -> (sum over each ceil-mode 2x2 window, number of in-bound cells) [N, ceil(H/2), ceil(W/2), *]"""
    n, h, w, c = x.shape
    xp = torch.zeros(n, h + h % 2, w + w % 2, c, dtype=x.dtype, device=x.device)
    xp[:, :h, :w] = x
    s = xp.view(n, (h + 1) // 2, 2, (w + 1) // 2, 2, c).sum((2, 4))
    one = torch.zeros(h + h % 2, w + w % 2, dtype=x.dtype, device=x.device)
    one[:h, :w] = 1
    cnt = one.view((h + 1) // 2, 2, (w + 1) // 2, 2).sum((1, 3))
    return s, cnt.view(1, (h + 1) // 2, (w + 1) // 2, 1)


def avgpool_reference(x):
    """fp64 (out, bound) of avgpool2_nhwc; x [N, H, W, C] (the values the kernel reads)"""
    s, cnt = _pool_windows(x.double())
    sa, _ = _pool_windows(x.double().abs())
    return s / cnt, 4 * U * sa / cnt


def pool_image_reference(img):
    """fp64 (out [Hq, Wq, 4], bound) of fgfa_pool_image; img [3, H, W] fp32"""
    x = img.double().reshape(1, 3, img.shape[-2], img.shape[-1]).permute(0, 2, 3, 1)
    s, cnt = _pool_windows(x)
    sa, _ = _pool_windows(x.abs())
    out = torch.zeros(s.shape[1], s.shape[2], 4, dtype=torch.float64, device=img.device)
    bound = torch.zeros_like(out)
    out[..., :3] = (s / cnt / 255.0)[0]
    bound[..., :3] = (6 * U * sa / cnt / 255.0)[0]
    return out, bound


def pairs_reference(ring, slots, key_pos):
    """fgfa_build_pairs exactly: [L, hq + 6, wq + 8, 8] in ring's dtype"""
    s_, hq, wq, _ = ring.shape
    out = torch.zeros(len(slots), hq + 6, wq + 8, 8, dtype=ring.dtype, device=ring.device)
    for f, s in enumerate(slots):
        out[f, 3:3 + hq, 3:3 + wq, 0:3] = ring[slots[key_pos], ..., 0:3]
        out[f, 3:3 + hq, 3:3 + wq, 4:7] = ring[s, ..., 0:3]
    return out


# ------------------------------------------------------------------------------------------------ case table
def exact_flow(h, w, rng, frac=0.5):
    """fp32 flow [h, w, 2] whose kernel positions land exactly on integer cells (0 and w - 1 / h - 1 among them) at
    most of a fraction `frac` of the pixels (a position (2k + 1) / w - 1 is not always one fp32 step away), random
    (sigma 3 cells) elsewhere"""
    flow = (rng.standard_normal((h, w, 2)) * 3).astype(F32)
    for ch, size in ((0, w), (1, h)):
        pos = np.broadcast_to(np.arange(w)[None, :] if ch == 0 else np.arange(h)[:, None], (h, w))
        target = rng.integers(0, size, (h, w))
        target[rng.random((h, w)) < 0.3] = 0
        target[rng.random((h, w)) < 0.3] = size - 1
        want = (rng.random((h, w)) < frac)
        base = ((2 * target + 1) * (size - 1) / (2.0 * size) - pos).astype(F32)
        done = np.zeros((h, w), bool)
        for j in [0] + [s * k for k in range(1, 200) for s in (1, -1)]:
            step = np.spacing(np.abs(base + pos).astype(F32)).astype(np.float64)     # one ulp of fx + x
            cand = (base.astype(np.float64) + j * step).astype(F32)
            lo, _, l, _, _ = _axis(cand, pos, size, "kernel")
            hit = want & ~done & (l == 0) & (lo == target)
            flow[..., ch] = np.where(hit, cand, flow[..., ch])
            done |= hit
        assert done[want].mean() > 0.5, "exact_flow: too few exact positions"
    return flow


def make_flow(mode, n, h, w, rng):
    """fp32 [n, h, w, 4]; channels 2 and 3 hold NaN (never read)"""
    f = np.full((n, h, w, 4), np.nan, F32)
    for i in range(n):
        if mode == "zero":
            f[i, ..., :2] = 0
        elif mode == "exact":
            f[i, ..., :2] = exact_flow(h, w, rng)
        elif mode == "far":
            v = (rng.standard_normal((h, w, 2)) * 3).astype(F32)
            far = rng.random((h, w, 2)) < 0.4
            v[far] = np.where(rng.random(int(far.sum())) < 0.5, -1e4, 1e4).astype(F32)
            f[i, ..., :2] = v
        else:
            f[i, ..., :2] = (rng.standard_normal((h, w, 2)) * 3).astype(F32)
    return f


def _values(kind, shape, g):
    if kind == "big":                      # fp16's top binades: |v| up to 6e4
        return (torch.rand(shape, generator=g) * 2 - 1) * 6e4
    if kind == "sub":                      # fp16 subnormals and the smallest normals (< 2^-14 ~ 6.1e-5)
        return (torch.rand(shape, generator=g) * 2 - 1) * 1.2e-4
    if kind == "tiny":                     # embeddings of norm ~ 1e-11: the + 1e-10 dominates (fp32 only)
        return torch.randn(shape, generator=g) * 1e-12
    return torch.randn(shape, generator=g)


def window(c):
    """the L ring slots of the window, by position"""
    L, key, n = c["L"], c["key"], c["n_slots"]
    if c["window"] == "first":             # the engine's first frame: slot 0 at positions 0..key, look-ahead after
        return [0] * (key + 1) + list(range(1, L - key))
    if c["window"] == "rot":               # the steady-state ring, rotated
        return [(c["seed"] % n + i) % n for i in range(L)]
    return [int(v) for v in np.random.default_rng(c["seed"]).permutation(n)[:L]]


def build_inputs(c):
    """CPU inputs of case c (fp32 values; an fp16 run uses their fp16 roundings)"""
    rng = np.random.default_rng(c["seed"])
    g = torch.Generator().manual_seed(c["seed"])
    k = c["kind"]
    if k == "agg":
        h, w, ld, cf, ce = c["h"], c["w"], c["ld"], c["cf"], c["ce"]
        ring = torch.full((c["n_slots"], h, w, ld), float("nan"))       # unused slots and padding: NaN, never read
        slots = window(c)
        used = sorted(set(slots))
        ring[used, ..., :cf] = _values(c["values"] if c["values"] != "tiny" else "randn", (len(used), h, w, cf), g)
        ring[used, ..., cf:cf + ce] = _values(c["values"], (len(used), h, w, ce), g)
        if c["values"] == "zero_frame":
            ring[slots[(c["key"] + 1) % c["L"]], ..., cf:cf + ce] = 0
        if c["values"] == "zero_key":
            ring[slots[c["key"]], ..., cf:cf + ce] = 0
        return dict(ring=ring, slots=slots, flow=make_flow(c["flow"], c["L"], h, w, rng))
    if k == "dff":
        h, w, ch = c["h"], c["w"], c["c"]
        key = torch.full((h, w, c["key_ld"]), float("nan"))
        key[..., c["key_off"]:c["key_off"] + ch] = _values(c["values"], (h, w, ch), g)
        scale = torch.full((h, w, ch + c["pad"]), float("nan"))
        sv = torch.rand(h, w, ch, generator=g) * 2 - 0.5               # FlowNetS' scale map + 1: around 1, both signs
        if c["values"] == "big":
            sv = sv * 0.66                                             # keeps |warp * scale| < 6e4
        scale[..., :ch] = sv
        return dict(key=key, scale=scale, flow=make_flow(c["flow"], 1, h, w, rng)[0])
    if k == "pool":
        x = torch.full((c["n"], c["h"], c["w"], c["c"] + c["pad"]), float("nan"))
        x[..., :c["c"]] = _values(c["values"], (c["n"], c["h"], c["w"], c["c"]), g)
        return dict(x=x)
    if k == "pool_image":
        img = torch.rand(3, c["h"], c["w"], generator=g) * 255 - 110  # the transformed frame: pixel - mean
        if c["values"] == "big":
            img = img * 64.0
        return dict(img=img)
    if k == "pairs":
        ring = torch.randn(c["n_slots"], c["h"], c["w"], 4, generator=g)  # channel 3 holds junk: never copied
        return dict(ring=ring, slots=window(c))
    raise ValueError(k)


def check_domain(c, inp):
    """the embeddings' sum of squares at each pixel is 0 or >= 2^-126 (see the module docstring)"""
    if c["kind"] != "agg":
        return
    e = inp["ring"][sorted(set(inp["slots"]))][..., c["cf"]:c["cf"] + c["ce"]].double()
    ss = (e * e).sum(-1)
    assert bool(((ss == 0) | (ss >= 2.0 ** -126)).all()), c["id"]


def _agg(cid, *, h=6, w=7, L=5, key=2, cf=64, ce=128, pad=8, n_slots=None, window="distinct", flow="randn",
         values="randn", out_pad=8, seed, dtypes=DTYPES):
    return dict(id=cid, kind="agg", h=h, w=w, L=L, key=key, cf=cf, ce=ce, ld=cf + ce + pad,
                n_slots=n_slots or L + 2, window=window, flow=flow, values=values, out_pad=out_pad, seed=seed,
                dtypes=dtypes)


def _dff(cid, *, h=6, w=7, c=64, key_ld=None, key_off=0, pad=8, flow="randn", values="randn", seed, dtypes=DTYPES):
    return dict(id=cid, kind="dff", h=h, w=w, c=c, key_ld=key_ld or c, key_off=key_off, pad=pad, flow=flow,
                values=values, seed=seed, dtypes=dtypes)


def _pool(cid, *, n=1, h, w, c=16, pad=8, values="randn", seed, dtypes=DTYPES):
    return dict(id=cid, kind="pool", n=n, h=h, w=w, c=c, pad=pad, values=values, seed=seed, dtypes=dtypes)


def _image(cid, *, h, w, values="randn", seed, dtypes=DTYPES):
    return dict(id=cid, kind="pool_image", h=h, w=w, values=values, seed=seed, dtypes=dtypes)


def _pairs(cid, *, h, w, L, key, n_slots, window="distinct", seed, dtypes=DTYPES):
    return dict(id=cid, kind="pairs", h=h, w=w, L=L, key=key, n_slots=n_slots, window=window, seed=seed,
                dtypes=dtypes)


def make_cases():
    """the committed case table (fixed seeds: every case is reproducible)"""
    C = []
    # production FGFA: 19-frame window, key 9, 1024 feats + 2048 embedding channels in a 3072-channel ring, at the
    # 600 x 1000 (38 x 63) and 192 x 320 (12 x 20) maps; the first frame's window and a rotated steady-state window
    for h, w in ((38, 63), (12, 20)):
        for win, s in (("first", 1), ("rot", 2)):
            C.append(_agg("prod_%s_%dx%d" % (win, h, w), h=h, w=w, L=19, key=9, cf=1024, ce=2048, pad=0, n_slots=19,
                          window=win, out_pad=0 if win == "first" else 16, seed=s + h))
    # embedding widths around the kernel's 256 threads x 16 channels
    for ce, s in ((1, 10), (200, 11), (256, 12), (1000, 13), (4096, 14)):
        C.append(_agg("ce%d" % ce, ce=ce, seed=s))
    for cf, s in ((1, 20), (100, 21), (1030, 22)):
        C.append(_agg("cf%d" % cf, cf=cf, seed=s))
    C.append(_agg("L1", L=1, key=0, seed=30))
    C.append(_agg("L32_key31", h=4, w=5, L=32, key=31, seed=31))
    C.append(_agg("key0", L=7, key=0, window="rot", n_slots=7, seed=32))
    C.append(_agg("key_last", L=7, key=6, seed=33))
    C.append(_agg("map_2x2", h=2, w=2, seed=40))
    C.append(_agg("map_2x9", h=2, w=9, flow="exact", seed=41))
    C.append(_agg("map_9x2", h=9, w=2, flow="exact", seed=42))
    C.append(_agg("flow_zero", flow="zero", seed=50))
    C.append(_agg("flow_exact", h=9, w=11, flow="exact", window="rot", n_slots=5, seed=51))
    C.append(_agg("flow_far", flow="far", seed=52))
    C.append(_agg("emb_zero_frame", values="zero_frame", seed=60))
    C.append(_agg("emb_zero_key", values="zero_key", seed=61))
    C.append(_agg("emb_tiny", ce=200, values="tiny", seed=62, dtypes=("f32",)))
    C.append(_agg("values_big", ce=200, values="big", seed=63))
    C.append(_agg("values_sub", ce=200, values="sub", seed=64))
    # DFF: the 1024-channel map, the key map as a channel slice of a 3072-channel buffer, padded scale / out rows
    C.append(_dff("dff_prod_38x63", h=38, w=63, c=1024, key_ld=3072, key_off=1024, pad=8, seed=100))
    C.append(_dff("dff_prod_12x20", h=12, w=20, c=1024, pad=0, seed=101))
    C.append(_dff("dff_grid_stride_64x80", h=64, w=80, c=1024, seed=102))  # 655,360 threads > 132 * 16 * 256
    C.append(_dff("dff_c8_2x2", h=2, w=2, c=8, key_ld=24, key_off=8, seed=103))
    C.append(_dff("dff_2x9_exact", h=2, w=9, c=16, flow="exact", seed=104))
    C.append(_dff("dff_9x2_exact", h=9, w=2, c=16, flow="exact", seed=105))
    C.append(_dff("dff_exact", h=9, w=11, c=32, flow="exact", seed=106))
    C.append(_dff("dff_zero", c=32, flow="zero", seed=107))
    C.append(_dff("dff_far", c=32, flow="far", seed=108))
    C.append(_dff("dff_big", c=32, values="big", seed=109))
    C.append(_dff("dff_sub", c=32, values="sub", seed=110))
    # NHWC 2x2 ceil-mode pool: FlowNetS' pool5 shape (grid-stride: 1,436,400 threads), odd / even / 1-cell sides
    C.append(_pool("pool_flownet", n=3, h=75, w=125, c=200, pad=0, seed=200))
    for (h, w), s in (((7, 9), 201), ((8, 10), 202), ((1, 1), 203), ((1, 9), 204), ((9, 1), 205), ((2, 2), 206)):
        C.append(_pool("pool_%dx%d" % (h, w), n=2, h=h, w=w, seed=s))
    C.append(_pool("pool_big", h=5, w=6, values="big", seed=207))
    C.append(_pool("pool_sub", h=5, w=6, values="sub", seed=208))
    # image pool: the 600 x 1000 frame, a 1500 x 1500 one (562,500 threads > 132 * 16 * 256), odd / even / 1-cell
    C.append(_image("image_600x1000", h=600, w=1000, seed=300))
    C.append(_image("image_grid_stride", h=1500, w=1500, seed=301))
    for (h, w), s in (((7, 9), 302), ((8, 10), 303), ((1, 1), 304), ((1, 9), 305), ((9, 1), 306)):
        C.append(_image("image_%dx%d" % (h, w), h=h, w=w, seed=s))
    C.append(_image("image_big", h=5, w=7, values="big", seed=307))
    # pairs: the 600 x 1000 frame's window (2,953,512 threads), the DFF pair, a small shuffled window
    C.append(_pairs("pairs_prod", h=300, w=500, L=19, key=9, n_slots=19, window="first", seed=400))
    C.append(_pairs("pairs_dff", h=48, w=80, L=2, key=0, n_slots=2, window="distinct", seed=401))
    C.append(_pairs("pairs_small", h=3, w=4, L=5, key=3, n_slots=7, seed=402))
    C.append(_pairs("pairs_rot", h=5, w=2, L=6, key=5, n_slots=6, window="rot", seed=403))
    return C


def threads(c):
    """threads the case's grid-stride kernel needs (None for the one-CTA-per-pixel aggregate)"""
    if c["kind"] == "dff":
        return c["h"] * c["w"] * c["c"] // 8
    if c["kind"] == "pool":
        return c["n"] * ((c["h"] + 1) // 2) * ((c["w"] + 1) // 2) * c["c"]
    if c["kind"] == "pool_image":
        return ((c["h"] + 1) // 2) * ((c["w"] + 1) // 2)
    if c["kind"] == "pairs":
        return c["L"] * (c["h"] + 6) * (c["w"] + 8)
    return None

