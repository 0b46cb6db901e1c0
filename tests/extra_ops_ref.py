"""Shared pieces of the conformance suite of csrc/deform.cu and csrc/train_ops.cu (test_extra_ops_conformance_cpu.py /
_gpu.py): fp64 references, per-element error bounds and the case table of the twelve kernels behind `mega_core._C`'s
focal loss, deformable convolution, deformable PSROI pooling, ROIAlign backward and ROIPool.

Decisions. Every value a decision depends on is taken exactly as the kernel computes it:
  * DCN (all four kernels): h = fl(float(h_col*stride - pad + i*dil) + offset) -- one fp32 add, which no compiler can
    contract -- then the gate `h > -1 && w > -1 && h < H && w < W`, floor(h) and the validity of each corner;
  * ROIPool: roundf(fl(r * scale)) (half away from zero), the bin size fl(roi_h / pooled), floorf(fl(ph * bin)) and
    ceilf(fl((ph + 1) * bin)), the clamp to the map, and the strict `>` of the maximum (ties: first index, row-major);
  * ROIAlign backward and PSROI pooling compute their sample positions through chains the compiler may contract into
    FMAs. The reference carries each position as an exact value v and an error bound e (class E below); a decision
    (the gates, `y <= 0`, the truncation, the `y_low >= H - 1` clamp, PSROI's rounded roi corners, its
    `-0.5 / W - 0.5` sample gate, floor and ceil after the clamp, ROIAlign's ceil of the adaptive grid) is taken at v
    and `check_domain` asserts that it is the same everywhere in [v - e, v + e]. A chain of exact operations has e = 0,
    so positions placed on a gate, on an integer or at x.5 are decided exactly;
  * focal loss: the `log(FLT_MIN)` clamp fmaxf(log p, -87.3365f) is continuous; it is applied to the fp64 log p.

Bounds. Everything else runs in fp64. E(v, e) propagates a first-order-exact error bound through each fp32 operation:
a product adds |a| e_b + |b| e_a + e_a e_b, a sum e_a + e_b, a quotient (e_a + |q| e_b) / (|b| - e_b), and every
rounding adds u (|v| + e) (u = 2^-24), except an operation on error-free operands whose exact result is an fp32 number.
So a deterministic chain of n operations gets the familiar sum of u |partial| terms. Each output must satisfy
    |got - ref| <= A[output] * bound,
with A calibrated on an H100 (test_extra_ops_conformance_gpu.py). Per output:
  * deterministic blends: im2col columns (tile, scalar and K-major kernels): lh = h - floor h, hh = 1 - lh,
    w00 = hh hw, ... each rounded once, then w00 v00 + w01 v01 + w10 v10 + w11 v11 (at most 4 roundings), times the
    mask for DCN v2 (one more rounding). PSROI forward: per sample (1 - dx)(1 - dy) v11 + ... (dx, dy carry the
    position's e), the samples summed in order, divided by the count. grad_offset / grad_mask are assigned sums over the
    channels of a deformable group, in channel order: per channel wh = -hw a1 - lw a2 + hw a3 + lw a4,
    (wh col) m, accumulated; grad_mask accumulates col (w00 a1 + ...). The channel sum: a lane sums ceil(P/32) B values,
    5 butterfly levels, one add into out[c]: (ceil(P/32) B + 6) u (sum |x| + |out[c]|).
  * atomic scatters (grad_input of ROIAlign, ROIPool, DCN and PSROI, and PSROI's grad_trans): the order is
    unspecified, so for each element e the reference counts n_e contributions t_j and bounds the accumulation by
    u n_e (|seed_e| + sum_j |t_j|), plus sum_j err(t_j), each term's own chain (ROIAlign (top w) / count, DCN
    w (col m), PSROI w diff_val with diff_val = top_diff / count, grad_trans's
    (u11 dy + u10 (1 - dy) - u01 dy - u00 (1 - dy)) trans_std diff_val roi_width). ROIPool's terms are exact.
  * focal loss: e = __expf(-|x|), whose maximum error the CUDA C++ Programming Guide documents as
    2 + floor(|1.173 x|) ulp (one ulp <= 2 u |value|), with results below 2^-126 flushed to zero; log1pf (1 ulp), the
    divide and the sums of the log-sigmoid identities follow. u^gamma = __expf(gamma log u): its argument carries
    |gamma| e(log u) + one rounding, and the intrinsic adds 2 + floor(1.173 |gamma log u|) ulp, so the term grows with
    |gamma log u|. The bound is relative to the fp64 value plus the 2^-126 floor of every flushed intrinsic; where
    fp32 pow would underflow to 0, the fp64 value is still the reference.
  * ROIPool forward: values and argmax are exact; an empty bin gives 0 and -1.
"""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

U = 2.0 ** -24
FLT_MIN = 2.0 ** -126
F32 = np.float32
LOG_FLT_MIN = float(F32(-87.3365))        # the kernels' fmaxf(log p, -87.3365f)
EXPF_ULP_SLOPE = 1.173                    # __expf: 2 + floor(|1.173 x|) ulp (CUDA C++ Programming Guide)

# A per output (calibration: test_extra_ops_conformance_gpu.py)
A = {"focal_fwd": 2.0, "focal_bwd": 2.0, "im2col": 2.0, "im2col_kq": 2.0, "deform_conv": 2.0, "psroi_fwd": 1.0,
     "roi_align_bwd": 2.0, "roi_pool_bwd": 2.0, "dcn_grad_input": 2.0, "dcn_grad_offset": 2.0, "dcn_grad_mask": 2.0,
     "channel_sum": 1.0, "psroi_grad_input": 2.0, "psroi_grad_trans": 1.0}

# constants of csrc/deform.cu / train_ops.cu / train_ops.cuh (test_extra_ops_conformance_cpu.py reads them back)
K_DCN_MAX_TAPS = 49
K_DCN_PIX = 32
K_DCN_CH = 16
K_ROI_BWD_STRIP = 8
GRID_CAP = 132 * 16                       # grid_dcn / grid_for: at most this many blocks
CHANNEL_SUM_BLOCKS = 132 * 8              # mega_channel_sum_nchw: at most this many blocks of CHANNEL_SUM_WARPS warps
CHANNEL_SUM_WARPS = 8
INSTANTIATIONS = ("focal_loss_kernel<false, false>", "focal_loss_kernel<false, true>",
                  "focal_loss_kernel<true, false>", "focal_loss_kernel<true, true>", "deform_im2col_tile_kernel",
                  "deform_im2col_kernel", "deform_psroi_fwd_kernel", "roi_align_bwd_kernel", "roi_pool_fwd_kernel",
                  "roi_pool_bwd_kernel", "dcn_im2col_kq_kernel", "dcn_col2im_fused_kernel",
                  "channel_sum_nchw_kernel", "deform_psroi_bwd_kernel")


# ------------------------------------------------------------------------------------------------ error arithmetic
def _t(x, like=None):
    if isinstance(x, torch.Tensor):
        return x.double()
    return torch.as_tensor(x, dtype=torch.float64, device=like.device if like is not None else None)


class E:
    """an fp64 value v and a bound e of |kernel's fp32 value - v| (see the module docstring)"""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = _t(v)
        self.e = torch.zeros_like(self.v) if e is None else torch.broadcast_to(_t(e, self.v), self.v.shape)

    @staticmethod
    def _rnd(v, e):
        exact = (e == 0) & (v.float().double() == v)
        return e + torch.where(exact, torch.zeros_like(v), U * (v.abs() + e) + 2.0 ** -150)

    def __add__(self, o):
        o = o if isinstance(o, E) else E(_t(o, self.v))
        v = self.v + o.v
        return E(v, self._rnd(v, self.e + o.e))

    def __sub__(self, o):
        o = o if isinstance(o, E) else E(_t(o, self.v))
        return self + E(-o.v, o.e)

    def __rsub__(self, o):
        return E(_t(o, self.v)) - self

    def __neg__(self):
        return E(-self.v, self.e)

    def __mul__(self, o):
        o = o if isinstance(o, E) else E(_t(o, self.v))
        v = self.v * o.v
        return E(v, self._rnd(v, self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = o if isinstance(o, E) else E(_t(o, self.v))
        v = self.v / o.v
        den = (o.v.abs() - o.e).clamp_min(1e-300)
        return E(v, self._rnd(v, (self.e + v.abs() * o.e) / den))

    def where(self, cond, other):
        other = other if isinstance(other, E) else E(_t(other, self.v).expand_as(self.v))
        return E(torch.where(cond, self.v, other.v), torch.where(cond, self.e, other.e))


def expf_fast(z):
    """__expf(z) (E in, E out): the argument's error propagates, the intrinsic adds 2 + floor(1.173 |z|) ulp, and
    results below 2^-126 may flush to zero"""
    v = torch.exp(z.v)
    grow = torch.expm1(z.e)
    ulps = 2.0 + torch.floor(EXPF_ULP_SLOPE * (z.v.abs() + z.e))
    return E(v, v * grow + 2 * U * ulps * v * (1 + grow) + FLT_MIN)


def log1pf(x):
    """log1pf(x) for x in [0, 1] (1 ulp)"""
    v = torch.log1p(x.v)
    return E(v, x.e / (1 + x.v - x.e).clamp_min(1e-300) + 2 * U * v.abs() + 2.0 ** -149)


def inside(got, ref, bound, a):
    return (got.double() - ref).abs() <= a * bound


def needed_a(got, ref, bound):
    """the smallest A every element passes with"""
    if got.numel() == 0:
        return 0.0
    err = (got.double().to(ref.device) - ref).abs()
    return (err / bound.clamp_min(1e-300)).max().item() if bool((err > 0).any()) else 0.0


# ------------------------------------------------------------------------------------------------ focal loss
def focal_reference(logits, targets, gamma, alpha, d_losses=None):
    """fp64 (ref, bound) of sigmoid_focalloss_forward (d_losses None) or _backward; logits [N, C] fp32, targets [N]"""
    x = E(logits.double())
    n, c = logits.shape
    t = targets.long().view(n, 1).to(logits.device)
    d = torch.arange(c, device=logits.device).view(1, c)
    g32, a32 = float(F32(gamma)), float(F32(alpha))
    one_m_a = float(F32(1.0) - F32(alpha))
    e = expf_fast(E(-x.v.abs()))
    lg = log1pf(e)
    inv = E(1.0 + 0 * x.v) / (e + 1.0)
    p = inv.where(x.v >= 0, e * inv)
    log_p = -(E(torch.clamp(-x.v, min=0)) + lg)
    log_1mp = -(E(torch.clamp(x.v, min=0)) + lg)
    clamped = E(torch.clamp(log_p.v, min=LOG_FLT_MIN), log_p.e)
    pow_1mp = expf_fast(log_1mp * g32)
    pow_p = expf_fast(log_p * g32)
    if d_losses is None:
        pos = (pow_1mp * (-a32)) * clamped
        neg = (pow_p * (-one_m_a)) * log_1mp
    else:
        f = (1.0 - p) - (p * g32) * clamped
        pos = (pow_1mp * (-a32)) * f
        gterm = ((log_1mp * (1.0 - p)) * g32) - p
        neg = (pow_p * (-one_m_a)) * gterm
    is_pos = (t == d + 1)
    is_neg = (~is_pos) & (t >= 0)
    r = pos.where(is_pos, neg.where(is_neg, torch.zeros_like(x.v)))
    if d_losses is not None:
        r = r * E(d_losses.double())
    return r.v, r.e


# ------------------------------------------------------------------------------------------------ DCN sampling
def dcn_positions(offset, b, dg, kh, kw, ho, wo, ph, pw, sh, sw, dh, dw):
    """fp32 sample positions (h, w) [B, dg, taps, Ho, Wo] exactly as the kernels compute them, as fp64 tensors"""
    off = offset.float().view(b, dg, kh * kw, 2, ho, wo)
    dev = offset.device
    i = torch.arange(kh, device=dev).repeat_interleave(kw).view(1, 1, -1, 1, 1)
    j = torch.arange(kw, device=dev).repeat(kh).view(1, 1, -1, 1, 1)
    hc = torch.arange(ho, device=dev).view(1, 1, 1, -1, 1)
    wc = torch.arange(wo, device=dev).view(1, 1, 1, 1, -1)
    hb = (hc * sh - ph + i * dh).float()
    wb = (wc * sw - pw + j * dw).float()
    return (hb + off[:, :, :, 0]).double(), (wb + off[:, :, :, 1]).double()


def dcn_geometry(h, w, height, width, mode="kernel"):
    """gate, corner validity [4] and E weights of the four corners at fp32 positions h, w"""
    gate = (h > -1) & (w > -1) & (h < height) & (w < width)
    hl, wl = torch.floor(h), torch.floor(w)
    lh, lw = E(h) - E(hl), E(w) - E(wl)
    hh, hw = 1.0 - lh, 1.0 - lw
    ok = [gate & (hl >= 0) & (wl >= 0), gate & (hl >= 0) & (wl + 1 <= width - 1),
          gate & (hl + 1 <= height - 1) & (wl >= 0), gate & (hl + 1 <= height - 1) & (wl + 1 <= width - 1)]
    if mode == "drop_far_corner":                 # deliberate bug: the bottom / right corner lost at the border
        ok[3] = ok[3] & (hl + 1 < height - 1) & (wl + 1 < width - 1)
    wts = [hh * hw, hh * lw, lh * hw, lh * lw]
    if mode == "swap_w01_w10":
        wts[1], wts[2] = wts[2], wts[1]
    idx = [hl * width + wl, hl * width + wl + 1, (hl + 1) * width + wl, (hl + 1) * width + wl + 1]
    idx = [torch.where(o, ix, torch.zeros_like(ix)).long() for o, ix in zip(ok, idx)]
    return gate, ok, idx, wts


def im2col_reference(x, offset, mask, kh, kw, ph, pw, sh, sw, dh, dw, dg, mode="kernel"):
    """fp64 (cols, bound), both [B, C, taps, Ho, Wo]: the column value of (channel, tap) at each output pixel"""
    b, c, height, width = x.shape
    ho = (height + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    wo = (width + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    taps, cpg = kh * kw, c // dg
    h, w = dcn_positions(offset, b, dg, kh, kw, ho, wo, ph, pw, sh, sw, dh, dw)
    gate, ok, idx, wts = dcn_geometry(h, w, height, width, mode)
    xs = x.double().view(b, dg, cpg, height * width)
    val = None
    for k in range(4):
        vk = torch.gather(xs, 3, idx[k].view(b, dg, 1, -1).expand(b, dg, cpg, -1)).view(b, dg, cpg, taps, ho, wo)
        vk = torch.where(ok[k].unsqueeze(2), vk, torch.zeros_like(vk))
        term = E(wts[k].v.unsqueeze(2), wts[k].e.unsqueeze(2)) * E(vk)
        val = term if val is None else val + term
    if mask is not None:
        val = val * E(mask.double().view(b, dg, 1, taps, ho, wo))
    z = gate.unsqueeze(2).expand_as(val.v)
    return (torch.where(z, val.v, torch.zeros_like(val.v)).reshape(b, c, taps, ho, wo),
            torch.where(z, val.e, torch.zeros_like(val.e)).reshape(b, c, taps, ho, wo))


# ------------------------------------------------------------------------------------------------ scatter bound
class Scatter:
    """accumulates terms t_j (E) into flat target indices: the atomic bound u n_e (|seed| + sum |t|) + sum err(t)"""

    def __init__(self, numel, dev, seed=None):
        z = torch.zeros(numel, dtype=torch.float64, device=dev)
        self.sum, self.abs, self.err, self.n = z.clone(), z.clone(), z.clone(), z.clone()
        self.seed = seed.double().reshape(-1).to(dev) if seed is not None else z.clone()

    def add(self, idx, term, mask=None):
        idx = idx.reshape(-1).long()
        v, e = term.v.reshape(-1), term.e.reshape(-1)
        if mask is not None:
            m = mask.reshape(-1)
            idx, v, e = idx[m], v[m], e[m]
        self.sum.index_add_(0, idx, v)
        self.abs.index_add_(0, idx, v.abs())
        self.err.index_add_(0, idx, e)
        self.n.index_add_(0, idx, torch.ones_like(v))

    def result(self):
        return self.seed + self.sum, self.err + U * self.n * (self.seed.abs() + self.abs)


# ------------------------------------------------------------------------------------------------ DCN backward
def col2im_reference(gcols, x, offset, mask, kh, kw, ph, pw, sh, sw, dh, dw, dg, ldp, seed_grad_in, mode="kernel"):
    """fp64 references and bounds of mega_deform_col2im_fused: (grad_input, bound), (grad_offset, bound),
    (grad_mask, bound) -- grad_mask None without a mask. gcols: [C*taps, B*ldp]."""
    b, c, height, width = x.shape
    ho = (height + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    wo = (width + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    taps, cpg, pt = kh * kw, c // dg, ho * wo
    h, w = dcn_positions(offset, b, dg, kh, kw, ho, wo, ph, pw, sh, sw, dh, dw)
    gate, ok, idx, wts = dcn_geometry(h, w, height, width)
    hl, wl = torch.floor(h), torch.floor(w)
    lh, lw = E(h) - E(hl), E(w) - E(wl)
    hh, hw = 1.0 - lh, 1.0 - lw
    m = E(mask.double().view(b, dg, taps, ho, wo)) if mask is not None else E(torch.ones_like(h))
    gc = gcols.double().view(c, taps, b, ldp)[..., :pt].permute(2, 0, 1, 3).reshape(b, dg, cpg, taps, ho, wo)
    xs = x.double().view(b, dg, cpg, height * width)
    zero = torch.zeros_like(h)
    acc_h = acc_w = acc_m = None
    sc = Scatter(x.numel(), x.device, seed_grad_in)
    base = (torch.arange(b, device=x.device).view(b, 1, 1) * c + torch.arange(dg, device=x.device).view(1, dg, 1) * cpg)
    for cc in range(cpg):
        col = E(gc[:, :, cc])
        a = [E(torch.where(ok[k], xs[:, :, cc].gather(2, idx[k].view(b, dg, -1)).view_as(h), zero)) for k in range(4)]
        wh = (((-hw) * a[0]) - lw * a[1]) + hw * a[2] + lw * a[3]
        ww = (((-hh) * a[0]) + hh * a[1]) - lh * a[2] + lh * a[3]
        th, tw = (wh * col) * m, (ww * col) * m
        if mode == "offset_without_mask":
            th, tw = wh * col, ww * col
        blend = wts[0] * a[0] + wts[1] * a[1] + wts[2] * a[2] + wts[3] * a[3]
        tm = col * blend
        acc_h = th if acc_h is None else acc_h + th
        acc_w = tw if acc_w is None else acc_w + tw
        acc_m = tm if acc_m is None else acc_m + tm
        top = col * m
        plane = ((base + cc) * height * width).view(b, dg, 1, 1, 1)
        for k in range(4):
            sc.add(plane + idx[k], wts[k] * top, ok[k])
    g_in, g_in_b = sc.result()
    gz = gate
    go_v = torch.stack([torch.where(gz, acc_h.v, zero), torch.where(gz, acc_w.v, zero)], 3)
    go_e = torch.stack([torch.where(gz, acc_h.e, zero), torch.where(gz, acc_w.e, zero)], 3)
    shape_off = (b, dg * 2 * taps, ho, wo)
    out = [(g_in.view(x.shape), g_in_b.view(x.shape)), (go_v.reshape(shape_off), go_e.reshape(shape_off)), None]
    if mask is not None:
        out[2] = (torch.where(gz, acc_m.v, zero).reshape(b, dg * taps, ho, wo),
                  torch.where(gz, acc_m.e, zero).reshape(b, dg * taps, ho, wo))
    return out


def channel_sum_reference(x, seed):
    """fp64 (out, bound) of mega_channel_sum_nchw on x [B, C, P] into out [C] seeded with `seed`"""
    b, c, p = x.shape
    xd = x.double()
    s = xd.sum((0, 2)) + seed.double()
    depth = math.ceil(p / 32) * b + 6
    return s, depth * U * (xd.abs().sum((0, 2)) + seed.double().abs())


# ------------------------------------------------------------------------------------------------ ROIAlign backward
def _f32(x):
    return float(F32(x))


def roi_align_bwd_reference(grad, rois, scale, pooled_h, pooled_w, batch, channels, height, width, sampling_ratio,
                            seed=None, mode="kernel"):
    """fp64 (grad_input, bound) of mega_roi_align_backward_nchw, and the positions' decision record for check_domain"""
    dev = grad.device
    sc = Scatter(batch * channels * height * width, dev, seed)
    decisions = []
    r32 = rois.float().cpu().numpy()
    for n in range(rois.shape[0]):
        rb = int(r32[n, 0])
        s = F32(scale)
        sw_, sh_, ew_, eh_ = (E(torch.tensor(float(r32[n, k]), dtype=torch.float64, device=dev)) * float(s)
                              for k in (1, 2, 3, 4))
        rw_, rh_ = ew_ - sw_, eh_ - sh_
        rw = E(max(rw_.v.item(), 1.0), rw_.e if rw_.v.item() > 1.0 else 0.0)
        rh = E(max(rh_.v.item(), 1.0), rh_.e if rh_.v.item() > 1.0 else 0.0)
        bh, bw = rh / float(pooled_h), rw / float(pooled_w)
        if sampling_ratio > 0:
            gh = gw = sampling_ratio
        else:
            qh, qw = rh / float(pooled_h), rw / float(pooled_w)
            decisions.append(("ceil", qh))
            decisions.append(("ceil", qw))
            gh, gw = int(math.ceil(qh.v.item())), int(math.ceil(qw.v.item()))
        cnt = float(gh * gw)
        php = torch.arange(pooled_h, device=dev, dtype=torch.float64).view(-1, 1, 1, 1)
        pwp = torch.arange(pooled_w, device=dev, dtype=torch.float64).view(1, -1, 1, 1)
        iy = torch.arange(gh, device=dev, dtype=torch.float64).view(1, 1, -1, 1)
        ix = torch.arange(gw, device=dev, dtype=torch.float64).view(1, 1, 1, -1)
        y = (sh_ + E(php) * bh) + (E(iy + 0.5) * bh) / float(gh)
        x = (sw_ + E(pwp) * bw) + (E(ix + 0.5) * bw) / float(gw)
        y = E(y.v.expand(pooled_h, pooled_w, gh, gw), y.e.expand(pooled_h, pooled_w, gh, gw))
        x = E(x.v.expand(pooled_h, pooled_w, gh, gw), x.e.expand(pooled_h, pooled_w, gh, gw))
        decisions += [("roi_align_y", y, height), ("roi_align_y", x, width)]
        valid = ~((y.v < -1.0) | (y.v > height) | (x.v < -1.0) | (x.v > width))
        yc = E(torch.clamp(y.v, min=0.0), torch.where(y.v <= 0, torch.zeros_like(y.e), y.e))
        xc = E(torch.clamp(x.v, min=0.0), torch.where(x.v <= 0, torch.zeros_like(x.e), x.e))
        yl, xl = torch.trunc(yc.v), torch.trunc(xc.v)
        ylim, xlim = yl >= height - 1, xl >= width - 1
        if mode == "drop_bottom_border":          # deliberate bug: samples clamped to the last row are lost
            valid = valid & ~ylim
        yl = torch.where(ylim, torch.full_like(yl, height - 1), yl)
        xl = torch.where(xlim, torch.full_like(xl, width - 1), xl)
        yh = torch.where(ylim, yl, yl + 1)
        xh = torch.where(xlim, xl, xl + 1)
        yc = yc.where(~ylim, yl)
        xc = xc.where(~xlim, xl)
        ly, lx = yc - E(yl), xc - E(xl)
        hy, hx = 1.0 - ly, 1.0 - lx
        wts = [hy * hx, hy * lx, ly * hx, ly * lx]
        offs = [yl * width + xl, yl * width + xh, yh * width + xl, yh * width + xh]
        c_hi = channels - 1 if mode == "strip_tail_loses_last" else channels
        shape = (c_hi, pooled_h, pooled_w, gh, gw)
        top = E(grad[n, :c_hi].double().view(c_hi, pooled_h, pooled_w, 1, 1).expand(shape))
        plane = ((rb * channels + torch.arange(c_hi, device=dev)) * height * width).view(-1, 1, 1, 1, 1)
        for k in range(4):
            t = (top * E(wts[k].v.expand(shape), wts[k].e.expand(shape))) / cnt
            sc.add(offs[k].long() + plane, t, valid.expand(shape))
    g, bnd = sc.result()
    shape = (batch, channels, height, width)
    return g.view(shape), bnd.view(shape), decisions


# ------------------------------------------------------------------------------------------------ ROIPool
def _roundf(v):
    """roundf: half away from zero"""
    return np.sign(v) * np.floor(np.abs(v) + F32(0.5))


def roi_pool_reference(x, rois, scale, pooled_h, pooled_w, mode="kernel"):
    """exact (out [K, C, ph, pw] fp32, argmax int32) of mega_roi_pool_forward; numpy, x on any device"""
    xn = x.float().cpu().numpy()
    r = rois.float().cpu().numpy()
    k = r.shape[0]
    n, c, height, width = xn.shape
    out = np.zeros((k, c, pooled_h, pooled_w), F32)
    arg = np.full((k, c, pooled_h, pooled_w), -1, np.int32)
    s = F32(scale)
    for i in range(k):
        b = int(r[i, 0])
        sw, sh, ew, eh = (int(_roundf(F32(r[i, j] * s))) for j in (1, 2, 3, 4))
        rw, rh = max(ew - sw + 1, 1), max(eh - sh + 1, 1)
        bh, bw = F32(F32(rh) / F32(pooled_h)), F32(F32(rw) / F32(pooled_w))
        for ph in range(pooled_h):
            hs = int(np.floor(F32(F32(ph) * bh)))
            he = int(np.ceil(F32(F32(ph + 1) * bh)))
            hs, he = min(max(hs + sh, 0), height), min(max(he + sh, 0), height)
            for pw in range(pooled_w):
                ws = int(np.floor(F32(F32(pw) * bw)))
                we = int(np.ceil(F32(F32(pw + 1) * bw)))
                ws, we = min(max(ws + sw, 0), width), min(max(we + sw, 0), width)
                if he <= hs or we <= ws:
                    continue
                win = xn[b, :, hs:he, ws:we].reshape(c, -1)
                j = win.argmax(1) if mode != "last_max" else win.shape[1] - 1 - win[:, ::-1].argmax(1)
                out[i, :, ph, pw] = win[np.arange(c), j]
                arg[i, :, ph, pw] = (j // (we - ws) + hs) * width + (j % (we - ws) + ws)
    return torch.from_numpy(out), torch.from_numpy(arg)


def roi_pool_bwd_reference(grad, argmax, rois, channels, height, width, batch, seed=None):
    """fp64 (grad_input, bound) of mega_roi_pool_backward"""
    dev = grad.device
    k, c, php, pwp = grad.shape
    sc = Scatter(batch * channels * height * width, dev, seed)
    rb = rois[:, 0].long().to(dev).view(k, 1, 1, 1)
    cc = torch.arange(c, device=dev).view(1, c, 1, 1)
    am = argmax.long().to(dev)
    idx = (rb * channels + cc) * height * width + am
    sc.add(torch.where(am >= 0, idx, torch.zeros_like(idx)), E(grad.double()), am >= 0)
    g, bnd = sc.result()
    return g.view(batch, channels, height, width), bnd.view(batch, channels, height, width)


# ------------------------------------------------------------------------------------------------ PSROI pooling
def psroi_geometry(rois, trans, no_trans, scale, output_dim, group_size, pooled, part_size, spp, trans_std,
                   num_classes):
    """per (roi, ctop, ph, pw, ih, iw): E positions (w, h), the input channel and the trans indices (fp64, torch)"""
    r = rois.float().cpu().numpy()
    k = r.shape[0]
    cec = output_dim if no_trans else output_dim // num_classes
    s = float(F32(scale))
    rs = lambda v: float(_roundf(F32(v)))                                     # noqa: E731
    sw_ = E(torch.tensor([rs(r[i, 1]) for i in range(k)], dtype=torch.float64)) * s - 0.5
    sh_ = E(torch.tensor([rs(r[i, 2]) for i in range(k)], dtype=torch.float64)) * s - 0.5
    ew_ = E(torch.tensor([rs(r[i, 3]) + 1.0 for i in range(k)], dtype=torch.float64)) * s - 0.5
    eh_ = E(torch.tensor([rs(r[i, 4]) + 1.0 for i in range(k)], dtype=torch.float64)) * s - 0.5
    c01 = float(F32(0.1))

    def clamp01(d):
        return E(torch.clamp(d.v, min=c01), torch.where(d.v > c01, d.e, torch.zeros_like(d.e)))
    rw, rh = clamp01(ew_ - sw_), clamp01(eh_ - sh_)
    bh, bw = rh / float(pooled), rw / float(pooled)
    sbh, sbw = bh / float(spp), bw / float(spp)
    ph = torch.arange(pooled, dtype=torch.float64)
    part = torch.floor(torch.tensor([float(F32(F32(F32(p) / F32(pooled)) * F32(part_size))) for p in range(pooled)],
                                    dtype=torch.float64)).long()
    grp = torch.tensor([min(max(int(np.floor(F32(F32(F32(p) * F32(group_size)) / F32(pooled)))), 0), group_size - 1)
                        for p in range(pooled)])
    ctop = torch.arange(output_dim).view(1, -1, 1, 1)
    cls = ctop // cec
    kk = torch.arange(k).view(-1, 1, 1, 1)
    pth, ptw = part.view(1, 1, -1, 1), part.view(1, 1, 1, -1)
    t_x = (((kk * num_classes + cls) * 2) * part_size + pth) * part_size + ptw
    t_y = (((kk * num_classes + cls) * 2 + 1) * part_size + pth) * part_size + ptw
    if no_trans:
        tx = ty = E(torch.zeros(k, output_dim, pooled, pooled, dtype=torch.float64))
    else:
        tf = trans.float().cpu().reshape(-1).double()
        tx, ty = E(tf[t_x]) * float(F32(trans_std)), E(tf[t_y]) * float(F32(trans_std))
    v4 = lambda e: E(e.v.view(-1, 1, 1, 1), e.e.view(-1, 1, 1, 1))           # noqa: E731
    ws = (E(ph.view(1, 1, 1, -1)) * v4(bw) + v4(sw_)) + tx * v4(rw)
    hs = (E(ph.view(1, 1, -1, 1)) * v4(bh) + v4(sh_)) + ty * v4(rh)
    sp = torch.arange(spp, dtype=torch.float64)
    w = E(ws.v.unsqueeze(-1).unsqueeze(-1), ws.e.unsqueeze(-1).unsqueeze(-1)) + \
        E(sp.view(1, -1)) * E(sbw.v.view(-1, 1, 1, 1, 1, 1), sbw.e.view(-1, 1, 1, 1, 1, 1))
    h = E(hs.v.unsqueeze(-1).unsqueeze(-1), hs.e.unsqueeze(-1).unsqueeze(-1)) + \
        E(sp.view(-1, 1)) * E(sbh.v.view(-1, 1, 1, 1, 1, 1), sbh.e.view(-1, 1, 1, 1, 1, 1))
    shape = (k, output_dim, pooled, pooled, spp, spp)
    w, h = E(w.v.expand(shape), w.e.expand(shape)), E(h.v.expand(shape), h.e.expand(shape))
    chan = (ctop * group_size + grp.view(1, 1, -1, 1)) * group_size + grp.view(1, 1, 1, -1)
    return dict(w=w, h=h, chan=chan.expand(k, output_dim, pooled, pooled), t_x=t_x.expand(k, output_dim, pooled, pooled),
                t_y=t_y.expand(k, output_dim, pooled, pooled), rw=rw, rh=rh,
                batch=torch.tensor([int(r[i, 0]) for i in range(k)]))


def _psroi_samples(g, height, width, mode="kernel"):
    w, h = g["w"], g["h"]
    keep = ~((w.v < -0.5) | (w.v > width - 0.5) | (h.v < -0.5) | (h.v > height - 0.5))
    wc = E(torch.clamp(w.v, 0.0, width - 1.0), torch.where((w.v > 0) & (w.v < width - 1), w.e, torch.zeros_like(w.e)))
    hc = E(torch.clamp(h.v, 0.0, height - 1.0), torch.where((h.v > 0) & (h.v < height - 1), h.e, torch.zeros_like(h.e)))
    if mode == "unclamped_h":
        hc = h
    x0, x1 = torch.floor(wc.v), torch.ceil(wc.v)
    y0, y1 = torch.floor(hc.v), torch.ceil(hc.v)
    dx, dy = wc - E(x0), hc - E(y0)
    return keep, x0.long(), x1.long(), y0.long(), y1.long(), dx, dy


def psroi_fwd_reference(x, rois, trans, no_trans, scale, output_dim, group_size, pooled, part_size, spp, trans_std,
                       mode="kernel"):
    """fp64 (out, bound, top_count) of mega_deform_psroi_pooling_forward, with the decision record"""
    n, c, height, width = x.shape
    num_classes = 1 if no_trans else trans.shape[1] // 2
    g = psroi_geometry(rois, trans, no_trans, scale, output_dim, group_size, pooled, part_size, spp, trans_std,
                       num_classes)
    keep, x0, x1, y0, y1, dx, dy = _psroi_samples(g, height, width)
    xd = x.double().cpu().reshape(-1)
    base = ((g["batch"].view(-1, 1, 1, 1) * c + g["chan"]) * height * width).unsqueeze(-1).unsqueeze(-1)
    vals = [E(xd[(base + yy * width + xx).clamp(0, xd.numel() - 1)]) for yy, xx in ((y0, x0), (y1, x0), (y0, x1),
                                                                                    (y1, x1))]
    s = ((1.0 - dx) * (1.0 - dy)) * vals[0] + ((1.0 - dx) * dy) * vals[1] + (dx * (1.0 - dy)) * vals[2] + \
        (dx * dy) * vals[3]
    s = s.where(keep, 0.0)
    acc = None
    spp_ = s.v.shape[-1]
    for ih in range(spp_):
        for iw in range(spp_):
            t = E(s.v[..., ih, iw], s.e[..., ih, iw])
            acc = t if acc is None else acc + t
    cnt = keep.sum((-1, -2)).double()
    div = cnt[:, :, :1, :1].expand_as(cnt) if mode == "first_bin_count" else cnt
    out = acc / E(div.clamp_min(1))
    out = out.where(cnt > 0, 0.0)
    decisions = [("psroi", g["w"], width), ("psroi", g["h"], height)]
    return out.v, out.e, cnt, decisions


def psroi_bwd_reference(top_diff, top_count, x, rois, trans, no_trans, scale, output_dim, group_size, pooled,
                        part_size, spp, trans_std, seed_in=None, seed_trans=None, mode="kernel"):
    """fp64 ((input_grad, bound), (trans_grad, bound) or None) of mega_deform_psroi_pooling_backward"""
    n, c, height, width = x.shape
    num_classes = 1 if no_trans else trans.shape[1] // 2
    g = psroi_geometry(rois, trans, no_trans, scale, output_dim, group_size, pooled, part_size, spp, trans_std,
                       num_classes)
    keep, x0, x1, y0, y1, dx, dy = _psroi_samples(g, height, width, mode)
    live = (top_count.cpu() > 0).view(*top_count.shape, 1, 1).expand_as(keep)
    keep = keep & live
    dv = E(top_diff.double().cpu()) / E(top_count.double().cpu().clamp_min(1))
    dv = E(dv.v.unsqueeze(-1).unsqueeze(-1).expand_as(dx.v), dv.e.unsqueeze(-1).unsqueeze(-1).expand_as(dx.v))
    base = ((g["batch"].view(-1, 1, 1, 1) * c + g["chan"]) * height * width).unsqueeze(-1).unsqueeze(-1)
    sc = Scatter(x.numel(), "cpu", seed_in.cpu() if seed_in is not None else None)
    terms = [((1.0 - dx) * (1.0 - dy), y0, x0), ((1.0 - dx) * dy, y1, x0), (dx * (1.0 - dy), y0, x1), (dx * dy, y1, x1)]
    for wgt, yy, xx in terms:
        sc.add((base + yy * width + xx).clamp(0, x.numel() - 1), wgt * dv, keep)
    gi, gib = sc.result()
    res = [(gi.view(x.shape), gib.view(x.shape)), None]
    if not no_trans:
        xd = x.double().cpu().reshape(-1)
        u = {}
        for key, (yy, xx) in (("00", (y0, x0)), ("01", (y1, x0)), ("10", (y0, x1)), ("11", (y1, x1))):
            u[key] = E(xd[(base + yy * width + xx).clamp(0, xd.numel() - 1)])
        tstd = float(F32(trans_std))
        ddx = ((((u["11"] * dy) + u["10"] * (1.0 - dy)) - u["01"] * dy) - u["00"] * (1.0 - dy)) * tstd * dv
        ddy = ((((u["11"] * dx) + u["01"] * (1.0 - dx)) - u["10"] * dx) - u["00"] * (1.0 - dx)) * tstd * dv
        rw = E(g["rw"].v.view(-1, 1, 1, 1, 1, 1), g["rw"].e.view(-1, 1, 1, 1, 1, 1))
        rh = E(g["rh"].v.view(-1, 1, 1, 1, 1, 1), g["rh"].e.view(-1, 1, 1, 1, 1, 1))
        ddx, ddy = ddx * rw, ddy * rh
        st = Scatter(trans.numel(), "cpu", seed_trans.cpu() if seed_trans is not None else None)
        sh6 = lambda t: t.unsqueeze(-1).unsqueeze(-1).expand_as(keep)         # noqa: E731
        st.add(sh6(g["t_x"]), ddx, keep)
        st.add(sh6(g["t_y"]), ddy, keep)
        gt, gtb = st.result()
        res[1] = (gt.view(trans.shape), gtb.view(trans.shape))
    return res


# ------------------------------------------------------------------------------------------------ domain
def decisions_stable(decisions):
    """True when every recorded decision is the same over [v - e, v + e] (e = 0: taken on the exact value)"""
    for d in decisions:
        kind, x = d[0], d[1]
        lo, hi = x.v - x.e, x.v + x.e
        if kind == "ceil":
            if not bool((torch.ceil(lo) == torch.ceil(hi)).all()):
                return False
        elif kind == "roi_align_y":
            n = d[2]
            for t in (-1.0, 0.0, float(n)):
                if not bool(((lo < t) == (hi < t)).all() & ((lo <= t) == (hi <= t)).all()):
                    return False
            lc, hc = lo.clamp_min(0), hi.clamp_min(0)
            if not bool((torch.trunc(lc) == torch.trunc(hc)).all()):
                return False
        elif kind == "psroi":
            n = d[2]
            for t in (-0.5, n - 0.5):
                if not bool(((lo < t) == (hi < t)).all() & ((lo > t) == (hi > t)).all()):
                    return False
            lc, hc = lo.clamp(0, n - 1), hi.clamp(0, n - 1)
            if not bool((torch.floor(lc) == torch.floor(hc)).all() & (torch.ceil(lc) == torch.ceil(hc)).all()):
                return False
    return True
