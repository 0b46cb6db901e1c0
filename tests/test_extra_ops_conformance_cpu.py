"""CPU half of the conformance suite of csrc/deform.cu and csrc/train_ops.cu (references: extra_ops_ref.py):

  1. the fp64 references equal the anchored oracles at fp64 to 1e-12 on small cases (torchvision's deform_conv2d and
     roi_pool, oracle/train_ops_oracle.py's restatements and their autograd, mega_oracle's focal loss and PSROI);
  2. the g++ builds of the kernels' bodies (tests/native/train_ops_host.cpp for train_ops.cuh, dcn_sample_host.cpp for
     the tile kernel's geometry and blend) and an fp32 emulation of the focal-loss kernel lie inside the bounds;
  3. the bounds reject deliberate bugs;
  4. the limits the references restate match the source;
  5. no wrapper hands `ptr` a temporary: `_lib.ptr` keeps no reference, so a converted copy made in the argument list
     is freed before the kernel runs and its block can be reused by the next conversion.
"""
import ast
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

import extra_ops_ref as R

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
CSRC = os.path.join(ROOT, "mega.pytorch_b200", "csrc")
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mega_oracle as mo  # noqa: E402
import train_ops_oracle as to  # noqa: E402
from test_train_ops_cpu import host_lib  # noqa: E402

AMAX = max(R.A.values())


def _close(a, b, tol=1e-12):
    scale = max(1.0, b.abs().max().item())
    assert (a - b).abs().max().item() <= tol * scale, (a - b).abs().max().item()


def _dyadic(t, bits=6):
    """values with few mantissa bits, so that fp32 sums of them are exact"""
    return torch.round(t * 2 ** bits) / 2 ** bits


# ------------------------------------------------------------------------------------------------ 1. oracle anchors
@pytest.mark.parametrize("bwd", [False, True])
def test_focal_reference_equals_oracle(bwd):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(64, 5, generator=g) * 4).float()
    t = torch.randint(-1, 6, (64,), generator=g)
    if not bwd:
        ref, _ = R.focal_reference(x, t, 1.5, 0.25)
        _close(ref, mo.sigmoid_focal_loss(x.double(), t, 1.5, 0.25))
    else:
        dl = torch.randn(64, 5, generator=g).float()
        ref, _ = R.focal_reference(x, t, 2.0, 0.25, dl)
        xl = x.double().requires_grad_(True)
        (mo.sigmoid_focal_loss(xl, t, 2.0, 0.25) * dl.double()).sum().backward()
        _close(ref, xl.grad, 1e-10)


def _dcn_inputs(seed, b=2, c=4, h=7, w=8, k=3, dg=2, modulated=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, c, h, w, generator=g).float()
    off = _dyadic(torch.randn(b, dg * 2 * k * k, h, w, generator=g) * 2).float()
    m = torch.rand(b, dg * k * k, h, w, generator=g).float() if modulated else None
    return x, off, m


def test_im2col_reference_equals_torchvision():
    import torchvision
    x, off, m = _dcn_inputs(2)
    cols, _ = R.im2col_reference(x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2)
    wt = torch.randn(6, 4, 3, 3, generator=torch.Generator().manual_seed(3)).double()
    out = torch.einsum("ok,bkp->bop", wt.reshape(6, 36), cols.reshape(2, 36, 56)).view(2, 6, 7, 8)
    _close(out, torchvision.ops.deform_conv2d(x.double(), off.double(), wt, padding=1, mask=m.double()))


def test_col2im_reference_equals_autograd():
    x, off, m = _dcn_inputs(4)
    k, dg, ldp = 3, 2, 56
    gcols = torch.randn(4 * 9, 2 * ldp, generator=torch.Generator().manual_seed(5)).float()
    (gi, _), (go, _), (gm, _) = R.col2im_reference(gcols, x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, dg, ldp, None)
    xl, ml = x.double().requires_grad_(True), m.double().requires_grad_(True)
    ol = off.double().requires_grad_(True)
    cols, _ = R.im2col_reference(xl.detach(), off, ml.detach(), 3, 3, 1, 1, 1, 1, 1, 1, dg)
    # autograd of the oracle's sampling (the same value as the column): d/d(x, offset, mask) of sum(cols * gcols)
    eye = torch.eye(4 * 9, dtype=torch.float64).view(4 * 9, 4, 3, 3)
    out = to.deform_conv2d(xl, ol, ml, eye, None, (1, 1), (1, 1), (1, 1), 1, dg)       # [B, C*taps, Ho, Wo]
    gc = gcols.double().view(36, 2, ldp).permute(1, 0, 2).reshape(2, 36, 7, 8)
    (out * gc).sum().backward()
    _close(cols.reshape(2, 36, 7, 8), out.detach())
    _close(gi, xl.grad)
    _close(go, ol.grad, 1e-11)
    _close(gm, ml.grad)


def _rois(seed, k, w_img, h_img, n_img=2):
    g = torch.Generator().manual_seed(seed)
    x1 = torch.rand(k, generator=g) * w_img * 0.7 - 3
    y1 = torch.rand(k, generator=g) * h_img * 0.7 - 3
    x2 = x1 + torch.rand(k, generator=g) * w_img * 0.6 + 1
    y2 = y1 + torch.rand(k, generator=g) * h_img * 0.6 + 1
    b = torch.randint(0, n_img, (k,), generator=g).float()
    return torch.stack([b, x1, y1, x2, y2], 1).float()


def _exact_rois(seed, k, bins, n_img=2):
    """rois whose sample positions are exact in fp32 at spatial scale 0.5: corners on a 1/2 grid and bin sizes (in
    scaled units) from `bins`, so the adaptive grid is a power of 2"""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for _ in range(k):
        bh, bw = (bins[int(torch.randint(0, len(bins), (1,), generator=g))] for _ in range(2))
        x1, y1 = (float(torch.randint(-6, 20, (1,), generator=g)) / 2 for _ in range(2))
        rows.append([float(torch.randint(0, n_img, (1,), generator=g)), x1, y1, x1 + 2 * bw * 2, y1 + 2 * bh * 3])
    return torch.tensor(rows).float()


@pytest.mark.parametrize("sr", [0, 2])
def test_roi_align_bwd_reference_equals_autograd(sr):
    rois = _exact_rois(6, 5, (1.5, 2.0, 3.5, 4.0))
    grad = torch.randn(5, 3, 3, 2, generator=torch.Generator().manual_seed(7)).float()
    ref, _, _ = R.roi_align_bwd_reference(grad, rois, 0.5, 3, 2, 2, 3, 12, 16, sr)
    xl = torch.zeros(2, 3, 12, 16, dtype=torch.float64, requires_grad=True)
    (to.roi_align(xl, rois, 0.5, 3, 2, sr) * grad.double()).sum().backward()
    _close(ref, xl.grad)


def test_roi_pool_reference_equals_torchvision():
    import torchvision
    x = torch.randn(2, 3, 12, 16, generator=torch.Generator().manual_seed(8)).float()
    rois = _rois(9, 7, 32, 24)
    out, arg = R.roi_pool_reference(x, rois, 0.5, 3, 4)
    tv = torchvision.ops.roi_pool(x, rois, (3, 4), 0.5)
    assert torch.equal(out, tv)
    o2, a2 = to.roi_pool(x, rois, 0.5, 3, 4)
    assert torch.equal(arg, a2)


@pytest.mark.parametrize("no_trans", [True, False])
def test_psroi_references_equal_oracles(no_trans):
    g = torch.Generator().manual_seed(10)
    gs, od, ps, part, spp, std = 2, 2, 2, 2, 2, 0.25
    x = torch.randn(2, od * gs * gs, 10, 12, generator=g).float()
    # integer corners with (x2 + 1 - x1) a multiple of 8: every position is exact in fp32 at scale 1/4
    x1 = torch.randint(-8, 40, (3, 2), generator=g).float()
    ext = torch.randint(1, 5, (3, 2), generator=g).float() * 8 - 1
    rois = torch.cat([torch.tensor([[0.0], [1.0], [1.0]]), x1, x1 + ext], 1)
    trans = _dyadic(torch.randn(3, 2, part, part, generator=g), 3).float()
    out, _, cnt, _ = R.psroi_fwd_reference(x, rois, trans, no_trans, 0.25, od, gs, ps, part, spp, std)
    o_ref, c_ref = to.deform_psroi_pool(x.double(), rois, trans.double(), no_trans, 0.25, od, gs, ps, part, spp, std)
    assert torch.equal(cnt.float(), c_ref)
    _close(out, o_ref.detach())
    o2, c2 = mo.deform_psroi_pool(x, rois, trans, no_trans, 0.25, od, gs, ps, part, spp, std)
    assert torch.equal(cnt.float(), c2)
    og = torch.randn(3, od, ps, ps, generator=g).float()
    (gi, _), gt = R.psroi_bwd_reference(og, cnt.float(), x, rois, trans, no_trans, 0.25, od, gs, ps, part, spp, std)
    xl = x.double().requires_grad_(True)
    tl = trans.double().requires_grad_(True)
    o3, _ = to.deform_psroi_pool(xl, rois, tl if not no_trans else None, no_trans, 0.25, od, gs, ps, part, spp, std)
    (o3 * og.double()).sum().backward()
    _close(gi, xl.grad)
    if not no_trans:
        _close(gt[0], tl.grad)


# ------------------------------------------------------------------------------------------------ 2. host builds
def _fp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _focal_emulation(x, t, gamma, alpha, dl=None, mode="kernel"):
    """fp32 emulation of focal_loss_kernel (np.exp for __expf); mode 'next_row_target' reads row n + 1's target in the
    float4 path"""
    f = np.float32
    xs = x.numpy().astype(f)
    n, c = xs.shape
    tt = t.numpy().astype(np.int64).reshape(n, 1)
    if mode == "next_row_target":
        tt = np.concatenate([tt[1:], tt[-1:]], 0)
    d = np.arange(c).reshape(1, c)
    e = np.exp(-np.abs(xs)).astype(f)
    lg = np.log1p(e).astype(f)
    inv = (f(1) / (f(1) + e)).astype(f)
    p = np.where(xs >= 0, inv, e * inv).astype(f)
    log_p = -(np.maximum(-xs, f(0)) + lg)
    log_1mp = -(np.maximum(xs, f(0)) + lg)
    g, a = f(gamma), f(alpha)
    pw1 = np.exp(g * log_1mp).astype(f)
    pwp = np.exp(g * log_p).astype(f)
    cl = np.maximum(log_p, f(-87.3365))
    if dl is None:
        pos = -a * pw1 * cl
        neg = -(f(1) - a) * pwp * log_1mp
    else:
        pos = -a * pw1 * (f(1) - p - p * g * cl)
        neg = -(f(1) - a) * pwp * (log_1mp * (f(1) - p) * g - p)
    r = np.where(tt == d + 1, pos, np.where(tt >= 0, neg, f(0))).astype(f)
    if dl is not None:
        r = (r * dl.numpy()).astype(f)
    return torch.from_numpy(r)


@pytest.mark.parametrize("bwd", [False, True])
def test_focal_emulation_inside_bound(bwd):
    for x, t, gamma, alpha in _focal_edges():
        dl = torch.linspace(-2, 2, x.numel()).view_as(x).float() if bwd else None
        ref, bnd = R.focal_reference(x, t, gamma, alpha, dl)
        got = _focal_emulation(x, t, gamma, alpha, dl)
        assert bool(R.inside(got, ref, bnd, AMAX).all()), (gamma, alpha, R.needed_a(got, ref, bnd))


def _focal_edges():
    vals = torch.tensor([0.0, 1e-3, -1e-3, 20, -20, 87.3, -87.3, 88, -88, 100, -100, 0.7, -2.5]).float()
    for c in (1, 3, 4, 30):
        n = 4 * len(vals)
        x = vals.repeat((n * c) // len(vals) + 1)[:n * c].view(n, c)
        t = torch.tensor([-1, 0, 1, c] * (n // 4), dtype=torch.int32)
        for gamma, alpha in ((0.0, 0.25), (1.0, 1.0), (1.5, 0.25), (2.0, 0.25)):
            yield x, t, gamma, alpha


def test_im2col_tile_blend_emulation_inside_bound():
    """the tile kernel's geometry (dcn_sample.cuh, its g++ build) and blend, on positions at the gate's edges"""
    from test_dcn_cpu import _host_lib
    lib = _host_lib()
    b, hgt, wid, ch = 1, 5, 6, 32
    x = torch.randn(b, hgt, wid, ch, generator=torch.Generator().manual_seed(12)).float()
    ho, wo = hgt, wid
    offs = torch.tensor([0.0, -1.0, 1.0, -0.5, 0.5, 4.0, 5.0, 6.0, 1e4, -1e4,
                         float(np.nextafter(np.float32(-1.0), np.float32(0))), 2.25]).float()
    off = offs[torch.randint(0, len(offs), (b * ho * wo * 18,), generator=torch.Generator().manual_seed(13))]
    off = off.view(b * ho * wo, 18)
    cols = torch.empty(b * ho * wo, 9, ch)
    assert lib.mega_dcn_sample_nhwc(_fp(x), 0, b, hgt, wid, ch, _fp(off), 18, 0, 1, 1, _fp(cols), None) == 0
    offset_nchw = off.view(b, ho, wo, 18).permute(0, 3, 1, 2).contiguous()
    ref, bnd = R.im2col_reference(x.permute(0, 3, 1, 2).contiguous(), offset_nchw, None, 3, 3, 1, 1, 1, 1, 1, 1, 1)
    got = cols.view(b, ho, wo, 9, ch).permute(0, 4, 3, 1, 2)
    assert bool(R.inside(got, ref, bnd, AMAX).all()), R.needed_a(got, ref, bnd)


def test_train_ops_host_build_inside_bounds():
    lib = host_lib()
    g = torch.Generator().manual_seed(14)
    # ROIAlign backward: strip tail (C = 9), rois past the border, sampling_ratio 0 and 2
    for sr in (0, 2):
        rois = _rois(15 + sr, 6, 40, 30)
        grad = torch.randn(6, 9, 3, 3, generator=g).float()
        seed = torch.randn(2, 9, 15, 20, generator=g).float()
        out = seed.clone()
        lib.mega_roi_align_backward_nchw(_fp(grad), _fp(rois), 6, ctypes.c_float(0.5), 3, 3, 2, 9, 15, 20, sr, _fp(out),
                                         None)
        ref, bnd, dec = R.roi_align_bwd_reference(grad, rois, 0.5, 3, 3, 2, 9, 15, 20, sr, seed)
        assert R.decisions_stable(dec)
        assert bool(R.inside(out, ref, bnd, AMAX).all()), R.needed_a(out, ref, bnd)
    # ROIPool forward / backward with ties (constant plane) and empty bins
    x = torch.randn(2, 3, 10, 12, generator=g).float()
    x[0, 1] = 0.5
    rois = _rois(17, 5, 24, 20)
    out = torch.empty(5, 3, 4, 4)
    arg = torch.empty(5, 3, 4, 4, dtype=torch.int32)
    lib.mega_roi_pool_forward(_fp(x), _fp(rois), 5, ctypes.c_float(0.5), 3, 10, 12, 4, 4, _fp(out), _fp(arg), None)
    ro, ra = R.roi_pool_reference(x, rois, 0.5, 4, 4)
    assert torch.equal(out, ro) and torch.equal(arg, ra)
    gr = torch.randn(5, 3, 4, 4, generator=g).float()
    gi = torch.zeros(2, 3, 10, 12)
    lib.mega_roi_pool_backward(_fp(gr), _fp(arg), _fp(rois), 5, 3, 10, 12, 4, 4, _fp(gi), None)
    ref, bnd = R.roi_pool_bwd_reference(gr, arg, rois, 3, 10, 12, 2)
    assert bool(R.inside(gi, ref, bnd, AMAX).all())
    # DCN: im2col (K-major), col2im, channel sum
    x, off, m = _dcn_inputs(18, b=2, c=4, h=6, w=7, k=3, dg=2)
    ldp = 44
    cols = torch.full((36, 2 * ldp), float("nan"))
    lib.mega_deform_im2col_kq(_fp(x), _fp(off), _fp(m), 2, 4, 6, 7, 3, 3, 1, 1, 1, 1, 1, 1, 2, ldp, _fp(cols), None)
    ref, bnd = R.im2col_reference(x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2)
    got = cols.view(4, 9, 2, ldp)[..., :42].permute(2, 0, 1, 3).reshape(ref.shape)
    assert bool(R.inside(got, ref, bnd, AMAX).all())
    assert bool(cols.view(4, 9, 2, ldp)[..., 42:].isnan().all())
    gcols = torch.randn(36, 2 * ldp, generator=g).float()
    gi0 = torch.randn(x.shape, generator=g).float()
    gi, go, gm = gi0.clone(), torch.full((2, 36, 6, 7), float("nan")), torch.full((2, 18, 6, 7), float("nan"))
    lib.mega_deform_col2im_fused(_fp(gcols), _fp(x), _fp(off), _fp(m), 2, 4, 6, 7, 3, 3, 1, 1, 1, 1, 1, 1, 2, ldp,
                                 _fp(gi), _fp(go), _fp(gm), None)
    refs = R.col2im_reference(gcols, x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2, ldp, gi0)
    for got, (ref, bnd) in zip((gi, go, gm), refs):
        assert bool(R.inside(got, ref, bnd, AMAX).all()), R.needed_a(got, ref, bnd)
    xs = torch.randn(3, 5, 37, generator=g).float()
    seed = torch.randn(5, generator=g).float()
    out = seed.clone()
    lib.mega_channel_sum_nchw(_fp(xs), 3, 5, 37, _fp(out), None)
    ref, bnd = R.channel_sum_reference(xs, seed)
    assert bool(R.inside(out, ref, bnd, AMAX).all())
    # PSROI backward
    gs, od, ps, part, spp = 3, 4, 3, 2, 2
    x = torch.randn(2, od * gs * gs, 10, 12, generator=g).float()
    rois = _rois(19, 4, 48, 40)
    trans = (torch.randn(4, 4, part, part, generator=g) * 0.5).float()
    _, _, cnt, _ = R.psroi_fwd_reference(x, rois, trans, False, 0.25, od, gs, ps, part, spp, 0.1)
    og = torch.randn(4, od, ps, ps, generator=g).float()
    gi0, gt0 = torch.randn(x.shape, generator=g).float(), torch.randn(trans.shape, generator=g).float()
    gi, gt = gi0.clone(), gt0.clone()
    cntf = cnt.float().contiguous()
    lib.mega_deform_psroi_pooling_backward(_fp(og), _fp(x), _fp(rois), _fp(trans), _fp(cntf), 4, od * gs * gs, 10, 12,
                                           0, ctypes.c_float(0.25), od, gs, ps, part, spp, ctypes.c_float(0.1), 2,
                                           _fp(gi), _fp(gt), None)
    (ri, bi), (rt, bt) = R.psroi_bwd_reference(og, cntf, x, rois, trans, False, 0.25, od, gs, ps, part, spp, 0.1, gi0,
                                               gt0)
    assert bool(R.inside(gi, ri, bi, AMAX).all()), R.needed_a(gi, ri, bi)
    assert bool(R.inside(gt, rt, bt, AMAX).all()), R.needed_a(gt, rt, bt)


# ------------------------------------------------------------------------------------------------ 3. mutations
def _rejects(got, ref, bnd):
    return not bool(R.inside(got, ref, bnd, AMAX).all())


def _border_offsets(b, dg, k, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(b, dg * 2 * k * k, h, w, generator=g) * 3 - 1.5).float()


@pytest.mark.parametrize("mode", ["drop_far_corner", "swap_w01_w10"])
def test_bound_rejects_im2col_bug(mode):
    x, _, m = _dcn_inputs(20)
    off = _border_offsets(2, 2, 3, 7, 8, 21)
    ref, bnd = R.im2col_reference(x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2)
    bad, _ = R.im2col_reference(x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2, mode=mode)
    assert _rejects(bad, ref, bnd)


def test_bound_rejects_im2col_without_mask():
    x, _, m = _dcn_inputs(22)
    off = _border_offsets(2, 2, 3, 7, 8, 23)
    ref, bnd = R.im2col_reference(x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2)
    bad, _ = R.im2col_reference(x, off, None, 3, 3, 1, 1, 1, 1, 1, 1, 2)
    assert _rejects(bad, ref, bnd)


@pytest.mark.parametrize("mode", ["strip_tail_loses_last", "drop_bottom_border"])
def test_bound_rejects_roi_align_bug(mode):
    rois = torch.tensor([[0, 2.0, 3.0, 30.0, 29.0], [0, 10.0, 20.0, 50.0, 40.0]]).float()   # past the bottom border
    grad = torch.randn(2, 9, 3, 3, generator=torch.Generator().manual_seed(24)).float()
    ref, bnd, _ = R.roi_align_bwd_reference(grad, rois, 0.5, 3, 3, 1, 9, 12, 30, 2)
    bad, _, _ = R.roi_align_bwd_reference(grad, rois, 0.5, 3, 3, 1, 9, 12, 30, 2, mode=mode)
    assert _rejects(bad, ref, bnd)


def test_bound_rejects_roi_pool_last_max():
    x = torch.zeros(1, 2, 8, 8)
    rois = torch.tensor([[0, 0.0, 0.0, 7.0, 7.0]])
    _, arg = R.roi_pool_reference(x, rois, 1.0, 2, 2)
    _, bad = R.roi_pool_reference(x, rois, 1.0, 2, 2, mode="last_max")
    assert not torch.equal(arg, bad)


def test_bound_rejects_psroi_first_bin_count():
    g = torch.Generator().manual_seed(25)
    x = torch.randn(1, 9, 10, 12, generator=g).float()
    rois = torch.tensor([[0, -6.0, -6.0, 20.0, 20.0]])         # bins at the top-left corner lose samples
    ref, bnd, _, _ = R.psroi_fwd_reference(x, rois, None, True, 0.5, 1, 3, 3, 3, 4, 0.1)
    bad, _, _, _ = R.psroi_fwd_reference(x, rois, None, True, 0.5, 1, 3, 3, 3, 4, 0.1, mode="first_bin_count")
    assert _rejects(bad, ref, bnd)


def test_bound_rejects_grad_offset_without_mask():
    x, off, m = _dcn_inputs(26)
    gcols = torch.randn(36, 2 * 56, generator=torch.Generator().manual_seed(27)).float()
    refs = R.col2im_reference(gcols, x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2, 56, None)
    bads = R.col2im_reference(gcols, x, off, m, 3, 3, 1, 1, 1, 1, 1, 1, 2, 56, None, mode="offset_without_mask")
    assert _rejects(bads[1][0], *refs[1])


def test_bound_rejects_psroi_unclamped_h():
    g = torch.Generator().manual_seed(28)
    x = torch.randn(1, 9, 10, 12, generator=g).float()
    rois = torch.tensor([[0, 2.0, 30.0, 30.0, 42.0]])          # samples between H - 1 and H - 0.5
    out, _, cnt, _ = R.psroi_fwd_reference(x, rois, None, True, 0.25, 1, 3, 3, 3, 4, 0.1)
    og = torch.ones(1, 1, 3, 3)
    (ref, bnd), _ = R.psroi_bwd_reference(og, cnt.float(), x, rois, None, True, 0.25, 1, 3, 3, 3, 4, 0.1)
    (bad, _), _ = R.psroi_bwd_reference(og, cnt.float(), x, rois, None, True, 0.25, 1, 3, 3, 3, 4, 0.1,
                                        mode="unclamped_h")
    assert _rejects(bad, ref, bnd)


def test_bound_rejects_focal_next_row_target():
    x = torch.randn(16, 8, generator=torch.Generator().manual_seed(29)).float()
    t = torch.arange(16, dtype=torch.int32) % 9
    ref, bnd = R.focal_reference(x, t, 2.0, 0.25)
    assert _rejects(_focal_emulation(x, t, 2.0, 0.25, mode="next_row_target"), ref, bnd)


def test_bound_rejects_focal_without_log_clamp():
    x = torch.tensor([[-100.0, -95.0]]).float()
    t = torch.tensor([1], dtype=torch.int32)
    ref, bnd = R.focal_reference(x, t, 0.0, 0.25)
    bad = torch.tensor([[0.25 * 100.0, 0.0]]).float()          # -alpha * log p unclamped
    assert _rejects(bad, ref, bnd)


def test_bound_rejects_grid_stride_skipping_its_last_pass():
    """a grid-stride loop that stops one pass early leaves the last items of a capped grid unwritten (NaN-guarded)"""
    n, c, block = 1100, 2000, 256                  # 2.2 M logits: past the 132 x 16 block cap
    stride = R.GRID_CAP * block
    total = n * c
    passes = -(-total // stride)
    assert passes >= 2
    x = torch.linspace(-5, 5, total).view(n, c).float()
    t = torch.arange(n, dtype=torch.int32) % (c + 1)
    ref, bnd = R.focal_reference(x, t, 2.0, 0.25)
    got = _focal_emulation(x, t, 2.0, 0.25).view(-1)
    assert bool(R.inside(got.view(n, c), ref, bnd, AMAX).all())
    got[(passes - 1) * stride:] = float("nan")
    assert _rejects(got.view(n, c), ref, bnd)


def test_bound_rejects_channel_sum_assign():
    xs = torch.randn(2, 3, 40, generator=torch.Generator().manual_seed(30)).float()
    seed = torch.tensor([1.0, -2.0, 3.0])
    ref, bnd = R.channel_sum_reference(xs, seed)
    assert _rejects(xs.double().sum((0, 2)).float(), ref, bnd)


# ------------------------------------------------------------------------------------------------ 4. restated limits
def _src(name):
    with open(os.path.join(CSRC, name)) as fh:
        return fh.read()


def test_restated_limits_match_source():
    deform, train, cuh = _src("deform.cu"), _src("train_ops.cu"), _src("train_ops.cuh")
    assert int(re.search(r"constexpr int kDcnMaxTaps = (\d+);", deform).group(1)) == R.K_DCN_MAX_TAPS
    assert int(re.search(r"constexpr int kDcnPix = (\d+);", deform).group(1)) == R.K_DCN_PIX
    assert int(re.search(r"constexpr int kDcnCh = (\d+);", deform).group(1)) == R.K_DCN_CH
    assert int(re.search(r"constexpr int kRoiBwdStrip = (\d+);", cuh).group(1)) == R.K_ROI_BWD_STRIP
    for src in (deform, train):
        m = re.search(r"const long long cap = (\d+)LL \* (\d+);", src)
        assert int(m.group(1)) * int(m.group(2)) == R.GRID_CAP
    m = re.search(r"const int warps = (\d+);.*?if \(blocks > (\d+) \* (\d+)\)", train, re.S)
    assert int(m.group(1)) == R.CHANNEL_SUM_WARPS and int(m.group(2)) * int(m.group(3)) == R.CHANNEL_SUM_BLOCKS
    assert "-87.3365f" in deform and R.LOG_FLT_MIN == float(np.float32(-87.3365))
    kernels = set(re.findall(r"__global__ void (?:__launch_bounds__\(\d+\)\s*)?(\w+_kernel)\(", deform + train))
    assert kernels == {re.sub(r"<.*", "", k) for k in R.INSTANTIATIONS}


# ------------------------------------------------------------------------------------------------ 5. ptr lint
def ptr_calls_with_temporaries(path):
    """(line, source) of every ptr(...) / _lib.ptr(...) call whose argument is a call expression"""
    with open(path) as fh:
        src = fh.read()
    bad = []
    for node in ast.walk(ast.parse(src)):
        if not isinstance(node, ast.Call):
            continue
        f = node.func
        name = f.id if isinstance(f, ast.Name) else f.attr if isinstance(f, ast.Attribute) else None
        if name == "ptr" and node.args and any(isinstance(a, (ast.Call, ast.IfExp, ast.BinOp)) for a in node.args):
            bad.append((node.lineno, ast.get_source_segment(src, node)))
    return bad


@pytest.mark.parametrize("rel", ["mega.pytorch_b200/mega_core/_C.py", "mega.pytorch_b200/mega_core/b200/ops.py"])
def test_no_pointer_to_a_temporary(rel):
    bad = ptr_calls_with_temporaries(os.path.join(ROOT, rel))
    assert not bad, "ptr() of a temporary (freed before the kernel runs): %s" % bad
