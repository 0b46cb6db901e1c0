"""CPU checks of the training-side half of `mega_core._C` (roi_align_backward, roi_pool_*, deform-conv backward,
deform_psroi_pooling_backward; SURVEY.md section 8b / 8f row 3):

  1. the oracles of oracle/train_ops_oracle.py are anchored -- against the C ROIAlign oracle (bit-pinned to the
     reference's ROIAlign_cpu.cpp), torchvision's roi_align / roi_pool / deform_conv2d (same lineage as the reference's
     kernels; forward and gradients) and the plain-Python PSROI restatement;
  2. the per-item device functions of csrc/train_ops.cuh, compiled for the host (tests/native/train_ops_host.cpp, same
     entry-point names and prototypes as the C ABI) and run item by item, reproduce those oracles when driven by the
     product's own host code: the tests patch the host build over the ctypes handles of libmega_b200.so (and a torch
     matmul over the wgmma GEMM wrapper) and call `mega_core._C.*` on CPU tensors. The index arithmetic and gradient
     formulas of the CUDA kernels, the argument order of every ctypes call and the operand re-layouts of _C.py are thus
     verified here; tests/test_zz_train_ops_gpu.py repeats the comparison on the GPU, where only the launch
     configuration and the GEMM calls are new. (The patching exists in this test only: the product has no CPU path.)
"""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import mega_oracle as mo  # noqa: E402
import train_ops_oracle as to  # noqa: E402

NATIVE = os.path.join(ROOT, "tests", "native")
_host = None


HOST_ENTRY_POINTS = ["mega_roi_align_backward_nchw", "mega_roi_pool_forward", "mega_roi_pool_backward",
                     "mega_deform_im2col_kq", "mega_deform_col2im_fused", "mega_channel_sum_nchw",
                     "mega_deform_psroi_pooling_backward"]


def host_lib():
    """g++ build of the item functions (rebuilt when the headers or the harness changed)"""
    global _host
    if _host is None:
        so = os.path.join(NATIVE, "libtrain_ops_host.so")
        srcs = [os.path.join(NATIVE, "train_ops_host.cpp"),
                os.path.join(ROOT, "mega.pytorch_b200", "csrc", "train_ops.cuh"),
                os.path.join(ROOT, "include", "mega_b200.h")]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-I",
                                   os.path.join(ROOT, "mega.pytorch_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                                   "-o", so, srcs[0]])
        _host = ctypes.CDLL(so)
    return _host


@pytest.fixture
def cpu_C(monkeypatch):
    """`mega_core._C` with the seven ABI v4 entry points served by the host build and ops.linear by torch.matmul"""
    from mega_core import _C, _lib
    from mega_core.b200 import ops
    host = host_lib()
    for name in HOST_ENTRY_POINTS:
        fn = getattr(host, name)
        real = getattr(_lib.lib, name)
        fn.argtypes, fn.restype = real.argtypes, real.restype
        monkeypatch.setattr(_lib.lib, name, fn)
    monkeypatch.setattr(_lib, "stream_ptr", lambda: None)
    monkeypatch.setattr(_C, "_cuda_only", lambda *a, **k: None)

    def linear(x, w, out, **kw):
        assert not kw and x.stride(1) == 1 and w.stride(1) == 1 and out.stride(1) == 1
        for t in (x, w, out):                       # the TMA alignment rules of the real GEMM
            assert t.data_ptr() % 16 == 0 and (t.stride(0) * 4) % 16 == 0, (t.shape, t.stride())
        out.copy_(x @ w.t())
        return out
    monkeypatch.setattr(ops, "linear", linear)
    return _C


def _rois(g, k, n_img, w_img, h_img):
    x1 = torch.rand(k, generator=g) * w_img * 0.7 - 10
    y1 = torch.rand(k, generator=g) * h_img * 0.7 - 10
    bw = torch.rand(k, generator=g) * w_img * 0.6 + 1
    bh = torch.rand(k, generator=g) * h_img * 0.6 + 1
    b = torch.randint(0, n_img, (k,), generator=g).float()
    return torch.stack([b, x1, y1, x1 + bw, y1 + bh], 1)


# ------------------------------------------------------------------------------------------------ oracle anchors
@pytest.mark.parametrize("sr", [0, 2])
def test_oracle_roi_align_is_anchored(sr):
    import torchvision
    g = torch.Generator().manual_seed(11)
    feat = torch.randn(2, 5, 12, 17, generator=g)
    rois = _rois(g, 5, 2, 17 * 16, 12 * 16)
    rois[4] = torch.tensor([1.0, 250.0, 170.0, 252.0, 500.0])       # partly outside, tiny width
    ref_c = mo.roi_align(feat, rois, 1 / 16.0, 7, 7, sr)
    got = to.roi_align(feat, rois, 1 / 16.0, 7, 7, sr)
    assert torch.allclose(got, ref_c, atol=2e-6, rtol=1e-6)
    tv = torchvision.ops.roi_align(feat, rois, (7, 7), 1 / 16.0, sr, aligned=False)
    assert torch.allclose(tv, ref_c, atol=2e-6, rtol=1e-6)
    # gradient: autograd of the restatement == torchvision's backward kernel
    grad = torch.randn(5, 5, 7, 7, generator=g)
    x = feat.clone().requires_grad_(True)
    (torchvision.ops.roi_align(x, rois, (7, 7), 1 / 16.0, sr, aligned=False) * grad).sum().backward()
    mine = to.roi_align_backward(grad, rois, 1 / 16.0, 7, 7, 2, 5, 12, 17, sr)
    assert torch.allclose(mine, x.grad, atol=1e-5, rtol=1e-5)


def test_oracle_roi_pool_is_anchored():
    import torchvision
    g = torch.Generator().manual_seed(12)
    feat = torch.randn(2, 4, 13, 19, generator=g)
    rois = _rois(g, 6, 2, 19 * 16, 13 * 16)
    rois[5] = torch.tensor([0.0, 400.0, 300.0, 420.0, 310.0])       # entirely outside: empty bins
    out, arg = to.roi_pool(feat, rois, 1 / 16.0, 7, 7)
    tv = torchvision.ops.roi_pool(feat, rois, (7, 7), 1 / 16.0)
    assert torch.equal(out, tv)
    assert (arg[5] == -1).all() and (out[5] == 0).all()
    grad = torch.randn(6, 4, 7, 7, generator=g)
    x = feat.clone().requires_grad_(True)
    (torchvision.ops.roi_pool(x, rois, (7, 7), 1 / 16.0) * grad).sum().backward()
    assert torch.allclose(to.roi_pool_backward(grad, feat, rois, 1 / 16.0, 7, 7), x.grad, atol=1e-6)


DCN_CASES = [
    # modulated, groups, dg, stride, pad, dil, k
    (False, 1, 1, 1, 1, 1, 3),
    (True, 1, 1, 1, 1, 1, 3),
    (True, 2, 2, 2, 1, 1, 3),
    (False, 2, 4, 1, 2, 2, 3),
    (True, 1, 2, 1, 0, 1, 1),
]


def _dcn_inputs(seed, modulated, groups, dg, stride, pad, dil, k, b=2, c=8, h=9, w=11, cout=12):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, c, h, w, generator=g)
    wt = torch.randn(cout, c // groups, k, k, generator=g) / (c * k * k / groups) ** 0.5
    bias = torch.randn(cout, generator=g) if modulated else None
    ho = (h + 2 * pad - (dil * (k - 1) + 1)) // stride + 1
    wo = (w + 2 * pad - (dil * (k - 1) + 1)) // stride + 1
    off = torch.randn(b, dg * 2 * k * k, ho, wo, generator=g) * 2.5      # many samples cross the border
    mask = torch.rand(b, dg * k * k, ho, wo, generator=g) if modulated else None
    go = torch.randn(b, cout, ho, wo, generator=g)
    return x, off, mask, wt, bias, go, ho, wo


@pytest.mark.parametrize("case", DCN_CASES)
def test_oracle_deform_conv_is_anchored(case):
    import torchvision
    modulated, groups, dg, stride, pad, dil, k = case
    x, off, mask, wt, bias, go, ho, wo = _dcn_inputs(21, *case)
    d = torch.float64
    leaves = [t.double().requires_grad_(True) if t is not None else None for t in (x, off, mask, wt, bias)]
    tv = torchvision.ops.deform_conv2d(leaves[0], leaves[1], leaves[3], leaves[4], stride=stride, padding=pad,
                                       dilation=dil, mask=leaves[2])
    mine = to.deform_conv2d(x.to(d), off.to(d), mask.to(d) if modulated else None, wt.to(d),
                            bias.to(d) if modulated else None, (stride, stride), (pad, pad), (dil, dil), groups, dg)
    assert torch.allclose(mine, tv.detach(), atol=1e-10)
    (tv * go.double()).sum().backward()
    grads = to.deform_conv2d_grads(x, off, mask, wt, bias, go, (stride, stride), (pad, pad), (dil, dil), groups, dg)
    for name, leaf in zip(("input", "offset", "mask", "weight", "bias"), leaves):
        if leaf is not None:
            assert torch.allclose(grads[name], leaf.grad.float(), atol=1e-5, rtol=1e-5), name


def test_oracle_deform_psroi_is_anchored():
    g = torch.Generator().manual_seed(3)
    gs, ps, od, ncls = 3, 3, 4, 2
    data = torch.randn(1, od * gs * gs, 11, 13, generator=g)
    rois = torch.tensor([[0, 8.0, 10.0, 120.0, 90.0], [0, 40.2, 33.7, 150.9, 160.1], [0, -10.0, -5.0, 30.0, 20.0]])
    trans = torch.randn(3, 2 * ncls, ps, ps, generator=g) * 0.5
    for no_trans in (True, False):
        ref, rc = mo.deform_psroi_pool(data, rois, trans, no_trans, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
        got, gc = to.deform_psroi_pool(data.double(), rois, trans.double(), no_trans, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
        assert torch.equal(gc, rc)
        assert torch.allclose(got.float(), ref, atol=1e-5, rtol=1e-5)


# ------------------------------------------- mega_core._C on the host build of the device code vs the oracles
@pytest.mark.parametrize("sr,c", [(0, 5), (2, 19), (0, 8)])
def test_C_roi_align_backward(cpu_C, sr, c):
    g = torch.Generator().manual_seed(31 + c)
    n, h, w, k = 2, 12, 17, 6
    rois = _rois(g, k, n, w * 16, h * 16)
    rois[5] = torch.tensor([1.0, 250.0, 170.0, 252.0, 500.0])
    grad = torch.randn(k, c, 7, 7, generator=g)
    ref = to.roi_align_backward(grad, rois, 1 / 16.0, 7, 7, n, c, h, w, sr)
    out = cpu_C.roi_align_backward(grad, rois, 1 / 16.0, 7, 7, n, c, h, w, sr)
    assert torch.allclose(out, ref, atol=2e-5, rtol=1e-5)
    assert out.abs().sum() > 0
    assert cpu_C.roi_align_backward(torch.zeros(0, c, 7, 7), torch.zeros(0, 5), 1 / 16.0, 7, 7, n, c, h, w, sr).sum() == 0


def test_C_roi_pool(cpu_C):
    g = torch.Generator().manual_seed(41)
    n, c, h, w, k = 2, 6, 13, 19, 7
    feat = torch.randn(n, c, h, w, generator=g)
    rois = _rois(g, k, n, w * 16, h * 16)
    rois[6] = torch.tensor([0.0, 400.0, 300.0, 420.0, 310.0])
    ref, ref_arg = to.roi_pool(feat, rois, 1 / 16.0, 7, 7)
    out, arg = cpu_C.roi_pool_forward(feat, rois, 1 / 16.0, 7, 7)
    assert torch.equal(out, ref) and torch.equal(arg, ref_arg)
    grad = torch.randn(k, c, 7, 7, generator=g)
    gin = cpu_C.roi_pool_backward(grad, feat, rois, arg, 1 / 16.0, 7, 7, n, c, h, w)
    assert torch.allclose(gin, to.roi_pool_backward(grad, feat, rois, 1 / 16.0, 7, 7), atol=1e-6)


@pytest.mark.parametrize("case", DCN_CASES)
def test_C_deform_conv_backward(cpu_C, case):
    modulated, groups, dg, stride, pad, dil, k = case
    x, off, mask, wt, bias, go, ho, wo = _dcn_inputs(51, *case, c=16, cout=24)
    ref = to.deform_conv2d_grads(x, off, mask, wt, bias, go, (stride, stride), (pad, pad), (dil, dil), groups, dg)
    gin, gw = torch.zeros_like(x), torch.zeros_like(wt)
    goff = torch.full_like(off, 7.0)                 # assigned, not accumulated
    b = x.shape[0]
    if modulated:
        gmask, gb = torch.full_like(mask, 7.0), torch.zeros_like(bias)
        cpu_C.modulated_deform_conv_backward(x, wt, bias, None, off, mask, None, gin, gw, gb, goff, gmask, go, k, k,
                                             stride, stride, pad, pad, dil, dil, groups, dg, True)
        assert torch.allclose(gmask, ref["mask"], atol=2e-4, rtol=1e-4)
        assert torch.allclose(gb, ref["bias"], atol=1e-4, rtol=1e-5)
    else:
        assert cpu_C.deform_conv_backward_input(x, off, go, gin, goff, wt, None, k, k, stride, stride, pad, pad, dil, dil,
                                                groups, dg, b) == 1
        assert cpu_C.deform_conv_backward_parameters(x, off, go, gw, None, None, k, k, stride, stride, pad, pad, dil, dil,
                                                     groups, dg, 0.5, b) == 1
        gw = gw * 2.0                                # scale = 0.5 above
    assert torch.allclose(gin, ref["input"], atol=2e-4, rtol=1e-4)
    assert torch.allclose(goff, ref["offset"], atol=2e-4, rtol=1e-4)
    assert torch.allclose(gw, ref["weight"], atol=2e-4, rtol=1e-4)


def test_C_deform_conv_backward_argument_errors(cpu_C):
    x, off, mask, wt, bias, go, ho, wo = _dcn_inputs(51, True, 1, 1, 1, 1, 1, 3, c=16, cout=24)
    with pytest.raises(RuntimeError, match="kernel shape"):
        cpu_C.deform_conv_backward_parameters(x, off, go, torch.zeros_like(wt), None, None, 5, 5, 1, 1, 1, 1, 1, 1, 1, 1,
                                              1.0, 2)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        cpu_C.deform_conv_backward_input(x, off, go[:, :22], torch.zeros_like(x), torch.zeros_like(off), wt[:22], None, 3,
                                         3, 1, 1, 1, 1, 1, 1, 1, 1, 2)


@pytest.mark.parametrize("no_trans", [True, False])
def test_C_deform_psroi_backward(cpu_C, no_trans):
    g = torch.Generator().manual_seed(3)
    gs, ps, od, ncls = 3, 3, 4, 2
    data = torch.randn(2, od * gs * gs, 11, 13, generator=g)
    rois = torch.tensor([[0, 8.0, 10.0, 120.0, 90.0], [1, 40.2, 33.7, 150.9, 160.1], [0, -10.0, -5.0, 30.0, 20.0],
                         [1, 300.0, 300.0, 320.0, 330.0]])
    k = rois.shape[0]
    trans = torch.randn(k, 2 * ncls, ps, ps, generator=g) * 0.5
    og = torch.randn(k, od, ps, ps, generator=g)
    _, cnt = to.deform_psroi_pool(data.double(), rois, trans.double(), no_trans, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
    ref_in, ref_tr = to.deform_psroi_pool_grads(data, rois, trans, og, no_trans, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
    gin = torch.zeros_like(data)
    gtr = torch.zeros_like(trans)
    cpu_C.deform_psroi_pooling_backward(og, data, rois, trans, cnt, gin, gtr, no_trans, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
    assert torch.allclose(gin, ref_in, atol=2e-5, rtol=1e-4)
    if no_trans:
        assert gtr.abs().sum() == 0
    else:
        assert torch.allclose(gtr, ref_tr, atol=2e-4, rtol=1e-3)
        assert ref_tr.abs().sum() > 0


# ------------------------------------------------ mega_core.layers autograd wrappers (backward on the host build)
@pytest.fixture
def cpu_layers(cpu_C, monkeypatch):
    """mega_core.layers on CPU tensors: backward ops as in cpu_C; the forward ops that have no host build are stood in
    by their oracles (test-only), so that the autograd plumbing of layers/train_ops.py can be exercised end to end"""
    from mega_core import layers

    def roi_align_forward(x, r, scale, ph, pw, sr):
        return mo.roi_align(x, r, scale, ph, pw, sr)

    def dcn_v1(x, w, off, out, cols, ones, kW, kH, dW, dH, pW, pH, dlW, dlH, group, dg, step):
        out.copy_(to.deform_conv2d(x, off, None, w, None, (dH, dW), (pH, pW), (dlH, dlW), group, dg))
        return 1

    def dcn_v2(x, w, b, ones, off, m, out, cols, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, with_bias):
        out.copy_(to.deform_conv2d(x, off, m, w, b if with_bias else None, (sh, sw), (ph, pw), (dh, dw), group, dg))

    def psroi(x, r, tr, out, cnt, no_trans, scale, od, gs, ps, part, spp, std):
        o, c = to.deform_psroi_pool(x, r, tr, no_trans, scale, od, gs, ps, part, spp, std)
        out.copy_(o)
        cnt.copy_(c)
    monkeypatch.setattr(cpu_C, "roi_align_forward", roi_align_forward)
    monkeypatch.setattr(cpu_C, "deform_conv_forward", dcn_v1)
    monkeypatch.setattr(cpu_C, "modulated_deform_conv_forward", dcn_v2)
    monkeypatch.setattr(cpu_C, "deform_psroi_pooling_forward", psroi)
    return layers


def test_layers_roi_align_and_pool_autograd(cpu_layers):
    import torchvision
    g = torch.Generator().manual_seed(71)
    feat = torch.randn(2, 6, 12, 17, generator=g)
    rois = _rois(g, 5, 2, 17 * 16, 12 * 16)
    wgt = torch.randn(5, 6, 7, 7, generator=g)
    x = feat.clone().requires_grad_(True)
    out = cpu_layers.ROIAlign((7, 7), 1 / 16.0, 2)(x, rois)
    (out * wgt).sum().backward()
    y = feat.clone().requires_grad_(True)
    ref = torchvision.ops.roi_align(y, rois, (7, 7), 1 / 16.0, 2, aligned=False)
    (ref * wgt).sum().backward()
    assert torch.allclose(out, ref, atol=2e-6) and torch.allclose(x.grad, y.grad, atol=1e-5)
    x = feat.clone().requires_grad_(True)
    out = cpu_layers.ROIPool(7, 1 / 16.0)(x, rois)
    (out * wgt).sum().backward()
    y = feat.clone().requires_grad_(True)
    ref = torchvision.ops.roi_pool(y, rois, 7, 1 / 16.0)
    (ref * wgt).sum().backward()
    assert torch.equal(out, ref) and torch.allclose(x.grad, y.grad, atol=1e-6)


@pytest.mark.parametrize("modulated", [False, True])
def test_layers_deform_conv_autograd(cpu_layers, modulated):
    import torchvision
    case = (modulated, 2, 2, 1, 1, 1, 3)
    x, off, mask, wt, bias, go, ho, wo = _dcn_inputs(81, *case, c=16, cout=24)
    mine = [t.clone().requires_grad_(True) if t is not None else None for t in (x, off, mask, wt, bias)]
    theirs = [t.clone().requires_grad_(True) if t is not None else None for t in (x, off, mask, wt, bias)]
    if modulated:
        out = cpu_layers.modulated_deform_conv(mine[0], mine[1], mine[2], mine[3], mine[4], 1, 1, 1, 2, 2)
    else:
        out = cpu_layers.deform_conv(mine[0], mine[1], mine[3], 1, 1, 1, 2, 2)
    ref = torchvision.ops.deform_conv2d(theirs[0], theirs[1], theirs[3], theirs[4], stride=1, padding=1, dilation=1,
                                        mask=theirs[2])
    assert torch.allclose(out, ref, atol=1e-4)
    (out * go).sum().backward()
    (ref * go).sum().backward()
    for a, b_ in zip(mine, theirs):
        if a is not None:
            assert torch.allclose(a.grad, b_.grad, atol=3e-4, rtol=1e-4)


def test_layers_modulated_pack_zero_init_is_half_a_convolution(cpu_layers):
    """ModulatedDeformConvPack starts with zero offsets and masks sigmoid(0) = 0.5: out = 0.5 * conv(x, w) + b"""
    torch.manual_seed(5)
    m = cpu_layers.ModulatedDeformConvPack(8, 12, 3, stride=1, padding=1, deformable_groups=2)
    with torch.no_grad():
        m.bias.normal_()
    x = torch.randn(2, 8, 9, 11, requires_grad=True)
    out = m(x)
    ref = 0.5 * torch.nn.functional.conv2d(x, m.weight, None, 1, 1) + m.bias.view(1, -1, 1, 1)
    assert torch.allclose(out, ref, atol=1e-5)
    out.sum().backward()
    assert m.conv_offset_mask.weight.grad is not None and m.weight.grad.abs().sum() > 0 and x.grad is not None
    gw = torch.autograd.grad(ref.sum(), m.weight)[0]
    assert torch.allclose(m.weight.grad, gw, atol=1e-4)


def test_layers_deform_roi_pooling_autograd(cpu_layers):
    g = torch.Generator().manual_seed(3)
    gs, ps, od = 3, 3, 4
    data = torch.randn(2, od * gs * gs, 11, 13, generator=g)
    rois = torch.tensor([[0, 8.0, 10.0, 120.0, 90.0], [1, 40.2, 33.7, 150.9, 160.1]])
    trans = torch.randn(2, 2, ps, ps, generator=g) * 0.5
    og = torch.randn(2, od, ps, ps, generator=g)
    x, t = data.clone().requires_grad_(True), trans.clone().requires_grad_(True)
    out = cpu_layers.DeformRoIPooling(1 / 16.0, ps, od, False, gs, ps, 4, 0.1)(x, rois, t)
    (out * og).sum().backward()
    ref_in, ref_tr = to.deform_psroi_pool_grads(data, rois, trans, og, False, 1 / 16.0, od, gs, ps, ps, 4, 0.1)
    assert torch.allclose(x.grad, ref_in, atol=2e-5, rtol=1e-4) and torch.allclose(t.grad, ref_tr, atol=2e-4, rtol=1e-3)
    pack = cpu_layers.ModulatedDeformRoIPoolingPack(1 / 16.0, ps, od * gs * gs, False, 1, ps, 4, 0.1, deform_fc_channels=32)
    y = pack(data.clone().requires_grad_(True), rois)
    assert y.shape == (2, od * gs * gs, ps, ps)
    y.sum().backward()
    assert pack.mask_fc[2].weight.grad is not None
