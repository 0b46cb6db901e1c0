"""Differentiable wrappers of the `_C` ops with the reference's layer names (layers/roi_align.py, roi_pool.py,
sigmoid_focal_loss.py, smooth_l1_loss.py, dcn/deform_conv_func.py, dcn/deform_conv_module.py, dcn/deform_pool_func.py,
dcn/deform_pool_module.py). Forward and backward both run on the sm_90a kernels of libmega_b200.so through
`mega_core._C`; nothing here has a CPU path. None of these layers is reached by the VID inference configs -- they
complete the operator API behind which `tools/train_net.py`-style callers find the same names (SURVEY.md 8b, 8f row 3).

One generic autograd.Function (`_COp`) carries every op: a wrapper hands it the forward closure, which returns the
output and the backward closure, so each op reads top to bottom in one place.
"""
import math

import torch
from torch import nn
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from .. import _C


class _COp(torch.autograd.Function):
    """forward(run, *tensors): `run(ctx_free_tensors...) -> (output, backward_fn)`; backward_fn(grad) returns one
    gradient (or None) per tensor argument."""

    @staticmethod
    def forward(ctx, run, *tensors):
        out, ctx.bwd = run(*[t.detach() if t is not None else None for t in tensors])
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad):
        return (None,) + tuple(ctx.bwd(grad.contiguous()))


# ------------------------------------------------------------------------------------------------ ROIAlign / ROIPool
def roi_align(input, rois, output_size, spatial_scale, sampling_ratio):
    """layers/roi_align.py:13-44; always fp32 (the reference wraps the module in amp.float_function, :57)"""
    oh, ow = _pair(output_size)
    shape = tuple(input.shape)

    def run(x, r):
        out = _C.roi_align_forward(x.float(), r.float(), spatial_scale, oh, ow, sampling_ratio)
        return out, lambda g: (_C.roi_align_backward(g, r.float(), spatial_scale, oh, ow, *shape, sampling_ratio), None)
    return _COp.apply(run, input, rois)


class ROIAlign(nn.Module):
    """layers/roi_align.py:47-69"""

    def __init__(self, output_size, spatial_scale, sampling_ratio):
        super().__init__()
        self.output_size, self.spatial_scale, self.sampling_ratio = output_size, spatial_scale, sampling_ratio

    def forward(self, input, rois):
        return roi_align(input, rois, self.output_size, self.spatial_scale, self.sampling_ratio)

    def __repr__(self):
        return "ROIAlign(output_size=%s, spatial_scale=%s, sampling_ratio=%s)" % (
            self.output_size, self.spatial_scale, self.sampling_ratio)


def roi_pool(input, rois, output_size, spatial_scale):
    """layers/roi_pool.py:12-49"""
    oh, ow = _pair(output_size)
    shape = tuple(input.shape)

    def run(x, r):
        out, argmax = _C.roi_pool_forward(x.float(), r.float(), spatial_scale, oh, ow)
        return out, lambda g: (_C.roi_pool_backward(g, x, r.float(), argmax, spatial_scale, oh, ow, *shape), None)
    return _COp.apply(run, input, rois)


class ROIPool(nn.Module):
    """layers/roi_pool.py:52-68"""

    def __init__(self, output_size, spatial_scale):
        super().__init__()
        self.output_size, self.spatial_scale = output_size, spatial_scale

    def forward(self, input, rois):
        return roi_pool(input, rois, self.output_size, self.spatial_scale)

    def __repr__(self):
        return "ROIPool(output_size=%s, spatial_scale=%s)" % (self.output_size, self.spatial_scale)


# --------------------------------------------------------------------------------------------------------- losses
def sigmoid_focal_loss_cuda(logits, targets, gamma, alpha):
    """layers/sigmoid_focal_loss.py:9-36: per-element losses [N, C]"""
    c = logits.shape[1]

    def run(x, t):
        return (_C.sigmoid_focalloss_forward(x, t, c, gamma, alpha),
                lambda g: (_C.sigmoid_focalloss_backward(x, t, g, c, gamma, alpha), None))
    return _COp.apply(run, logits, targets)


class SigmoidFocalLoss(nn.Module):
    """layers/sigmoid_focal_loss.py:52-76 (sum of the element losses); device tensors only"""

    def __init__(self, gamma, alpha):
        super().__init__()
        self.gamma, self.alpha = gamma, alpha

    def forward(self, logits, targets):
        return sigmoid_focal_loss_cuda(logits, targets, self.gamma, self.alpha).sum()

    def __repr__(self):
        return "SigmoidFocalLoss(gamma=%s, alpha=%s)" % (self.gamma, self.alpha)


def smooth_l1_loss(input, target, beta=1. / 9, size_average=True):
    """layers/smooth_l1_loss.py:6-16 (plain tensor arithmetic in the reference too)"""
    d = (input - target).abs()
    loss = torch.where(d < beta, d * d * (0.5 / beta), d - 0.5 * beta)
    return loss.mean() if size_average else loss.sum()


# ------------------------------------------------------------------------------------------ deformable convolution
def _dcn_out_shape(x, weight, stride, padding, dilation):
    dims = []
    for d in range(2):
        k = dilation[d] * (weight.shape[d + 2] - 1) + 1
        dims.append((x.shape[d + 2] + 2 * padding[d] - k) // stride[d] + 1)
    if min(dims) <= 0:
        raise ValueError("convolution input is too small (output would be %s)" % "x".join(map(str, dims)))
    return (x.shape[0], weight.shape[0]) + tuple(dims)


def deform_conv(input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1, im2col_step=64):
    """dcn/deform_conv_func.py:9-118 (v1). `im2col_step` only has to divide the batch, as in the reference; the B200
    kernels always process the whole batch."""
    if input is not None and input.dim() != 4:
        raise ValueError("Expected 4D tensor as input, got %dD tensor instead." % input.dim())
    (sh, sw), (ph, pw), (dh, dw) = _pair(stride), _pair(padding), _pair(dilation)
    step = min(im2col_step, input.shape[0])
    assert input.shape[0] % step == 0, "im2col step must divide batchsize"
    need = (input.requires_grad or offset.requires_grad, weight.requires_grad)

    def run(x, off, w):
        kh, kw = w.shape[2], w.shape[3]
        geo = (kw, kh, sw, sh, pw, ph, dw, dh, groups, deformable_groups)
        out = x.new_empty(_dcn_out_shape(x, w, (sh, sw), (ph, pw), (dh, dw)), dtype=torch.float32)
        _C.deform_conv_forward(x, w, off, out, None, None, *geo, step)

        def bwd(g):
            gx = goff = gw = None
            if need[0]:
                gx, goff = torch.zeros_like(x, dtype=torch.float32), torch.zeros_like(off, dtype=torch.float32)
                _C.deform_conv_backward_input(x, off, g, gx, goff, w, None, *geo, step)
            if need[1]:
                gw = torch.zeros_like(w, dtype=torch.float32)
                _C.deform_conv_backward_parameters(x, off, g, gw, None, None, *geo, 1, step)
            return gx, goff, gw
        return out, bwd
    return _COp.apply(run, input, offset, weight)


def modulated_deform_conv(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                          deformable_groups=1):
    """dcn/deform_conv_func.py:121-259 (v2; scalar stride / padding / dilation as in the reference)"""
    with_bias = bias is not None

    def run(x, off, m, w, b):
        kh, kw = w.shape[2], w.shape[3]
        geo = (kh, kw, stride, stride, padding, padding, dilation, dilation, groups, deformable_groups, with_bias)
        out = x.new_empty(_dcn_out_shape(x, w, _pair(stride), _pair(padding), _pair(dilation)), dtype=torch.float32)
        _C.modulated_deform_conv_forward(x, w, b, None, off, m, out, None, *geo)

        def bwd(g):
            gx, goff, gm = (torch.zeros_like(t, dtype=torch.float32) for t in (x, off, m))
            gw = torch.zeros_like(w, dtype=torch.float32)
            gb = torch.zeros_like(b, dtype=torch.float32) if with_bias else None
            _C.modulated_deform_conv_backward(x, w, b, None, off, m, None, gx, gw, gb, goff, gm, g, *geo)
            return gx, goff, gm, gw, gb
        return out, bwd
    return _COp.apply(run, input, offset, mask, weight, bias)


class DeformConv(nn.Module):
    """dcn/deform_conv_module.py:10-73"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=False):
        assert not bias
        assert in_channels % groups == 0, "in_channels %d cannot be divisible by groups %d" % (in_channels, groups)
        assert out_channels % groups == 0, "out_channels %d cannot be divisible by groups %d" % (out_channels, groups)
        super().__init__()
        self.with_bias = bias
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = (_pair(v) for v in
                                                                      (kernel_size, stride, padding, dilation))
        self.groups, self.deformable_groups = groups, deformable_groups
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, *self.kernel_size))
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1. / math.sqrt(self.in_channels * self.kernel_size[0] * self.kernel_size[1])
        nn.init.uniform_(self.weight, -bound, bound)
        if getattr(self, "bias", None) is not None:
            nn.init.zeros_(self.bias)

    def forward(self, input, offset):
        return deform_conv(input, offset, self.weight, self.stride, self.padding, self.dilation, self.groups,
                           self.deformable_groups)

    def extra_repr(self):
        return ("in_channels=%d, out_channels=%d, kernel_size=%s, stride=%s, dilation=%s, padding=%s, groups=%d, "
                "deformable_groups=%d, bias=%s" % (self.in_channels, self.out_channels, self.kernel_size, self.stride,
                                                   self.dilation, self.padding, self.groups, self.deformable_groups,
                                                   self.with_bias))


class ModulatedDeformConv(DeformConv):
    """dcn/deform_conv_module.py:76-137 (scalar stride / padding / dilation)"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, deformable_groups)
        self.stride, self.padding, self.dilation, self.with_bias = stride, padding, dilation, bias
        if bias:
            self.bias = nn.Parameter(torch.zeros(out_channels))
        else:
            self.register_parameter("bias", None)

    def forward(self, input, offset, mask):
        return modulated_deform_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding,
                                     self.dilation, self.groups, self.deformable_groups)


class ModulatedDeformConvPack(ModulatedDeformConv):
    """dcn/deform_conv_module.py:140-177: offsets and masks predicted by a zero-initialised ordinary convolution"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, deformable_groups,
                         bias)
        taps = self.kernel_size[0] * self.kernel_size[1]
        self.conv_offset_mask = nn.Conv2d(in_channels // groups, deformable_groups * 3 * taps, self.kernel_size,
                                          stride=_pair(stride), padding=_pair(padding), bias=True)
        self.init_offset()

    def init_offset(self):
        nn.init.zeros_(self.conv_offset_mask.weight)
        nn.init.zeros_(self.conv_offset_mask.bias)

    def forward(self, input):
        o1, o2, m = self.conv_offset_mask(input).chunk(3, dim=1)
        return super().forward(input, torch.cat((o1, o2), 1), torch.sigmoid(m))


# ------------------------------------------------------------------------------------- deformable PSROI pooling
def deform_roi_pooling(data, rois, offset, spatial_scale, out_size, out_channels, no_trans, group_size=1,
                       part_size=None, sample_per_part=4, trans_std=.0):
    """dcn/deform_pool_func.py:8-92"""
    part_size = out_size if part_size is None else part_size
    assert 0.0 <= trans_std <= 1.0
    args = (no_trans, spatial_scale, out_channels, group_size, out_size, part_size, sample_per_part, trans_std)

    def run(x, r, off):
        n = r.shape[0]
        out = x.new_empty(n, out_channels, out_size, out_size, dtype=torch.float32)
        count = torch.empty_like(out)
        _C.deform_psroi_pooling_forward(x, r, off, out, count, *args)

        def bwd(g):
            gx = torch.zeros_like(x, dtype=torch.float32)
            goff = torch.zeros_like(off, dtype=torch.float32)
            _C.deform_psroi_pooling_backward(g, x, r, off, count, gx, goff, *args)
            return gx, None, goff
        return out, bwd
    return _COp.apply(run, data, rois, offset)


class DeformRoIPooling(nn.Module):
    """dcn/deform_pool_module.py:6-33"""

    def __init__(self, spatial_scale, out_size, out_channels, no_trans, group_size=1, part_size=None, sample_per_part=4,
                 trans_std=.0):
        super().__init__()
        self.spatial_scale, self.out_size, self.out_channels, self.no_trans = spatial_scale, out_size, out_channels, no_trans
        self.group_size, self.part_size = group_size, (out_size if part_size is None else part_size)
        self.sample_per_part, self.trans_std = sample_per_part, trans_std

    def _pool(self, data, rois, offset, no_trans):
        return deform_roi_pooling(data, rois, offset, self.spatial_scale, self.out_size, self.out_channels, no_trans,
                                  self.group_size, self.part_size, self.sample_per_part, self.trans_std)

    def forward(self, data, rois, offset):
        return self._pool(data, rois, data.new_empty(0) if self.no_trans else offset, self.no_trans)


def _fc_stack(sizes, final_zero=True, sigmoid=False):
    layers = []
    for i in range(len(sizes) - 1):
        layers.append(nn.Linear(sizes[i], sizes[i + 1]))
        if i < len(sizes) - 2:
            layers.append(nn.ReLU(inplace=True))
    if final_zero:
        nn.init.zeros_(layers[-1].weight)
        nn.init.zeros_(layers[-1].bias)
    if sigmoid:
        layers.append(nn.Sigmoid())
    return nn.Sequential(*layers)


class DeformRoIPoolingPack(DeformRoIPooling):
    """dcn/deform_pool_module.py:36-86: offsets predicted from an undeformed pooling pass by three FC layers"""

    def __init__(self, spatial_scale, out_size, out_channels, no_trans, group_size=1, part_size=None, sample_per_part=4,
                 trans_std=.0, deform_fc_channels=1024):
        super().__init__(spatial_scale, out_size, out_channels, no_trans, group_size, part_size, sample_per_part,
                         trans_std)
        self.deform_fc_channels = deform_fc_channels
        if not no_trans:
            flat = out_size * out_size
            self.offset_fc = _fc_stack([flat * out_channels, deform_fc_channels, deform_fc_channels, flat * 2])

    def _offsets(self, data, rois):
        n = rois.shape[0]
        x = self._pool(data, rois, data.new_empty(0), True)
        return x, self.offset_fc(x.view(n, -1)).view(n, 2, self.out_size, self.out_size)

    def forward(self, data, rois):
        assert data.size(1) == self.out_channels
        if self.no_trans:
            return self._pool(data, rois, data.new_empty(0), True)
        return self._pool(data, rois, self._offsets(data, rois)[1], False)


class ModulatedDeformRoIPoolingPack(DeformRoIPoolingPack):
    """dcn/deform_pool_module.py:89-150: as above, times a predicted per-bin mask"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if not self.no_trans:
            flat = self.out_size * self.out_size
            self.mask_fc = _fc_stack([flat * self.out_channels, self.deform_fc_channels, flat], sigmoid=True)

    def forward(self, data, rois):
        assert data.size(1) == self.out_channels
        if self.no_trans:
            return self._pool(data, rois, data.new_empty(0), True)
        x, offset = self._offsets(data, rois)
        n = rois.shape[0]
        mask = self.mask_fc(x.view(n, -1)).view(n, 1, self.out_size, self.out_size)
        return self._pool(data, rois, offset, False) * mask
