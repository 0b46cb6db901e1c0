"""Layer wrappers with the reference's names (mega_core/layers/__init__.py:4-46): nms and the parameter holders here,
the differentiable `_C` ops (ROIAlign / ROIPool / focal loss / deformable convolution and pooling) in train_ops.py."""
import torch
from torch import nn

from .. import _C


def nms(boxes, scores, threshold):
    """layers/nms.py:8 of the reference (`amp.float_function(_C.nms)`): always fp32"""
    return _C.nms(boxes.float(), scores.float(), threshold)


from .train_ops import (ROIAlign, ROIPool, SigmoidFocalLoss, DeformConv, ModulatedDeformConv,  # noqa: E402,F401
                        ModulatedDeformConvPack, DeformRoIPooling, DeformRoIPoolingPack,
                        ModulatedDeformRoIPoolingPack, deform_conv, modulated_deform_conv, deform_roi_pooling,
                        roi_align, roi_pool, sigmoid_focal_loss_cuda, smooth_l1_loss)


class FrozenBatchNorm2d(nn.Module):
    """buffer holder with the reference's names (layers/batch_norm.py:5-31); the arithmetic
    (scale = weight * rsqrt(running_var), no eps) is folded into the conv epilogue on the device."""

    def __init__(self, n):
        super().__init__()
        self.register_buffer("weight", torch.ones(n))
        self.register_buffer("bias", torch.zeros(n))
        self.register_buffer("running_mean", torch.zeros(n))
        self.register_buffer("running_var", torch.ones(n))


Conv2d = nn.Conv2d   # the reference's empty-batch-safe subclass (layers/misc.py:30-43) is a parameter holder here


class DFConv2d(nn.Module):
    """parameter holder with the reference's names (layers/misc.py:114-189): `offset`, a Conv2d with bias predicting
    deformable_groups * 18 offsets (v1) or * 27 offsets and mask logits (with_modulated_dcn), and `conv`, the
    DeformConv / ModulatedDeformConv without bias. The engines run the deformable backbone convolutions on the
    device (mega_core/b200/engine.py, ResNetStages)."""

    def __init__(self, in_channels, out_channels, with_modulated_dcn=True, kernel_size=3, stride=1, groups=1,
                 dilation=1, deformable_groups=1, bias=False):
        super().__init__()
        padding = dilation * (kernel_size - 1) // 2
        per_group = kernel_size * kernel_size * (3 if with_modulated_dcn else 2)
        self.offset = Conv2d(in_channels, deformable_groups * per_group, kernel_size, stride=stride, padding=padding,
                             dilation=dilation)
        conv = ModulatedDeformConv if with_modulated_dcn else DeformConv
        self.conv = conv(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                         groups=groups, deformable_groups=deformable_groups, bias=bias)
        self.with_modulated_dcn = with_modulated_dcn
        self.kernel_size, self.stride, self.padding, self.dilation = kernel_size, stride, padding, dilation


__all__ = ["nms", "roi_align", "ROIAlign", "roi_pool", "ROIPool", "smooth_l1_loss", "Conv2d", "DFConv2d", "FrozenBatchNorm2d",
           "SigmoidFocalLoss", "deform_conv", "modulated_deform_conv", "DeformConv", "ModulatedDeformConv",
           "ModulatedDeformConvPack", "deform_roi_pooling", "DeformRoIPooling", "DeformRoIPoolingPack",
           "ModulatedDeformRoIPoolingPack"]
