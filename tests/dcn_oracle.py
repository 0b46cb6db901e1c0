"""The oracle's bottleneck (oracle/mega_oracle.py) with a deformable conv2 where the state dict has one: DFConv2d of
MODEL.RESNETS.STAGE_WITH_DCN (modeling/backbone/resnet.py:286-299, layers/misc.py:114-189). conv2.offset is a 3x3 conv
with bias (padding = dilation, the conv2 stride); its first 18 channels are the offsets, and for DCN v2 (27 channels)
the sigmoid of the last 9 is the mask; conv2.conv is the deformable conv without bias, restated by
oracle/train_ops_oracle.deform_conv2d. stride_in_1x1 picks the stride layout as tests/stride3x3_oracle.py does.
deformable() makes the oracle's bodies (and the oracles built on them) use it."""
import contextlib

import torch.nn.functional as F


def deform_conv2(x, sd, p, stride, dilation):
    """DFConv2d.forward (layers/misc.py:176-187) on x [B,C,H,W]"""
    import train_ops_oracle as to
    wo, bo = sd[p + "conv2.offset.weight"], sd[p + "conv2.offset.bias"]
    om = F.conv2d(x, wo, bo, stride, dilation, dilation)
    offset, mask = (om[:, :18], om[:, -9:].sigmoid()) if wo.shape[0] == 27 else (om, None)
    return to.deform_conv2d(x, offset, mask, sd[p + "conv2.conv.weight"], None, (stride, stride),
                            (dilation, dilation), (dilation, dilation), 1, 1)


def make_bottleneck(stride_in_1x1=True):
    def bottleneck(x, sd, p, stride, dilation):
        """modeling/backbone/resnet.py:239-344 with a DFConv2d conv2 when the state dict has conv2.conv.weight"""
        import mega_oracle as mo
        identity = x
        if dilation > 1:
            stride = 1
        s1, s3 = (stride, 1) if stride_in_1x1 else (1, stride)
        out = F.conv2d(x, sd[p + "conv1.weight"], None, s1)
        out = mo.frozen_bn(out, sd, p + "bn1.").relu()
        if (p + "conv2.conv.weight") in sd:
            out = deform_conv2(out, sd, p, s3, dilation)
        else:
            out = F.conv2d(out, sd[p + "conv2.weight"], None, s3, dilation, dilation)
        out = mo.frozen_bn(out, sd, p + "bn2.").relu()
        out = F.conv2d(out, sd[p + "conv3.weight"], None, 1)
        out = mo.frozen_bn(out, sd, p + "bn3.")
        if (p + "downsample.0.weight") in sd:
            identity = F.conv2d(x, sd[p + "downsample.0.weight"], None, stride)
            identity = mo.frozen_bn(identity, sd, p + "downsample.1.")
        return (out + identity).relu()
    return bottleneck


@contextlib.contextmanager
def deformable(stride_in_1x1=True):
    """inside: mega_oracle's resnet_c4_body / res5_head use the bottleneck above"""
    import mega_oracle as mo
    saved = mo.bottleneck
    mo.bottleneck = make_bottleneck(stride_in_1x1)
    try:
        yield
    finally:
        mo.bottleneck = saved
