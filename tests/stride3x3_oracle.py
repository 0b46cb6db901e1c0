"""The oracle's bottleneck (oracle/mega_oracle.py) with MODEL.RESNETS.STRIDE_IN_1X1 = False: a block's stride on its 3x3
conv2 instead of its 1x1 conv1 (modeling/backbone/resnet.py:272-275; the downsample keeps the stride, a dilated block
runs at stride 1). conv2 is grouped with NUM_GROUPS = conv1 width / conv2.weight.shape[1] (resnet.py:296-309), so the
same block serves the dense and the ResNeXt bodies. strided_3x3() makes the oracle's bodies and res5 heads use it."""
import contextlib

import torch.nn.functional as F


def bottleneck(x, sd, p, stride, dilation):
    """modeling/backbone/resnet.py:239-344 with STRIDE_IN_1X1=False"""
    import mega_oracle as mo
    identity = x
    stride3, down_stride = (1, 1) if dilation > 1 else (stride, stride)
    out = F.conv2d(x, sd[p + "conv1.weight"], None, 1)
    out = mo.frozen_bn(out, sd, p + "bn1.").relu()
    w2 = sd[p + "conv2.weight"]
    out = F.conv2d(out, w2, None, stride3, dilation, dilation, out.shape[1] // w2.shape[1])
    out = mo.frozen_bn(out, sd, p + "bn2.").relu()
    out = F.conv2d(out, sd[p + "conv3.weight"], None, 1)
    out = mo.frozen_bn(out, sd, p + "bn3.")
    if (p + "downsample.0.weight") in sd:
        identity = F.conv2d(x, sd[p + "downsample.0.weight"], None, down_stride)
        identity = mo.frozen_bn(identity, sd, p + "downsample.1.")
    return (out + identity).relu()


@contextlib.contextmanager
def strided_3x3():
    """inside: mega_oracle's resnet_c4_body / res5_head (and the oracles built on them) use the 3x3-strided bottleneck"""
    import mega_oracle as mo
    saved = mo.bottleneck
    mo.bottleneck = bottleneck
    try:
        yield
    finally:
        mo.bottleneck = saved
