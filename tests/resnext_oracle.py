"""The oracle's bottleneck (oracle/mega_oracle.py) for ResNeXt bodies: conv2 grouped with
NUM_GROUPS = conv1 width / conv2.weight.shape[1] (modeling/backbone/resnet.py:296-309). For NUM_GROUPS = 1 it computes
what mega_oracle.bottleneck computes. grouped_bottlenecks() makes the oracle's bodies and res5 heads use it."""
import contextlib

import torch.nn.functional as F


def bottleneck(x, sd, p, stride, dilation):
    """modeling/backbone/resnet.py:239-344 with STRIDE_IN_1X1=True (config/defaults.py:273) and a grouped conv2"""
    import mega_oracle as mo
    identity = x
    if dilation > 1:
        stride_eff, down_stride = 1, 1
    else:
        stride_eff, down_stride = stride, stride
    out = F.conv2d(x, sd[p + "conv1.weight"], None, stride_eff)
    out = mo.frozen_bn(out, sd, p + "bn1.").relu()
    w2 = sd[p + "conv2.weight"]
    out = F.conv2d(out, w2, None, 1, dilation, dilation, out.shape[1] // w2.shape[1])
    out = mo.frozen_bn(out, sd, p + "bn2.").relu()
    out = F.conv2d(out, sd[p + "conv3.weight"], None, 1)
    out = mo.frozen_bn(out, sd, p + "bn3.")
    if (p + "downsample.0.weight") in sd:
        identity = F.conv2d(x, sd[p + "downsample.0.weight"], None, down_stride)
        identity = mo.frozen_bn(identity, sd, p + "downsample.1.")
    return (out + identity).relu()


@contextlib.contextmanager
def grouped_bottlenecks():
    """inside: mega_oracle's resnet_c4_body / res5_head (and the oracles built on them) use the grouped bottleneck"""
    import mega_oracle as mo
    saved = mo.bottleneck
    mo.bottleneck = bottleneck
    try:
        yield
    finally:
        mo.bottleneck = saved
