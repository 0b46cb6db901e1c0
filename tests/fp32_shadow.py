"""Test harness: an fp32 'shadow' of ops.conv_gemm built from torch ops (cuBLAS/cuDNN with TF32 off).

Used only by tests/tools to separate LOGIC errors of the engine orchestration from TF32 rounding
of the wgmma kernel: with the shadow installed every dense contraction is exact fp32 while all
other kernels (NMS, RPN selection, ROIAlign, relation soft-max, post-processing) stay ours."""
import contextlib

import torch
import torch.nn.functional as F


def _shadow_conv_gemm(a, w, out, *, taps=(1, 1), dil=1, pad=0, scale=None, bias=None, residual=None, relu=False,
                      tile=None, block_n=None, cout=None, k=None, batch=1, a_c_off=0, a_n_off=0, b_k_off=0, b_n_off=0,
                      out_c_off=0, out_n_off=0, res_c_off=0, res_n_off=0, bias_z_off=0, max_ctas=0, stream_k=None,
                      out_hw=None, n_img=None, stride=(1, 1), pad_w=None):
    t, rows, kk = w.shape
    cout = rows if cout is None else cout
    k = kk if k is None else k
    on, oh, ow, oc = out.shape
    if n_img is not None:
        on = n_img
    ld = out.stride(2)
    out_z_off = out_c_off + out_n_off * out.stride(0)
    res_z_off = res_c_off + (res_n_off * residual.stride(0) if residual is not None else 0)
    for z in range(batch):
        az = a[z * a_n_off: z * a_n_off + on] if a_n_off else a
        az = az[..., z * a_c_off: z * a_c_off + k]                       # [n,h,w,k]
        wz = w[:, z * b_n_off: z * b_n_off + cout, z * b_k_off: z * b_k_off + k]   # [t, cout, k]
        pw_ = pad if pad_w is None else pad_w
        if taps[0] == 1 and taps[1] == az.shape[2] and pad == 0 and pw_ == 0 and tuple(stride) == (1, 1) and ow == 1 \
                and dil == 1:
            # a kernel as wide as the map (the l_fcs[0] GEMM written as a convolution): one dot product per row
            y = (az.reshape(az.shape[0], az.shape[1], -1).double()
                 @ wz.permute(1, 0, 2).reshape(cout, -1).double().t()).view(az.shape[0], az.shape[1], 1, cout)[:, :oh]
        else:
            x = az.permute(0, 3, 1, 2).double()
            wt = wz.reshape(taps[0], taps[1], cout, k).permute(2, 3, 0, 1).double()
            extra_h, extra_w = taps[0] * dil + stride[0], taps[1] * dil + stride[1]     # zero fill beyond the map, like TMA
            x = F.pad(x, (pw_, extra_w, pad, extra_h))
            y = F.conv2d(x, wt, None, stride, 0, dil)[:, :, :oh, :ow].permute(0, 2, 3, 1)   # [n,oh,ow,cout]
        if scale is not None:
            y = y * scale[z * bias_z_off: z * bias_z_off + cout].double()
        if bias is not None:
            y = y + bias[z * bias_z_off: z * bias_z_off + cout].double()
        flat = out.reshape(-1) if out.is_contiguous() else None
        if residual is not None:
            r = torch.as_strided(residual, (on, oh, ow, cout),
                                 (residual.stride(0), residual.stride(1), residual.stride(2), 1),
                                 residual.storage_offset() + z * res_z_off)
            y = y + r.double()
        if relu == "leaky":
            y = F.leaky_relu(y, 0.1)
        elif relu:
            y = y.relu()
        o = torch.as_strided(out, (on, oh, ow, cout), (out.stride(0), out.stride(1), ld, 1),
                             out.storage_offset() + z * out_z_off)
        o.copy_(y.float())
    return out


@contextlib.contextmanager
def fp32_shadow():
    from mega_core.b200 import ops
    saved = ops.conv_gemm
    ops.conv_gemm = _shadow_conv_gemm
    try:
        yield
    finally:
        ops.conv_gemm = saved
