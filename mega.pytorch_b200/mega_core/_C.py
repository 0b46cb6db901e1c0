"""`mega_core._C` -- the reference's native-op module (csrc/vision.cpp:9-25), served by the sm_90a
kernels of libmega_b200.so. Signatures are positional and identical to the reference's pybind
functions. Device tensors run the CUDA kernels; like the reference (csrc/nms.h:10-28, csrc/ROIAlign.h:11-25) `nms` and
`roi_align_forward` also accept CPU tensors (host implementations in csrc/host_ops.cu, bit-identical to the reference's
cpu/*.cpp); every other name is CUDA-only, as in the reference ("Not implemented on the CPU")."""
import torch

from . import _lib
from .b200 import ops


def _cuda_only(name, *tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("%s: Not implemented on the CPU (mega_core._C is the B200 build; "
                               "the CPU path of the reference lives only in the test oracle)" % name)


def nms(dets, scores, threshold):
    """nms(Tensor dets[n,4], Tensor scores[n], float thr) -> LongTensor (csrc/nms.h:10-28).
    Kept original indices in ascending order, on the input's device (nms.cu:127-130); an empty
    input returns an empty long tensor."""
    if dets.numel() == 0:
        return torch.empty(0, dtype=torch.int64, device="cpu")            # nms.h:17-18 / nms_cpu.cpp:13-15
    if not dets.is_cuda:
        return _nms_cpu(dets, scores, float(threshold))
    _cuda_only("nms", dets, scores)
    keep, count = ops.nms_device(dets, scores, float(threshold))
    return keep[: int(count.item())]        # the one host read the dynamic output size requires


def _nms_cpu(dets, scores, threshold):
    """nms_cpu (cpu/nms_cpu.cpp:6-75): suppress when IoU >= threshold, kept original indices ascending"""
    if scores.is_cuda:
        raise RuntimeError("scores must be a CPU tensor")
    if dets.dtype != scores.dtype:
        raise RuntimeError("dets should have the same type as scores")
    if dets.dtype not in (torch.float32, torch.float64):
        raise RuntimeError("nms: \"nms\" not implemented for '%s'" % dets.dtype)
    d, s = dets.contiguous(), scores.contiguous()
    n = d.shape[0]
    keep = torch.empty(n, dtype=torch.int64)
    count = torch.zeros(1, dtype=torch.int32)
    _lib.check(_lib.lib.mega_nms_host(d.data_ptr(), s.data_ptr(), n, threshold, 1 if d.dtype == torch.float64 else 0,
                                      keep.data_ptr(), count.data_ptr()), "mega_nms_host")
    return keep[: int(count[0])]


def roi_align_forward(input, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio):
    """(csrc/ROIAlign.h:11-25) NCHW fp32 input, rois [K,5] = (batch, x1, y1, x2, y2) -> [K,C,ph,pw]"""
    if not input.is_cuda:
        if rois.is_cuda:
            raise RuntimeError("rois must be a CPU tensor")
        if input.dtype not in (torch.float32, torch.float64) or rois.dtype != input.dtype:
            raise RuntimeError("ROIAlign_forward: input and rois must both be float32 or both float64 CPU tensors")
        x, r = input.contiguous(), rois.contiguous()
        out = torch.empty(r.shape[0], x.shape[1], int(pooled_height), int(pooled_width), dtype=x.dtype)
        if out.numel() == 0:
            return out
        _lib.check(_lib.lib.mega_roi_align_forward_nchw_host(x.data_ptr(), x.shape[0], x.shape[1], x.shape[2], x.shape[3],
                                                             r.data_ptr(), r.shape[0], float(spatial_scale),
                                                             int(pooled_height), int(pooled_width), int(sampling_ratio),
                                                             1 if x.dtype == torch.float64 else 0, out.data_ptr()),
                   "mega_roi_align_forward_nchw_host")
        return out
    _cuda_only("roi_align_forward", input, rois)
    return ops.roi_align_nchw(input, rois, float(spatial_scale), int(pooled_height), int(pooled_width),
                              int(sampling_ratio))


def sigmoid_focalloss_forward(logits, targets, num_classes, gamma, alpha):
    """(csrc/SigmoidFocalLoss.h:10-15) logits [N,C], int32 targets [N] -> losses [N,C]"""
    _cuda_only("sigmoid_focalloss_forward", logits, targets)
    logits = logits.contiguous().float()
    targets = targets.contiguous().to(torch.int32)
    out = torch.empty_like(logits)
    _lib.check(_lib.lib.mega_sigmoid_focalloss_forward(_lib.ptr(logits), _lib.ptr(targets), logits.shape[0],
                                                       int(num_classes), float(gamma), float(alpha), _lib.ptr(out),
                                                       _lib.stream_ptr()), "mega_sigmoid_focalloss_forward")
    return out


def sigmoid_focalloss_backward(logits, targets, d_losses, num_classes, gamma, alpha):
    """(csrc/SigmoidFocalLoss.h:26-32)"""
    _cuda_only("sigmoid_focalloss_backward", logits, targets, d_losses)
    logits = logits.contiguous().float()
    targets = targets.contiguous().to(torch.int32)
    d_losses = d_losses.contiguous().float()
    out = torch.empty_like(logits)
    _lib.check(_lib.lib.mega_sigmoid_focalloss_backward(_lib.ptr(logits), _lib.ptr(targets), _lib.ptr(d_losses),
                                                        logits.shape[0], int(num_classes), float(gamma), float(alpha),
                                                        _lib.ptr(out), _lib.stream_ptr()),
               "mega_sigmoid_focalloss_backward")
    return out


def _deform_conv(input, weight, bias, offset, mask, output, kh, kw, sh, sw, ph, pw, dh, dw, group, deformable_group):
    """bilinear im2col kernel + wgmma GEMM per group; writes `output` (NCHW) in place"""
    _cuda_only("deform_conv", input, weight, offset, output)
    if not (input.is_contiguous() and weight.is_contiguous()):
        raise RuntimeError("input / weight tensor has to be contiguous")     # deform_conv_cuda.cu:504-505
    b, c, h, w = input.shape
    cout, cpg = weight.shape[0], weight.shape[1]
    if tuple(weight.shape[2:]) != (kh, kw):
        raise RuntimeError("Input shape and kernel shape wont match: (%d x %d vs %d x %d)." % (kh, kw, weight.shape[2], weight.shape[3]))
    if c != cpg * group:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (c, cpg * group))
    ho = (h + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    wo = (w + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    kg = cpg * kh * kw
    cog = cout // group
    if kg % 4 or cog % 4:
        raise RuntimeError("deform_conv (B200 build): per-group C*kh*kw and Cout must be multiples of 4")
    if output.dtype != torch.float32 or not output.is_contiguous() or tuple(output.shape) != (b, cout, ho, wo):
        raise RuntimeError("deform_conv: output must be a contiguous float32 tensor of shape %s, got %s %s" % (
            (b, cout, ho, wo), output.dtype, tuple(output.shape)))
    kpad = c * kh * kw
    cols = torch.empty(b, ho * wo, kpad, device=input.device)
    # the converted operands stay bound until the launch is enqueued: a temporary freed earlier could be handed to the
    # next conversion by the caching allocator, and the kernel would read one operand through another's pointer
    x = input.float()
    off = offset.contiguous().float()
    msk = mask.contiguous().float() if mask is not None else None
    _lib.check(_lib.lib.mega_deform_im2col(_lib.ptr(x), _lib.ptr(off), _lib.ptr(msk), b, c, h, w, kh, kw, ph, pw, sh,
                                           sw, dh, dw, deformable_group, kpad, _lib.ptr(cols), _lib.stream_ptr()),
               "mega_deform_im2col")
    nhwc = torch.empty(b, 1, ho * wo, cout, device=input.device)
    w2 = weight.float().reshape(cout, kg)
    for g in range(group):
        a = cols.view(b, 1, ho * wo, kpad)[..., g * kg:(g + 1) * kg]
        wg = w2[g * cog:(g + 1) * cog].contiguous().view(1, cog, kg)
        bg = bias[g * cog:(g + 1) * cog].contiguous().float() if bias is not None else None
        ops.conv_gemm(a, wg, nhwc[..., g * cog:(g + 1) * cog], bias=bg, tile=(1, 128))
    out = output.view(b, cout, ho * wo)
    ops.transpose_2d(nhwc.view(b, ho * wo, cout), out, b, ho * wo, cout)
    return ho, wo


def deform_conv_forward(input, weight, offset, output, columns, ones, kW, kH, dW, dH, padW, padH, dilationW, dilationH,
                        group, deformable_group, im2col_step):
    """(csrc/deform_conv.h:11-28) v1; `output` [B,Cout,Ho,Wo] is written in place, returns 1"""
    _deform_conv(input, weight, None, offset, None, output, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group,
                 deformable_group)
    return 1


def modulated_deform_conv_forward(input, weight, bias, ones, offset, mask, output, columns, kernel_h, kernel_w,
                                  stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group, deformable_group,
                                  with_bias):
    """(csrc/deform_conv.h:115-150) v2; `output` is written in place"""
    _deform_conv(input, weight, bias if with_bias else None, offset, mask, output, kernel_h, kernel_w, stride_h, stride_w,
                 pad_h, pad_w, dilation_h, dilation_w, group, deformable_group)


def deform_psroi_pooling_forward(input, bbox, trans, out, top_count, no_trans, spatial_scale, output_dim, group_size,
                                 pooled_size, part_size, sample_per_part, trans_std):
    """(csrc/deform_pool.h:11-37) writes `out` [K,output_dim,ps,ps] and `top_count` in place"""
    _cuda_only("deform_psroi_pooling_forward", input, bbox, out, top_count)
    if not input.is_contiguous():
        raise RuntimeError("input must be contiguous")
    n, c, h, w = input.shape
    shape = (bbox.shape[0], int(output_dim), int(pooled_size), int(pooled_size))
    for name, t in (("out", out), ("top_count", top_count)):
        _writable(name, t)
        if tuple(t.shape) != shape:
            raise RuntimeError("%s must have shape %s, got %s" % (name, shape, tuple(t.shape)))
    num_classes = 1 if no_trans else trans.shape[1] // 2
    x = input.float()
    rois = bbox.contiguous().float()
    tr = trans.contiguous().float() if not no_trans else None
    _lib.check(_lib.lib.mega_deform_psroi_pooling_forward(
        _lib.ptr(x), _lib.ptr(rois), _lib.ptr(tr), bbox.shape[0], c, h, w,
        int(bool(no_trans)), float(spatial_scale), int(output_dim), int(group_size), int(pooled_size), int(part_size),
        int(sample_per_part), float(trans_std), num_classes, _lib.ptr(out), _lib.ptr(top_count), _lib.stream_ptr()),
        "mega_deform_psroi_pooling_forward")


def roi_align_backward(grad, rois, spatial_scale, pooled_height, pooled_width, batch_size, channels, height, width,
                       sampling_ratio):
    """(csrc/ROIAlign.h:27-45) grad [K,C,ph,pw], rois [K,5] -> grad_input [batch,C,H,W] (newly allocated, zeros + scatter)"""
    _cuda_only("roi_align_backward", grad, rois)
    grad_input = torch.zeros(int(batch_size), int(channels), int(height), int(width), device=grad.device)
    if grad.numel() == 0:                                   # ROIAlign_cuda.cu:324-327
        return grad_input
    grad = grad.contiguous().float()
    rois = rois.contiguous().float()
    _lib.check(_lib.lib.mega_roi_align_backward_nchw(
        _lib.ptr(grad), _lib.ptr(rois), rois.shape[0], float(spatial_scale), int(pooled_height), int(pooled_width),
        int(batch_size), int(channels), int(height), int(width), int(sampling_ratio), _lib.ptr(grad_input),
        _lib.stream_ptr()), "mega_roi_align_backward_nchw")
    return grad_input


def roi_pool_forward(input, rois, spatial_scale, pooled_height, pooled_width):
    """(csrc/ROIPool.h:11-24) -> (output [K,C,ph,pw], argmax int32 [K,C,ph,pw])"""
    _cuda_only("roi_pool_forward", input, rois)
    input = input.contiguous().float()
    rois = rois.contiguous().float()
    k, (n, c, h, w) = rois.shape[0], input.shape
    out = torch.empty(k, c, int(pooled_height), int(pooled_width), device=input.device)
    argmax = torch.zeros(k, c, int(pooled_height), int(pooled_width), device=input.device, dtype=torch.int32)
    if out.numel():
        _lib.check(_lib.lib.mega_roi_pool_forward(_lib.ptr(input), _lib.ptr(rois), k, float(spatial_scale), c, h, w,
                                                  int(pooled_height), int(pooled_width), _lib.ptr(out),
                                                  _lib.ptr(argmax), _lib.stream_ptr()), "mega_roi_pool_forward")
    return out, argmax


def roi_pool_backward(grad, input, rois, argmax, spatial_scale, pooled_height, pooled_width, batch_size, channels,
                      height, width):
    """(csrc/ROIPool.h:26-47) -> grad_input [batch,C,H,W]"""
    _cuda_only("roi_pool_backward", grad, rois, argmax)
    grad_input = torch.zeros(int(batch_size), int(channels), int(height), int(width), device=grad.device)
    if grad.numel() == 0:
        return grad_input
    grad = grad.contiguous().float()
    rois = rois.contiguous().float()
    argmax = argmax.contiguous().to(torch.int32)
    _lib.check(_lib.lib.mega_roi_pool_backward(_lib.ptr(grad), _lib.ptr(argmax), _lib.ptr(rois), rois.shape[0],
                                               int(channels), int(height), int(width), int(pooled_height),
                                               int(pooled_width), _lib.ptr(grad_input), _lib.stream_ptr()),
               "mega_roi_pool_backward")
    return grad_input


def _writable(name, t):
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise RuntimeError("%s must be a contiguous float32 tensor (it is written in place)" % name)


def _dcn_backward(input, offset, mask, weight_shape, weight, grad_output, grad_input, grad_offset, grad_mask,
                  grad_weight, grad_bias, scale, kh, kw, sh, sw, ph, pw, dh, dw, group, deformable_group):
    """Backward of (modulated) deformable convolution on the reference's column layout cols[k][b*ldp + p]
    (deform_conv_cuda.cu:300-302):
      input / offset / mask gradients: gcols = W^T . grad_out (one wgmma GEMM per group), then ONE fused pass
        (mega_deform_col2im_fused) instead of the reference's col2im_coord + col2im kernels;
      weight gradient: cols = deformable im2col of the input, grad_W += scale * grad_out . cols^T (one GEMM per group
        with K = batch * Ho * Wo, where the reference loops over im2col_step slices of the batch);
      bias gradient: per-channel sum of grad_out.
    Operand re-layouts (NCHW <-> pixel-major, zero padding of Ho*Wo to a multiple of 4 for TMA) are torch copies."""
    _cuda_only("deform_conv_backward", input, offset, grad_output)
    if not input.is_contiguous():
        raise RuntimeError("input tensor has to be contiguous")                 # deform_conv_cuda.cu:586
    b, c, h, w = input.shape
    cout, cpg_w = weight_shape[0], weight_shape[1]
    if tuple(weight_shape[2:]) != (kh, kw):
        raise RuntimeError("Input shape and kernel shape wont match: (%d x %d vs %d x %d)." % (kh, kw, weight_shape[2], weight_shape[3]))
    if c != cpg_w * group:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (c, cpg_w * group))
    ho = (h + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    wo = (w + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    if tuple(grad_output.shape) != (b, cout, ho, wo):
        raise RuntimeError("invalid spatial size of gradOutput: expected %s, got %s" % ((b, cout, ho, wo), tuple(grad_output.shape)))
    if offset.shape[0] != b:
        raise RuntimeError("invalid batch size of offset")                      # deform_conv_cuda.cu:306
    cog = cout // group
    if cog % 4:
        raise RuntimeError("deform_conv backward (B200 build): Cout / group must be a multiple of 4")
    taps, pt = kh * kw, ho * wo
    ldp = (pt + 3) // 4 * 4
    kg = cpg_w * taps
    dev = input.device
    x = input.float()
    off = offset.contiguous().float()
    msk = mask.contiguous().float() if mask is not None else None
    go = grad_output.contiguous().float().view(b, cout, pt)
    geo = (b, c, h, w, kh, kw, ph, pw, sh, sw, dh, dw, deformable_group, ldp)
    if grad_input is not None:
        _writable("grad_input", grad_input)
        _writable("grad_offset", grad_offset)
        if grad_mask is not None:
            _writable("grad_mask", grad_mask)
        go_t = torch.zeros(b, ldp, cout, device=dev)                # pixel-major grad_out: [b*ldp, cout]
        go_t[:, :pt] = go.transpose(1, 2)
        go_t = go_t.view(b * ldp, cout)
        gcols = torch.empty(c * taps, b * ldp, device=dev)
        w2 = weight.float().reshape(cout, kg)
        for g in range(group):
            wt_g = w2[g * cog:(g + 1) * cog].t().contiguous()                   # [kg, cog]
            ops.linear(wt_g, go_t[:, g * cog:(g + 1) * cog], gcols[g * kg:(g + 1) * kg])
        _lib.check(_lib.lib.mega_deform_col2im_fused(_lib.ptr(gcols), _lib.ptr(x), _lib.ptr(off), _lib.ptr(msk), *geo,
                                                     _lib.ptr(grad_input), _lib.ptr(grad_offset), _lib.ptr(grad_mask),
                                                     _lib.stream_ptr()), "mega_deform_col2im_fused")
    if grad_weight is not None:
        _writable("grad_weight", grad_weight)
        cols = torch.zeros(c * taps, b * ldp, device=dev)
        _lib.check(_lib.lib.mega_deform_im2col_kq(_lib.ptr(x), _lib.ptr(off), _lib.ptr(msk), *geo, _lib.ptr(cols),
                                                  _lib.stream_ptr()), "mega_deform_im2col_kq")
        go_p = torch.zeros(cout, b, ldp, device=dev)                # channel-major grad_out: [cout, b*ldp]
        go_p[:, :, :pt] = go.permute(1, 0, 2)
        go_p = go_p.view(cout, b * ldp)
        kgp = (kg + 3) // 4 * 4
        tmp = torch.empty(cout, kgp, device=dev)
        for g in range(group):
            ops.linear(go_p[g * cog:(g + 1) * cog], cols[g * kg:(g + 1) * kg], tmp[g * cog:(g + 1) * cog, :kg])
        grad_weight.view(cout, kg).add_(tmp[:, :kg], alpha=float(scale))        # addmm_(..., beta=1, alpha=scale)
    if grad_bias is not None:
        _writable("grad_bias", grad_bias)
        _lib.check(_lib.lib.mega_channel_sum_nchw(_lib.ptr(go), b, cout, pt, _lib.ptr(grad_bias), _lib.stream_ptr()),
                   "mega_channel_sum_nchw")


def deform_conv_backward_input(input, offset, gradOutput, gradInput, gradOffset, weight, columns, kW, kH, dW, dH, padW,
                               padH, dilationW, dilationH, group, deformable_group, im2col_step):
    """(csrc/deform_conv.h:45-77) v1: accumulates into `gradInput`, assigns `gradOffset` (both caller-allocated,
    deform_conv_func.py:87-88), returns 1. `columns` / im2col_step are the reference's scratch management: unused."""
    if not weight.is_contiguous():
        raise RuntimeError("weight tensor has to be contiguous")
    _dcn_backward(input.contiguous(), offset, None, weight.shape, weight, gradOutput, gradInput, gradOffset, None, None,
                  None, 1.0, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group, deformable_group)
    return 1


def deform_conv_backward_parameters(input, offset, gradOutput, gradWeight, columns, ones, kW, kH, dW, dH, padW, padH,
                                    dilationW, dilationH, group, deformable_group, scale, im2col_step):
    """(csrc/deform_conv.h:79-113) v1: gradWeight += scale * grad_out . cols^T, returns 1"""
    _dcn_backward(input.contiguous(), offset, None, gradWeight.shape, None, gradOutput, None, None, None, gradWeight,
                  None, scale, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group, deformable_group)
    return 1


def modulated_deform_conv_backward(input, weight, bias, ones, offset, mask, columns, grad_input, grad_weight, grad_bias,
                                   grad_offset, grad_mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                                   pad_w, dilation_h, dilation_w, group, deformable_group, with_bias):
    """(csrc/deform_conv.h:152-190) v2: accumulates grad_input / grad_weight / grad_bias, assigns grad_offset /
    grad_mask (all caller-allocated, deform_conv_func.py:206-210)"""
    if not weight.is_contiguous():
        raise RuntimeError("weight tensor has to be contiguous")                # deform_conv_cuda.cu:587
    _dcn_backward(input, offset, mask, weight.shape, weight, grad_output, grad_input, grad_offset, grad_mask,
                  grad_weight, grad_bias if with_bias else None, 1.0, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                  pad_w, dilation_h, dilation_w, group, deformable_group)


def deform_psroi_pooling_backward(out_grad, input, bbox, trans, top_count, input_grad, trans_grad, no_trans,
                                  spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part,
                                  trans_std):
    """(csrc/deform_pool.h:41-69) accumulates `input_grad` and `trans_grad` in place"""
    _cuda_only("deform_psroi_pooling_backward", out_grad, input, bbox, top_count, input_grad)
    if not out_grad.is_contiguous():
        raise RuntimeError("out_grad tensor has to be contiguous")              # deform_pool_cuda.cu:66
    if not input.is_contiguous():
        raise RuntimeError("input tensor has to be contiguous")
    n, c, h, w = input.shape
    if bbox.shape[0] != out_grad.shape[0]:
        raise RuntimeError("Output shape and bbox number wont match: (%d vs %d)." % (out_grad.shape[0], bbox.shape[0]))
    _writable("input_grad", input_grad)
    num_classes = 1 if no_trans else trans.shape[1] // 2
    tr = tg = None
    if not no_trans:
        _writable("trans_grad", trans_grad)
        tr, tg = trans.contiguous().float(), trans_grad
    og = out_grad.float()
    x = input.float()
    rois = bbox.contiguous().float()
    cnt = top_count.contiguous().float()
    _lib.check(_lib.lib.mega_deform_psroi_pooling_backward(
        _lib.ptr(og), _lib.ptr(x), _lib.ptr(rois), _lib.ptr(tr), _lib.ptr(cnt), bbox.shape[0], c, h, w, int(bool(no_trans)), float(spatial_scale),
        int(output_dim), int(group_size), int(pooled_size), int(part_size), int(sample_per_part), float(trans_std),
        num_classes, _lib.ptr(input_grad), _lib.ptr(tg), _lib.stream_ptr()), "mega_deform_psroi_pooling_backward")
