"""Three representative contractions of the strict mode (3xTF32; --split16: 3xFP16 on split-fp16 tensors) at the sizes of a 4-key-frame step
(8 images of 600x1000), timed with CUDA events and -- under `ncu --profile-from-start off` -- profiled one launch each:
res4 3x3 (K = 2304 -> 256), RPN head 3x3 (K = 9216 -> 1024), res4 1x1 expand (K = 256 -> 1024, residual).
    ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/strict python tools/strict_gemm_probe.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "mega.pytorch_b200"))
import torch  # noqa: E402

from mega_core.b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
n, h, w = 8, 38, 63
ops.AUTOTUNE[0] = True


def mk(*s):
    return (torch.randn(*s, generator=g) * 0.5).to(dev)


x256, x1024 = mk(n, h, w, 256), mk(n, h, w, 1024)
w33, wrpn, wexp = mk(9, 256, 256) * 0.05, mk(9, 1024, 1024) * 0.02, mk(1, 1024, 256) * 0.1
o256, o1024, o1024b = torch.zeros(n, h, w, 256, device=dev), torch.zeros(n, h, w, 1024, device=dev), torch.zeros(n, h, w, 1024, device=dev)
sc, bi = torch.ones(1024, device=dev), torch.zeros(1024, device=dev)
S256, S1024 = sc[:256], sc
cases = [("res4 3x3 256->256", lambda: ops.conv_gemm(x256, w33, o256, taps=(3, 3), pad=1, scale=S256, bias=bi[:256], relu=True), 2 * n * h * w * 256 * 2304),
         ("rpn 3x3 1024->1024", lambda: ops.conv_gemm(x1024, wrpn, o1024, taps=(3, 3), pad=1, bias=bi, relu=True), 2 * n * h * w * 1024 * 9216),
         ("res4 1x1 256->1024 + residual", lambda: ops.conv_gemm(x256, wexp, o1024b, scale=S1024, bias=bi, residual=x1024, relu=True), 2 * n * h * w * 1024 * 256)]
if "--split16" in sys.argv:      # the same three layers in the split-fp16 format ("3xFP16": no split work in the kernel)
    ops.pack_split16(x256), ops.pack_split16(x1024)
    ops.mark_split16(o256), ops.mark_split16(o1024b)
    w33, wrpn, wexp = ops.pack_weights_split16(w33, scale=S256), ops.pack_weights_split16(wrpn), ops.pack_weights_split16(wexp, scale=S1024)
    S256 = S1024 = None      # (folded into the packed weights)
    ops.mark_split16(o1024)
if "--split16" in sys.argv and "--more" in sys.argv:
    # two layers that ran slower than their shapes explain inside the step: the RPN head's 1x1 (75 of 80 output columns, block_n
    # 64 as the engine launches it / 128) and res5's dilated 3x3
    x512 = ops.pack_split16(mk(n, h, w, 512))
    whead, w5 = ops.pack_weights_split16(mk(1, 75, 1024) * 0.02), ops.pack_weights_split16(mk(9, 512, 512) * 0.02)
    ohead, o512 = torch.zeros(n, h, w, 80, device=dev), ops.mark_split16(torch.zeros(n, h, w, 512, device=dev))
    cases += [("rpn head 1x1 1024->75, block_n 64", lambda: ops.conv_gemm(x1024, whead, ohead, bias=bi[:75], cout=75, block_n=64), 2 * n * h * w * 75 * 1024),
              ("rpn head 1x1 1024->75, block_n 128", lambda: ops.conv_gemm(x1024, whead, ohead, bias=bi[:75], cout=75, block_n=128), 2 * n * h * w * 75 * 1024),
              ("res5 3x3 dil 2 512->512", lambda: ops.conv_gemm(x512, w5, o512, taps=(3, 3), dil=2, pad=2, bias=bi[:512], relu=True), 2 * n * h * w * 512 * 4608),
              ("res5 3x3 dil 2 512->512, 124 CTAs", lambda: ops.conv_gemm(x512, w5, o512, taps=(3, 3), dil=2, pad=2, bias=bi[:512], relu=True, max_ctas=124), 2 * n * h * w * 512 * 4608)]
with ops.precision("fp32x3"):
    for name, fn, flops in cases:
        for _ in range(3):
            fn()
        ts = []
        for _ in range(10):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ms = float(np.median(ts))
        print("%-32s %8.1f us  %7.1f GFLOP  %6.1f TFLOP/s (x3 MMAs: %6.1f executed)" % (name, ms * 1e3, flops / 1e9, flops / ms / 1e9, 3 * flops / ms / 1e9))
    torch.cuda.profiler.start()
    for name, fn, flops in cases[:3]:
        fn()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
