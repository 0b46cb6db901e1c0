// Sample geometry of a deformable convolution tap, shared by the NCHW im2col tile kernel of deform.cu and the NHWC
// column kernel of dcn_sample.cu, and compiled by g++ for the CPU tests (tests/native/dcn_sample_host.cpp).
//
// The arithmetic is the reference's deformable_im2col_bilinear behind the `h > -1 && w > -1 && h < H && w < W` gate
// (csrc/cuda/deform_conv_kernel_cuda.cu:92-120, :197-250, :578-640): floor, the four bilinear weights, and the four
// corner indices (h * width + w) with each corner's validity folded in (-1: that corner reads 0; all four -2: the whole
// sample is outside the gate and its value is 0).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define DCN_HD __host__ __device__ __forceinline__
#else
#define DCN_HD static inline
#endif

namespace mega {

struct DcnTap {          // geometry of one (tap, pixel) sample
  int i00, i01, i10, i11;
  float w00, w01, w10, w11;
};

constexpr int kDcnOutside = -2;

DCN_HD DcnTap dcn_tap_geometry(float h_im, float w_im, int height, int width) {
  DcnTap g = {0, 0, 0, 0, 0.f, 0.f, 0.f, 0.f};
  if (h_im > -1 && w_im > -1 && h_im < height && w_im < width) {
    const int h_low = static_cast<int>(floorf(h_im)), w_low = static_cast<int>(floorf(w_im));
    const int h_high = h_low + 1, w_high = w_low + 1;
    const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
    const bool t0 = h_low >= 0, t1 = h_high <= height - 1, l0 = w_low >= 0, l1 = w_high <= width - 1;
    g.i00 = (t0 && l0) ? h_low * width + w_low : -1;
    g.i01 = (t0 && l1) ? h_low * width + w_high : -1;
    g.i10 = (t1 && l0) ? h_high * width + w_low : -1;
    g.i11 = (t1 && l1) ? h_high * width + w_high : -1;
    g.w00 = hh * hw; g.w01 = hh * lw; g.w10 = lh * hw; g.w11 = lh * lw;
  } else {
    g.i00 = g.i01 = g.i10 = g.i11 = kDcnOutside;
  }
  return g;
}

// the interpolated value w00 v00 + w01 v01 + w10 v10 + w11 v11, as the reference's sum compiles for the GPU (one
// multiply, three fused multiply-adds, left to right); fmaf rounds once on the host too, so the g++ build gives the
// same bits
DCN_HD float dcn_blend(const DcnTap& g, float v00, float v01, float v10, float v11) {
  return fmaf(g.w11, v11, fmaf(g.w10, v10, fmaf(g.w01, v01, g.w00 * v00)));
}

// DCN v2 (DFConv2d.forward, layers/misc.py:182-184): the modulation scalar is the sigmoid of the offset conv's last 9
// channels
DCN_HD float dcn_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

}  // namespace mega
