// Per-item body of the test-time input transform (SURVEY.md section 8f row 1): the reference's
//   Resize (PIL bilinear, data/transforms/transforms.py:27-63) -> ToTensor (:117-119) -> Normalize with to_bgr255
//   (:122-135)
// applied to a decoded uint8 RGB frame, fused into one pass with the reference's exact arithmetic:
//   * PIL's resize (Pillow 12.2 src/libImaging/Resample.c, a third-party dependency the reference does not pin) is a
//     horizontal then a vertical pass of 8-bit fixed-point convolutions: coefficients scaled by 2^22 and truncated
//     ((int)(0.5 + k * 2^22)), accumulator seeded with 2^21, result >> 22 clipped to 0..255, and -- the part a float
//     bilinear resize cannot reproduce -- the horizontal result is ROUNDED TO UINT8 before the vertical pass. The
//     coefficient / bounds tables are computed on the host in double exactly as precompute_coeffs() does
//     (mega_core/data/transforms: resample_tables) and passed in; the integer work happens here;
//   * ToTensor + Normalize: x = u8 / 255 (fp32 division), x * 255 when to_bgr255 (with the channel order reversed),
//     (x - mean) / std, each op rounded separately (no FMA contraction).
// Output: fp32 [3, out_h, out_w], the tensor `ImageList` wraps in the reference -- bit-identical to the CPU pipeline.
// Same __host__ __device__ arrangement as train_ops.cuh: the CPU tests run this body through a g++ build.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define MEGA_IMG_HD __host__ __device__ __forceinline__
#else
#define MEGA_IMG_HD static inline
#endif
#if defined(__CUDA_ARCH__)      // device pass: IEEE round-to-nearest ops that ptxas never contracts into FMAs
#define MEGA_FDIV(a, b) __fdiv_rn((a), (b))
#define MEGA_FMUL(a, b) __fmul_rn((a), (b))
#define MEGA_FSUB(a, b) __fsub_rn((a), (b))
#else                           // host pass (x86-64 without -mfma: no contraction either)
#define MEGA_FDIV(a, b) ((a) / (b))
#define MEGA_FMUL(a, b) ((a) * (b))
#define MEGA_FSUB(a, b) ((a) - (b))
#endif

namespace mega_image {

constexpr int kPrecisionBits = 32 - 8 - 2;   // Resample.c: PRECISION_BITS

struct ResizeGeom {
  int src_h, src_w, out_h, out_w;
  long long src_row_stride;   // bytes between source rows
  long long src_pix_stride;   // bytes between pixels of a row: 3 for interleaved HWC, 1 for planar CHW
  long long src_ch_stride;    // bytes between the R, G, B samples of a pixel: 1 for HWC, H * W for planar CHW
  int ksize_h, ksize_v;       // coefficients per output column / row (0: that pass is skipped, sizes equal)
  // device tables: bounds_* [2 * out] = (first source index, count), kk_* [out * ksize] fixed-point coefficients
  const int* bounds_h;
  const int* kk_h;
  const int* bounds_v;
  const int* kk_v;
  float mean[3], stdv[3];     // in OUTPUT channel order
  int to_bgr255;
  int hflip = 0;              // output column x takes resized column out_w - 1 - x (FLIP_LEFT_RIGHT after Resize)
};

MEGA_IMG_HD int clip8(int v) {
  v >>= kPrecisionBits;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// horizontal pass value of source row `row` at output column x (3 channels), rounded to uint8 like imTemp
MEGA_IMG_HD void horiz_rgb(const ResizeGeom& g, const uint8_t* src, int row, int x, int rgb[3]) {
  const uint8_t* line = src + row * g.src_row_stride;
  const long long ps = g.src_pix_stride, cs = g.src_ch_stride;
  if (g.ksize_h == 0) {
    rgb[0] = line[x * ps], rgb[1] = line[x * ps + cs], rgb[2] = line[x * ps + 2 * cs];
    return;
  }
  const int xmin = g.bounds_h[2 * x], n = g.bounds_h[2 * x + 1];
  const int* k = g.kk_h + static_cast<long long>(x) * g.ksize_h;
  int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
  const uint8_t* p = line + xmin * ps;
  for (int i = 0; i < n; ++i) {
    s0 += p[i * ps] * k[i];
    s1 += p[i * ps + cs] * k[i];
    s2 += p[i * ps + 2 * cs] * k[i];
  }
  rgb[0] = clip8(s0), rgb[1] = clip8(s1), rgb[2] = clip8(s2);
}

// one item = one output pixel (y, x), x fastest: three coalesced fp32 stores, neighbouring source bytes
MEGA_IMG_HD void image_transform_item(long long index, const ResizeGeom& g, const uint8_t* src, float* out) {
  const int x = static_cast<int>(index % g.out_w);
  const int y = static_cast<int>(index / g.out_w);
  const int xs = g.hflip ? g.out_w - 1 - x : x;
  int rgb[3];
  if (g.ksize_v == 0) {
    horiz_rgb(g, src, y, xs, rgb);
  } else {
    const int ymin = g.bounds_v[2 * y], n = g.bounds_v[2 * y + 1];
    const int* k = g.kk_v + static_cast<long long>(y) * g.ksize_v;
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int j = 0; j < n; ++j) {
      int h[3];
      horiz_rgb(g, src, ymin + j, xs, h);
      s0 += h[0] * k[j];
      s1 += h[1] * k[j];
      s2 += h[2] * k[j];
    }
    rgb[0] = clip8(s0), rgb[1] = clip8(s1), rgb[2] = clip8(s2);
  }
  const long long plane = static_cast<long long>(g.out_h) * g.out_w;
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int c = 0; c < 3; ++c) {
    const int u = g.to_bgr255 ? rgb[2 - c] : rgb[c];
    float v = MEGA_FDIV(static_cast<float>(u), 255.0f);          // F.to_tensor: byte -> float, div(255)
    if (g.to_bgr255) v = MEGA_FMUL(v, 255.0f);                   // image[[2, 1, 0]] * 255
    v = MEGA_FDIV(MEGA_FSUB(v, g.mean[c]), g.stdv[c]);           // F.normalize: sub_(mean).div_(std)
    out[c * plane + index] = v;
  }
}

}  // namespace mega_image
