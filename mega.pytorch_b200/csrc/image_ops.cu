// mega_image_transform_u8: decoded uint8 RGB frame (HWC, device) -> the fp32 [3, H', W'] tensor the reference's
// test-time transform produces (Resize + ToTensor + Normalize, data/transforms/build.py:5-49), bit-identical to the
// CPU pipeline. Replaces, per frame, PIL's two resize passes over the image, two float conversions and a
// normalisation on the host (SURVEY.md section 8f row 1: the step immediately before the hot path), and shrinks the
// host->device copy of a frame from 7.2 MB of fp32 to the 1.8-2.8 MB of the decoded bytes. HBM-side the kernel reads
// the source once (neighbouring outputs share taps through L1/L2) and writes 12 bytes per output pixel.
#include "common.cuh"
#include "image_ops.cuh"
#include "mega_b200.h"

namespace mega {

__global__ void image_transform_kernel(long long total, mega_image::ResizeGeom g, const uint8_t* __restrict__ src,
                                       float* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    mega_image::image_transform_item(i, g, src, out);
}

}  // namespace mega

extern "C" int mega_image_transform_u8_ex(const unsigned char* src, int src_h, int src_w, long long src_row_stride,
                                          long long src_pix_stride, long long src_ch_stride, const int* bounds_h,
                                          const int* kk_h, int ksize_h, const int* bounds_v, const int* kk_v, int ksize_v,
                                          int out_h, int out_w, const float* mean_host, const float* std_host,
                                          int to_bgr255, int hflip, float* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  MEGA_ARG_CHECK(src_h > 0 && src_w > 0 && out_h > 0 && out_w > 0, "image_transform: empty image");
  MEGA_ARG_CHECK((src_pix_stride == 3 && src_ch_stride == 1 && src_row_stride >= 3LL * src_w) ||
                     (src_pix_stride == 1 && src_ch_stride >= static_cast<long long>(src_h) * src_row_stride &&
                      src_row_stride >= src_w),
                 "image_transform: source must be interleaved HWC (pixel stride 3, channel stride 1) or planar CHW "
                 "(pixel stride 1, channel stride >= H * row stride)");
  MEGA_ARG_CHECK(ksize_h >= 0 && ksize_v >= 0, "image_transform: negative kernel size");
  MEGA_ARG_CHECK(ksize_h > 0 || out_w == src_w, "image_transform: horizontal pass skipped but widths differ");
  MEGA_ARG_CHECK(ksize_v > 0 || out_h == src_h, "image_transform: vertical pass skipped but heights differ");
  MEGA_ARG_CHECK((ksize_h == 0 || (bounds_h && kk_h)) && (ksize_v == 0 || (bounds_v && kk_v)),
                 "image_transform: coefficient tables missing");
  MEGA_ARG_CHECK(mean_host && std_host, "image_transform: mean / std missing");
  mega_image::ResizeGeom g;
  g.src_h = src_h, g.src_w = src_w, g.out_h = out_h, g.out_w = out_w, g.src_row_stride = src_row_stride;
  g.src_pix_stride = src_pix_stride, g.src_ch_stride = src_ch_stride;
  g.ksize_h = ksize_h, g.ksize_v = ksize_v;
  g.bounds_h = bounds_h, g.kk_h = kk_h, g.bounds_v = bounds_v, g.kk_v = kk_v;
  for (int c = 0; c < 3; ++c) g.mean[c] = mean_host[c], g.stdv[c] = std_host[c];
  g.to_bgr255 = to_bgr255 ? 1 : 0;
  g.hflip = hflip ? 1 : 0;
  const long long total = static_cast<long long>(out_h) * out_w;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  mega::image_transform_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(total, g, src, out);
  MEGA_CUDA_CHECK(cudaGetLastError());
  return MEGA_OK;
}

extern "C" int mega_image_transform_u8(const unsigned char* src, int src_h, int src_w, long long src_row_stride,
                                       long long src_pix_stride, long long src_ch_stride, const int* bounds_h, const int* kk_h, int ksize_h, const int* bounds_v,
                                       const int* kk_v, int ksize_v, int out_h, int out_w, const float* mean_host,
                                       const float* std_host, int to_bgr255, float* out, void* stream_v) {
  return mega_image_transform_u8_ex(src, src_h, src_w, src_row_stride, src_pix_stride, src_ch_stride, bounds_h, kk_h,
                                    ksize_h, bounds_v, kk_v, ksize_v, out_h, out_w, mean_host, std_host, to_bgr255, 0,
                                    out, stream_v);
}
